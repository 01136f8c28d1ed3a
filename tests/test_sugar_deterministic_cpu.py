"""The deterministic SuGaR backwards' C ABI without a GPU: the six symbols are exported, the _bytes queries follow their documented
formulas in size_t at large sizes, and the entries reject a NULL, misaligned or short scratch and ids at or above 2^32 before any
device call (the pointers passed here are never dereferenced)."""
from __future__ import annotations

import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import pytest  # noqa: E402

SYMBOLS = ("gsr_sugar_field_backward_det_bytes", "gsr_sugar_field_backward_det", "gsr_sugar_sdf_normal_backward_det_bytes",
           "gsr_sugar_sdf_normal_backward_det", "gsr_sugar_sample_backward_det_bytes", "gsr_sugar_sample_backward_det")


@pytest.fixture(scope="module")
def L():
    from autovfx_b200 import _lib
    return _lib


def A(x):
    return -(-x // 256) * 256


def group(M, P):  # the grouping of M partial ids over P Gaussians (include/gsr_b200.h)
    c = -(-M // 2048)
    return 4 * A(4 * M) + A(1024 * c) + A(4 * (-(-max(256 * c, P + 1) // 1024))) + A(4 * (P + 1))


def field_bytes(N, K, P):
    return A(128 * P) + 2 * A(4 * N) + group(N * K, P)


def normal_bytes(N, K, P, with_loss):
    return A(64 * P) + A(16 * N) + A(32 * N) + group(N * (K + 1) if with_loss else N, P)


def test_symbols_are_exported(L):
    for s in SYMBOLS:
        assert s in L.EXPORTS and hasattr(L.lib, s), s
    assert L.lib.gsr_abi_version() == 4


SIZES = [(0, 1, 0), (1, 1, 1), (1000, 16, 4000), (1_000_000, 16, 3_000_000), (2**31 - 1, 32, 2**31 - 1), (134_217_728, 32, 7)]


@pytest.mark.parametrize("N,K,P", SIZES)
def test_bytes_formulas(L, N, K, P):
    assert L.lib.gsr_sugar_field_backward_det_bytes(N, K, P) == field_bytes(N, K, P)
    for wl in (0, 1):
        assert L.lib.gsr_sugar_sdf_normal_backward_det_bytes(N, K, P, wl) == normal_bytes(N, K, P, wl)
    assert L.lib.gsr_sugar_sample_backward_det_bytes(N, max(P, 1)) == group(N, max(P, 1))


FAKE = 0x100000  # 16-byte aligned, never dereferenced: every rejection below happens before a device call


def _err(L):
    return L.lib.gsr_last_error().decode()


def _field(L, N=1000, K=16, P=4000, scratch=FAKE, nbytes=None):
    nbytes = L.lib.gsr_sugar_field_backward_det_bytes(N, K, P) if nbytes is None else nbytes
    return L.lib.gsr_sugar_field_backward_det(N, K, P, N, FAKE, FAKE, None, FAKE, FAKE, FAKE, FAKE, 1.0, 1e-16, 0.0, FAKE, None, None,
                                              None, FAKE, FAKE, FAKE, FAKE, FAKE, scratch, nbytes, None)


def _normal(L, N=1000, K=16, P=4000, loss=True, scratch=FAKE, nbytes=None):
    nbytes = L.lib.gsr_sugar_sdf_normal_backward_det_bytes(N, K, P, int(loss)) if nbytes is None else nbytes
    return L.lib.gsr_sugar_sdf_normal_backward_det(N, K, P, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE if loss else None,
                                                   None if loss else FAKE, FAKE, FAKE, FAKE, scratch, nbytes, None)


def _sample(L, N=1000, P=4000, scratch=FAKE, nbytes=None):
    nbytes = L.lib.gsr_sugar_sample_backward_det_bytes(N, P) if nbytes is None else nbytes
    return L.lib.gsr_sugar_sample_backward_det(N, P, 1.5, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, scratch, nbytes, None)


CALLS = {"field": _field, "normal_loss": _normal, "normal_estimate": lambda L, **kw: _normal(L, loss=False, **kw), "sample": _sample}


@pytest.mark.parametrize("which", sorted(CALLS))
def test_null_misaligned_and_short_scratch(L, which):
    call = CALLS[which]
    assert call(L, scratch=None) == -1 and "scratch is NULL" in _err(L)
    assert call(L, scratch=FAKE + 4) == -1 and "16-byte aligned" in _err(L)
    need = {"field": lambda: L.lib.gsr_sugar_field_backward_det_bytes(1000, 16, 4000),
            "normal_loss": lambda: L.lib.gsr_sugar_sdf_normal_backward_det_bytes(1000, 16, 4000, 1),
            "normal_estimate": lambda: L.lib.gsr_sugar_sdf_normal_backward_det_bytes(1000, 16, 4000, 0),
            "sample": lambda: L.lib.gsr_sugar_sample_backward_det_bytes(1000, 4000)}[which]()
    assert call(L, nbytes=need - 1) == -2 and "too small" in _err(L)


def test_ids_at_or_above_two_to_the_32(L):
    # N * K = 2^27 * 32 = 2^32 field ids; N * (K + 1) = (2^32 / 17 + 1) * 17 > 2^32 normal ids, one fewer sample stays below
    assert _field(L, N=2**27, K=32) == -1 and "2^32" in _err(L)
    n = 2**32 // 17 + 1
    assert _normal(L, N=n, K=16) == -1 and "2^32" in _err(L)
    # just below: the id check passes and a one-byte-short scratch is what is reported
    need = L.lib.gsr_sugar_field_backward_det_bytes(2**27 - 1, 32, 4000)
    assert _field(L, N=2**27 - 1, K=32, nbytes=need - 1) == -2
    assert _normal(L, N=n - 1, K=16, nbytes=L.lib.gsr_sugar_sdf_normal_backward_det_bytes(n - 1, 16, 4000, 1) - 1) == -2
    # without the loss a sample has one id, so the same N is accepted as far as the size check
    assert _normal(L, N=n, K=16, loss=False, nbytes=L.lib.gsr_sugar_sdf_normal_backward_det_bytes(n, 16, 4000, 0) - 1) == -2
