"""The deterministic backward's C ABI without a GPU: the two symbols are exported, gsr_backward_det_bytes follows its formula, and
gsr_backward_det rejects a NULL or misaligned scratch, one too small for the frame's tiles and NULL arguments before any device
call (the pointers passed here are never dereferenced)."""
from __future__ import annotations

import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import pytest  # noqa: E402


@pytest.fixture(scope="module")
def L():
    from autovfx_b200 import _lib
    return _lib


def _formula(R, W, H, extra):
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    table = -(-tiles * 8 * 4 // 256) * 256  # [tiles][8] u32 warp_last, 256-byte aligned
    return table + R * 8 * (13 if extra else 10) * 4


def test_symbols_are_exported(L):
    assert "gsr_backward_det" in L.EXPORTS and "gsr_backward_det_bytes" in L.EXPORTS
    assert hasattr(L.lib, "gsr_backward_det") and hasattr(L.lib, "gsr_backward_det_bytes")
    assert L.lib.gsr_abi_version() == 4


@pytest.mark.parametrize("R", [0, 1, 31, 6_900_000, 3_000_000_000])
@pytest.mark.parametrize("W,H", [(1, 1), (16, 16), (17, 9), (1920, 1080), (8192, 4096)])
@pytest.mark.parametrize("extra", [0, 1])
def test_bytes_formula(L, R, W, H, extra):
    assert L.lib.gsr_backward_det_bytes(R, W, H, extra) == _formula(R, W, H, extra)


def _frame(L, P=10, W=64, H=48):
    fr = L.gsr_frame()
    fr.P, fr.D, fr.M, fr.W, fr.H = P, 0, 0, W, H
    fr.bg, fr.means3D = 0x1000, 0x2000
    return fr


FAKE = 0x100000  # 16-byte aligned, never dereferenced: every rejection below happens before a device call


def _grads(L):
    return L.gsr_grads(*([FAKE] * 7 + [None, None, None]))


def _call(L, fr=True, ws=True, gr=True, inputs=FAKE, scratch=FAKE, nbytes=1 << 20, extras=(None, None, None)):
    f = _frame(L) if fr is True else None
    w = L.gsr_workspace(FAKE, 1 << 20, FAKE, 1 << 20, FAKE, 1 << 20) if ws else None
    g = _grads(L) if gr else None
    return L.lib.gsr_backward_det(C.byref(f) if f is not None else None, C.byref(w) if w is not None else None, inputs, inputs, inputs,
                                  inputs, inputs, *extras, C.byref(g) if g is not None else None, scratch, nbytes, None)


def _err(L):
    return L.lib.gsr_last_error().decode()


def test_null_and_misaligned_scratch(L):
    assert _call(L, scratch=None) == -1 and "scratch is NULL" in _err(L)
    assert _call(L, scratch=FAKE + 4) == -1 and "16-byte aligned" in _err(L)


def test_scratch_smaller_than_the_tile_table(L):
    need = L.lib.gsr_backward_det_bytes(0, 64, 48, 0)
    assert _call(L, nbytes=need - 1) == -2 and "too small" in _err(L)
    need_x = L.lib.gsr_backward_det_bytes(0, 64, 48, 1)
    assert _call(L, nbytes=need_x - 1, extras=(FAKE, FAKE, FAKE)) == -2 and "too small" in _err(L)


def test_null_arguments(L):
    assert _call(L, fr=False) == -1 and "null argument" in _err(L)
    assert _call(L, ws=False) == -1 and "null argument" in _err(L)
    assert _call(L, gr=False) == -1 and "null argument" in _err(L)
    assert _call(L, inputs=None) == -1 and "null input" in _err(L)
    assert _call(L, extras=(FAKE, None, FAKE)) == -1 and "all given or all NULL" in _err(L)
