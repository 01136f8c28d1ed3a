"""CPU tests of the host's slab sizing and selection (rasterizer.slab_stride, _DeviceState.grow_slab) and of the C ABI's slab
workspace queries.  No compute calls."""
from autovfx_b200 import _lib
from autovfx_b200 import rasterizer as R

TILES_1080P = 120 * 68


def test_first_guess_fills_the_budget_and_overflow_sets_the_stride():
    cap = 12_000_000
    S = R.slab_stride(3_000_000, 1920, 1080, cap, 0)
    assert S % R.SLAB_ALIGN == 0 and TILES_1080P * S <= R.SLAB_BUDGET * cap < TILES_1080P * (S + R.SLAB_ALIGN)
    st = object.__new__(R._DeviceState)  # host bookkeeping only: no pinned ring, no device
    st.capacity, st.slab_want = cap, 0
    st.grow_slab(2000)
    assert st.slab_want == 2528 and st.slab_stride(3_000_000, 1920, 1080) == 2528  # 1.25 x 2000 rounded up to 32
    st.grow_slab(1000)  # never shrinks
    assert st.slab_want == 2528


def test_crowded_tiles_and_wide_ids_select_the_ranked_emission():
    cap = 12_000_000
    assert R.slab_stride(3_000_000, 1920, 1080, cap, 32 * ((R.SLAB_BUDGET * cap // TILES_1080P) // 32 + 1)) == 0  # over budget
    assert R.slab_stride((1 << 24) + 1, 1920, 1080, cap, 64) == 0  # ids wider than 24 bits: no packed keys
    assert R.slab_stride(0, 1920, 1080, cap, 64) == 0
    assert R.slab_stride(1000, 64, 64, 1 << 20, 64, _lib.GSR_FLAG_TIGHT_TILES) == 0  # tight tiles keep the ranked emission
    assert R.slab_stride(1000, 64, 64, 1 << 20, 64) == 64


def test_flags_carry_the_stride_above_the_mode_bits():
    assert R.slab_flags(0) == 0
    f = R.slab_flags(2528)
    assert f >> _lib.GSR_SLAB_SHIFT == 2528 // 32 and f & ((1 << _lib.GSR_SLAB_SHIFT) - 1) == 0
    assert _lib.GSR_FLAG_RESUME < (1 << _lib.GSR_SLAB_SHIFT)


def test_slab_workspace_queries():
    L = _lib.lib
    for cap, W, H, S in ((1, 64, 48, 32), (12345, 256, 256, 96), (12_000_000, 1920, 1080, 2528)):
        tiles = ((W + 15) // 16) * ((H + 15) // 16)
        nbytes = L.gsr_binning_bytes_slab(cap, W, H, S)
        assert L.gsr_binning_capacity_slab(nbytes, W, H, S) >= cap
        assert nbytes - L.gsr_binning_bytes(cap) < 13 * (tiles * S + 64)
    assert L.gsr_binning_bytes_slab(1000, 64, 64, 0) == L.gsr_binning_bytes(1000)
    assert L.gsr_binning_capacity_slab(L.gsr_binning_bytes(1000), 64, 64, 0) == 1000
    assert L.gsr_binning_capacity_slab(L.gsr_binning_bytes(1000), 1920, 1080, 32) == 0  # the slab does not fit
