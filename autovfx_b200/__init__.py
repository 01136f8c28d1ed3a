"""autovfx_b200 — H100-native (sm_90a) 3D-Gaussian-splatting rasterizer hot path for haoyuhsu/autovfx.

Only what the path needs: ``csrc/`` (hand-written CUDA + the C ABI of include/gsr_b200.h), the host-side
mirror of the reference's Python interface (``rasterizer``, ``knn``), the per-frame loop (``render_loop``) and
caller-contract helpers (``scene``).  Importing the operators requires the compiled library; there is no
CPU or PyTorch fallback.
"""
__version__ = "0.1.0"


def load_ops():
    """Import the CUDA-backed operators (raises ImportError if libgsr_b200.so is unavailable)."""
    from . import rasterizer, knn  # noqa: F401
    return rasterizer, knn
