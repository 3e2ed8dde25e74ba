"""Argument checks of the mode-P silhouette entry points, which reject a bad workspace before any CUDA call (no device
needed), and the workspace size they ask for."""
import ctypes

import pytest


@pytest.fixture(scope="module")
def lib():
    import b3d
    return b3d.lib


def _taps(n=21):
    return ctypes.cast((ctypes.c_float * n)(*([1.0 / n] * n)), ctypes.c_void_p)


FAKE = ctypes.c_void_p(1 << 20)     # a device address that is never dereferenced: the calls fail their checks first


def test_workspace_bytes(lib):
    for B, V in [(1, 2), (2, 32), (16, 128), (64, 128)]:
        assert lib.b3d_pc_silhouette_workspace_bytes(B, V, 0) == 0
        assert lib.b3d_pc_silhouette_workspace_bytes(B, V, 1) == 2 * B * V ** 3 * 4


@pytest.mark.parametrize("direction", ["fwd", "bwd"])
def test_mode_p_rejects_a_missing_or_small_workspace(lib, direction):
    B, N, V = 2, 100, 32
    need = lib.b3d_pc_silhouette_workspace_bytes(B, V, 1)

    def call(mode, ws, nbytes, batch=B):
        if direction == "fwd":
            return lib.b3d_pc_silhouette_fwd_hosttaps(FAKE, FAKE, _taps(), 21, None, batch, N, V, mode, FAKE, ws, nbytes, None)
        return lib.b3d_pc_silhouette_bwd_hosttaps(FAKE, FAKE, _taps(), 21, None, FAKE, batch, N, V, mode, FAKE, None, ws,
                                                  nbytes, None)

    for ws, nbytes in [(None, 0), (None, need), (FAKE, need - 4), (FAKE, 0)]:
        assert call(1, ws, nbytes) == -1
        msg = lib.b3d_last_error().decode()
        assert "workspace" in msg and str(need) in msg, msg
    assert call(1, ctypes.c_void_p((1 << 20) + 4), need) == -2         # 16-byte alignment, as every buffer of the ABI
    # an empty batch needs no workspace in either mode; mode R never needs one
    assert call(1, None, 0, batch=0) == 0
    assert call(0, None, 0, batch=0) == 0
    assert call(2, FAKE, need) == -1 and "mode" in lib.b3d_last_error().decode()
