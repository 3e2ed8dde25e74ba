"""Texture filters and kaolin's linear_rasterizer arguments without a GPU: the oracle composition against the reference's
Renderer (tests/golden/filtering_reference.npz), argument errors in Python and at the C ABI."""
import os
import sys
import tempfile
import warnings

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import mesh as M

sys.path.insert(0, GOLDEN)
import filtering_common as FC        # noqa: E402


@pytest.mark.parametrize("si", [0, 1])
@pytest.mark.parametrize("filtering", ["nearest", "bicubic"])
def test_oracle_render_reproduces_reference_filtering(si, filtering):
    z = np.load(os.path.join(GOLDEN, "filtering_reference.npz"))
    path = M.write_uvsphere_obj(os.path.join(tempfile.mkdtemp(), "uvsphere_16rings.obj"), rings=16)
    T = M.TemplateData(M.load_obj(path), path)
    H = int(z["H"][0])
    vtx, uvs, tex, bg = (torch.from_numpy(z[f"s{si}_{k}"]) for k in ("vtx", "uvs", "tex", "bg"))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)      # grid_sample's align_corners default notice
        img, alpha, _, _ = FC.render(vtx, T.faces, uvs, tex, T.face_textures, H, H, filtering=filtering)
        img_bg, hard, _, _ = FC.render(vtx, T.faces, uvs, tex, T.face_textures, H, H, background_image=bg,
                                       return_hardmask=True, filtering=filtering)
    for got, key in ((img, "img"), (alpha, "alpha"), (img_bg, "img_bg"), (hard, "hard")):
        assert torch.equal(got, torch.from_numpy(z[f"s{si}_{filtering}_{key}"])), key
    if si == 1:
        assert float(uvs.min()) < 0 and float(uvs.max()) > 1          # zero padding is exercised


def test_unknown_filter_is_a_value_error():
    from rendering.renderer import Renderer
    for f in ("bilinear", "nearest", "bicubic"):
        Renderer(16, 16, filtering=f)
    for f in ("area", "Bilinear", None):
        with pytest.raises(ValueError, match="filtering"):
            Renderer(16, 16, filtering=f)


def kaolin_args(B=2, F=5, d=3):
    return (torch.zeros(B, F, 9), torch.zeros(B, F, 6), torch.zeros(B, F, 1), torch.zeros(B, F, 3 * d))


@pytest.mark.parametrize("bad,match", [
    (dict(knum=0), "knum"), (dict(knum=2.5), "knum"), (dict(expand=-0.01), "expand"),
    (dict(multiplier=0.0), "multiplier"), (dict(delta=-1.0), "delta"),
])
def test_linear_rasterizer_bad_parameters(bad, match):
    import b3d
    from rendering.renderer import linear_rasterizer
    with pytest.raises(b3d.B3DError, match=match):
        linear_rasterizer(8, 8, *kaolin_args(), **bad)


@pytest.mark.parametrize("which,shape", [
    (3, (2, 5, 0)), (3, (2, 5, 4)), (3, (2, 4, 3)), (1, (2, 5, 4)), (1, (2, 5)), (2, (2, 5, 3)), (2, (2, 5)),
    (0, (2, 5, 6)),
])
def test_linear_rasterizer_misshaped_inputs(which, shape):
    import b3d
    from rendering.renderer import linear_rasterizer
    args = list(kaolin_args())
    args[which] = torch.zeros(shape)
    with pytest.raises(b3d.B3DError, match="points3d|points2d|normalz|vertex_attr"):
        linear_rasterizer(8, 8, *args)


def test_cpu_tensors_are_rejected():
    import b3d
    from rendering.renderer import linear_rasterizer
    with pytest.raises(b3d.B3DError, match="no CPU fallback"):
        linear_rasterizer(8, 8, *kaolin_args(d=4))


def test_c_abi_rejects_bad_arguments():
    import b3d
    lib = b3d.lib
    # (d, expand, knum, multiplier, delta) -> message
    cases = [((0, 0.02, 30, 1000.0, 7000.0), b"d=0"), ((3, 0.02, 0, 1000.0, 7000.0), b"knum=0"),
             ((3, 0.02, 30, 0.0, 7000.0), b"multiplier"), ((3, 0.02, 30, 1000.0, 0.0), b"delta"),
             ((3, -0.5, 30, 1000.0, 7000.0), b"expand")]
    for (d, e, k, m, dl), msg in cases:
        assert lib.b3d_mesh_raster_attr_fwd(None, None, d, 1, 1, 8, 8, e, k, m, dl, None, None, None, None, None) == -1
        assert msg in lib.b3d_last_error()
        assert lib.b3d_mesh_raster_attr_bwd(None, None, d, 1, 1, 8, 8, e, k, m, dl, None, None, None, None, None, None,
                                            None) == -1
        assert msg in lib.b3d_last_error()
    assert lib.b3d_mesh_face_pack(None, None, None, -1.0, 1, 1, None, None) == -1
    assert b"multiplier" in lib.b3d_last_error()
    for filt in (-1, 3):
        assert lib.b3d_mesh_render_filtered_fwd(None, None, None, None, 1, 1, 8, 8, 4, 4, filt, None, None, None, None,
                                                None) == -1
        assert b"unknown filter" in lib.b3d_last_error()
        assert lib.b3d_mesh_render_filtered_bwd(None, None, None, 0, 1, 1, 8, 8, 4, 4, filt, None, None, None, None,
                                                None, None, None, None) == -1
        assert b"unknown filter" in lib.b3d_last_error()
