"""The host side of the sample export (sample_export.py, rendering/mesh_template.py ObjWriter, b3d.data.sample_pack's
argument checks) against tests/golden/samples_reference.npz, which make_golden_samples.py recorded by executing the
`--save_results` block of the reference's main.py (CPU)."""
import gzip
import os
import sys

import numpy as np
import pytest
import torch
from PIL import Image

from conftest import GOLDEN

sys.path.insert(0, GOLDEN)
import samples_common as SC        # noqa: E402


@pytest.fixture(scope="module")
def golden():
    d = dict(np.load(os.path.join(GOLDEN, "samples_reference.npz")))
    d["obj"], d["mtl"], d["grid"] = SC.unpack_files(d)
    return d


def template(tmp_path, rings=16):
    from rendering.mesh_template import MeshTemplate
    path = os.path.join(str(tmp_path), f"uvsphere_{rings}rings.obj")
    with gzip.open(os.path.join(GOLDEN, f"uvsphere_{rings}rings.obj.gz"), "rb") as src, open(path, "wb") as dst:
        dst.write(src.read())
    return MeshTemplate(path, device="cpu")


def test_draws_equal_the_reference_draws(golden):
    from sample_export import sample_draws
    indices, classes, noise = sample_draws(SC.PoseSet(), SC.N, SC.LATENT, SC.SIGMA, True, seed=SC.SEED)
    assert np.array_equal(indices, golden["indices"])
    assert torch.equal(noise, torch.from_numpy(golden["noise"]))
    assert torch.equal(classes, torch.from_numpy(golden["classes"]))
    # the batches slice one draw of all N: 4 + 4 + 2 rows are the rows of the single draw
    parts = [noise[s] for s in (slice(0, 4), slice(4, 8), slice(8, 10))]
    assert [p.shape[0] for p in parts] == [4, 4, 2] and torch.equal(torch.cat(parts), torch.from_numpy(golden["noise"]))
    # an unconditional generator draws no classes and the same indices and noise
    i2, c2, n2 = sample_draws(SC.PoseSet(), SC.N, SC.LATENT, SC.SIGMA, False, seed=SC.SEED)
    assert c2 is None and np.array_equal(i2, indices) and torch.equal(n2, noise)
    assert float(noise.abs().max()) <= SC.SIGMA


def test_more_samples_than_the_dataset_raise():
    from sample_export import sample_draws
    with pytest.raises(ValueError):
        sample_draws(SC.PoseSet(n=5), 6, SC.LATENT, SC.SIGMA, False, seed=0)


def test_obj_writer_reproduces_the_reference_files(golden, tmp_path):
    from rendering.mesh_template import ObjWriter
    tpl = template(tmp_path)
    writer = ObjWriter(tpl.mesh)
    for i in range(SC.N):
        verts = golden["vertices"][i][:, [0, 2, 1]]              # main.py:870, Y and Z swapped
        writer.write(str(tmp_path / f"mesh_{i}"), np.ascontiguousarray(verts), golden["textures"][i])
        assert open(tmp_path / f"mesh_{i}.obj").read() == str(golden["obj"][i])
        assert open(tmp_path / f"mesh_{i}.mtl").read() == str(golden["mtl"][i])
        assert np.array_equal(np.asarray(Image.open(tmp_path / f"mesh_{i}.png")), golden["textures"][i])


def test_grid_assembly_reproduces_the_reference_grid(golden):
    from sample_export import assemble_grid, grid_shape
    g = golden["grid"]
    h = w = SC.RENDER // 2
    tiles = np.stack([g[(k // 8) * h:(k // 8 + 1) * h, (k % 8) * w:(k % 8 + 1) * w] for k in range(SC.N)])
    assert np.array_equal(assemble_grid(tiles), g)
    assert not g[h:, 2 * w:].any()                               # the cells after the last sample are 0
    assert grid_shape(16, h, w) == ((2 * h, 8 * w, 3), 8) and grid_shape(3, h, w) == ((h, 3 * w, 3), 3)
    assert grid_shape(17, h, w) == ((3 * h, 8 * w, 3), 8)


def test_export_obj_writes_the_png_its_mtl_names(golden, tmp_path):
    tpl = template(tmp_path)
    tex = torch.from_numpy(golden["pred_tex"][0]) / 2 + 0.5
    verts = torch.from_numpy(golden["vertices"][0][:, [0, 2, 1]].copy())
    tpl.export_obj(str(tmp_path / "mesh_0"), verts, tex)
    assert open(tmp_path / "mesh_0.obj").read() == str(golden["obj"][0])
    assert open(tmp_path / "mesh_0.mtl").read() == str(golden["mtl"][0])
    assert "map_Kd mesh_0.png" in str(golden["mtl"][0])
    assert np.array_equal(np.asarray(Image.open(tmp_path / "mesh_0.png")), golden["textures"][0])


def test_texture_only_generator_is_rejected():
    from sample_export import SampleExporter

    class TextureOnly(torch.nn.Module):
        mesh_head = False
    with pytest.raises(ValueError, match="mesh head"):
        SampleExporter(TextureOnly(), None, SC.PoseSet(), SC.SIGMA)


def test_sample_pack_validates_arguments_without_gpu():
    import b3d
    from b3d import lib
    from b3d.data import sample_pack
    B, H, W, T = 2, 8, 6, 4

    def args(**kw):
        a = dict(image=torch.zeros(B, H, W, 3), imidx=torch.zeros(B, H, W, dtype=torch.int32), tex=torch.zeros(B, 3, T, T),
                 tiles_out=torch.empty(B, H // 2, W // 2, 3, dtype=torch.uint8),
                 tex8_out=torch.empty(B, T, T, 3, dtype=torch.uint8))
        a.update(kw)
        return a
    with pytest.raises(b3d.B3DError, match="no CPU fallback"):
        sample_pack(**args())
    bad = {"odd height": args(image=torch.zeros(B, 7, W, 3), imidx=torch.zeros(B, 7, W, dtype=torch.int32)),
           "odd width": args(image=torch.zeros(B, H, 5, 3), imidx=torch.zeros(B, H, 5, dtype=torch.int32)),
           "image shape": args(image=torch.zeros(B, H, W, 4)),
           "tex shape": args(tex=torch.zeros(B, 3, T, T + 1)),
           "tiles shape": args(tiles_out=torch.empty(B, H, W, 3, dtype=torch.uint8)),
           "tex8 shape": args(tex8_out=torch.empty(B, T, T, 4, dtype=torch.uint8)),
           "image dtype": args(image=torch.zeros(B, H, W, 3, dtype=torch.float64)),
           "imidx dtype": args(imidx=torch.zeros(B, H, W, dtype=torch.int64)),
           "non-contiguous image": args(image=torch.zeros(B, W, H, 3).transpose(1, 2)),
           "non-contiguous tex": args(tex=torch.zeros(B, 3, T, T).transpose(2, 3))}
    for name, a in bad.items():
        with pytest.raises(b3d.B3DError) as e:
            sample_pack(**a)
        assert "no CPU fallback" not in str(e.value), name
    # the C entry checks sizes before any CUDA call
    assert lib.b3d_sample_pack(None, None, 2, 7, 6, None, 4, None, None, None) != 0
    assert b"even height and width" in lib.b3d_last_error()
    assert lib.b3d_sample_pack(None, None, 2, 8, 6, None, 0, None, None, None) != 0
    assert b"bad sizes" in lib.b3d_last_error()
    assert lib.b3d_version() >= 410
