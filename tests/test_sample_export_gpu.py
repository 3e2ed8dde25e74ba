"""The sample export on the GPU (sample_export.py, b3d_sample_pack):

1. b3d_sample_pack bit-exact against the torch composition of main.py:886-895 and export_obj's texture bytes, on the same
   GPU tensors: real renders of the 16- and 31-ring templates, empty and fully covered renders, values beyond +-1, on the
   quantisation boundaries, -0.0, and pool windows whose sum depends on the order of the additions;
2. the exporter against tests/golden/samples_reference.npz (the reference's --save_results block), through a stand-in
   generator that returns the golden's outputs for the golden's noise;
3. the files do not depend on the batch size;
4. the README's first command as library calls: a random-weight 512^2 generator saved in the shipped checkpoints' format,
   loaded with GANTrainer.load_checkpoint(path, 'evaluate') and exported at B 16 on a synthetic CUB-like cache, with one
   host synchronisation per batch and none per sample."""
import gzip
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from PIL import Image

from conftest import GOLDEN

sys.path.insert(0, GOLDEN)
import samples_common as SC                                   # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def template(tmp_dir, rings=16):
    from rendering.mesh_template import MeshTemplate
    path = os.path.join(str(tmp_dir), f"uvsphere_{rings}rings.obj")
    with gzip.open(os.path.join(GOLDEN, f"uvsphere_{rings}rings.obj.gz"), "rb") as src, open(path, "wb") as dst:
        dst.write(src.read())
    return MeshTemplate(path, is_symmetric=True, device=DEV)


def torch_composition(image, imidx, tex):
    """main.py:886-895 per tile (make_grid only places them) and export_obj's bytes of pred_tex / 2 + 0.5."""
    img = image.clone()
    alpha = (imidx > 0).to(img.dtype).unsqueeze(-1)              # Renderer(return_hardmask=True)
    img[alpha.expand_as(img) == 0] = 1
    img = F.avg_pool2d(img.permute(0, 3, 1, 2) / 2 + 0.5, 2)
    tiles = (img.permute(0, 2, 3, 1) * 255).clamp(0, 255).byte()
    tex8 = ((tex / 2 + 0.5).permute(0, 2, 3, 1) * 255).clamp(0, 255).byte()
    return tiles, tex8


def rendered(tpl, B, H, T, seed):
    from rendering.renderer import Renderer
    g = torch.Generator().manual_seed(seed)
    mm = (torch.randn(B, 3, 32, 32, generator=g) * 0.05).to(DEV)
    scale = (0.6 + 0.3 * torch.rand(B, 1, generator=g)).to(DEV)
    trans = torch.cat(((torch.rand(B, 2, generator=g) - 0.5) * 0.2, torch.zeros(B, 1)), 1).to(DEV)
    rot = F.normalize(torch.randn(B, 4, generator=g), dim=1).to(DEV)
    tex = (torch.rand(B, 3, T, T, generator=g) * 2.4 - 1.2).to(DEV)     # beyond +-1: the clamp acts
    r = Renderer(H, H)
    with torch.no_grad():
        image, _ = tpl.forward_renderer(r, tpl.vertices_and_pose(mm, scale, trans, rot)[1], tex)
    return image.contiguous(), r.last_face_index.contiguous(), tex


def edge_values(image, imidx, tex, seed):
    """Overwrite parts of a batch with the values where a different rounding or summation order shows."""
    g = torch.Generator().manual_seed(seed)
    B, H, W, _ = image.shape
    img, idx, t = image.clone(), imidx.clone(), tex.clone()
    k = torch.arange(256, dtype=torch.float32)
    bounds = 2 * (k / 255) - 1                                   # x / 2 + 0.5 lands on (or next to) a multiple of 1/255
    near = torch.cat([bounds, torch.nextafter(bounds, torch.tensor(2.0)), torch.nextafter(bounds, torch.tensor(-2.0))])
    specials = torch.cat([near, torch.tensor([-0.0, 0.0, 1.0, -1.0, 1.5, -1.5, 3e38, -3e38, 1e-30, -1e-30])])
    # four rows of texels: the boundary values; the rest of the row is left as it was
    flat = t[0].reshape(3, -1)
    n = min(specials.numel(), flat.shape[1])
    flat[:, :n] = specials[:n].to(DEV)
    # pool windows (covered) whose exact sum differs from the order ((((0 + a) + b) + c) + d)
    windows = torch.tensor([[1.0, -1 + 2e-8, -3.0, -1 + 2e-8], [1e-8, 1.0, 1e-8, -1.0], [-0.0, -0.0, -0.0, -0.0],
                            [0.9921875, 1e-7, 0.0078125, -1e-7], [-1 + 1e-7, 1.0, -1.0, 1 - 1e-7]])
    ys = torch.randint(0, H // 2, (64,), generator=g)
    xs = torch.randint(0, W // 2, (64,), generator=g)
    for j in range(64):
        b = j % B
        w = windows[j % len(windows)] if j < 40 else near[torch.randint(0, near.numel(), (4,), generator=g)]
        y, x = 2 * int(ys[j]), 2 * int(xs[j])
        for q, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
            img[b, y + dy, x + dx, :] = w[q]
            idx[b, y + dy, x + dx] = 1
    return img, idx, t


def check_pack(image, imidx, tex):
    from b3d.data import sample_pack
    B, H, W, _ = image.shape
    T = tex.shape[2]
    tiles = torch.full((B, H // 2, W // 2, 3), 7, dtype=torch.uint8, device=DEV)
    tex8 = torch.full((B, T, T, 3), 7, dtype=torch.uint8, device=DEV)
    sample_pack(image, imidx, tex, tiles, tex8)
    ref_tiles, ref_tex8 = torch_composition(image, imidx, tex)
    assert torch.equal(tiles, ref_tiles), int((tiles != ref_tiles).sum())
    assert torch.equal(tex8, ref_tex8), int((tex8 != ref_tex8).sum())
    return tiles


# ---------------------------------------------------------------------------------------------------- 1. the kernel
@pytest.mark.parametrize("B,H,T,rings", [(1, 512, 512, 16), (7, 512, 512, 31), (16, 512, 512, 16), (7, 64, 64, 31),
                                         (16, 64, 64, 16)])
def test_sample_pack_is_bit_exact_on_renders(tmp_path, B, H, T, rings):
    tpl = template(tmp_path, rings)
    image, imidx, tex = rendered(tpl, B, H, T, seed=B + H + rings)
    cov = float((imidx > 0).float().mean())
    assert 0.05 < cov < 0.95, cov
    check_pack(image, imidx, tex)
    check_pack(*edge_values(image, imidx, tex, seed=B))


@pytest.mark.parametrize("H", [512, 64])
def test_sample_pack_empty_and_fully_covered(H):
    g = torch.Generator().manual_seed(H)
    B, T = 3, 16
    image = (torch.randn(B, H, H, 3, generator=g) * 1.5).to(DEV)
    tex = (torch.randn(B, 3, T, T, generator=g) * 1.5).to(DEV)
    empty = torch.zeros(B, H, H, dtype=torch.int32, device=DEV)
    tiles = check_pack(image, empty, tex)
    assert bool((tiles == 255).all())                            # background: 1.0 -> 255
    full = torch.randint(1, 900, (B, H, H), generator=g, dtype=torch.int32).to(DEV)
    check_pack(image, full, tex)


# ---------------------------------------------------------------------------------------------------- 2. the golden
class GoldenGenerator(torch.nn.Module):
    """Returns the golden's generator outputs for the golden's noise rows, and fails on any other input."""
    mesh_head = True

    def __init__(self, d):
        super().__init__()
        self.anchor = torch.nn.Parameter(torch.zeros(1))
        self.args = types.SimpleNamespace(conditional_class=True)
        for k in ("noise", "classes", "pred_tex", "pred_mesh"):
            self.register_buffer(k, torch.from_numpy(d[k]))

    def forward(self, z, c=None, caption=None, return_attention=False):
        eq = (z[:, None, :] == self.noise[None]).all(-1)
        assert bool((eq.sum(1) == 1).all()), "the exporter passed noise the golden does not hold"
        k = eq.to(torch.int64).argmax(1)
        assert torch.equal(c, self.classes[k])
        return self.pred_tex[k], self.pred_mesh[k], None


def read_files(out_dir, n):
    objs = [open(os.path.join(out_dir, f"mesh_{i}.obj")).read() for i in range(n)]
    mtls = [open(os.path.join(out_dir, f"mesh_{i}.mtl")).read() for i in range(n)]
    pngs = [np.asarray(Image.open(os.path.join(out_dir, f"mesh_{i}.png"))) for i in range(n)]
    return objs, mtls, pngs


def test_exporter_reproduces_the_reference_export(tmp_path):
    from rendering.renderer import Renderer
    from sample_export import SampleExporter
    from oracle import mesh as M
    d = dict(np.load(os.path.join(GOLDEN, "samples_reference.npz")))
    d["obj"], d["mtl"], d["grid"] = SC.unpack_files(d)
    tpl = template(tmp_path)
    gen = GoldenGenerator(d).to(DEV)
    exp = SampleExporter(gen, tpl, SC.PoseSet(), SC.SIGMA, latent_dim=SC.LATENT)
    out_dir, grid_path = str(tmp_path / "results" / "golden"), str(tmp_path / "results" / "golden.png")
    res = exp.export(out_dir, grid_path, SC.N, 4, seed=SC.SEED, writers=3)
    assert np.array_equal(res["indices"], d["indices"])
    assert torch.equal(res["noise"], torch.from_numpy(d["noise"]))
    objs, mtls, pngs = read_files(out_dir, SC.N)
    for i in range(SC.N):
        ours, ref = objs[i].splitlines(), str(d["obj"][i]).splitlines()
        assert len(ours) == len(ref)
        assert [l for l in ours if not l.startswith("v ")] == [l for l in ref if not l.startswith("v ")]
        v_ours = np.array([[float(x) for x in l.split()[1:]] for l in ours if l.startswith("v ")])
        v_ref = np.array([[float(x) for x in l.split()[1:]] for l in ref if l.startswith("v ")])
        assert np.abs(v_ours - v_ref).max() <= 1e-5 + 1e-9
        assert mtls[i] == str(d["mtl"][i])
        assert np.array_equal(pngs[i], d["textures"][i])
    # the render of the reference's posed vertices: the same pixels covered by the same faces as the oracle's rasteriser
    # (the golden's render came from it)
    obj_path = os.path.join(str(tmp_path), "uvsphere_16rings.obj")
    T = M.TemplateData(M.load_obj(obj_path), obj_path)
    ref_index = M.forward_renderer(T, torch.from_numpy(d["posed"]), torch.from_numpy(d["pred_tex"]), SC.RENDER,
                                   SC.RENDER)[2].numpy()
    r = Renderer(SC.RENDER, SC.RENDER)
    with torch.no_grad():
        tpl.forward_renderer(r, torch.from_numpy(d["posed"]).to(DEV), gen.pred_tex)
    assert np.array_equal(r.last_face_index.cpu().numpy(), ref_index)
    # the exporter's own posed vertices (one fused launch) are a few fp32 ulps from the reference's qrot composition: a
    # pixel centre lying on a face edge may change sides; the grid is within 1 LSB in every tile those pixels leave alone
    ds = SC.PoseSet()
    sel = torch.as_tensor(d["indices"])
    with torch.no_grad():
        _, vtx = tpl.vertices_and_pose(gen.pred_mesh, ds.data['scale'][sel].to(DEV), ds.data['translation'][sel].to(DEV),
                                       ds.data['rotation'][sel].to(DEV))
        assert np.abs(vtx.cpu().numpy() - d["posed"]).max() < 1e-5
        tpl.forward_renderer(r, vtx, gen.pred_tex)
    flipped = np.argwhere(r.last_face_index.cpu().numpy() != ref_index)
    assert len(flipped) <= 8, len(flipped)
    grid = np.asarray(Image.open(grid_path))
    assert grid.shape == d["grid"].shape == (512, 2048, 3)
    ok = np.ones(grid.shape[:2], dtype=bool)
    for b, y, x in flipped:                                       # the grid cell of the tile pixel that pools it
        row, col = divmod(int(b), 8)
        ok[row * 256 + y // 2, col * 256 + x // 2] = False
    assert np.abs(grid.astype(np.int16) - d["grid"])[ok].max() <= 1
    assert ok.sum() >= ok.size - 8


# ---------------------------------------------------------------------------------------------------- 3. batch size
class RowwiseGenerator(torch.nn.Module):
    """Output of a sample from its own noise row only, elementwise (no reduction whose order could depend on B)."""
    mesh_head = True

    def __init__(self):
        super().__init__()
        self.anchor = torch.nn.Parameter(torch.zeros(1))
        yy, xx = torch.meshgrid(torch.linspace(-3, 3, 64), torch.linspace(-3, 3, 64), indexing="ij")
        self.register_buffer("pattern", torch.stack((torch.sin(xx), torch.cos(yy), torch.sin(xx + yy))))
        self.register_buffer("mesh_pattern", F.avg_pool2d(self.pattern[None], 2)[0])

    def forward(self, z, c=None, caption=None, return_attention=False):
        tex = torch.tanh(2 * z[:, :3, None, None] * self.pattern)
        mesh = 0.05 * z[:, 3:6, None, None] * self.mesh_pattern
        return tex, mesh, None


def test_files_do_not_depend_on_the_batch_size(tmp_path):
    from sample_export import SampleExporter
    tpl = template(tmp_path)
    exp = SampleExporter(RowwiseGenerator().to(DEV), tpl, SC.PoseSet(n=50), 2.0, latent_dim=8)
    got = []
    for B in (8, 16, 37):
        out = str(tmp_path / f"b{B}")
        exp.export(out, os.path.join(out, "grid.png"), 37, B, seed=11, writers=4)
        got.append(read_files(out, 37) + ([np.asarray(Image.open(os.path.join(out, "grid.png")))],))
    for other in got[1:]:
        assert other[0] == got[0][0] and other[1] == got[0][1]
        for a, b in zip(other[2] + other[3], got[0][2] + got[0][3]):
            assert np.array_equal(a, b)
    assert got[0][3][0].shape == (5 * 256, 8 * 256, 3)


# ---------------------------------------------------------------------------------------------------- 4. end to end
def write_cub_cache(root, n):
    from data.pseudo_gt import save_poses_metadata
    g = torch.Generator().manual_seed(3)
    paths = [f"{i:03d}.Bird/img_{i}.jpg" for i in range(n)]
    save_poses_metadata(os.path.join(root, "cache", "cub"), 0.6 + 0.3 * torch.rand(n, 1, generator=g),
                        torch.cat(((torch.rand(n, 2, generator=g) - 0.5) * 0.2, torch.zeros(n, 1)), 1),
                        F.normalize(torch.randn(n, 4, generator=g), dim=1), paths)
    labels = os.path.join(root, "datasets", "cub", "CUB_200_2011")
    os.makedirs(labels)
    with open(os.path.join(labels, "images.txt"), "w") as f:
        f.writelines(f"{i + 1} {p}\n" for i, p in enumerate(paths))
    with open(os.path.join(labels, "image_class_labels.txt"), "w") as f:
        f.writelines(f"{i + 1} {i % 200 + 1}\n" for i in range(n))


def test_readme_command_as_library_calls(tmp_path, monkeypatch):
    import bench
    from data.cub_200_2011_dataset import CubDataset
    from gan_training import GANTrainer
    from sample_export import SampleExporter
    root = str(tmp_path)
    write_cub_cache(root, 40)
    args = bench.gan_args(512, 3)
    args.dataset, args.evaluate = "cub", True
    ds = CubDataset(args, root=root)
    tpl = template(tmp_path)
    torch.manual_seed(0)
    tr = GANTrainer(args, mesh_template=tpl, device=DEV)
    saved = {k: v.clone() for k, v in tr.trainer.generator_running_avg.state_dict().items()}
    ckpt = str(tmp_path / "checkpoint_latest.pth")
    torch.save({"generator_running_avg": saved}, ckpt)               # the shipped checkpoints' layout
    torch.manual_seed(1)
    tr = GANTrainer(args, mesh_template=tpl, device=DEV)
    tr.load_checkpoint(ckpt, "evaluate")
    gen = tr.trainer.generator_running_avg
    assert all(torch.equal(v, saved[k]) for k, v in gen.state_dict().items())
    gen.train()

    counts = {"event": 0, "device": 0, "stream": 0}
    event_sync, device_sync, stream_sync = torch.cuda.Event.synchronize, torch.cuda.synchronize, torch.cuda.Stream.synchronize

    def counting(key, fn):
        def wrapped(*a, **k):
            counts[key] += 1
            return fn(*a, **k)
        return wrapped
    monkeypatch.setattr(torch.cuda.Event, "synchronize", counting("event", event_sync))
    monkeypatch.setattr(torch.cuda, "synchronize", counting("device", device_sync))
    monkeypatch.setattr(torch.cuda.Stream, "synchronize", counting("stream", stream_sync))
    exp = SampleExporter(gen, tpl, ds, ds.suggest_truncation_sigma(), latent_dim=args.latent_dim)
    out_dir, grid_path = str(tmp_path / "results" / "w"), str(tmp_path / "results" / "w.png")
    exp.export(out_dir, grid_path, 16, 16, seed=0, writers=8)
    monkeypatch.undo()
    assert counts == {"event": 1, "device": 0, "stream": 0}, counts          # one batch: one wait, for its copy
    assert not gen.training
    for i in range(16):
        for ext in ("obj", "mtl", "png"):
            assert os.path.getsize(os.path.join(out_dir, f"mesh_{i}.{ext}")) > 0
        tex = np.asarray(Image.open(os.path.join(out_dir, f"mesh_{i}.png")))
        assert tex.shape == (512, 512, 3) and tex.dtype == np.uint8
        assert open(os.path.join(out_dir, f"mesh_{i}.obj")).read().count("\nv ") == tpl.mesh.vertices.shape[0]
    grid = np.asarray(Image.open(grid_path))
    assert grid.shape == (512, 2048, 3) and grid.dtype == np.uint8
    assert 0 < float((grid != 255).any(-1).mean()) < 0.9         # the undeformed template covers part of each tile

    # two batches of 8: two waits, still none per sample
    counts.update(event=0, device=0, stream=0)
    monkeypatch.setattr(torch.cuda.Event, "synchronize", counting("event", event_sync))
    monkeypatch.setattr(torch.cuda, "synchronize", counting("device", device_sync))
    exp.export(str(tmp_path / "b8"), str(tmp_path / "b8.png"), 16, 8, seed=0, writers=8)
    monkeypatch.undo()
    assert counts["event"] == 2 and counts["device"] == 0, counts


def test_errors(tmp_path):
    import b3d
    from sample_export import SampleExporter
    tpl = template(tmp_path)
    with pytest.raises(b3d.B3DError, match="CUDA device"):
        SampleExporter(RowwiseGenerator(), tpl, SC.PoseSet(), 1.0, latent_dim=8)
    exp = SampleExporter(RowwiseGenerator().to(DEV), tpl, SC.PoseSet(n=5), 1.0, latent_dim=8)
    with pytest.raises(ValueError):
        exp.export(str(tmp_path / "o"), str(tmp_path / "g.png"), 6, 2, seed=0)
