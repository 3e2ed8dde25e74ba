"""The reconstruction export on the GPU (reconstruction_export.py, b3d_recon_texture_pack, cmr_data/photos.py,
reconstruct.py):

1. the texture pack against the torch composition visibility_to_mask / mirror_tex / F.interpolate, and at its edges;
2. the export agrees with the pseudo-ground-truth export on the same network and batch;
3. a known symmetric texture rendered at a known pose comes back from the export, and the exported model re-renders the
   photo;
4. the files do not depend on the batch size or the number of writer threads;
5. PhotoFolder gives the CMR dataset path's network input bit for bit;
6. a network on the CPU is refused; the README command writes every file."""
import gzip
import os
import shutil
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from PIL import Image

from conftest import GOLDEN

sys.path.insert(0, GOLDEN)
import recon_data_common as RD                                # noqa: E402
from test_pseudo_gt_export_gpu import cfg_batches, cfg_trainer, template   # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


# ---------------------------------------------------------------------------------------------------- 1. the kernel
def pack_inputs(B, Th, R, T, seed, vis_mode="random"):
    g = torch.Generator().manual_seed(seed)
    vis = torch.rand(B, Th, Th, generator=g) < 0.1
    vis[:, Th // 4:Th // 2, Th // 8:Th // 3] = True
    if vis_mode == "none":
        vis[:] = False
    alpha = (torch.rand(B, R, R, 1, generator=g) > 0.2).float()
    if vis_mode == "all":
        vis[:], alpha[:] = True, 1.0
    proj = torch.rand(B, R, R, 3, generator=g) * 2.4 - 1.2          # beyond [-1, 1]: the clamp
    pred = torch.rand(B, 3, T, T, generator=g) * 2.2 - 1.1
    return [t.to(DEV).contiguous() for t in (vis.to(torch.uint8), proj, alpha, pred)]


def mirror_batch(t):
    """data.pseudo_gt.mirror_tex over [B,R,R,C] (or [B,R,R])."""
    from data.pseudo_gt import mirror_tex
    if t.dim() == 3:
        return mirror_tex(t)
    B, R, _, C = t.shape
    return mirror_tex(t.permute(0, 3, 1, 2).reshape(B * C, R, R)).reshape(B, C, R, R).permute(0, 2, 3, 1)


def reference_pack(vis, proj, alpha, pred, symmetric):
    from data.pseudo_gt import visibility_to_mask
    B, R = proj.shape[0], proj.shape[1]
    mask = visibility_to_mask(vis.float().unsqueeze(1).expand(-1, 3, -1, -1).contiguous(), R)
    valid = (mask[..., 0] > 0) & (alpha[..., 0] > 0)
    tex = F.interpolate(pred, size=(R, R), mode='bilinear', align_corners=False).permute(0, 2, 3, 1)
    src = torch.zeros(B, R, R, dtype=torch.uint8, device=DEV)
    if symmetric:
        mvalid = mirror_batch(valid)
        tex = torch.where(mvalid.unsqueeze(-1), mirror_batch(proj), tex)
        src = torch.where(mvalid, torch.full_like(src, 2), src)
    tex = torch.where(valid.unsqueeze(-1), proj, tex)
    src = torch.where(valid, torch.ones_like(src), src)
    return ((tex / 2 + 0.5) * 255).clamp(0, 255).byte(), src


def run_pack(vis, proj, alpha, pred, symmetric):
    from b3d.data import recon_texture_pack
    B, R = proj.shape[0], proj.shape[1]
    tex8 = torch.empty(B, R, R, 3, dtype=torch.uint8, device=DEV)
    src8 = torch.empty(B, R, R, dtype=torch.uint8, device=DEV)
    recon_texture_pack(vis, proj, alpha, pred, symmetric, tex8, src8)
    return tex8, src8


@pytest.mark.parametrize("symmetric", [True, False], ids=["symmetric", "asymmetric"])
@pytest.mark.parametrize("R,T", [(512, 128), (256, 64)])
def test_pack_matches_the_torch_composition(R, T, symmetric):
    vis, proj, alpha, pred = pack_inputs(3, T, R, T, seed=R + T + symmetric)
    tex8, src8 = run_pack(vis, proj, alpha, pred, symmetric)
    ref8, ref_src = reference_pack(vis, proj, alpha, pred, symmetric)
    assert torch.equal(src8, ref_src), int((src8 != ref_src).sum())
    counts = [int((ref_src == k).sum()) for k in range(3)]
    assert counts[0] > 0 and counts[1] > 0 and (counts[2] > 0) == symmetric, counts
    projected = (ref_src > 0).unsqueeze(-1).expand_as(tex8)
    assert torch.equal(tex8[projected], ref8[projected])
    diff = (tex8.int() - ref8.int()).abs()
    print(f"R {R} T {T} symmetric {symmetric}: {int((diff > 0).sum())} of {diff[~projected].numel()} predicted "
          f"texel channels differ by 1 LSB")
    assert int(diff.max()) <= 1


@pytest.mark.parametrize("mode", ["none", "all"])
def test_pack_with_nothing_or_everything_visible(mode):
    vis, proj, alpha, pred = pack_inputs(2, 64, 256, 64, seed=7, vis_mode=mode)
    tex8, src8 = run_pack(vis, proj, alpha, pred, True)
    ref8, ref_src = reference_pack(vis, proj, alpha, pred, True)
    assert torch.equal(src8, ref_src)
    assert bool((src8 == (0 if mode == "none" else 1)).all())
    if mode == "all":
        assert torch.equal(tex8, ref8)
    else:
        assert int((tex8.int() - ref8.int()).abs().max()) <= 1


def test_pack_single_sample_equals_its_row_of_a_batch():
    vis, proj, alpha, pred = pack_inputs(4, 64, 256, 64, seed=3)
    tex8, src8 = run_pack(vis, proj, alpha, pred, True)
    one8, one_src = run_pack(vis[2:3], proj[2:3], alpha[2:3], pred[2:3], True)
    assert torch.equal(one8, tex8[2:3]) and torch.equal(one_src, src8[2:3])


def test_pack_rejects_bad_arguments():
    import b3d
    from b3d import lib, ptr
    from b3d.data import recon_texture_pack
    vis, proj, alpha, pred = pack_inputs(2, 32, 64, 32, seed=1)
    tex8 = torch.empty(2, 64, 64, 3, dtype=torch.uint8, device=DEV)
    src8 = torch.empty(2, 64, 64, dtype=torch.uint8, device=DEV)
    bad = [(vis.float(), proj, alpha, pred, tex8, src8), (vis, proj.double(), alpha, pred, tex8, src8),
           (vis, proj[:1].contiguous(), alpha, pred, tex8, src8), (vis, proj, alpha, pred.cpu(), tex8, src8),
           (vis, proj, alpha, pred, tex8[..., :2], src8), (vis, proj, alpha, pred, tex8, src8[:1])]
    for v, p, a, t, o8, os8 in bad:
        with pytest.raises(b3d.B3DError):
            recon_texture_pack(v, p, a, t, True, o8, os8)
    odd = pack_inputs(1, 32, 63, 32, seed=2)
    with pytest.raises(b3d.B3DError, match="odd"):
        recon_texture_pack(*odd, True, torch.empty(1, 63, 63, 3, dtype=torch.uint8, device=DEV),
                           torch.empty(1, 63, 63, dtype=torch.uint8, device=DEV))
    # the C entry point checks the same before any launch
    rc = lib.b3d_recon_texture_pack(ptr(vis), 32, 32, ptr(proj), ptr(alpha), 2, 63, ptr(pred), 32, 1, ptr(tex8),
                                    ptr(src8), None)
    assert rc != 0 and b"odd" in lib.b3d_last_error()
    host = torch.empty(2, 64, 64, dtype=torch.uint8)
    rc = lib.b3d_recon_texture_pack(ptr(vis), 32, 32, ptr(proj), ptr(alpha), 2, 64, ptr(pred), 32, 1, ptr(tex8),
                                    ptr(host), None)
    assert rc != 0 and b"not device memory" in lib.b3d_last_error()


# ---------------------------------------------------------------------------------------------------- 2. cross path
def staged_batch(exp, batch, posed=True, per_index=True):
    """The staged bytes of one batch, as the export's drain sees them."""
    from staging import Staging, views
    exp._staging = Staging(exp.device, 'test')
    lay, nbytes = exp._device_batch(batch, posed, per_index)
    return {k: t.cpu() for k, t in views(exp._staging.buffer, lay).items()}


def obj_vertices(path):
    with open(path) as fh:
        return [line for line in fh if line.startswith('v ')]


def test_export_agrees_with_the_pseudo_gt_export(tmp_path):
    from fid_common import randomize_inception
    from pseudo_gt_export import PseudoGTExporter
    from reconstruction_export import ReconstructionExporter
    from utils.inception import InceptionV3
    tpl = template(tmp_path)
    B, R = 6, 512
    tr = cfg_trainer(tpl, B)
    batch = cfg_batches(1, B, seed=11)[0]
    X, img299, hd, scale, trans, rot, ind = batch
    cache = str(tmp_path / "cache")
    PseudoGTExporter(tr, tpl, R, inception=randomize_inception(InceptionV3([0], weights=None), 1)).export(
        [batch], [f"img{i}" for i in range(B)], cache, 'cub', writers=2)
    exp = ReconstructionExporter(tr, tpl, R)
    rbatch = (X, hd, scale, trans, rot, ind)
    names = [f"img{i}" for i in range(B)]
    out = exp.export([rbatch], names, str(tmp_path / "out"), posed=True, writers=2, per_index=True)
    staged = staged_batch(exp, rbatch)
    with torch.no_grad():
        _, mesh_map = tr.generator(X)
        td, sd = tr.dataset_params(ind, 'deltas')
        raw = tpl.vertices_and_pose(mesh_map, scale + sd, trans + td, rot)[0]
    assert out['names'] == names
    for i in range(B):
        rec = np.load(os.path.join(cache, f"pseudogt_{R}x{R}", f"{i}.npz"), allow_pickle=True)['data'].item()
        seen = rec['texture_alpha'][0] > 0
        assert torch.equal(staged['src8'][i] == 1, seen), i
        assert int(out['sources'][i, 1]) == int(seen.sum()) > 0
        assert int(out['sources'][i].sum()) == R * R
        ref = raw[i][..., [0, 2, 1]].cpu()
        assert torch.equal(staged['vertices'][i], ref)
        lines = ['v {:.5f} {:.5f} {:.5f}\n'.format(*p) for p in ref.tolist()]
        assert obj_vertices(str(tmp_path / "out" / f"img{i}.obj")) == lines


# ---------------------------------------------------------------------------------------------------- 3. orientation
class FixedNet(torch.nn.Module):
    """Stands in for the reconstruction network: a fixed displacement map and a flat grey texture for every input."""

    def __init__(self, mesh_map, T):
        super().__init__()
        self.anchor = torch.nn.Parameter(torch.zeros(1))
        self.mesh_map, self.T = mesh_map, T

    def forward(self, X):
        B = X.shape[0]
        return (torch.zeros(B, 3, self.T, self.T, device=X.device),
                self.mesh_map.expand(B, -1, -1, -1).contiguous())


def symmetric_texture(R):
    """A smooth texture with K(y, x) = K(y, mx), mx = R-1-((x + R/2) mod R): the template's mirror image of itself."""
    x = torch.arange(R, dtype=torch.float64)
    mx = R - 1 - (x + R // 2) % R
    y = torch.arange(R, dtype=torch.float64)[:, None]
    h = lambda u, k, p: torch.cos(2 * np.pi * k * (u + 0.5) / R + p)          # noqa: E731
    chans = [0.4 * (h(x, 1, 0.3) + h(mx, 1, 0.3)) * torch.cos(np.pi * y / R) + 0.1,
             0.3 * (h(x, 2, 1.1) + h(mx, 2, 1.1)) + 0.3 * torch.cos(2 * np.pi * y / R),
             0.4 * (h(x, 3, 2.0) + h(mx, 3, 2.0)) + 0.2 * torch.sin(np.pi * y / R)]
    return torch.stack([c.expand(R, R) for c in chans]).float().clamp(-0.95, 0.95).unsqueeze(0)


def test_known_texture_and_pose_round_trip(tmp_path):
    from oracle import mesh as OM
    from reconstruction_export import ReconstructionExporter
    from rendering.renderer import Renderer
    tpl = template(tmp_path)
    R = 256
    H = 1024
    K = symmetric_texture(R).to(DEV)
    g = torch.Generator().manual_seed(5)
    mesh_map = (torch.randn(1, 3, 32, 32, generator=g) * 0.02).to(DEV)
    scale = torch.tensor([[0.8]], device=DEV)
    trans = torch.tensor([[0.05, -0.03, 0.0]], device=DEV)
    rot = F.normalize(torch.tensor([[0.9, 0.2, 0.35, 0.1]]), dim=1).to(DEV)
    with torch.no_grad():
        raw, vtx = tpl.vertices_and_pose(mesh_map, scale, trans, rot)
        image, alpha = tpl.forward_renderer(Renderer(H, H), vtx, K)
    photo = (image * alpha).permute(0, 3, 1, 2).contiguous()
    X = torch.zeros(1, 4, 256, 256, device=DEV)
    trainer = types.SimpleNamespace(generator=FixedNet(mesh_map, 64).to(DEV), dataset_params=None,
                                    args=types.SimpleNamespace(optimize_deltas=False, optimize_z0=False))
    exp = ReconstructionExporter(trainer, tpl, R)
    batch = (X, photo, scale, trans, rot, torch.zeros(1, dtype=torch.int64, device=DEV))
    out_dir = str(tmp_path / "out")
    exp.export([batch], ["known"], out_dir, posed=True, writers=1)
    staged = staged_batch(exp, batch, per_index=False)
    src = staged['src8'][0]
    tex8 = np.array(Image.open(os.path.join(out_dir, "known.png")))
    assert np.array_equal(tex8, staged['tex8'][0].numpy())
    truth = ((K[0].permute(1, 2, 0) / 2 + 0.5) * 255).clamp(0, 255).byte().cpu().numpy().astype(int)
    err = np.abs(tex8.astype(int) - truth).max(axis=-1)
    stats = {}
    for k in (1, 2):
        e = err[(src == k).numpy()]
        stats[k] = (e.size, np.median(e), e.mean())
        print(f"source {k}: {e.size} texels, median {np.median(e)}, mean {e.mean():.2f}, 95th {np.percentile(e, 95)}")
    for k, (size, median, mean) in stats.items():
        # a smooth texture re-sampled twice (render, projection) is a level or two off, more where the surface is seen
        # edge-on (H100: source 1 median 1, mean 5.2); a wrong orientation costs ~100 levels
        assert size > 0.05 * R * R and median <= 4 and mean <= 12, (k, size, median, mean)

    # the exported model, read back from its files, re-renders the photo
    raw_obj = torch.tensor([[float(c) for c in line.split()[1:]] for line in
                            obj_vertices(os.path.join(out_dir, "known.obj"))])[:, [0, 2, 1]].unsqueeze(0)
    assert float((raw_obj - raw[0].cpu()).abs().max()) <= 1e-5
    vtx2 = OM.transform_vertices(raw_obj, scale.cpu(), trans.cpu(), rot.cpu()).to(DEV)
    tex = torch.from_numpy(tex8).to(DEV).permute(2, 0, 1).unsqueeze(0).float() / 127.5 - 1
    with torch.no_grad():
        image2, alpha2 = tpl.forward_renderer(Renderer(H, H), vtx2.contiguous(), tex)
    inside = (F.max_pool2d(1 - alpha.permute(0, 3, 1, 2), 5, 1, 2) == 0)[0, 0]      # the mask, eroded by 2 pixels
    d = (image2 - image)[0][inside].abs().max(dim=-1).values.cpu().numpy()
    print(f"re-render: {d.size} pixels, median {np.median(d):.4f}, mean {d.mean():.4f}, 99th {np.percentile(d, 99):.4f}")
    assert d.size > 0.05 * H * H
    assert np.median(d) <= 0.05 and d.mean() <= 0.1


# ---------------------------------------------------------------------------------------------------- 4. batching
def test_files_do_not_depend_on_batch_size_or_writers(tmp_path):
    from reconstruction_export import ReconstructionExporter
    tpl = template(tmp_path)
    n = 8
    tr = cfg_trainer(tpl, n, seed=2)
    X, _, hd, scale, trans, rot, ind = cfg_batches(1, n, seed=6)[0]
    names = [f"im{i}" for i in range(n)]
    exp = ReconstructionExporter(tr, tpl, 512)

    def split(B):
        return [(X[a:a + B], hd[a:a + B], scale[a:a + B], trans[a:a + B], rot[a:a + B], ind[a:a + B])
                for a in range(0, n, B)]

    runs = {}
    for key, B, writers in (("b8w8", 8, 8), ("b3w8", 3, 8), ("b8w1", 8, 1)):
        d = str(tmp_path / key)
        out = exp.export(split(B), names, d, posed=True, writers=writers, per_index=True)
        assert out['names'] == names
        runs[key] = (d, out['sources'])
    files = sorted(os.listdir(runs["b8w8"][0]))
    assert len(files) == 4 * n
    for key in ("b3w8", "b8w1"):
        assert sorted(os.listdir(runs[key][0])) == files
        assert np.array_equal(runs[key][1], runs["b8w8"][1])
        for f in files:
            with open(os.path.join(runs[key][0], f), 'rb') as a, open(os.path.join(runs["b8w8"][0], f), 'rb') as b:
                assert a.read() == b.read(), (key, f)


# ---------------------------------------------------------------------------------------------------- 5. photos
def tight_box_tree(root):
    """The synthetic CUB tree with every annotated box replaced by the tight box of its mask (1-based)."""
    inp = RD.make_inputs(0)
    for i in range(int(inp['cub_n'])):
        ys, xs = np.nonzero(inp[f'cub_mask{i}'])
        inp[f'cub_bbox{i}'] = np.array([xs.min(), ys.min(), xs.max(), ys.max()]) + 1
    RD.write_tree(root, inp)
    return inp


def test_photo_folder_gives_the_dataset_input(tmp_path):
    from cmr_data.cub import CUBDataset
    from cmr_data.photos import PhotoFolder
    root = str(tmp_path)
    inp = tight_box_tree(root)
    n = int(inp['cub_n'])
    photos = tmp_path / "photos"
    photos.mkdir()
    for i in range(n):
        photo, mask = inp[f'cub_photo{i}'], inp[f'cub_mask{i}']
        if i == 2 and photo.ndim == 3:                   # one RGBA photo, the others with a mask file
            Image.fromarray(np.dstack([photo, mask * 255]).astype(np.uint8), 'RGBA').save(photos / f"p{i}.png")
        else:
            Image.fromarray(photo, 'L' if photo.ndim == 2 else 'RGB').save(photos / f"p{i}.png")
            Image.fromarray(mask * 255).save(photos / f"p{i}_mask.png")
    ds = CUBDataset('train', False, 256, root=root).to_device(DEV)
    pf = PhotoFolder(str(photos), 256).to_device(DEV)
    assert pf.names == [f"p{i}" for i in range(n)]
    for a, b in zip(ds.eval_batches(3), pf.eval_batches(3)):
        assert torch.equal(a[0].view(torch.int32), b[0].view(torch.int32))
        assert bool(torch.isnan(b[1]).all()) and torch.equal(a[-1], b[-1])


def test_a_network_on_the_cpu_is_refused(tmp_path):
    import b3d
    from reconstruction_export import ReconstructionExporter
    tpl = template(tmp_path)
    trainer = types.SimpleNamespace(generator=torch.nn.Linear(2, 2), dataset_params=None,
                                    args=types.SimpleNamespace(optimize_deltas=False, optimize_z0=False))
    with pytest.raises(b3d.B3DError, match="move it to a CUDA device"):
        ReconstructionExporter(trainer, tpl)


# ---------------------------------------------------------------------------------------------------- 6. the command
def test_the_readme_command_writes_every_file(tmp_path, monkeypatch):
    import reconstruct
    from reconstruction_training import ReconTrainer, default_args
    from rendering.mesh_template import MeshTemplate
    root = str(tmp_path)
    inp = tight_box_tree(root)
    n = int(inp['cub_n'])
    os.makedirs(os.path.join(root, 'mesh_templates'))
    mesh = os.path.join(root, 'mesh_templates', 'uvsphere_16rings.obj')
    with gzip.open(os.path.join(GOLDEN, "uvsphere_16rings.obj.gz"), "rb") as src, open(mesh, "wb") as dst:
        shutil.copyfileobj(src, dst)
    torch.manual_seed(3)
    tr = ReconTrainer(default_args(), MeshTemplate(mesh, device=DEV), n, device=DEV)
    with torch.no_grad():
        tr.dataset_params.ds_translation.normal_(0, 0.02)
    os.makedirs(os.path.join(root, 'checkpoints_recon', 'birds'))
    tr.save_checkpoint(os.path.join(root, 'checkpoints_recon', 'birds', 'checkpoint_latest.pth'))
    photos = tmp_path / "photos"
    photos.mkdir()
    for i in range(3):
        photo, mask = inp[f'cub_photo{i}'], inp[f'cub_mask{i}']
        Image.fromarray(np.dstack([photo, mask * 255]).astype(np.uint8), 'RGBA').save(photos / f"bird{i}.png")
    monkeypatch.chdir(root)

    out = reconstruct.main(['--name', 'birds', '--dataset', 'cub', '--split', 'train', '--batch_size', '3'])
    from cmr_data.cub import CUBDataset
    expect = [reconstruct.output_name(p) for p in CUBDataset('train', False, 32, root=root).get_paths()]
    assert out['names'] == expect and out['sources'].shape == (n, 3)
    assert int(out['sources'][:, 1].sum()) > 0
    files = set(os.listdir(os.path.join('results_recon', 'birds')))
    assert files == {f"{m}{ext}" for m in expect for ext in ('.obj', '.mtl', '.png', '_views.png')}
    sheet = np.asarray(Image.open(os.path.join('results_recon', 'birds', f"{expect[0]}_views.png")))
    assert sheet.shape == (512, 1280, 3)

    out = reconstruct.main(['--name', 'birds', '--dataset', 'cub', '--photos', str(photos), '--output', 'mine',
                            '--export_resolution', '256', '--indices', '2', '0'])
    assert out['names'] == ['bird2', 'bird0'] and bool((out['sources'][:, 1:] == 0).all())
    assert set(os.listdir('mine')) == {f"bird{i}{ext}" for i in (0, 2) for ext in ('.obj', '.mtl', '.png', '_views.png')}
    sheet = np.asarray(Image.open(os.path.join('mine', "bird0_views.png")))
    assert (sheet[256:, :256] == 255).all()                   # no pose: no render at the input pose
