"""The pseudo-ground-truth export on the GPU (pseudo_gt_export.py, b3d_texel_visibility, b3d_pseudogt_pack):

1. texel visibility bit-exact against d(render)/d(texture) > 0 (autograd through the CUDA renderer, or the adjoint kernel on
   hand-made index buffers): toy scene, full size, the non-symmetric seam, texel-centre UVs, u / v at 0 and 1, empty render;
2. the record packing: mask bit-exact against visibility_to_mask at R 16 / 64 / 512 / 300, fp16 planes bit-exact against
   .half() of the existing composition, bad arguments rejected on the host;
3. the exporter reproduces tests/golden/pseudogt_reference.npz (the reference's export loop);
4. full-size records bit-exact against texel_visibility -> visibility_to_mask -> InverseRenderer -> make_record;
5. a whole synthetic CUB / P3D set: one file per image, poses metadata, real-image statistics, and a GAN step on the cache;
6. the staging buffers are allocated once per export."""
import gzip
import os
import sys
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN

sys.path.insert(0, GOLDEN)
import pseudogt_common as PC                                  # noqa: E402
import recon_data_common as RD                                # noqa: E402
from fid_common import randomize_inception                    # noqa: E402
from test_recon_dataset_hostlogic import make                 # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def template(tmp_dir, symmetric=True, rings=16):
    from rendering.mesh_template import MeshTemplate
    path = os.path.join(str(tmp_dir), f"uvsphere_{rings}rings.obj")
    with gzip.open(os.path.join(GOLDEN, f"uvsphere_{rings}rings.obj.gz"), "rb") as src, open(path, "wb") as dst:
        dst.write(src.read())
    return MeshTemplate(path, is_symmetric=symmetric, device=DEV)


def scene(tpl, B, tex_res, seed):
    """Posed vertices of a randomly deformed template and a texture, as the reconstruction network would give them."""
    g = torch.Generator().manual_seed(seed)
    mm = (torch.randn(B, 3, 32, 32, generator=g) * 0.05).to(DEV)
    scale = (0.6 + 0.3 * torch.rand(B, 1, generator=g)).to(DEV)
    trans = torch.cat(((torch.rand(B, 2, generator=g) - 0.5) * 0.2, torch.zeros(B, 1)), 1).to(DEV)
    rot = torch.nn.functional.normalize(torch.randn(B, 4, generator=g), dim=1).to(DEV)
    tex = (torch.rand(B, 3, tex_res, tex_res, generator=g) * 2 - 1).to(DEV)
    return tpl.vertices_and_pose(mm, scale, trans, rot)[1], tex


def kernel_visibility(tpl, vtx, tex, H):
    from b3d.mesh import render_indices, texel_visibility
    uvs, padded = tpl.adjust_uv_and_texture(tex)
    imidx, imwei, fuv = render_indices(vtx, tpl.mesh.faces, uvs, tpl.mesh.face_textures, H, H)
    return texel_visibility(imidx, imwei, fuv, padded.shape[2], padded.shape[3], tpl.is_symmetric)


def autograd_visibility(tpl, vtx, tex, H):
    from rendering.inverse_renderer import texel_visibility
    from rendering.renderer import Renderer
    vis, _, _ = texel_visibility(tpl, Renderer(H, H), vtx, tex)
    return (vis > 0).any(dim=1).to(torch.uint8)


# ---------------------------------------------------------------------------------------------------- 1. visibility
@pytest.mark.parametrize("B,H,tex_res,symmetric", [(2, 64, 16, True), (10, 1024, 128, True), (3, 256, 32, False)],
                         ids=["toy", "full_size", "non_symmetric"])
def test_visibility_matches_the_texture_gradient(tmp_path, B, H, tex_res, symmetric):
    tpl = template(tmp_path, symmetric)
    vtx, tex = scene(tpl, B, tex_res, seed=B + H)
    ours = kernel_visibility(tpl, vtx, tex, H)
    ref = autograd_visibility(tpl, vtx, tex, H)
    assert ours.shape == ref.shape == (B, tex_res, tex_res) and ours.dtype == torch.uint8
    assert 0 < int(ref.sum()) < ref.numel()
    assert torch.equal(ours, ref), int((ours != ref).sum())


def adjoint_visibility(imidx, imwei, fuv, Th, Tw, symmetric):
    """dtex of b3d_mesh_render_bwd under d_imout = 1, summed back through the seam padding, > 0."""
    from b3d import check, lib, ptr, stream_ptr
    B, H, W = imidx.shape
    F = fuv.shape[1]
    # every face covers the whole image, so every tile bins every face the index buffer names
    fgeo = torch.tensor([-5000., -5000., 5000., -5000., 0., 5000., 0., 0., 0., 1., 0., 0.], device=DEV).repeat(B, F, 1)
    tex = torch.zeros(B, 3, Th, Tw, device=DEV)
    dtex, dfp, dfuv = torch.empty_like(tex), torch.empty(B, F, 6, device=DEV), torch.empty(B, F, 6, device=DEV)
    ones = torch.ones(B, H, W, 3, device=DEV)
    check(lib.b3d_mesh_render_bwd(ptr(fgeo), ptr(fuv), ptr(tex), 0, B, F, H, W, Th, Tw, ptr(imidx), ptr(imwei), ptr(ones),
                                  None, ptr(dfp), ptr(dfuv), ptr(dtex), stream_ptr(fgeo)))
    if symmetric:
        src = dtex[..., 1:-1].clone()
        src[..., -1] += dtex[..., 0]
        src[..., 0] += dtex[..., -1]
    else:
        src = dtex[..., :-1].clone()
        src[..., 0] += dtex[..., -1]
    return (src > 0).any(dim=1).to(torch.uint8)


def edge_buffers(Th, Tw, seed, empty=False):
    """Index buffers whose pixels sample exactly on texel centres (zero-weight taps), at u / v = 0 and 1 (the seam columns
    and the last row), and at random points."""
    g = torch.Generator().manual_seed(seed)
    B, H, W, F = 2, 48, 40, 96
    corners = []
    for f in range(F):
        if f < 64:                       # one point per face, on a texel centre or the borders
            k = [0, Tw - 1, 1, Tw - 2][f % 4] if f < 16 else int(torch.randint(0, Tw, (1,), generator=g))
            j = [0, Th - 1][f % 2] if f < 32 else int(torch.randint(0, Th, (1,), generator=g))
            u = torch.tensor(k / (Tw - 1), dtype=torch.float32)
            v = 1 - torch.tensor(j / (Th - 1), dtype=torch.float32)
            corners.append(torch.stack((u, v)).repeat(3))
        else:
            corners.append(torch.rand(6, generator=g))
    fuv = torch.stack(corners).unsqueeze(0).repeat(B, 1, 1).to(DEV).contiguous()
    imidx = torch.randint(0, F + 1, (B, H, W), generator=g, dtype=torch.int32)
    if empty:
        imidx.zero_()
    w = torch.rand(B, H, W, 3, generator=g)
    w = w / w.sum(-1, keepdim=True)
    pinned = imidx.long() - 1 < 64                 # texel-centre faces: all weight on the first corner, u = corner u exactly
    w[pinned] = torch.tensor([1.0, 0.0, 0.0])
    return imidx.to(DEV), w.to(DEV).contiguous(), fuv


@pytest.mark.parametrize("symmetric", [True, False])
@pytest.mark.parametrize("empty", [False, True], ids=["edges", "empty"])
def test_visibility_at_texel_centres_seams_and_empty(symmetric, empty):
    from b3d.mesh import texel_visibility
    Th, Tw_out = 16, 16
    Tw = Tw_out + (2 if symmetric else 1)
    imidx, imwei, fuv = edge_buffers(Th, Tw, seed=5 + symmetric, empty=empty)
    ours = texel_visibility(imidx, imwei, fuv, Th, Tw, symmetric)
    ref = adjoint_visibility(imidx, imwei, fuv, Th, Tw, symmetric)
    assert ours.shape == (2, Th, Tw_out)
    assert torch.equal(ours, ref), int((ours != ref).sum())
    if empty:
        assert int(ours.sum()) == 0
    else:
        assert int(ref.sum()) > 0


def test_visibility_rejects_bad_arguments():
    import b3d
    from b3d.mesh import texel_visibility
    imidx, imwei, fuv = edge_buffers(16, 18, seed=1)
    with pytest.raises(b3d.B3DError):
        texel_visibility(imidx.float(), imwei, fuv, 16, 18, True)
    with pytest.raises(b3d.B3DError):
        texel_visibility(imidx, imwei[..., :2].contiguous(), fuv, 16, 18, True)
    with pytest.raises(b3d.B3DError):
        texel_visibility(imidx, imwei, fuv, 16, 2, True)
    with pytest.raises(b3d.B3DError, match="no CPU fallback"):
        texel_visibility(imidx.cpu(), imwei, fuv, 16, 18, True)
    with pytest.raises(b3d.B3DError):
        texel_visibility(imidx, imwei, fuv, 16, 18, True, out=torch.empty(1, 16, 16, dtype=torch.uint8, device=DEV))


# ---------------------------------------------------------------------------------------------------- 2. packing
def pack_inputs(B, Th, R, C, seed, img=(3, 20, 24)):
    g = torch.Generator().manual_seed(seed)
    vis = (torch.rand(B, Th, Th, generator=g) < 0.05)
    vis[:, Th // 4:Th // 2, Th // 3:Th // 2] = True
    vis[:, :, 0] |= torch.rand(B, Th, generator=g) < 0.5            # first / last row and column
    vis[:, -1, :] |= torch.rand(B, Th, generator=g) < 0.5
    tex = torch.rand(B, R, R, C, generator=g) * 2 - 1
    tex[0, 0, 0, 0] = 70000.0                                        # beyond fp16: inf, as .half() rounds it
    alpha = (torch.rand(B, R, R, 1, generator=g) > 0.3).float()
    image = torch.randn(B, *img, generator=g)
    return [t.to(DEV).contiguous() for t in (vis.to(torch.uint8), tex, alpha, image)]


def fp16_outputs(B, C, R, img):
    return (torch.empty(B, C, R, R, dtype=torch.float16, device=DEV), torch.empty(B, 1, R, R, dtype=torch.float16, device=DEV),
            torch.empty(B, *img, dtype=torch.float16, device=DEV))


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int16), b.view(torch.int16))


@pytest.mark.parametrize("R", [16, 64, 512, 300])
def test_pack_matches_the_reference_composition(R):
    from b3d.data import pseudogt_pack
    from data.pseudo_gt import visibility_to_mask
    B, Th, C = 3, 128, 4
    vis, tex, alpha, image = pack_inputs(B, Th, R, C, seed=R)
    mask = visibility_to_mask(vis.float().unsqueeze(1).expand(-1, 3, -1, -1).contiguous(), R)
    # the mask alone: with an all-ones alpha the packed alpha is the mask
    outs = fp16_outputs(B, C, R, image.shape[1:])
    pseudogt_pack(vis, tex, torch.ones_like(alpha), image, *outs)
    assert torch.equal(outs[1].float(), mask.permute(0, 3, 1, 2)), int((outs[1].float() != mask.permute(0, 3, 1, 2)).sum())
    assert 0 < float(mask.mean()) < 1
    # the planes: bit for bit what the reference's masking, permute and .half() give (including -0.0 and inf)
    pseudogt_pack(vis, tex, alpha, image, *outs)
    assert same_bits(outs[0], (tex * mask).permute(0, 3, 1, 2).half())
    assert same_bits(outs[1], (alpha * mask).permute(0, 3, 1, 2).half())
    assert same_bits(outs[2], image.half())


def test_pack_rejects_bad_arguments():
    import b3d
    from b3d import lib, ptr
    from b3d.data import pseudogt_pack
    vis, tex, alpha, image = pack_inputs(2, 32, 16, 3, seed=0)
    outs = fp16_outputs(2, 3, 16, image.shape[1:])
    bad = [((vis.float(), tex, alpha, image), outs), ((vis, tex.double(), alpha, image), outs),
           ((vis, tex[:1].contiguous(), alpha, image), outs), ((vis, tex, alpha[..., :0], image), outs),
           ((vis, tex, alpha, image.cpu()), outs), ((vis, tex, alpha, image), (outs[0].float(), outs[1], outs[2])),
           ((vis, tex, alpha, image), (outs[0][:, :2], outs[1], outs[2])),
           ((vis, tex, alpha, image), (outs[0], outs[1], outs[2][:1]))]
    for args, o in bad:
        with pytest.raises(b3d.B3DError):
            pseudogt_pack(*args, *o)
    # the C entry rejects host memory before any launch
    host = torch.empty(outs[2].shape, dtype=torch.float16)
    rc = lib.b3d_pseudogt_pack(ptr(vis), 32, 32, ptr(tex), ptr(alpha), 2, 16, 3, ptr(image), 3, 20, 24, ptr(outs[0]),
                               ptr(outs[1]), ptr(host), None)
    assert rc != 0 and b"not device memory" in lib.b3d_last_error()
    rc = lib.b3d_pseudogt_pack(ptr(vis), 32, 32, ptr(tex), ptr(alpha), 2, 0, 3, ptr(image), 3, 20, 24, ptr(outs[0]),
                               ptr(outs[1]), ptr(outs[2]), None)
    assert rc != 0 and b"bad sizes" in lib.b3d_last_error()


# ---------------------------------------------------------------------------------------------------- 3. golden
def test_exporter_reproduces_the_reference_export(tmp_path):
    from models.reconstruction import DatasetParams
    from oracle import mesh as M
    from pseudo_gt_export import PseudoGTExporter
    from rendering.mesh_template import MeshTemplate
    d = np.load(os.path.join(GOLDEN, "pseudogt_reference.npz"))
    tpl = MeshTemplate(M.write_uvsphere_obj(str(tmp_path / "uvsphere_16rings.obj"), rings=16), device=DEV)
    opts = types.SimpleNamespace(optimize_deltas=True, optimize_z0=False)
    dp = DatasetParams(opts, 10)
    with torch.no_grad():
        dp.ds_translation.copy_(torch.tensor(d["ds_translation"]))
        dp.ds_scale.copy_(torch.tensor(d["ds_scale"]))
    trainer = types.SimpleNamespace(generator=PC.build_net().to(DEV), dataset_params=dp.to(DEV), args=opts)
    exp = PseudoGTExporter(trainer, tpl, PC.PSEUDO, inception=PC.Extractor())
    exp.renderer_res = PC.RENDER                      # the golden's render resolution (the reference's rule gives 1024)
    cache = str(tmp_path / "cache")
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False   # TinyNet's convolutions in fp32
    try:
        res = exp.export(PC.batches(), [f"img{i}" for i in range(20)], cache, 'cub', writers=2)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved
    out_dir = os.path.join(cache, f"pseudogt_{PC.PSEUDO}x{PC.PSEUDO}")
    assert sorted(int(f[:-4]) for f in os.listdir(out_dir)) == [0, 1, 2, 13] and res['records'] == 4
    for idx in (0, 1, 2, 13):
        rec = np.load(os.path.join(out_dir, f"{idx}.npz"), allow_pickle=True)['data'].item()
        # the displacement map comes from cuDNN's fp32 convolution instead of the CPU's: a few fp32 ulps apart
        assert np.abs(rec['mesh'].numpy() - d[f"{idx}.mesh"]).max() < 1e-6
        assert rec['mesh'].dtype == torch.float32 and rec['texture'].dtype == torch.float16
        assert np.array_equal(rec['image'].numpy(), d[f"{idx}.image"])
        assert np.array_equal(rec['texture_alpha'].numpy(), d[f"{idx}.texture_alpha"])
        assert np.abs(rec['texture'].float().numpy() - d[f"{idx}.texture"].astype(np.float32)).max() <= 1e-3


# ---------------------------------------------------------------------------------------------------- 4. full size
def cfg_trainer(tpl, n, seed=0):
    from reconstruction_training import ReconTrainer, default_args
    torch.manual_seed(seed)
    tr = ReconTrainer(default_args(), tpl, n, device=DEV)
    with torch.no_grad():
        tr.dataset_params.ds_translation.normal_(0, 0.02)
        tr.dataset_params.ds_scale.normal_(0, 0.02)
    return tr


def cfg_batches(n_batches, B, seed=0, hd=1024):
    g = torch.Generator().manual_seed(seed)
    out = []
    for k in range(n_batches):
        out.append(tuple(t.to(DEV) for t in (
            torch.rand(B, 4, 256, 256, generator=g) * 2 - 1, torch.rand(B, 3, 299, 299, generator=g) * 2 - 1,
            torch.rand(B, 3, hd, hd, generator=g) * 2 - 1, 0.6 + 0.3 * torch.rand(B, 1, generator=g),
            torch.cat(((torch.rand(B, 2, generator=g) - 0.5) * 0.2, torch.zeros(B, 1)), 1),
            torch.nn.functional.normalize(torch.randn(B, 4, generator=g), dim=1), torch.arange(k * B, (k + 1) * B))))
    return out


def test_full_size_records_equal_the_autograd_construction(tmp_path):
    from data.pseudo_gt import make_record, visibility_to_mask
    from pseudo_gt_export import PseudoGTExporter
    from rendering.inverse_renderer import InverseRenderer, texel_visibility
    from rendering.renderer import Renderer
    from utils.inception import InceptionV3
    tpl = template(tmp_path)
    B, R = 10, 512
    tr = cfg_trainer(tpl, B)
    batch = cfg_batches(1, B, seed=3)[0]
    exp = PseudoGTExporter(tr, tpl, R, inception=randomize_inception(InceptionV3([0], weights=None), 1))
    cache = str(tmp_path / "cache")
    exp.export([batch], [f"img{i}" for i in range(B)], cache, 'cub', writers=4)

    X, img299, hd, scale, trans, rot, ind = batch
    with torch.no_grad():
        pred_tex, mesh_map = tr.generator(X)
        td, sd = tr.dataset_params(ind, 'deltas')
        vtx = tpl.vertices_and_pose(mesh_map, scale + sd, trans + td, rot)[1]
    vis, _, _ = texel_visibility(tpl, Renderer(1024, 1024), vtx, pred_tex)
    with torch.no_grad():
        mask = visibility_to_mask(vis, R)
        inv_tex, inv_alpha = InverseRenderer(tpl.mesh, R, R)(vtx, hd)
        inv_tex, inv_alpha = (inv_tex * mask).permute(0, 3, 1, 2), (inv_alpha * mask).permute(0, 3, 1, 2)
    assert 0.05 < float(mask.mean()) < 0.95
    for i in range(B):
        ref = make_record(mesh_map[i], inv_tex[i], inv_alpha[i], img299[i])
        rec = np.load(os.path.join(cache, f"pseudogt_{R}x{R}", f"{i}.npz"), allow_pickle=True)['data'].item()
        assert torch.equal(rec['mesh'], ref['mesh'])
        for k in ('texture', 'texture_alpha', 'image'):
            assert same_bits(rec[k], ref[k]), (i, k)


# ---------------------------------------------------------------------------------------------------- 5. whole set
def write_cub_labels(root, paths):
    labels = os.path.join(root, 'datasets', 'cub', 'CUB_200_2011')
    with open(os.path.join(labels, 'images.txt'), 'w') as f:
        f.writelines(f"{i + 1} {p}\n" for i, p in enumerate(paths))
    with open(os.path.join(labels, 'image_class_labels.txt'), 'w') as f:
        f.writelines(f"{i + 1} {i % 3 + 1}\n" for i in range(len(paths)))


@pytest.mark.parametrize("name", ["cub", "p3d"])
def test_whole_synthetic_set(tmp_path, name):
    from data.pseudo_gt import load_poses_metadata
    from fid_evaluation import load_real_statistics
    from pseudo_gt_export import PseudoGTExporter, imagenet_rows
    from utils.fid import forward_inception_features
    from utils.inception import InceptionV3
    root = str(tmp_path)
    RD.write_tree(root, RD.make_inputs(0))
    tpl = template(tmp_path)
    ds = make(root, name, [256, 299, 1024], is_train=False).to_device(DEV)
    n, B, R = len(ds), 3, 256
    assert n % B != 0                                   # a ragged last batch
    tr = cfg_trainer(tpl, n, seed=1)
    inc = randomize_inception(InceptionV3([0], weights=None), 2)
    val = make(root, 'cub', 299, is_train=False).to_device(DEV) if name == 'cub' else None
    cache = os.path.join(root, 'cache', name)
    res = PseudoGTExporter(tr, tpl, R, inception=inc).export(
        ds.eval_batches(B), ds.get_paths(), cache, name, val_batches=val.eval_batches(B) if val else None, writers=4)

    files = sorted(os.listdir(os.path.join(cache, f"pseudogt_{R}x{R}")))
    assert files == sorted(f"{i}.npz" for i in range(n)) and res['records'] == n
    meta = load_poses_metadata(cache)
    rows = ds.store['poses'][:, 0].cpu()
    assert meta['path'] == ds.get_paths()
    assert torch.equal(meta['scale'], rows[:, :1]) and torch.equal(meta['translation'], rows[:, 1:4])
    assert torch.equal(meta['rotation'], rows[:, 4:])

    with torch.no_grad():
        feats = torch.cat([forward_inception_features(inc, b[1] / 2 + 0.5) for b in ds.eval_batches(B)]).double().cpu().numpy()
    if name == 'p3d':
        feats = feats[imagenet_rows(ds.get_paths())]
        assert 0 < len(feats) < n
    mu, sigma, count = load_real_statistics(res['fid_train'], 299, expect_images=len(feats))
    np.testing.assert_allclose(mu, feats.mean(axis=0), rtol=0, atol=1e-12)
    np.testing.assert_allclose(sigma, np.cov(feats, rowvar=False), rtol=0, atol=1e-9)
    if name == 'cub':
        with torch.no_grad():
            vf = torch.cat([forward_inception_features(inc, b[0][:, :3] / 2 + 0.5)
                            for b in val.eval_batches(B)]).double().cpu().numpy()
        mu, sigma, count = load_real_statistics(res['fid_testval'], 299, expect_images=len(vf))
        np.testing.assert_allclose(mu, vf.mean(axis=0), rtol=0, atol=1e-12)
        np.testing.assert_allclose(sigma, np.cov(vf, rowvar=False), rtol=0, atol=1e-9)
    else:
        assert res['fid_testval'] is None

    if name == 'cub':                                   # the GAN stage trains on the written cache
        import bench
        from data.cub_200_2011_dataset import CubDataset
        from gan_training import GANTrainer
        import dataset_common as DC
        write_cub_labels(root, ds.get_paths())
        gds = CubDataset(DC.make_args('cub', texture_resolution=R), root=root).to_device(DEV)
        batch = next(iter(gds.train_batches(2, 0)))
        torch.manual_seed(0)
        gan = GANTrainer(bench.gan_args(R, 2), mesh_template=tpl, device=DEV)
        losses = [float(x) for x in gan.train_epoch([batch])]
        assert losses and all(np.isfinite(losses)), losses


# ---------------------------------------------------------------------------------------------------- 6. memory
def test_staging_buffers_are_allocated_once(tmp_path):
    from pseudo_gt_export import PseudoGTExporter
    from utils.inception import InceptionV3
    tpl = template(tmp_path)
    B = 10
    tr = cfg_trainer(tpl, 3 * B)
    inc = randomize_inception(InceptionV3([0], weights=None), 1)
    batches = cfg_batches(3, B, seed=4)
    peaks = []
    for k in (2, 3):
        exp = PseudoGTExporter(tr, tpl, 512, inception=inc)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        exp.export(batches[:k], [f"img{i}" for i in range(3 * B)], str(tmp_path / f"c{k}"), 'cub', writers=4)
        torch.cuda.synchronize()
        peaks.append(torch.cuda.max_memory_allocated() - base)
        del exp
    # B 10 at 1024^2 / R 512: render buffers 0.34 GB, the inverse render and staging about 0.1 GB, the network's and
    # Inception's activations (0.55 GB measured on an H100); a third batch must not need more than the first two
    assert peaks[1] < 2 ** 30, peaks
    assert peaks[1] <= peaks[0] + 16 * 2 ** 20, peaks
