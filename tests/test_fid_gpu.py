"""FID evaluation path on the GPU (SURVEY §8f rank 4): the kernels of csrc/fid_kernels.cu against torch, the Inception
convolution geometries on the wgmma kernel against an fp64 convolution, the whole CUDA Inception against the oracle's
restatement of the network (same state dict), a 299 x 299 render (the evaluation resolution, main.py:156) against the mesh
oracle, and the evaluation loop end to end.

Tolerances: fp32 kernels 1e-5 (resampling: 2e-4, the fp32 source coordinate); single tf32 convolutions 4e-3 of the largest magnitude (as tests/test_bench_shapes_gpu.py);
the full network — 47 stacked tf32 convolutions — 2e-2 of the largest activation of each block; feature statistics
(fp64 sums) 1e-9; face-index buffer of the render exact."""
import os
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN
from fid_common import randomize_inception
from oracle import fid as OF
from oracle import mesh as M

sys.path.insert(0, GOLDEN)
import gan_common as GC          # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _lib():
    import b3d
    return b3d


def test_input_transform_and_pools():
    b3d = _lib()
    from b3d import check, lib, ptr, stream_ptr
    g = torch.Generator().manual_seed(1)
    for H, W in ((256, 256), (299, 299), (64, 80)):
        img = torch.rand(2, 3, H, W, generator=g)
        ref = (2 * F.interpolate(img.double(), size=(299, 299), mode="bilinear", align_corners=False) - 1).permute(0, 2, 3, 1)
        x = img.to(DEV)
        out = torch.full((2, 299, 299, 32), 7.0, device=DEV)
        check(lib.b3d_inception_input(ptr(x), 2, H, W, 299, 299, 32, 1, ptr(out), stream_ptr(x)))
        assert float((out[..., :3].cpu().double() - ref).abs().max()) < 2e-4     # fp32 source coordinates
        assert float(out[..., 3:].abs().max()) == 0.0
        if (H, W) == (299, 299):
            assert torch.equal(out[..., :3].cpu(), (2 * img - 1).permute(0, 2, 3, 1))       # no resampling at the native size
    x = torch.randn(3, 35, 35, 288, generator=g)
    ref = F.max_pool2d(x.permute(0, 3, 1, 2), 3, 2).permute(0, 2, 3, 1)
    out = torch.zeros(3, 17, 17, 768, device=DEV)
    xd = x.to(DEV)
    check(lib.b3d_maxpool3x3s2_nhwc(ptr(xd), 3, 35, 35, 288, out.data_ptr() + 4 * 480, 768, stream_ptr(xd)))
    assert torch.equal(out[..., 480:].cpu(), ref) and float(out[..., :480].abs().max()) == 0.0
    x = torch.randn(2, 8, 8, 2048, generator=g)
    out = torch.empty(2, 2048, device=DEV)
    xd = x.to(DEV)
    check(lib.b3d_mean_hw_nhwc(ptr(xd), 2, 64, 2048, ptr(out), stream_ptr(xd)))
    assert float((out.cpu() - x.mean(dim=(1, 2))).abs().max()) < 1e-5
    assert b3d.launch_count() > 0


def test_feature_statistics_match_numpy():
    from utils.fid import FIDStatistics, calculate_stats
    g = torch.Generator().manual_seed(2)
    for D in (2048, 100):
        a = torch.randn(37, D, generator=g) * 0.7 + 0.2
        b = torch.randn(50, D, generator=g) * 1.3 - 0.1
        st = FIDStatistics(D, DEV)
        st.update(a.to(DEV))
        st.update(b.to(DEV))
        mu, sigma = st.finalize()
        full = torch.cat([a, b]).double().numpy()
        np.testing.assert_allclose(mu, full.mean(axis=0), rtol=0, atol=1e-12)
        np.testing.assert_allclose(sigma, np.cov(full, rowvar=False), rtol=0, atol=1e-9)
    m2, s2 = calculate_stats(a.to(DEV))
    np.testing.assert_allclose(s2, np.cov(a.double().numpy(), rowvar=False), rtol=0, atol=1e-9)


# (cin, cout, kernel, stride, padding, H = W, avg_fold): the distinct convolution geometries of Inception-v3
GEOMETRIES = [(3, 32, 3, 2, 0, 299, False), (32, 32, 3, 1, 0, 149, False), (32, 64, 3, 1, 1, 147, False), (64, 80, 1, 1, 0, 73, False),
              (80, 192, 3, 1, 0, 73, False), (48, 64, 5, 1, 2, 35, False), (192, 32, 1, 1, 0, 35, True), (288, 384, 3, 2, 0, 35, False),
              (128, 128, (1, 7), 1, (0, 3), 17, False), (160, 192, (7, 1), 1, (3, 0), 17, False), (192, 320, 3, 2, 0, 17, False),
              (384, 384, (1, 3), 1, (0, 1), 8, False), (448, 384, 3, 1, 1, 8, False), (2048, 192, 1, 1, 0, 8, True)]


@pytest.mark.parametrize("geo", GEOMETRIES, ids=lambda g: "x".join(str(v) for v in g[:6]).replace(" ", ""))
def test_inception_convolution_geometries(geo):
    from utils import inception as I
    cin, cout, k, stride, pad, HW, avg = geo
    torch.manual_seed(cin + cout)
    net = I.InceptionV3([0], weights=None)
    m = I.BasicConv2d(cin, cout, k, stride=stride, padding=pad)
    holder = torch.nn.Sequential(m)
    randomize_inception(holder, 3)
    B = 2
    x = torch.randn(B, cin, HW, HW)
    cinp = -(-cin // 32) * 32
    xh = F.pad(x.permute(0, 2, 3, 1), (0, cinp - cin)).contiguous().to(DEV)
    sd = {"u." + kk: v.double() for kk, v in m.state_dict().items()}
    xin = F.avg_pool2d(x.double(), 3, 1, 1) if avg else x.double()
    ref = OF._unit(sd, "u", xin, stride, pad).permute(0, 2, 3, 1)
    # 1. own tensor (padded channel count, pad channels exactly zero)
    y = net._conv(xh, m, avg_fold=avg)
    assert y.shape[3] % 32 == 0 and y.shape[:3] == ref.shape[:3]
    lim = 4e-3 * float(ref.abs().max())
    assert float((y[..., :cout].cpu().double() - ref).abs().max()) <= lim
    assert float(y[..., cout:].abs().max()) == 0.0 if y.shape[3] > cout else True
    # 2. into a channel slice of a wider tensor
    if cout % 32 == 0:
        out = torch.full((B, ref.shape[1], ref.shape[2], cout + 96), -3.0, device=DEV)
        net._conv(xh, m, avg_fold=avg, out=out, coff=64)
        assert float((out[..., 64:64 + cout].cpu().double() - ref).abs().max()) <= lim
        assert float((out[..., :64] + 3).abs().max()) == 0.0 and float((out[..., 64 + cout:] + 3).abs().max()) == 0.0


def test_inception_forward_matches_oracle():
    from utils.inception import InceptionV3
    m = randomize_inception(InceptionV3([0, 1, 2, 3], weights=None), 4)
    x = torch.rand(2, 3, 256, 256, generator=torch.Generator().manual_seed(8))
    ref = OF.inception_forward(m.state_dict(), x.double(), (0, 1, 2, 3))
    got = m.to(DEV)(x.to(DEV))
    assert [tuple(g.shape) for g in got] == [tuple(r.shape) for r in ref]
    for g, r in zip(got, ref):
        err = float((g.cpu().double() - r).abs().max()) / float(r.abs().max())
        assert err < 2e-2, err
    # the drop-in call of utils/fid.py
    from utils.fid import forward_inception_batch
    m.output_blocks = [3]                          # what init_inception() selects: the 2048-d pool features
    emb = forward_inception_batch(m, x.to(DEV))
    assert emb.shape == (2, 2048) and np.isfinite(emb).all()
    np.testing.assert_allclose(emb, got[3].reshape(2, -1).cpu().numpy(), rtol=0, atol=1e-6)
    with pytest.raises(Exception):
        m(x)                                       # CPU tensor: no fallback


def test_render_at_evaluation_resolution_matches_oracle():
    """299 x 299 is not a multiple of the rasteriser's 16-pixel tiles: partial tiles on both edges."""
    from rendering.mesh_template import MeshTemplate
    from rendering.renderer import Renderer
    path = M.write_uvsphere_obj(os.path.join(tempfile.mkdtemp(), "uvsphere_16rings.obj"), rings=16)
    mt, T = MeshTemplate(path, device=DEV), M.TemplateData(M.load_obj(path), path)
    g = torch.Generator().manual_seed(12)
    mesh_map = torch.randn(1, 3, 32, 32, generator=g) * 0.05
    q = F.normalize(torch.randn(1, 4, generator=g), dim=-1)
    s, t = torch.tensor([[0.7]]), torch.tensor([[0.1, -0.05, 0.0]])
    tex = torch.rand(1, 3, 64, 64, generator=g) * 2 - 1
    vtx = M.transform_vertices(M.get_vertex_positions(T, mesh_map), s, t, q)
    img_o, alpha_o, idx_o = M.forward_renderer(T, vtx, tex, 299, 299)
    r = Renderer(299, 299)
    img, alpha = mt.forward_renderer(r, vtx.to(DEV), tex.to(DEV))
    assert torch.equal(r.last_face_index.cpu(), idx_o)
    assert float((img.cpu() - img_o).abs().max()) < 1e-4 and float((alpha.cpu() - alpha_o).abs().max()) < 2e-5
    # ... and the fused vertex pipeline used by the evaluation loop gives the same vertices
    _, vtx2 = mt.vertices_and_pose(mesh_map.to(DEV), s.to(DEV), t.to(DEV), q.to(DEV))
    assert float((vtx2.cpu() - vtx).abs().max()) < 5e-6


def test_evaluation_loop():
    from fid_evaluation import FIDEvaluator, load_real_statistics, save_real_statistics
    from models import gan
    from rendering.mesh_template import MeshTemplate
    from utils.fid import calculate_frechet_distance
    from utils.inception import InceptionV3
    args = GC.make_args(256, 2)
    G, _ = GC.build(gan, args)
    G.to(DEV).eval()
    path = M.write_uvsphere_obj(os.path.join(tempfile.mkdtemp(), "uvsphere_16rings.obj"), rings=16)
    mt = MeshTemplate(path, device=DEV)
    # the 768-d block keeps the host-side eigendecompositions of this test short (2048-d: ~4 s per distance); the 2048-d
    # pool features are covered by test_inception_forward_matches_oracle
    inc = randomize_inception(InceptionV3([2], weights=None), 6)
    ev = FIDEvaluator(G, mt, inception=inc, truncation_sigma=1.0, device=DEV)
    g = torch.Generator().manual_seed(21)

    def batches(n, B=3, pseudo=True, image=True):
        for i in range(n):
            d = {"idx": torch.arange(i * B, (i + 1) * B), "class": torch.randint(0, 200, (B, 1), generator=g),
                 "rotation": F.normalize(torch.randn(B, 4, generator=g), dim=-1), "scale": 0.5 + 0.3 * torch.rand(B, generator=g),
                 "translation": (torch.rand(B, 3, generator=g) - 0.5) * 0.2}
            if image:
                d["image"] = torch.rand(B, 3, 299, 299, generator=g)
            if pseudo:
                d["texture"] = torch.rand(B, 3, 256, 256, generator=g) * 2 - 1
                d["mesh"] = torch.randn(B, 3, 32, 32, generator=g) * 0.05
            yield d

    out = ev.evaluate(batches(2), seed=1234, keep_features=True)
    assert out["num_generated"] == 6 and ev.m_real is not None and ev.m_real.shape == (768,)
    for k in ("fid", "fid_texture_only", "fid_mesh_only"):
        assert np.isfinite(out[k]) and out[k] > 0
    f = out["features"]["combined"].cpu().double().numpy()
    assert f.shape == (6, 768)
    ref = calculate_frechet_distance(f.mean(axis=0), np.cov(f, rowvar=False), ev.m_real, ev.s_real)
    assert abs(ref - out["fid"]) <= 1e-4 * abs(ref)      # 6 samples: rank-5 covariances, sqrt of ~2000 noise-level eigenvalues
    # the three renders of a batch differ (generated vs pseudo-ground-truth mesh / texture)
    assert float((out["features"]["combined"] - out["features"]["texture_only"]).abs().max()) > 0
    # cached real statistics (the reference's npz format) -> a `fast` evaluation needs no real images; same seed, same score
    p = os.path.join(tempfile.mkdtemp(), "precomputed_fid_299x299_train.npz")
    save_real_statistics(p, ev.m_real, ev.s_real, 6)
    ev2 = FIDEvaluator(G, mt, inception=inc, truncation_sigma=1.0, device=DEV)
    mu, sigma, n = load_real_statistics(p, 299, expect_images=6)
    ev2.set_real_statistics(mu, sigma)
    g.manual_seed(21)
    out2 = ev2.evaluate(batches(2, image=True), fast=True, seed=1234)
    assert set(out2) == {"fid", "num_generated"}
    assert abs(out2["fid"] - out["fid"]) <= 1e-4 * abs(out["fid"])
