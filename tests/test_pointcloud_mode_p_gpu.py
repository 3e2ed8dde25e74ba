"""The fused mode-P silhouette (paper semantics: (1 - r, r) corner weights, a real Gaussian chained along x, y and z, no
epsilon pads) through b3d_pc_silhouette_{fwd,bwd}_hosttaps: against the fp64 oracle, against the dense-grid path, at its
edges, in the K-candidate pipeline and under CUDA-graph capture.

Tolerance against the oracle: the rule of test_pointcloud_dense_gpu.py, |cuda - oracle64| <= 4 x the fp32-vs-fp64 oracle
gap + 2e-5 of the largest magnitude."""
import pytest
import torch

from oracle import pointcloud as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EPS = 1e-5


def cloud(B, N, seed, sphere=False):
    g = torch.Generator().manual_seed(seed)
    p = (torch.rand(B, N, 3, generator=g) * 2 - 1) * 0.45
    if sphere:      # noisy sphere shell: the collision pattern of a real shape
        d = torch.nn.functional.normalize(torch.randn(B, N, 3, generator=g), dim=-1)
        p = d * (0.35 + 0.01 * torch.randn(B, N, 1, generator=g))
    return p, torch.randn(B, 4, generator=g), 0.5 + 0.5 * torch.rand(B, 1, generator=g), g


def oracle_both(p, q, s, wts, V, ksize, sigma):
    out = {}
    for dt in (torch.float32, torch.float64):
        po, qo = p.to(dt).requires_grad_(True), q.to(dt).requires_grad_(True)
        so = s.to(dt).requires_grad_(True) if s is not None else None
        sil = O.effective_loss_forward(po, qo, so, V=V, kernel_size=ksize, sigma=sigma, mode="P")
        grads = torch.autograd.grad((sil * wts.to(dt)).sum(), [po, qo] + ([so] if s is not None else []))
        out[dt] = [sil.detach()] + list(grads)
    return out


def fused(p, q, s, wts, V, ksize, sigma):
    from utils.effective_loss_function import EffectiveLossFunction
    m = EffectiveLossFunction(voxel_size=V, kernel_size=ksize, smooth_sigma=sigma, semantics="P").to(DEV)
    pc, qc = p.to(DEV).requires_grad_(True), q.to(DEV).requires_grad_(True)
    sc = s.to(DEV).requires_grad_(True) if s is not None else None
    sil = m(pc, qc, sc)
    grads = torch.autograd.grad((sil * wts.to(DEV)).sum(), [pc, qc] + ([sc] if s is not None else []))
    return [sil.detach()] + list(grads)


def assert_oracle_rule(got, orc):
    for v, o32, o64, name in zip(got, orc[torch.float32], orc[torch.float64], ["sil", "dp", "dq", "ds"]):
        gap = float((o32.double() - o64).abs().max())
        tol = 4 * gap + 2e-5 * max(1.0, float(o64.abs().max()))
        err = float((v.cpu().double() - o64).abs().max())
        assert err <= tol, (name, err, tol)


@pytest.mark.parametrize("B,N,V,ksize,sigma,with_scale", [
    (2, 300, 2, 21, 3.0, True),        # the smallest grid: every tap but the centre falls in the zero padding
    (2, 700, 33, 21, 3.0, False),      # V not a multiple of any tile
    (2, 500, 40, 21, 0.2, True),       # the sigma schedule's end: taps ~ (0, .., 1, .., 0)
    (1, 3000, 64, 21, 3.0, True),
    (2, 800, 33, 1, 3.0, True),        # ktaps 1: no blur
    (1, 2000, 64, 63, 3.0, True),      # the widest kernel the ABI takes: halo 31
    (2, 600, 40, 63, 0.2, False),
])
def test_against_fp64_oracle(B, N, V, ksize, sigma, with_scale):
    p, q, s, g = cloud(B, N, 100 * V + ksize)
    s = s if with_scale else None
    wts = torch.rand(B, V, V, generator=g)
    assert_oracle_rule(fused(p, q, s, wts, V, ksize, sigma), oracle_both(p, q, s, wts, V, ksize, sigma))


def test_v128_noisy_sphere_against_fp64_oracle():
    """cfg2's point size (B 16, N 8000, V 128) in one launch; samples are independent, so two of them are checked."""
    B, N, V = 16, 8000, 128
    p, q, s, g = cloud(B, N, 128, sphere=True)
    wts = torch.rand(B, V, V, generator=g)
    got = fused(p, q, s, wts, V, 21, 3.0)
    pick = [3, 12]
    orc = oracle_both(p[pick], q[pick], s[pick], wts[pick], V, 21, 3.0)
    assert_oracle_rule([t[pick] for t in got], orc)


def test_fused_matches_dense_path_at_cfg2_size():
    from b3d.pointcloud import effective_loss, effective_loss_dense, smoothing_taps
    B, N, V = 16, 8000, 128
    p, q, s, g = cloud(B, N, 7, sphere=True)
    wts = torch.rand(B, V, V, generator=g).to(DEV)
    taps = smoothing_taps(3.0, 21, "P")
    res = []
    for fn in (effective_loss, effective_loss_dense):
        pc, qc, sc = p.to(DEV).requires_grad_(True), q.to(DEV).requires_grad_(True), s.to(DEV).requires_grad_(True)
        sil = fn(pc, qc, sc, V=V, taps=taps, mode="P")
        res.append([sil.detach()] + list(torch.autograd.grad((sil * wts).sum(), [pc, qc, sc])))
    for a, b, name in zip(res[0], res[1], ["sil", "dp", "dq", "ds"]):
        err, mag = float((a - b).abs().max()), float(b.abs().max())
        assert err <= 1e-4 * max(mag, 1e-3), (name, err, mag)     # fp32 summation order only


def test_edges():
    from b3d.pointcloud import effective_loss, smoothing_taps
    V = 32
    taps = smoothing_taps(3.0, 21, "P")
    q = torch.tensor([[1.0, 0, 0, 0], [0.3, -0.2, 0.9, 0.1]], device=DEV)
    empty_value = 1 - (1 - EPS) ** V          # no occupancy: o = eps in every cell, no pad terms
    # B 0
    z = torch.zeros(0, 10, 3, device=DEV, requires_grad=True)
    out = effective_loss(z, torch.zeros(0, 4, device=DEV), None, V=V, taps=taps, mode="P")
    assert out.shape == (0, V, V)
    out.sum().backward()
    # N 0 and all points out of bounds: the analytic image, zero gradients
    for pts in (torch.zeros(2, 0, 3, device=DEV), torch.full((2, 64, 3), 3.0, device=DEV)):
        pts = pts.requires_grad_(True)
        qq, ss = q.clone().requires_grad_(True), torch.ones(2, 1, device=DEV, requires_grad=True)
        sil = effective_loss(pts, qq, ss, V=V, taps=taps, mode="P")
        assert torch.allclose(sil, torch.full_like(sil, empty_value), rtol=0, atol=1e-6)
        gp, gq, gs = torch.autograd.grad((sil * torch.rand_like(sil)).sum(), [pts, qq, ss])
        assert not gp.any() and not gq.any() and not gs.any()
    # many points in one voxel: raw occupancy far above 1, the clamp mask is active
    p, qr, s, g = cloud(1, 400, 3)
    p[0, :300] = torch.tensor([0.05, -0.02, 0.11]) + 1e-4 * torch.randn(300, 3, generator=g)
    wts = torch.rand(1, V, V, generator=g)
    assert_oracle_rule(fused(p, qr, s, wts, V, 21, 3.0), oracle_both(p, qr, s, wts, V, 21, 3.0))
    # non-finite taps propagate (no skip of empty cells then)
    bad = list(taps)
    bad[10] = float("nan")
    out = effective_loss(p.to(DEV), qr.to(DEV), None, V=V, taps=bad, mode="P")
    assert torch.isnan(out).all()


def test_k_candidate_pipeline_picks_the_dense_path_candidates():
    from b3d.pointcloud import effective_loss, effective_loss_dense, smoothing_taps
    from models.unsupervised_part import UnsupervisedLoss
    B, K, N, V = 3, 4, 600, 32
    p, _, _, g = cloud(B, N, 21)
    cand = torch.randn(B * K, 4, generator=g)
    student = torch.randn(B, 4, generator=g)
    pk = p.repeat_interleave(K, dim=0).to(DEV)
    taps = smoothing_taps(3.0, 21, "P")
    sil_f = effective_loss(pk, cand.to(DEV), None, V=V, taps=taps, mode="P")
    sil_d = effective_loss_dense(pk, cand.to(DEV), None, V=V, taps=taps, mode="P")
    # target masks: a perturbed silhouette of one candidate per sample, at twice the resolution
    best = torch.randint(0, K, (B,), generator=g)
    tgt = sil_d.view(B, K, V, V)[torch.arange(B, device=DEV), best.to(DEV)]
    masks = (tgt + 0.05 * torch.rand(B, V, V, generator=g).to(DEV)).repeat_interleave(2, 1).repeat_interleave(2, 2)
    idx = []
    for sil in (sil_f, sil_d):
        loss = UnsupervisedLoss(K, 20.0)
        loss((sil, cand.to(DEV), student.to(DEV)), masks, True)
        idx.append(loss.minimum_indexes.cpu())
    assert torch.equal(idx[0], idx[1])
    assert torch.equal(idx[0], best)


def test_cuda_graph_replay_matches_eager():
    from b3d.pointcloud import effective_loss, smoothing_taps
    B, N, V = 4, 3000, 64
    p, q, s, g = cloud(B, N, 33, sphere=True)
    taps = smoothing_taps(2.0, 21, "P")
    wts = torch.rand(B, V, V, generator=g).to(DEV)
    pc, qc, sc = p.to(DEV).requires_grad_(True), q.to(DEV).requires_grad_(True), s.to(DEV).requires_grad_(True)

    def step():
        sil = effective_loss(pc, qc, sc, V=V, taps=taps, mode="P")
        (sil * wts).sum().backward()
        return sil

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            for t in (pc, qc, sc):
                t.grad = None
            eager = step().detach().clone()
            eager_grads = [t.grad.clone() for t in (pc, qc, sc)]
    torch.cuda.current_stream().wait_stream(side)
    for t in (pc, qc, sc):
        t.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        sil = step()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip([sil] + [t.grad for t in (pc, qc, sc)], [eager] + eager_grads):
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-6 * float(b.abs().max()))


def test_second_backward_through_the_same_graph():
    """The backward overwrites the workspace with its gradients; a retained graph refills it before a second backward."""
    from b3d.pointcloud import effective_loss, smoothing_taps
    p, q, s, g = cloud(2, 1000, 5)
    pc, qc, sc = p.to(DEV).requires_grad_(True), q.to(DEV).requires_grad_(True), s.to(DEV).requires_grad_(True)
    sil = effective_loss(pc, qc, sc, V=40, taps=smoothing_taps(3.0, 21, "P"), mode="P")
    w = torch.rand(sil.shape, generator=g).to(DEV)
    first = torch.autograd.grad((sil * w).sum(), [pc, qc, sc], retain_graph=True)
    second = torch.autograd.grad((sil * w).sum(), [pc, qc, sc])
    for a, b in zip(first, second):
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-6 * float(b.abs().max()))
