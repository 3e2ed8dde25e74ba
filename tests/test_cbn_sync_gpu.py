"""Mode 2 of b3d_cbn_prepare (the reference's SyncBN formulas) and the all-reduced coupling terms of the fused backward on
one GPU: a two-rank gloo world with both processes on cuda:0.  gloo has no peer-memory path (b3d.sync.peer_sync returns
None), so _CBNActPad all-reduces the fp64 sums and the backward's `red` with torch.distributed.  Outputs, input gradients,
the gamma / beta parameter gradients (summed over the ranks) and the running buffers must equal the SyncBN formulas in fp64
on the whole batch: inv_std = clamp(var, eps)^-1/2, running variance unbiased with the GLOBAL count."""
import os
import queue
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import PKG, ROOT

pytestmark = pytest.mark.gpu
N, C, H, W, UP, PAD = 8, 64, 8, 6, 2, 1


def _inputs():
    """The global batch (fp32 values held in fp64), seeded; channel 1 is near constant (variance ~ eps / 4).  Pixels on the
    LeakyReLU kink are moved off it (cbn_common.clear_kinks)."""
    import torch.nn.functional as F
    from cbn_common import EMB, EPS, clear_kinks, make_cbn
    g = torch.Generator().manual_seed(21)
    y = torch.randn(N, C, H, W, generator=g, dtype=torch.float64) * 1.3 + 0.2
    y[:, 1] = (EPS / 4) ** 0.5 * torch.randn(N, H, W, generator=g, dtype=torch.float64)
    skip = torch.randn(N, C, H, W + 2, generator=g, dtype=torch.float64)
    z = torch.randn(N, EMB, generator=g, dtype=torch.float64)
    w = torch.randn(N, C, UP * H, UP * W + 2 * PAD, generator=g, dtype=torch.float64)
    y, skip, z = y.float().double(), skip.float().double(), z.float().double()
    cbn = make_cbn(C, 4, norm_g='syncbatch')
    gam, bet = (F.linear(z, m.weight.double(), m.bias.double()).detach() for m in (cbn.fc_gamma, cbn.fc_beta))
    dy, _ = clear_kinks(y, gam, bet, clamp=True)
    return (y + dy).float().double(), skip, z, w


def _worker(rank, world, port, q):
    for p in (PKG, ROOT, os.path.join(ROOT, "tests")):
        if p not in sys.path:
            sys.path.insert(0, p)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from b3d.ew import cbn_act_pad
        from cbn_common import make_cbn
        dev = torch.device("cuda:0")
        # gloo all-reduces CUDA tensors itself; should this build not, the sums are staged through host memory
        staged = False
        try:
            probe = torch.ones(4, device=dev, dtype=torch.float64)
            dist.all_reduce(probe)
            assert float(probe[0]) == world
        except Exception:                                   # noqa: BLE001 — any refusal of CUDA tensors
            staged = True
            plain = dist.all_reduce

            def all_reduce(t, *a, **kw):
                h = t.cpu()
                plain(h, *a, **kw)
                t.copy_(h)
            dist.all_reduce = all_reduce
        cbn = make_cbn(C, 4, norm_g='syncbatch').to(dev).train()
        y, skip, z, w = _inputs()
        lo, hi = rank * N // world, (rank + 1) * N // world
        yr = y[lo:hi].float().to(dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
        sr = skip[lo:hi].float().to(dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
        zr = z[lo:hi].float().to(dev).requires_grad_(True)
        out = cbn_act_pad(yr, cbn, zr, skip_nchw=sr, skip_off=1, up=UP, pad=PAD)
        (out * w[lo:hi].float().to(dev)).sum().backward()
        torch.cuda.synchronize()
        grads = [p.grad.cpu().numpy() for p in (cbn.fc_gamma.weight, cbn.fc_gamma.bias, cbn.fc_beta.weight, cbn.fc_beta.bias)]
        q.put((rank, staged, out.detach().cpu().numpy(), yr.grad.cpu().numpy(), sr.grad.cpu().numpy(), zr.grad.cpu().numpy(),
               grads, cbn.norm.running_mean.cpu().numpy(), cbn.norm.running_var.cpu().numpy(), int(cbn.norm.num_batches_tracked)))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_syncbn_mode2_on_one_gpu_world2():
    import torch.nn.functional as F
    from cbn_common import EPS, make_cbn, ref_glue
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 35000 + os.getpid() % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    try:
        for p in procs:
            p.start()
        res = {}
        for _ in procs:
            try:
                r = q.get(timeout=180)
            except queue.Empty:
                pytest.fail(f"a rank did not report; exit codes {[p.exitcode for p in procs]}")
            res[r[0]] = r[1:]
        for p in procs:
            p.join(timeout=60)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(timeout=10)
    print(f"  gloo all-reduce of CUDA fp64 tensors: {'staged through host memory' if res[0][0] else 'direct'}")

    cbn = make_cbn(C, 4, norm_g='syncbatch')
    rm0, rv0 = cbn.norm.running_mean.double(), cbn.norm.running_var.double()
    P = [p.detach().double().requires_grad_(True) for p in (cbn.fc_gamma.weight, cbn.fc_gamma.bias, cbn.fc_beta.weight, cbn.fc_beta.bias)]
    y, skip, z, w = _inputs()
    y, skip, z = (t.requires_grad_(True) for t in (y, skip, z))
    out, _, _, m, v = ref_glue(y, F.linear(z, P[0], P[1]), F.linear(z, P[2], P[3]), skip, 1, UP, PAD, clamp=True)
    (out * w).sum().backward()

    def close(name, got, want, rel):
        got, want = torch.as_tensor(got).double(), want.detach()
        e = float((got - want).abs().max())
        print(f"  {name:16s} rel {e / float(want.abs().max()):.2e}")
        assert e <= rel * float(want.abs().max()), f"{name}: {e:.3e} > {rel:g} x {float(want.abs().max()):.3e}"

    close("out", torch.cat([torch.as_tensor(res[r][1]) for r in range(2)]), out, 1e-5)
    close("d y", torch.cat([torch.as_tensor(res[r][2]) for r in range(2)]), y.grad, 1e-4)
    close("d skip", torch.cat([torch.as_tensor(res[r][3]) for r in range(2)]), skip.grad, 1e-5)
    close("d z", torch.cat([torch.as_tensor(res[r][4]) for r in range(2)]), z.grad, 1e-4)
    for j, name in enumerate(("d fc_gamma.w", "d fc_gamma.b", "d fc_beta.w", "d fc_beta.b")):
        close(name, sum(torch.as_tensor(res[r][5][j]) for r in range(2)), P[j].grad, 1e-4)
    n = N * H * W                                                # the global count
    rm_ref = 0.9 * rm0 + 0.1 * m.detach()
    rv_ref = 0.9 * rv0 + 0.1 * v.detach() * n / (n - 1)
    for r in range(2):
        close("running_mean", res[r][6], rm_ref, 2e-6)
        close("running_var", res[r][7], rv_ref, 2e-6)
        assert res[r][8] == 1
    # the near-constant channel normalises with clamp(var, eps), not var + eps
    assert float(v[1]) < EPS / 2
