"""Multi-process validation pass on CPU (gloo, world size 2): rank r evaluates batches r::2 with distributed=True and the
per-sample sums are all-reduced, so both ranks return the single-process totals of the whole validation set.  Stand-ins
of recon_step_common replace the network, template and renderer; the fused losses are their torch definitions."""
import os
import sys

import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import GOLDEN, PKG, ROOT


def run(shard, distributed):
    import pytest
    for p in (PKG, ROOT, GOLDEN, os.path.join(ROOT, "tests")):
        if p not in sys.path:
            sys.path.insert(0, p)
    import recon_eval_common as RE
    import test_recon_eval_hostlogic as H
    mp_ = pytest.MonkeyPatch()
    try:
        RT = H.torch_criteria(mp_)
        out = {}
        for loss in RE.CRITERIA:
            tr = H.eval_trainer(RT, True, True, loss)
            batches = RE.eval_batches() + RE.eval_batches()[:1]          # four batches: two per rank
            out[loss] = tr.evaluate(batches if shard is None else batches[shard::2], distributed=distributed)
        return out
    finally:
        mp_.undo()


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    q.put((rank, run(rank, True)))
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_validation_pass_equals_single_process():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33000 + os.getpid() % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=180) for _ in procs], key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    ref = run(None, False)
    for loss in ref:
        assert ref[loss]["N"] == 16
        for rank, out in res:
            assert out[loss]["N"] == 16
            for k in ("recon_loss", "flat_loss", "miou"):
                assert abs(out[loss][k] - ref[loss][k]) <= 1e-9 * abs(ref[loss][k]), (rank, loss, k, out[loss][k], ref[loss][k])
