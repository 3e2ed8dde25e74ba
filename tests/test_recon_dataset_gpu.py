"""The device path of the reconstruction datasets on the GPU: b3d_image_batch batches against the reference loaders
(tests/golden/recon_data_reference.npz) for every (index, flip), single and list img_size; against the host restatement at
cfg4 size and at 1024^2 from a 3141-pixel window; bad arguments; ReconTrainer.step and .evaluate fed by the device batches
against the same calls on the host ImageDataset batches; graph capture; the last partial batch."""
import os
import sys
import tempfile

import numpy as np
import pytest
import torch

from conftest import GOLDEN

sys.path.insert(0, GOLDEN)
import recon_data_common as RD                                # noqa: E402
from test_recon_dataset_hostlogic import bits, golden_img, make, ordered, ulps  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope='module')
def gold():
    return np.load(os.path.join(GOLDEN, 'recon_data_reference.npz'))


@pytest.fixture(scope='module')
def root(gold, tmp_path_factory):
    r = str(tmp_path_factory.mktemp('recon_data_gpu'))
    RD.write_tree(r, {k[3:]: gold[k] for k in gold.files if k.startswith('in_')})
    return r


def not_identical(a, b):
    return int((ordered(a) != ordered(b)).sum())


def host_batch(ds, idx, flips, img_size):
    """ImageDataset's collated batch of (idx, flip) pairs, the mirror draw forced per item."""
    from cmr_data.image_dataset import ImageDataset
    wrap = ImageDataset(ds, img_size)
    saved = torch.randint
    it = iter([int(f) for f in flips])
    torch.randint = lambda *a, **k: torch.tensor([next(it)])
    try:
        items = [wrap[int(i)] for i in idx]
    finally:
        torch.randint = saved
    out = [torch.stack([t[k] for t in items]) for k in range(len(items[0]))]
    out[-1] = out[-1].squeeze(-1)
    return out


@pytest.mark.parametrize('sizes', [RD.R, list(RD.SIZES)], ids=['single', 'list'])
@pytest.mark.parametrize('name', ['cub', 'p3d'])
def test_kernel_batches_match_the_reference(gold, root, name, sizes):
    ds = make(root, name, sizes).to_device(DEV)
    n = len(ds)
    idx = torch.arange(n, dtype=torch.int32, device=DEV)
    diff, total = 0, 0
    for f in (0, 1):
        out = [t.cpu() for t in ds.gather(idx, torch.full((n,), f, dtype=torch.uint8, device=DEV))]
        extra = len(sizes) - 1 if isinstance(sizes, list) else 0
        X, scale, trans, rot, ind = out[0], *out[1 + extra:]
        img, mask = golden_img(gold, name, f), golden_img(gold, name, f, 'mask')
        want = np.concatenate([(img * 2 - 1) * mask[:, None], mask[:, None]], axis=1)
        assert ulps(X.numpy(), want) <= 1
        diff, total = diff + not_identical(X.numpy(), want), total + want.size
        for k, e in zip(RD.SIZES[1:], out[1:1 + extra]):
            ik, mk = golden_img(gold, name, f, f'img_{k}'), golden_img(gold, name, f, f'mask_{k}')
            w = (ik * 2 - 1) * mk[:, None]
            assert ulps(e.numpy(), w) <= 1
            diff, total = diff + not_identical(e.numpy(), w), total + w.size
        pose = gold[f'{name}_flip{f}_sfm_pose']
        assert np.array_equal(bits(scale.numpy()), bits(pose[:, :1].astype(np.float32)))
        assert np.array_equal(bits(trans.numpy()), bits(np.concatenate([pose[:, 1:3], np.zeros((n, 1))], 1).astype(np.float32)))
        assert np.array_equal(bits(rot.numpy()), bits(pose[:, 3:].astype(np.float32)))
        assert ind.dtype == torch.int64 and ind.tolist() == [i + n * f for i in range(n)]
    print(f'{name} {sizes}: {diff} of {total} image elements not bit-identical to the reference (all within 1 ulp)')
    # mixed flips and repeated indices
    sel, fl = [3, 0, 3, n - 1, 1], [1, 0, 0, 1, 1]
    out = ds.gather(torch.tensor(sel, dtype=torch.int32, device=DEV), torch.tensor(fl, dtype=torch.uint8, device=DEV))
    ref = host_batch(make(root, name, sizes), sel, fl, sizes)
    for a, b in zip(out, ref):
        assert a.dtype == b.dtype and ulps(a.cpu().float().numpy(), b.float().numpy()) <= 1


def test_kernel_equals_the_host_restatement_at_cfg4():
    from cmr_data.cub import CUBDataset
    from tools.time_recon_data import write_cub_like_tree
    root = write_cub_like_tree(tempfile.mkdtemp(), 50, seed=5)
    ds = CUBDataset('train', True, 256, root=root).to_device(DEV)
    assert ds.windows()[:, 4].max() > 256 and ds.windows()[:, 4].min() < 256          # down- and upscaled crops
    g = torch.Generator().manual_seed(1)
    idx, fl = torch.randperm(50, generator=g), torch.randint(0, 2, (50,), generator=g)
    out = ds.gather(idx.to(torch.int32).to(DEV), fl.to(torch.uint8).to(DEV))
    ref = host_batch(CUBDataset('train', True, 256, root=root), idx, fl, 256)
    assert out[0].shape == (50, 4, 256, 256)
    assert not_identical(out[0].cpu().numpy(), ref[0].numpy()) == 0                    # same taps, same products
    for a, b in zip(out[1:], ref[1:]):
        assert torch.equal(a.cpu(), b)


def test_kernel_equals_the_host_restatement_at_1024_from_a_3141_window():
    from cmr_data.cub import CUBDataset
    from tools.time_recon_data import write_cub_like_tree
    root = write_cub_like_tree(tempfile.mkdtemp(), 2, seed=2, hw=(3141, 3141), ext='png', boxes=[(1, 1, 3141, 3141)] * 2)
    ds = CUBDataset('train', True, [1024, 299], root=root).to_device(DEV)
    ww, wh, _, _, S = ds.windows()[0, :5]
    assert (ww, wh) == (3141, 3141) and S > 3141
    for f in (0, 1):
        out = ds.gather(torch.zeros(1, dtype=torch.int32, device=DEV), torch.full((1,), f, dtype=torch.uint8, device=DEV))
        ref = host_batch(CUBDataset('train', True, [1024, 299], root=root), [0], [f], [1024, 299])
        for a, b in zip(out, ref):
            assert a.shape == b.shape and not_identical(a.cpu().float().numpy(), b.float().numpy()) == 0


def test_bad_arguments_are_errors(root):
    import ctypes
    import b3d
    from b3d.data import image_batch
    ds = make(root, 'cub').to_device(DEV)
    st, n = ds.store, len(ds)
    out = list(ds.batch_outputs(2))
    idx = torch.zeros(2, dtype=torch.int32, device=DEV)
    with pytest.raises(b3d.B3DError, match='pixels must be a contiguous'):
        image_batch(st['pixels'].cpu(), st['offsets'], st['geometry'], st['poses'], idx, None, out[:1], *out[1:])
    with pytest.raises(b3d.B3DError, match='image output 0'):
        image_batch(st['pixels'], st['offsets'], st['geometry'], st['poses'], idx, None, [out[0][:, :3]], *out[1:])
    with pytest.raises(b3d.B3DError, match='idx'):
        image_batch(st['pixels'], st['offsets'], st['geometry'], st['poses'], idx.long(), None, out[:1], *out[1:])
    # the C entry itself: a host pointer, a null pointer
    res = (ctypes.c_int32 * 1)(RD.R)
    imgs = (ctypes.c_void_p * 1)(out[0].data_ptr())
    host = st['geometry'].cpu()
    args = [st['pixels'].data_ptr(), st['offsets'].data_ptr(), host.data_ptr(), st['poses'].data_ptr(), n, idx.data_ptr(),
            None, 2, 1, ctypes.cast(res, ctypes.c_void_p), ctypes.cast(imgs, ctypes.c_void_p)] + \
        [t.data_ptr() for t in out[1:]] + [torch.cuda.current_stream().cuda_stream]
    assert b3d.lib.b3d_image_batch(*args) == -1 and b'geometry is not device memory' in b3d.lib.b3d_last_error()
    args[2] = None
    assert b3d.lib.b3d_image_batch(*args) == -1 and b'null store pointer' in b3d.lib.b3d_last_error()
    # an index outside the store, or a record with S < 1: NaN rows and ind -1, the other rows untouched
    with pytest.raises(b3d.B3DError, match='index range'):
        ds.gather(torch.tensor([0, n], dtype=torch.int32, device=DEV))
    o = ds.batch_outputs(3)
    st['geometry'][2, 4] = 0
    ds._gather(torch.tensor([1, n + 5, 2], dtype=torch.int32, device=DEV), None, o)
    for b in (1, 2):
        assert torch.isnan(o[0][b]).all() and torch.isnan(o[1][b]).all() and torch.isnan(o[3][b]).all()
        assert int(o[4][b]) == -1
    assert not torch.isnan(o[0][0]).any() and int(o[4][0]) == 1
    with pytest.raises(b3d.B3DError, match='CUDA device'):
        make(root, 'cub').to_device('cpu')
    torch.cuda.synchronize()


def test_train_batches_keep_the_last_partial_batch(root):
    from data.abstract_dataset import epoch_flips, epoch_order
    ds = make(root, 'cub').to_device(DEV)
    n = len(ds)
    got = list(ds.train_batches(3, 4, seed=2))
    assert [b[0].shape[0] for b in got] == [3] * (n // 3) + [n % 3]
    order, flips = epoch_order(n, 4, seed=2), epoch_flips(n, 4, seed=2)
    ind = torch.cat([b[4].cpu() for b in got])
    assert torch.equal(ind, order + n * flips.long())
    ref = host_batch(make(root, 'cub'), order, flips, RD.R)
    X = torch.cat([b[0].cpu() for b in got])
    assert ulps(X.numpy(), ref[0].numpy()) <= 1
    # a validation split: never mirrored
    val = make(root, 'cub', is_train=False).to_device(DEV)
    assert (torch.cat([b[4].cpu() for b in val.train_batches(4, 0)]) < n).all()
    ev = list(val.eval_batches(4, rank=1, world=2))
    a, b = n // 2, n
    assert torch.cat([e[4].cpu() for e in ev]).tolist() == list(range(a, b))


@pytest.fixture(scope='module')
def cfg4_root():
    from tools.time_recon_data import write_cub_like_tree
    return write_cub_like_tree(tempfile.mkdtemp(), 12, seed=7)


@pytest.fixture(scope='module')
def tpl16():
    from rendering.mesh_template import MeshTemplate
    from tools.uvsphere import write_uvsphere_obj
    return MeshTemplate(write_uvsphere_obj(os.path.join(tempfile.mkdtemp(), "uvsphere_16rings.obj"), rings=16), device=DEV)


def test_training_step_on_device_batches_equals_host_batches(cfg4_root, tpl16):
    from cmr_data.cub import CUBDataset
    from reconstruction_training import ReconTrainer, default_args
    ds = CUBDataset('train', True, 256, root=cfg4_root).to_device(DEV)
    sel, fl = [4, 0, 9, 4, 11, 2, 7, 1], [1, 0, 1, 0, 0, 1, 1, 0]
    dev_batch = ds.gather(torch.tensor(sel, dtype=torch.int32, device=DEV), torch.tensor(fl, dtype=torch.uint8, device=DEV))
    host = [t.to(DEV) for t in host_batch(CUBDataset('train', True, 256, root=cfg4_root), sel, fl, 256)]
    out = []
    for batch in (dev_batch, host):
        torch.manual_seed(4321)
        tr = ReconTrainer(default_args(), tpl16, dataset_size=len(ds), device=DEV)
        loss, recon, flat, miou = tr.step(*batch)
        out.append((float(loss), float(recon), float(miou),
                    {k: float(p.grad.norm()) for k, p in tr.generator.named_parameters() if p.grad is not None}))
    (l_k, r_k, m_k, g_k), (l_t, r_t, m_t, g_t) = out
    assert abs(l_k - l_t) <= 1e-5 * abs(l_t) and abs(r_k - r_t) <= 1e-5 * abs(r_t) and abs(m_k - m_t) < 1e-4
    floor = 1e-5 * max(g_t.values())
    for k in g_t:
        assert abs(g_k[k] - g_t[k]) <= 1e-4 * g_t[k] + floor, (k, g_k[k], g_t[k])


def test_evaluate_on_eval_batches_equals_host_batches(cfg4_root, tpl16):
    from cmr_data.cub import CUBDataset
    from cmr_data.image_dataset import ImageDataset
    from reconstruction_training import ReconTrainer, default_args
    ds = CUBDataset('train', False, 256, root=cfg4_root).to_device(DEV)
    torch.manual_seed(4321)
    tr = ReconTrainer(default_args(), tpl16, dataset_size=len(ds), device=DEV)
    a = tr.evaluate(ds.eval_batches(5))
    loader = torch.utils.data.DataLoader(ImageDataset(CUBDataset('train', False, 256, root=cfg4_root), 256), batch_size=5)
    b = tr.evaluate([[t.to(DEV) for t in batch] for batch in loader])
    assert a['N'] == b['N'] == len(ds)
    for k in ('recon_loss', 'flat_loss', 'miou'):
        assert abs(a[k] - b[k]) <= 1e-5 * abs(b[k]), (k, a[k], b[k])


def test_graph_capture_replays_on_new_indices(root):
    ds = make(root, 'p3d', list(RD.SIZES)).to_device(DEV)
    B = 4
    idx = torch.zeros(B, dtype=torch.int32, device=DEV)
    flip = torch.zeros(B, dtype=torch.uint8, device=DEV)
    out = ds.batch_outputs(B)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ds.gather(idx, flip, out)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ds.gather(idx, flip, out)
    for sel, fl in (([3, 0, 4, 4], [1, 0, 1, 0]), ([2, 1, 0, 3], [0, 0, 1, 1])):
        idx.copy_(torch.tensor(sel, dtype=torch.int32, device=DEV))
        flip.copy_(torch.tensor(fl, dtype=torch.uint8, device=DEV))
        graph.replay()
        torch.cuda.synchronize()
        eager = ds.gather(idx.clone(), flip.clone())
        for a, b in zip(out, eager):
            assert torch.equal(a, b)
