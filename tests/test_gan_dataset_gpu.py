"""The device path of the GAN datasets on the GPU: b3d_gather_fields batches equal the reference loader's batches bit for
bit (tests/golden/dataset_reference.npz), host storage equals device storage, bad arguments are errors, and the batches feed
GANTrainer, FIDEvaluator and a captured CUDA graph exactly like the tensors torch builds from the records."""
import os
import sys
import tempfile

import numpy as np
import pytest
import torch

from conftest import GOLDEN

sys.path.insert(0, GOLDEN)
import dataset_common as DC                                    # noqa: E402
from test_gan_dataset_hostlogic import CLASSES, batch, bits, items, torch_batch  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope='module')
def gold():
    return np.load(os.path.join(GOLDEN, 'dataset_reference.npz'))


@pytest.fixture(scope='module')
def root(gold, tmp_path_factory):
    r = str(tmp_path_factory.mktemp('gan_data_gpu'))
    DC.write_tree(r, {k[3:]: gold[k] for k in gold.files if k.startswith('in_')})
    return r


def packed(root, name, storage='device', include_image=False, **kw):
    return CLASSES[name](DC.make_args(name, **kw), root=root).to_device(DEV, storage=storage, include_image=include_image)


def same_bits(a, b):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a
    return np.array_equal(bits(a), bits(b))


@pytest.mark.parametrize('storage', ['device', 'host'])
@pytest.mark.parametrize('name', ['cub', 'p3d'])
def test_gather_is_bit_exact(gold, root, name, storage):
    ds = packed(root, name, storage)
    n = len(ds)
    idx = torch.arange(n, dtype=torch.int32, device=DEV)
    for f in (1, 0):
        out = ds.gather(idx, torch.full((n,), f, dtype=torch.uint8, device=DEV))
        for key, k in (('X_tex', 'texture'), ('X_alpha', 'texture_alpha'), ('X_mesh', 'mesh')):
            assert out[key].dtype == torch.float32 and same_bits(out[key], items(gold, name, k, f)), (f, k)
        assert torch.equal(out['C'].cpu(), torch.from_numpy(gold[f'{name}_flip{f}_class']))
    # the reference loader's batch: repeated indices, mixed flips
    bi = torch.tensor(gold[f'{name}_batch_idx'], dtype=torch.int32, device=DEV)
    bf = torch.tensor(gold[f'{name}_batch_flip'], dtype=torch.uint8, device=DEV)
    out = ds.gather(bi, bf)
    for key, k in (('X_tex', 'texture'), ('X_alpha', 'texture_alpha'), ('X_mesh', 'mesh')):
        assert same_bits(out[key], batch(gold, name, k)), k
    assert torch.equal(out['C'].cpu(), torch.from_numpy(gold[f'{name}_batch_class']))
    # B = 1, no flip tensor
    out = ds.gather(bi[:1])
    assert same_bits(out['X_tex'], items(gold, name, 'texture', 0)[int(bi[0])][None])


@pytest.mark.parametrize('name', ['cub', 'p3d'])
def test_host_storage_equals_device_storage(root, name):
    a, b = packed(root, name, 'device', True), packed(root, name, 'host', True)
    assert a.store['texture'].is_cuda and b.store['texture'].is_pinned()
    for x, y in zip(a.train_batches(5, 3, seed=2), b.train_batches(5, 3, seed=2)):
        for k in x:
            assert torch.equal(x[k], y[k]), k
    for x, y in zip(a.eval_batches(5), b.eval_batches(5)):
        for k in x:
            assert torch.equal(x[k], y[k]), k


@pytest.mark.parametrize('kw', [dict(), dict(texture_only=True), dict(conditional_class=False)])
@pytest.mark.parametrize('name', ['cub', 'p3d'])
def test_train_batches_equal_the_torch_batches(root, name, kw):
    from data.abstract_dataset import epoch_flips, epoch_order
    ds = packed(root, name, **kw)
    B = 3
    for epoch in (0, 1):
        order = epoch_order(len(ds), epoch, seed=5)
        flips = epoch_flips(len(order), epoch, seed=5)
        got = list(ds.train_batches(B, epoch, seed=5))
        assert len(got) == len(ds) // B
        for k, b in enumerate(got):
            ref = torch_batch(ds, order[k * B:(k + 1) * B], flips[k * B:(k + 1) * B], kw.get('texture_only', False))
            assert sorted(b) == ['C', 'X_alpha', 'X_mesh', 'X_tex']
            for key in ('X_tex', 'X_alpha', 'X_mesh'):
                if ref[key] is None:
                    assert b[key] is None
                else:
                    assert torch.equal(b[key].cpu().view(torch.int32), ref[key].view(torch.int32)), key
            if kw.get('conditional_class', True):
                assert torch.equal(b['C'].cpu(), ref['C'])
            else:
                assert b['C'] is None
    # augmentation off: never mirrored
    ds.args.evaluate = True
    order = epoch_order(len(ds), 0)
    b = next(ds.train_batches(B, 0))
    assert torch.equal(b['X_tex'].cpu(), torch_batch(ds, order[:B], [0] * B)['X_tex'])


@pytest.mark.parametrize('name', ['cub', 'p3d'])
def test_eval_batches_equal_the_reference_items(gold, root, name):
    ds = packed(root, name, include_image=True)
    n = len(ds)
    for world in (1, 2):
        seen = []
        for rank in range(world):
            for d in ds.eval_batches(5, rank, world):
                i = d['idx'].cpu().numpy()
                seen.extend(i.tolist())
                assert sorted(d) == ['class', 'idx', 'image', 'mesh', 'rotation', 'scale', 'texture', 'texture_alpha',
                                     'translation']
                for k in ('scale', 'translation', 'rotation', 'image'):
                    assert same_bits(d[k], gold[f'{name}_eval_{k}'][i]), k
                for k in ('texture', 'texture_alpha', 'mesh'):
                    assert same_bits(d[k], items(gold, name, k, 0)[i]), k
                assert np.array_equal(d['class'].cpu().numpy(), gold[f'{name}_eval_class'][i])
        assert seen == list(range(n))
    sizes = [d['idx'].numel() for d in ds.eval_batches(5)]
    assert sizes == [5] * (n // 5) + ([n % 5] if n % 5 else [])
    assert 'image' not in next(packed(root, name).eval_batches(4))


def test_bad_arguments_are_errors(root):
    import b3d
    from b3d.data import gather_fields
    ds = packed(root, 'cub')
    n = len(ds)
    idx = torch.zeros(2, dtype=torch.int32, device=DEV)
    out = torch.empty(2, 3, DC.R, DC.R, device=DEV)
    with pytest.raises(b3d.B3DError, match='not device-accessible'):
        gather_fields([(ds.store['texture'].cpu(), out, True, 1.0, 0.0)], idx)           # pageable host store
    with pytest.raises(b3d.B3DError, match='dtype'):
        gather_fields([(ds.store['texture'].double(), out, True, 1.0, 0.0)], idx)
    with pytest.raises(b3d.B3DError, match='output'):
        gather_fields([(ds.store['texture'], out.half(), True, 1.0, 0.0)], idx)
    with pytest.raises(b3d.B3DError, match='idx'):
        gather_fields([(ds.store['texture'], out, True, 1.0, 0.0)], idx.long())
    with pytest.raises(b3d.B3DError, match='index range'):
        ds.gather(torch.tensor([0, n], dtype=torch.int32, device=DEV))
    with pytest.raises(b3d.B3DError, match='index range'):
        ds.gather(torch.tensor([-1, 0], dtype=torch.int32, device=DEV))
    # without the host-side check the kernel writes NaN / -1 rows for an index outside the store
    o = ds.batch_outputs(2)
    ds._gather_train(torch.tensor([1, n + 5], dtype=torch.int32, device=DEV), None, o)
    assert torch.isnan(o['X_tex'][1]).all() and not torch.isnan(o['X_tex'][0]).any() and int(o['C'][1, 0]) == -1
    with pytest.raises(ValueError, match='storage'):
        ds.to_device(DEV, storage='disk')
    torch.cuda.synchronize()


@pytest.fixture(scope='module')
def root256():
    """4 CUB records at 256^2 with 299^2 images: the GAN and the FID evaluation run at their real sizes."""
    r = tempfile.mkdtemp()
    DC.write_tree(r, DC.make_inputs(seed=3, res=256, n=4, img=299), datasets=('cub',))
    return r


@pytest.fixture(scope='module')
def tpl16():
    from rendering.mesh_template import MeshTemplate
    from tools.uvsphere import write_uvsphere_obj
    return MeshTemplate(write_uvsphere_obj(os.path.join(tempfile.mkdtemp(), "uvsphere_16rings.obj"), rings=16), device=DEV)


def test_training_steps_equal_the_torch_fed_steps(root256, tpl16):
    import bench
    from data.abstract_dataset import epoch_flips, epoch_order
    from gan_training import GANTrainer
    args = bench.gan_args(256, 2)
    ds = CLASSES['cub'](DC.make_args('cub', texture_resolution=256), root=root256).to_device(DEV)
    B = 2
    order, flips = epoch_order(len(ds), 0, seed=1), epoch_flips(len(ds), 0, seed=1)
    g = torch.Generator().manual_seed(9)
    noise = [torch.randn(B, args.latent_dim, generator=g).to(DEV) for _ in range(2)]
    fed = [dict(b, noise=z) for b, z in zip(ds.train_batches(B, 0, seed=1), noise)]
    ref = []
    for k, z in enumerate(noise):
        t = torch_batch(ds, order[k * B:(k + 1) * B], flips[k * B:(k + 1) * B])
        ref.append({key: v.to(DEV) for key, v in t.items()} | {'noise': z})
    assert any(bool(f) for f in flips[:2 * B]) and not all(bool(f) for f in flips[:2 * B])
    losses = []
    for batches in (fed, ref, fed):
        torch.manual_seed(4)
        tr = GANTrainer(args, mesh_template=tpl16, device=DEV)
        losses.append([float(x) for x in tr.train_epoch(batches)])          # one G step, one D step
    # identical inputs: the losses differ at most by the trainer's own run-to-run spread (zero when deterministic)
    spread = max(abs(a - b) for a, b in zip(losses[0], losses[2]))
    assert len(losses[0]) == 2 and all(abs(a - b) <= 4 * spread for a, b in zip(losses[0], losses[1])), losses


def test_fid_evaluation_equals_the_loader_dicts(root256, tpl16):
    import bench
    from fid_common import randomize_inception
    from fid_evaluation import FIDEvaluator
    from data.abstract_dataset import AbstractDatasetForEvaluation
    from models.gan import Generator
    from utils.inception import InceptionV3
    args = bench.gan_args(256, 2)
    torch.manual_seed(2)
    G = Generator(args, args.latent_dim, symmetric=True, mesh_head=True).to(DEV).eval()
    inc = randomize_inception(InceptionV3([2], weights=None), 6)
    ds = CLASSES['cub'](DC.make_args('cub', texture_resolution=256), root=root256).to_device(DEV, include_image=True)
    loader = torch.utils.data.DataLoader(AbstractDatasetForEvaluation(ds), batch_size=3, shuffle=False)
    a = FIDEvaluator(G, tpl16, inception=inc, device=DEV).evaluate(ds.eval_batches(3), seed=1234, keep_features=True)
    b = FIDEvaluator(G, tpl16, inception=inc, device=DEV).evaluate(loader, seed=1234, keep_features=True)
    assert a['num_generated'] == b['num_generated'] == len(ds)
    for k in b['features']:
        x, y = a['features'][k], b['features'][k]
        assert float((x - y).abs().max()) <= 1e-5 * float(y.abs().max()), k
    for k in ('fid', 'fid_texture_only', 'fid_mesh_only'):
        assert abs(a[k] - b[k]) <= 1e-5 * abs(b[k]), k


def test_graph_capture_replays_on_new_indices(gold, root):
    ds = packed(root, 'cub')
    B = 4
    idx = torch.zeros(B, dtype=torch.int32, device=DEV)
    flip = torch.zeros(B, dtype=torch.uint8, device=DEV)
    out = ds.batch_outputs(B)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ds.gather(idx, flip, out)
        y = out['X_tex'] * out['X_alpha'] + out['X_mesh'].sum()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ds.gather(idx, flip, out)
        y = out['X_tex'] * out['X_alpha'] + out['X_mesh'].sum()
    for sel, fl in (([3, 0, 7, 7], [1, 0, 1, 0]), ([11, 2, 5, 9], [0, 0, 1, 1])):
        idx.copy_(torch.tensor(sel, dtype=torch.int32, device=DEV))
        flip.copy_(torch.tensor(fl, dtype=torch.uint8, device=DEV))
        graph.replay()
        torch.cuda.synchronize()
        tex = np.stack([items(gold, 'cub', 'texture', f)[i] for i, f in zip(sel, fl)])
        alpha = np.stack([items(gold, 'cub', 'texture_alpha', f)[i] for i, f in zip(sel, fl)])
        mesh = np.stack([items(gold, 'cub', 'mesh', f)[i] for i, f in zip(sel, fl)])
        assert same_bits(out['X_tex'], tex) and same_bits(out['X_alpha'], alpha) and same_bits(out['X_mesh'], mesh)
        expect = out['X_tex'] * out['X_alpha'] + out['X_mesh'].sum()
        assert torch.equal(y, expect)
