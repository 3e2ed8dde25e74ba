"""The drop-in GAN datasets (data/abstract_dataset.py, cub_200_2011_dataset.py, pascal3d_plus_dataset.py) against the
reference's own classes run on a synthetic cache (tests/golden/dataset_reference.npz, make_golden_dataset.py), and the host
side of their device path: sampler orders, evaluation shards, the packed-store size.  No GPU."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN

sys.path.insert(0, GOLDEN)
import dataset_common as DC                                    # noqa: E402
from data.abstract_dataset import (AbstractDatasetForEvaluation, epoch_flips, epoch_order,  # noqa: E402
                                   epoch_seed, eval_shard)
from data.cub_200_2011_dataset import CubDataset               # noqa: E402
from data.pascal3d_plus_dataset import Pascal3DPlusDataset     # noqa: E402
from data.pseudo_gt import mirror_tex                          # noqa: E402

CLASSES = {'cub': CubDataset, 'p3d': Pascal3DPlusDataset}


@pytest.fixture(scope='module')
def gold():
    return np.load(os.path.join(GOLDEN, 'dataset_reference.npz'))


@pytest.fixture(scope='module')
def root(gold, tmp_path_factory):
    r = str(tmp_path_factory.mktemp('gan_data'))
    DC.write_tree(r, {k[3:]: gold[k] for k in gold.files if k.startswith('in_')})
    return r


def bits(t):
    return np.asarray(t, dtype=np.float32).view(np.int32)


def items(gold, name, k, flip):
    """The reference's __getitem__ planes k of every index (fp32): mirrored ones as recorded, unmirrored ones = the records
    (the generator checked that the reference returns them widened, bit for bit)."""
    if flip:
        return gold[f'{name}_flip1_{k}'].astype(np.float32)
    rec = gold[f'in_{name}_{k}']
    if name == 'p3d':
        rec = rec[[i for i, p in enumerate(gold['in_p3d_path']) if str(p).startswith('car_imagenet')]]
    return rec.astype(np.float32)


def batch(gold, name, k):
    """The reference loader's recorded batch: the items of its (index, flip) pairs."""
    return np.stack([items(gold, name, k, f)[i] for i, f in zip(gold[f'{name}_batch_idx'], gold[f'{name}_batch_flip'])])


def fixed_randint(monkeypatch, values):
    it = iter(values)
    monkeypatch.setattr(torch, 'randint', lambda *a, **k: torch.tensor([next(it)]))


@pytest.mark.parametrize('name', ['cub', 'p3d'])
def test_items_match_the_reference(gold, root, monkeypatch, name):
    args = DC.make_args(name)
    ds = CLASSES[name](args, root=root)
    n = int(gold[f'{name}_len'])
    assert len(ds) == n
    assert np.array_equal(np.stack(ds.classes), gold[f'{name}_classes'])
    assert tuple(ds.n_classes) == tuple(gold[f'{name}_n_classes']) and args.n_classes == ds.n_classes
    for f in (1, 0):
        fixed_randint(monkeypatch, [f] * n)
        its = [ds[i] for i in range(n)]
        for k in ('texture', 'texture_alpha', 'mesh'):
            got = np.stack([it[k].numpy() for it in its])
            assert got.dtype == np.float32
            assert np.array_equal(bits(got), bits(items(gold, name, k, f))), (f, k)
        assert np.array_equal(np.stack([it['class'] for it in its]), gold[f'{name}_flip{f}_class'])
        assert [it['idx'] for it in its] == list(range(n))
        assert sorted(its[0]) == ['class', 'idx', 'mesh', 'texture', 'texture_alpha']


@pytest.mark.parametrize('name', ['cub', 'p3d'])
def test_evaluation_items_match_the_reference(gold, root, name):
    ds = CLASSES[name](DC.make_args(name), root=root)
    its = [AbstractDatasetForEvaluation(ds)[i] for i in range(len(ds))]
    assert sorted(its[0]) == ['class', 'idx', 'image', 'mesh', 'rotation', 'scale', 'texture', 'texture_alpha',
                                'translation']
    for k in ('scale', 'translation', 'rotation', 'image'):
        assert np.array_equal(bits(np.stack([it[k].numpy() for it in its])), bits(gold[f'{name}_eval_{k}'])), k
    for k in ('texture', 'texture_alpha', 'mesh'):
        assert np.array_equal(bits(np.stack([it[k].numpy() for it in its])), bits(items(gold, name, k, 0))), k
    assert np.array_equal(np.stack([it['class'] for it in its]), gold[f'{name}_eval_class'])


@pytest.mark.parametrize('name', ['cub', 'p3d'])
def test_suggestions_match_the_reference(gold, root, name):
    args = DC.make_args(name)
    ds = CLASSES[name](args, root=root)
    sig = []
    for cc, col in ((False, False), (True, False), (True, True)):
        args.conditional_class, args.conditional_color = cc, col
        sig.append(ds.suggest_truncation_sigma())
    assert sig == list(gold[f'{name}_sigma'])
    nd = []
    for r in (32, 256, 512, 1024):
        args.texture_resolution = r
        nd.append(ds.suggest_num_discriminators())
    assert nd == list(gold[f'{name}_num_disc'])
    assert ds.suggest_mesh_template() == str(gold[f'{name}_template'])


@pytest.mark.parametrize('name', ['cub', 'p3d'])
def test_errors_match_the_reference(gold, tmp_path, name):
    inp = {k[3:]: gold[k] for k in gold.files if k.startswith('in_')}
    DC.write_tree(str(tmp_path / 'count'), inp, datasets=(name,), drop_file=(name, 4))
    assert str(gold[f'{name}_err_count']) == 'ValueError'
    with pytest.raises(ValueError, match='pseudo-ground-truth'):
        CLASSES[name](DC.make_args(name), root=str(tmp_path / 'count'))
    DC.write_tree(str(tmp_path / 'none'), inp, datasets=(name,), with_pseudo_gt=False)
    assert str(gold[f'{name}_err_nopgt']) == 'ValueError'
    with pytest.raises(ValueError, match='pseudo-ground-truth'):
        CLASSES[name](DC.make_args(name), root=str(tmp_path / 'none'))
    ds = CLASSES[name](DC.make_args(name, evaluate=True), root=str(tmp_path / 'none'))
    assert ds.has_pseudo_ground_truth == bool(gold[f'{name}_nopgt_has'])
    assert len(ds) == int(gold[f'{name}_nopgt_eval_len'])
    assert sorted(AbstractDatasetForEvaluation(ds)[0]) == list(gold[f'{name}_nopgt_eval_keys'])
    with pytest.raises(ValueError, match='conditional_text'):
        CLASSES[name](DC.make_args(name, conditional_text=True), root=str(tmp_path / 'none'))


def torch_batch(ds, idx, flip, texture_only=False):
    """The batch restated in torch from the records: gather + mirror_tex + collate, as main.py's loader yields it."""
    recs = [ds.load_pseudo_ground_truth(int(i)) for i in idx]
    out = {}
    for key, k in (('X_tex', 'texture'), ('X_alpha', 'texture_alpha'), ('X_mesh', 'mesh')):
        out[key] = torch.stack([mirror_tex(r[k]) if f else r[k] for r, f in zip(recs, flip)])
    if texture_only:
        out['X_mesh'] = None
    out['C'] = torch.as_tensor(np.stack([ds.classes[int(i)] for i in idx]))
    return out


@pytest.mark.parametrize('name', ['cub', 'p3d'])
def test_torch_restatement_equals_the_reference_batch(gold, root, name):
    ds = CLASSES[name](DC.make_args(name), root=root)
    b = torch_batch(ds, gold[f'{name}_batch_idx'], gold[f'{name}_batch_flip'])
    for key, k in (('X_tex', 'texture'), ('X_alpha', 'texture_alpha'), ('X_mesh', 'mesh')):
        assert np.array_equal(bits(b[key].numpy()), bits(batch(gold, name, k))), k
    assert np.array_equal(b['C'].numpy(), gold[f'{name}_batch_class'])
    assert b['C'].dtype == torch.int64


@pytest.mark.parametrize('n,batch', [(12, 4), (37, 5), (100, 32)])
@pytest.mark.parametrize('seed', [0, 7])
def test_order_is_torchs_sampler(n, batch, seed):
    for epoch in range(3):
        # single process: RandomSampler with a generator seeded from (seed, epoch)
        order = epoch_order(n, epoch, seed)
        g = torch.Generator()
        g.manual_seed(epoch_seed(seed, epoch))
        ref = list(torch.utils.data.BatchSampler(torch.utils.data.RandomSampler(range(n), generator=g), batch, True))
        assert [order[k * batch:(k + 1) * batch].tolist() for k in range(len(order) // batch)] == ref
        assert sorted(order.tolist()) == list(range(n))
        for world in (2, 3):
            per_rank = []
            for rank in range(world):
                s = torch.utils.data.DistributedSampler(range(n), num_replicas=world, rank=rank, shuffle=True, seed=seed)
                s.set_epoch(epoch)
                ref = list(torch.utils.data.BatchSampler(s, batch, True))
                o = epoch_order(n, epoch, seed, rank, world)
                assert [o[k * batch:(k + 1) * batch].tolist() for k in range(len(o) // batch)] == ref
                per_rank.append(o)
            assert set(torch.cat(per_rank).tolist()) == set(range(n))
    assert not torch.equal(epoch_order(n, 0, seed), epoch_order(n, 1, seed))


def test_flips_are_seeded_bernoulli():
    f = epoch_flips(4000, 3, seed=1)
    assert f.dtype == torch.uint8 and set(f.unique().tolist()) == {0, 1}
    assert abs(f.float().mean().item() - 0.5) < 0.04
    assert torch.equal(f, epoch_flips(4000, 3, seed=1))
    assert not torch.equal(f, epoch_flips(4000, 4, seed=1)) and not torch.equal(f, epoch_flips(4000, 3, seed=1, rank=1))


@pytest.mark.parametrize('n', [1, 7, 12, 100])
@pytest.mark.parametrize('world', [1, 2, 3, 8])
def test_eval_shards_partition_the_index_set(n, world):
    seen = []
    for rank in range(world):
        a, b = eval_shard(n, rank, world)
        assert a <= b
        seen.extend(range(a, b))
    assert seen == list(range(n))


@pytest.mark.parametrize('name', ['cub', 'p3d'])
def test_memory_estimate_matches_the_records(gold, root, name):
    ds = CLASSES[name](DC.make_args(name), root=root)
    n = len(ds)
    rec = {k: gold[f'in_{name}_{k}'][0] for k in ('texture', 'texture_alpha', 'mesh', 'image')}
    planes = n * (rec['texture'].nbytes + rec['texture_alpha'].nbytes + rec['mesh'].nbytes)
    cls = n * 8 * len(ds.classes[0])
    assert ds.packed_bytes() == planes + cls
    assert ds.packed_bytes(include_image=True) == planes + cls + n * rec['image'][:3].nbytes
    lay = ds.store_layout(include_image=True)
    assert lay['texture'] == ((n, 3, DC.R, DC.R), torch.float16) and lay['mesh'] == ((n, 3, 32, 32), torch.float32)
    assert lay['image'][0] == (n, 3, DC.IMG, DC.IMG) and lay['class'] == ((n, len(ds.classes[0])), torch.int64)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the CPU-only behaviour")
def test_to_device_without_a_gpu_raises(root):
    import b3d
    ds = CubDataset(DC.make_args('cub'), root=root)
    with pytest.raises(b3d.B3DError, match='no CPU fallback'):
        ds.to_device()
    with pytest.raises(ValueError, match='storage'):
        ds.to_device(storage='disk')
