"""Host logic of the pseudo-ground-truth export (pseudo_gt_export.py) on the CPU: the render-resolution and texture-resize
rule, the P3D ImageNet subset, poses metadata in index order, records cloned out of a staged batch (readable by the
reference's dataset class, one sample per file), and that the exporter refuses to run without CUDA."""
import os
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN


def test_renderer_resolution_and_texture_resize():
    from pseudo_gt_export import renderer_resolution, resize_texture
    assert renderer_resolution(512) == 1024 and renderer_resolution(256) == 1024 and renderer_resolution(16) == 1024
    assert renderer_resolution(600) == 1200
    t = torch.rand(2, 3, 128, 128)
    assert resize_texture(t, 1024) is t                       # 128 = 1024 // 8: kept as it is
    big = torch.rand(2, 3, 256, 256)
    r = resize_texture(big, 1024)
    assert r.shape == (2, 3, 128, 128)
    assert torch.equal(r, F.interpolate(big, size=(128, 128), mode='bilinear', align_corners=False))
    assert resize_texture(big, 2048) is big


def test_p3d_imagenet_subset():
    from pseudo_gt_export import imagenet_rows
    paths = ['car_imagenet/n1.JPEG', 'car_pascal/2008_1.jpg', 'car_imagenet/n2.JPEG', 'x/car_imagenet.jpg']
    assert imagenet_rows(paths) == [0, 2]


def _staged(B=3, R=8, C=3, seed=0):
    """A host byte buffer laid out like one staged batch, with seeded contents."""
    from pseudo_gt_export import _layout, _views
    lay, nbytes = _layout(B, C, R, (3, 6, 6), (3, 32, 32))
    buf = torch.zeros(nbytes, dtype=torch.uint8)
    v = _views(buf, lay)
    g = torch.Generator().manual_seed(seed)
    for k in ('texture', 'texture_alpha', 'image'):
        v[k].copy_((torch.rand(v[k].shape, generator=g) * 2 - 1).half())
    v['mesh'].copy_(torch.randn(v['mesh'].shape, generator=g) * 0.05)
    v['pose'].copy_(torch.rand(B, 8, generator=g))
    v['ind'].copy_(torch.tensor([7, 2, 5][:B]))
    return buf, lay, v


def test_layout_is_aligned_and_disjoint():
    from pseudo_gt_export import _layout
    lay, nbytes = _layout(5, 4, 16, (3, 12, 12), (3, 32, 32))
    spans = sorted((o, o + int(np.prod(s)) * torch.empty(0, dtype=dt).element_size()) for o, dt, s in lay.values())
    assert all(o % 16 == 0 for o, _ in spans)
    assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:])) and spans[-1][1] <= nbytes


def test_poses_metadata_in_index_order_with_the_dataset_paths(tmp_path):
    from data.pseudo_gt import load_poses_metadata
    from pseudo_gt_export import staged_records, write_poses_metadata
    _, _, v = _staged()
    poses = {idx: pose for idx, _, pose in staged_records(v)}
    paths = [f'img{i}.jpg' for i in range(10)]
    ordered = write_poses_metadata(str(tmp_path), poses, paths)
    assert ordered == ['img2.jpg', 'img5.jpg', 'img7.jpg']
    d = load_poses_metadata(str(tmp_path))
    rows = v['pose'][[1, 2, 0]]
    assert d['path'] == ordered
    assert torch.equal(d['scale'], rows[:, :1]) and torch.equal(d['translation'], rows[:, 1:4])
    assert torch.equal(d['rotation'], rows[:, 4:])
    assert d['scale'].shape == (3, 1) and d['translation'].shape == (3, 3) and d['rotation'].shape == (3, 4)


def test_staged_records_are_per_sample_clones(tmp_path):
    """A record sliced out of the slot would pickle the slot's whole storage; the clones carry one sample each, so a written
    file is about one record's size whatever the batch size."""
    from data.pseudo_gt import load_pseudo_ground_truth, pseudo_gt_dir, save_pseudo_gt
    from pseudo_gt_export import staged_records
    sizes = {}
    for B in (1, 3):
        _, _, v = _staged(B=B, R=32)
        recs = staged_records(v)
        for idx, rec, _ in recs:
            for k, t in rec.items():
                assert t.untyped_storage().nbytes() == t.numel() * t.element_size(), k
        idx, rec, _ = recs[0]
        assert rec['mesh'].dtype == torch.float32 and rec['texture'].dtype == torch.float16
        d = pseudo_gt_dir(str(tmp_path / f'b{B}'), 32)
        save_pseudo_gt(d, idx, rec)
        sizes[B] = os.path.getsize(os.path.join(d, f'{idx}.npz'))
        back = load_pseudo_ground_truth(str(tmp_path / f'b{B}'), 32, idx)
        assert torch.equal(back['texture'], v['texture'][0].float())
        assert torch.equal(back['mesh'], v['mesh'][0])
    assert sizes[3] < 1.2 * sizes[1], sizes


def test_staged_record_reads_back_as_the_reference_dataset_reads_it(tmp_path):
    """reference_pins.npz holds what the reference's AbstractDataset.load_pseudo_ground_truth / mirror_tex returned for the
    record of test_pseudo_gt_format._record(seed=3); the same planes staged in a batch buffer and written from there must read
    back identically."""
    from data.pseudo_gt import load_pseudo_ground_truth, mirror_tex, pseudo_gt_dir, save_pseudo_gt
    from pseudo_gt_export import _layout, _views, staged_records
    from test_pseudo_gt_format import _record
    pins = np.load(os.path.join(GOLDEN, "reference_pins.npz"))
    rec = _record(seed=3)
    lay, nbytes = _layout(2, rec['texture'].shape[0], rec['texture'].shape[1], rec['image'].shape, rec['mesh'].shape)
    buf = torch.zeros(nbytes, dtype=torch.uint8)
    v = _views(buf, lay)
    for k in ('mesh', 'texture', 'texture_alpha', 'image'):
        v[k][1].copy_(rec[k])
    v['ind'].copy_(torch.tensor([4, 0]))
    idx, staged, _ = staged_records(v)[1]
    assert idx == 0
    cache = os.path.join(str(tmp_path), "cache", "cub")
    save_pseudo_gt(pseudo_gt_dir(cache, 32), idx, staged)
    ours = load_pseudo_ground_truth(cache, 32, 0)
    assert sorted(ours) == [str(k) for k in pins["pgt_keys"]]
    for k in ours:
        theirs = pins["pgt_" + k]
        assert ours[k].shape == theirs.shape and ours[k].numpy().dtype == theirs.dtype and np.array_equal(ours[k].numpy(), theirs), k
    assert np.array_equal(mirror_tex(ours['texture']).numpy(), pins["pgt_mirror_tex"])


def test_exporter_refuses_without_cuda():
    import b3d
    from pseudo_gt_export import PseudoGTExporter
    trainer = types.SimpleNamespace(generator=torch.nn.Linear(1, 1), dataset_params=None,
                                    args=types.SimpleNamespace(optimize_deltas=False, optimize_z0=False))
    with pytest.raises(b3d.B3DError, match="CUDA"):
        PseudoGTExporter(trainer, mesh_template=None, pseudogt_resolution=16, inception=torch.nn.Identity())
