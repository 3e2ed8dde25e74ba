"""The reconstruction stage's image datasets on the host (cmr_data/): the drop-in CUBDataset / P3dDataset items and
ImageDataset tuples against the reference loaders run on a synthetic tree (tests/golden/recon_data_reference.npz, made by
make_golden_recon_data.py with OpenCV's resize), the pose table and crop windows of the device store, and the store sizes of
the shipped annotations' layout."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN

sys.path.insert(0, GOLDEN)
import recon_data_common as RD                                # noqa: E402


def classes():
    from cmr_data.cub import CUBDataset
    from cmr_data.p3d import P3dDataset
    return {'cub': CUBDataset, 'p3d': P3dDataset}


@pytest.fixture(scope='module')
def gold():
    return np.load(os.path.join(GOLDEN, 'recon_data_reference.npz'))


@pytest.fixture(scope='module')
def root(gold, tmp_path_factory):
    r = str(tmp_path_factory.mktemp('recon_data'))
    RD.write_tree(r, {k[3:]: gold[k] for k in gold.files if k.startswith('in_')})
    return r


def make(root, name, img_size=RD.R, is_train=True):
    return classes()[name]('train', is_train, img_size, root=root)


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view({4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def ordered(a):
    """fp32 -> int64 on a line where adjacent floats are adjacent integers (-0 and +0 both 0)."""
    i = np.ascontiguousarray(a, np.float32).view(np.int32).astype(np.int64)
    return np.where(i < 0, -(i & 0x7FFFFFFF), i)


def ulps(a, b):
    """Largest distance between two fp32 arrays in units in the last place, not counting differences below 1e-14: OpenCV
    and the restatement may differ by ~1e-15 in double (a tap weight of ~1e-15 in one, 0 in the other), which is a
    huge number of ulps around 0 and far below fp32's resolution of these [-1, 1] values."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    d = np.abs(ordered(a) - ordered(b))
    d[np.abs(a.astype(np.float64) - b) <= 1e-14] = 0
    return int(d.max())


def forced_items(ds, f, monkeypatch):
    monkeypatch.setattr(torch, 'randint', lambda *a, **k: torch.tensor([f]))
    try:
        return [ds[i] for i in range(len(ds))]
    finally:
        monkeypatch.undo()


def golden_img(gold, name, f, key='img'):
    v = gold[f'{name}_{key}']
    return v[..., ::-1] if f else v


@pytest.mark.parametrize('name', ['cub', 'p3d'])
def test_items_equal_the_reference_loader(gold, root, name, monkeypatch):
    ds = make(root, name)
    n = int(gold[f'in_{name}_n'])
    assert len(ds) == n and ds.get_paths() == [str(p) for p in gold[f'{name}_paths']]
    for f in (0, 1):
        items = forced_items(ds, f, monkeypatch)
        assert [it['mirrored'] for it in items] == [bool(f)] * n and [it['inds'] for it in items] == list(range(n))
        assert [it['path'] for it in items] == ds.get_paths()
        assert np.array_equal(bits(np.stack([it['sfm_pose'] for it in items])), bits(gold[f'{name}_flip{f}_sfm_pose']))
        assert np.array_equal(bits(np.stack([it['kp'] for it in items])), bits(gold[f'{name}_flip{f}_kp']))
        img = np.stack([it['img'] for it in items])
        mask = np.stack([it['mask'] for it in items])
        assert img.dtype == np.float64 and img.shape == (n, 3, RD.R, RD.R) and mask.shape == (n, RD.R, RD.R)
        assert ulps(img.astype(np.float32), golden_img(gold, name, f)) <= 1
        assert ulps(mask.astype(np.float32), golden_img(gold, name, f, 'mask')) <= 1


@pytest.mark.parametrize('name', ['cub', 'p3d'])
def test_image_dataset_tuples_equal_the_reference(gold, root, name, monkeypatch):
    from cmr_data.image_dataset import ImageDataset
    n = int(gold[f'in_{name}_n'])
    for img_size in (RD.R, list(RD.SIZES)):
        wrap = ImageDataset(make(root, name, img_size), img_size)
        for f in (0, 1):
            monkeypatch.setattr(torch, 'randint', lambda *a, **k: torch.tensor([f]))
            tuples = [wrap[i] for i in range(n)]
            monkeypatch.undo()
            img, mask = golden_img(gold, name, f), golden_img(gold, name, f, 'mask')
            pose = gold[f'{name}_flip{f}_sfm_pose']
            for i, t in enumerate(tuples):
                extra = len(img_size) - 1 if isinstance(img_size, list) else 0
                assert len(t) == 5 + extra
                X, scale, trans, rot, ind = t[0], *t[1 + extra:]
                want = (img[i] * 2 - 1) * mask[i][None]
                assert ulps(X[:3].numpy(), want) <= 1 and ulps(X[3].numpy(), mask[i]) <= 1
                assert np.array_equal(bits(scale.numpy()), bits(pose[i, :1].astype(np.float32)))
                assert np.array_equal(bits(trans.numpy()), bits(np.array([pose[i, 1], pose[i, 2], 0], np.float32)))
                assert np.array_equal(bits(rot.numpy()), bits(pose[i, 3:].astype(np.float32)))
                assert ind.tolist() == [i + n * f]
                for k, e in zip(RD.SIZES[1:], t[1:1 + extra]):
                    ik, mk = golden_img(gold, name, f, f'img_{k}')[i], golden_img(gold, name, f, f'mask_{k}')[i]
                    assert e.shape == (3, k, k) and ulps(e.numpy(), (ik * 2 - 1) * mk[None]) <= 1


def test_a_plain_dataloader_collates_the_tuples(root):
    from cmr_data.image_dataset import ImageDataset
    wrap = ImageDataset(make(root, 'cub'), RD.R)
    X, scale, trans, rot, ind = next(iter(torch.utils.data.DataLoader(wrap, batch_size=3, shuffle=False)))
    assert X.shape == (3, 4, RD.R, RD.R) and scale.shape == (3, 1) and trans.shape == (3, 3) and rot.shape == (3, 4)
    assert ind.shape == (3, 1)


@pytest.mark.parametrize('name', ['cub', 'p3d'])
def test_validation_items_are_never_mirrored(root, name):
    ds = make(root, name, is_train=False)
    assert not any(ds[i]['mirrored'] for i in range(len(ds)))


@pytest.mark.parametrize('name', ['cub', 'p3d'])
def test_pose_table_equals_the_item_poses(gold, root, name):
    ds = make(root, name)
    t = ds.pose_table()
    assert t.dtype == np.float32 and t.shape == (len(ds), 2, 8)
    for f in (0, 1):
        p = gold[f'{name}_flip{f}_sfm_pose']
        want = np.zeros((len(ds), 8), np.float32)
        want[:, :3], want[:, 4:] = p[:, :3], p[:, 3:]
        assert np.array_equal(bits(t[:, f]), bits(want))
    # the list form poses with its first size
    assert np.array_equal(bits(make(root, name, list(RD.SIZES)).pose_table()), bits(t))


@pytest.mark.parametrize('name', ['cub', 'p3d'])
def test_crop_windows_and_store_size(gold, root, name):
    from cmr_data.image_utils import crop
    ds = make(root, name)
    win = ds.windows()
    total = 0
    for i in range(len(ds)):
        ww, wh, wx0, wy0, S, px, py = (int(v) for v in win[i])
        mask = gold[f'in_{name}_mask{i}']
        # the window is exactly where the crop of an index image lands inside the photo
        h, w = mask.shape
        index = (np.arange(h * w).reshape(h, w) + 1).astype(np.float64)
        c = crop(index, ds.crop_box(i), bgval=0)[..., 0]
        assert c.shape == (S, S)
        inside = np.argwhere(c > 0)
        assert (inside.min(0).tolist(), (inside.max(0) - inside.min(0) + 1).tolist()) == ([wy0, wx0], [wh, ww])
        assert c[wy0, wx0] == py * w + px + 1
        total += ww * wh
    assert ds.packed_bytes() == 4 * total
    if name == 'cub':
        assert {20, 64, 83} <= set(win[:, 4].tolist())           # upscaled, halved exactly, non-integer downscale


def test_quaternion_conversions_round_trip():
    from cmr_data.transformations import quaternion_from_matrix, quaternion_matrix
    g = np.random.default_rng(3)
    for _ in range(200):
        q = g.normal(size=4)
        q /= np.linalg.norm(q)
        q *= np.sign(q[0])
        M = quaternion_matrix(q)
        assert np.allclose(M[:3, :3] @ M[:3, :3].T, np.eye(3), atol=1e-12)
        assert np.allclose(quaternion_from_matrix(M), q, atol=1e-12)
    assert np.array_equal(quaternion_from_matrix(np.identity(4)), [1, 0, 0, 0])
    with pytest.raises(NotImplementedError):
        quaternion_from_matrix(np.identity(4), isprecise=False)


def test_resize_restatement_matches_its_definition():
    """image_utils.resize against a per-pixel evaluation of the bilinear rule (independent of the vectorised form)."""
    from cmr_data.image_utils import resize
    g = np.random.default_rng(1)
    for S, R in ((83, 37), (64, 32), (20, 64), (7, 7)):
        img = g.random((S, S, 3))
        got = resize(img, R, R)
        scale = 1.0 / (R / S)

        def taps(d):
            fx = (d + 0.5) * scale - 0.5
            s = int(np.floor(fx))
            fx -= s
            if s < 0:
                s, fx = 0, 0.0
            if s >= S - 1:
                s, fx = S - 1, 0.0
            return s, min(s + 1, S - 1), 1.0 - fx, fx
        for y in (0, R // 2, R - 1):
            y0, y1, b0, b1 = taps(y)
            for x in (0, R // 3, R - 1):
                x0, x1, a0, a1 = taps(x)
                want = (img[y0, x0] * a0 + img[y0, x1] * a1) * b0 + (img[y1, x0] * a0 + img[y1, x1] * a1) * b1
                assert np.array_equal(got[y, x], want)
    assert resize(g.random((5, 5, 1)), 3, 3).shape == (3, 3)


def test_crop_window_lies_inside_photo_and_crop():
    """Boxes of the shipped annotations' kind (inside, the whole photo, past three borders): the window is never larger
    than its photo or its crop square."""
    from cmr_data.image_utils import crop_window, peturb_bbox, square_bbox
    for (h, w, box) in ((336, 500, (60, 27, 325, 304)), (188, 312, (1, 1, 312, 188)), (375, 500, (-40, 10, 560, 380))):
        sq = square_bbox(peturb_bbox(np.array(box, float) - 1, pf=0.05))
        x0, y0, wx0, wy0, ww, wh = crop_window(sq, h, w)
        S = int(round(sq[2])) - x0 + 1
        assert 0 < ww <= min(w, S) and 0 < wh <= min(h, S) and wx0 + ww <= S and wy0 + wh <= S
