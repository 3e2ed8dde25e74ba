"""Host logic of the reconstruction export: the photo crop square, the mirrored column map, PhotoFolder's files and the
flags of reconstruct.py."""
import types

import numpy as np
import pytest
import torch
from PIL import Image


def synthetic_masks():
    g = np.random.default_rng(4)
    out = []
    for h, w, box in ((40, 60, (5, 7, 30, 22)), (64, 48, (0, 10, 47, 63)), (30, 30, (12, 12, 12, 12)),
                      (50, 70, (1, 2, 68, 9)), (33, 45, (20, 3, 27, 31))):
        m = np.zeros((h, w), np.uint8)
        x0, y0, x1, y1 = box
        m[y0:y1 + 1, x0:x1 + 1] = g.random((y1 - y0 + 1, x1 - x0 + 1)) < 0.6
        m[y0, x0] = m[y1, x1] = 1                     # the box's corners are set
        out.append((m, box))
    return out


def test_crop_square_follows_the_cmr_rule():
    from cmr_data import image_utils
    from cmr_data.base import BaseDataset
    from cmr_data.photos import photo_crop_box, tight_box
    for mask, box in synthetic_masks():
        assert list(tight_box(mask)) == list(box)
        # a CMR dataset item whose annotated (1-based) box is the mask's tight box
        fake = types.SimpleNamespace(anno=[types.SimpleNamespace(bbox=types.SimpleNamespace(
            x1=box[0] + 1, y1=box[1] + 1, x2=box[2] + 1, y2=box[3] + 1))], padding_frac=0.05, jitter_frac=0,
            is_train=False)
        assert photo_crop_box(mask) == BaseDataset.crop_box(fake, 0)
        assert photo_crop_box(mask) == image_utils.square_bbox(image_utils.peturb_bbox(list(map(float, box)), pf=0.05))
    assert photo_crop_box(np.zeros((4, 4), np.uint8)) is None


@pytest.mark.parametrize("R", [2, 4, 8, 64, 256, 512])
def test_mirrored_column_map_equals_mirror_tex(R):
    from data.pseudo_gt import mirror_tex
    x = np.arange(R)
    mx = R - 1 - (x + R // 2) % R                    # b3d_recon_texture_pack's column map
    cols = mirror_tex(torch.arange(R).view(1, 1, R))[0, 0].numpy()
    assert np.array_equal(cols, mx)
    assert np.array_equal(mx[mx], x)                  # a reflection: mirrored twice is the identity


def write_photo(path, h=24, w=32, rgba=False, box=(4, 5, 20, 18)):
    rgb = (np.arange(h * w * 3) % 251).reshape(h, w, 3).astype(np.uint8)
    mask = np.zeros((h, w), np.uint8)
    x0, y0, x1, y1 = box
    mask[y0:y1 + 1, x0:x1 + 1] = 200
    if rgba:
        Image.fromarray(np.dstack([rgb, mask]), 'RGBA').save(path)
    else:
        Image.fromarray(rgb).save(path)
    return mask


def test_photo_folder_reads_masks_and_alpha(tmp_path):
    from cmr_data.photos import PhotoFolder, list_photos
    write_photo(tmp_path / "b.png", rgba=True)
    write_photo(tmp_path / "a.jpg", box=(0, 0, 31, 10))
    Image.fromarray(write_photo(tmp_path / "unused.png", box=(0, 0, 31, 10))).save(tmp_path / "a_mask.png")
    (tmp_path / "notes.txt").write_text("not a photo")
    (tmp_path / "unused.png").unlink()
    assert list_photos(str(tmp_path)) == [("a", "a.jpg", "a_mask.png"), ("b", "b.png", None)]
    ds = PhotoFolder(str(tmp_path), [256, 64])
    assert ds.names == ["a", "b"] and len(ds) == 2 and ds.get_paths() == ["a.jpg", "b.png"]
    assert set(np.unique(ds.anno[0].mask)) == {0, 1} and int(ds.anno[1].mask.sum()) == 17 * 14
    assert ds.crop_box(1)[2] - ds.crop_box(1)[0] == ds.crop_box(1)[3] - ds.crop_box(1)[1]
    poses = ds.pose_table()
    assert poses.shape == (2, 2, 8) and poses.dtype == np.float32 and np.isnan(poses).all()
    win = ds.windows()
    assert (win[:, 4] >= 1).all() and (win[:, :2] >= 1).all()


def test_photo_folder_errors_name_the_file(tmp_path):
    from cmr_data.photos import PhotoFolder
    write_photo(tmp_path / "empty.png", rgba=True, box=(0, 0, -1, -1))
    with pytest.raises(ValueError, match="empty.png: the foreground mask is empty"):
        PhotoFolder(str(tmp_path), 256)
    (tmp_path / "empty.png").unlink()
    write_photo(tmp_path / "plain.png")
    with pytest.raises(ValueError, match="plain.png: no alpha channel and no plain_mask.png"):
        PhotoFolder(str(tmp_path), 256)
    Image.fromarray(np.ones((5, 5), np.uint8)).save(tmp_path / "plain_mask.png")
    with pytest.raises(ValueError, match="plain_mask.png: the mask is 5x5, its photo 32x24"):
        PhotoFolder(str(tmp_path), 256)
    (tmp_path / "plain.png").unlink()
    (tmp_path / "plain_mask.png").unlink()
    with pytest.raises(ValueError, match="no photos"):
        PhotoFolder(str(tmp_path), 256)


def test_flags_and_defaults(tmp_path):
    import reconstruct
    a = reconstruct.parse_args(['--name', 'birds', '--dataset', 'cub'])
    assert (a.split, a.mesh_path, a.output) == ('testval', 'mesh_templates/uvsphere_16rings.obj', 'results_recon/birds')
    assert (a.export_resolution, a.batch_size, a.writers, a.which_epoch) == (512, 16, 8, 'latest')
    assert a.symmetric is True and a.optimize_deltas is True and a.optimize_z0 is False
    assert a.indices is None and a.num_images is None and a.photos is None
    a = reconstruct.parse_args(['--name', 'cars', '--dataset', 'p3d', '--split', 'train', '--indices', '4', '1',
                                '--num_images', '1', '--output', 'o', '--texture_resolution', '64'])
    assert (a.split, a.indices, a.num_images, a.output, a.mesh_path) == ('train', [4, 1], 1, 'o',
                                                                         'mesh_templates/uvsphere_31rings.obj')
    assert a.texture_resolution == 64
    a = reconstruct.parse_args(['--name', 'x', '--dataset', 'cub', '--photos', str(tmp_path)])
    assert a.photos == str(tmp_path) and a.split is None


@pytest.mark.parametrize("argv", [
    ['--dataset', 'cub'],
    ['--name', 'x', '--dataset', 'shapenet'],
    ['--name', 'x', '--dataset', 'cub', '--split', 'val'],
    ['--name', 'x', '--dataset', 'p3d', '--split', 'testval'],
    ['--name', 'x', '--dataset', 'cub', '--photos', 'no_such_directory'],
    ['--name', 'x', '--dataset', 'cub', '--export_resolution', '511'],
    ['--name', 'x', '--dataset', 'cub', '--batch_size', '0'],
    ['--name', 'x', '--dataset', 'cub', '--writers', '0'],
    ['--name', 'x', '--dataset', 'cub', '--num_images', '0'],
    ['--name', 'x', '--dataset', 'cub', '--indices', '-1'],
], ids=["no_name", "dataset", "cub_val", "p3d_testval", "photos_missing", "odd_resolution", "batch", "writers",
        "num_images", "negative_index"])
def test_argument_errors(argv, capsys):
    import reconstruct
    with pytest.raises(SystemExit) as e:
        reconstruct.parse_args(argv)
    assert e.value.code == 2
    assert 'error' in capsys.readouterr().err


def test_photos_and_split_together_are_refused(tmp_path, capsys):
    import reconstruct
    with pytest.raises(SystemExit):
        reconstruct.parse_args(['--name', 'x', '--dataset', 'cub', '--photos', str(tmp_path), '--split', 'train'])
    assert '--photos exports a folder' in capsys.readouterr().err


def test_selection_names_and_checkpoint_size():
    import reconstruct
    assert reconstruct.select(5, None, None) == [0, 1, 2, 3, 4]
    assert reconstruct.select(5, None, 2) == [0, 1]
    assert reconstruct.select(5, [4, 0, 2], 2) == [4, 0]
    with pytest.raises(SystemExit, match="--indices 5 outside the 5 images"):
        reconstruct.select(5, [1, 5], None)
    assert reconstruct.output_name('001.Black_footed_Albatross/Black_Footed_Albatross_0009_34.jpg') == \
        '001.Black_footed_Albatross_Black_Footed_Albatross_0009_34'
    assert reconstruct.output_name('car_imagenet\\n02814533_1.JPEG') == 'car_imagenet_n02814533_1'
    assert reconstruct.checkpoint_dataset_size({'dataset_params': {'ds_translation': torch.zeros(7, 2),
                                                                   'ds_scale': torch.zeros(7, 1)}}) == 7
    assert reconstruct.checkpoint_dataset_size({'dataset_params': None}) == 1


def test_importing_the_command_does_nothing():
    import importlib
    import reconstruct
    importlib.reload(reconstruct)
    assert reconstruct.build_parser().prog


def test_exporter_without_cuda_raises(monkeypatch):
    import b3d
    from reconstruction_export import ReconstructionExporter
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: False)
    trainer = types.SimpleNamespace(generator=torch.nn.Linear(2, 2))
    with pytest.raises(b3d.B3DError, match="needs a CUDA device"):
        ReconstructionExporter(trainer, None)
