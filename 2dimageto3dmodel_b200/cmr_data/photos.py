"""User photos for the reconstruction export: a folder of images that are not in CUB-200-2011 or PASCAL3D+, with a
foreground mask but no annotation and no SfM pose.

Each photo is either an RGBA PNG (the mask is alpha > 0) or an RGB image with a `<stem>_mask.png` beside it (the mask is
that image's grey level > 0).  The crop square follows BaseDataset.crop_box with the tight box of the mask in place of the
annotated one: the box of mask > 0, padded by 5 % (peturb_bbox, pf=0.05, jf=0), squared (square_bbox).  The device
store and its batches are BaseDataset's, so `to_device()` / `eval_batches(B)` build the network input of a whole batch in
one b3d_image_batch launch.  The pose rows are NaN: there is no camera to place the prediction in."""
import os
import types

import numpy as np
from PIL import Image

from . import image_utils
from .base import BaseDataset

IMAGE_EXTENSIONS = ('.png', '.jpg', '.jpeg', '.bmp', '.webp')
MASK_SUFFIX = '_mask'


def tight_box(mask):
    """Zero-indexed [x0, y0, x1, y1] (float) of the pixels of mask > 0, or None when there are none."""
    ys, xs = np.nonzero(mask)
    if len(xs) == 0:
        return None
    return np.array([xs.min(), ys.min(), xs.max(), ys.max()], float)


def photo_crop_box(mask, padding_frac=0.05):
    """The crop square of a photo with foreground mask > 0, by the rule of BaseDataset.crop_box.  None for an empty
    mask."""
    box = tight_box(mask)
    if box is None:
        return None
    return image_utils.square_bbox(image_utils.peturb_bbox(box, pf=padding_frac, jf=0))


def list_photos(directory):
    """-> sorted [(name, photo file, mask file or None)] of the photos in directory: every image whose name does not end
    in `_mask.png`, with its `<stem>_mask.png` when there is one."""
    files = set(os.listdir(directory))
    out = []
    for f in sorted(files):
        stem, ext = os.path.splitext(f)
        if ext.lower() not in IMAGE_EXTENSIONS or f.endswith(MASK_SUFFIX + '.png'):
            continue
        mask = stem + MASK_SUFFIX + '.png'
        out.append((stem, f, mask if mask in files else None))
    return out


def read_mask(directory, photo, mask_file):
    """uint8 0 / 1 foreground mask of one photo (its alpha, or its mask file's grey level, > 0)."""
    path = os.path.join(directory, photo)
    if mask_file is None:
        with Image.open(path) as im:
            if im.mode not in ('RGBA', 'LA', 'PA') and not (im.mode == 'P' and 'transparency' in im.info):
                raise ValueError(f'{path}: no alpha channel and no {os.path.splitext(photo)[0]}{MASK_SUFFIX}.png beside it')
            alpha = np.asarray(im.convert('RGBA'))[..., 3]
        return (alpha > 0).astype(np.uint8)
    mpath = os.path.join(directory, mask_file)
    with Image.open(mpath) as im:
        m = (np.asarray(im.convert('L')) > 0).astype(np.uint8)
    with Image.open(path) as im:
        size = im.size
    if m.shape != (size[1], size[0]):
        raise ValueError(f'{mpath}: the mask is {m.shape[1]}x{m.shape[0]}, its photo {size[0]}x{size[1]}')
    return m


class PhotoFolder(BaseDataset):
    """directory: the photos (see the module docstring); img_size: the network input's side, or a list of sides (the first
    is the network's).  Items are in file-name order; `names` holds their stems.  An empty mask raises ValueError naming
    the file."""

    def __init__(self, directory, img_size):
        super().__init__(False, img_size)
        self.img_dir = directory
        self.anno, self.names, self._boxes = [], [], []
        for name, photo, mask_file in list_photos(directory):
            mask = read_mask(directory, photo, mask_file)
            box = photo_crop_box(mask, self.padding_frac)
            if box is None:
                raise ValueError(f'{os.path.join(directory, mask_file or photo)}: the foreground mask is empty')
            self.anno.append(types.SimpleNamespace(rel_path=photo, mask=mask))
            self.names.append(name)
            self._boxes.append(box)
        if not self.anno:
            raise ValueError(f'{directory}: no photos ({", ".join(IMAGE_EXTENSIONS)})')
        self.num_imgs = len(self.anno)

    def crop_box(self, index):
        return self._boxes[index]

    def pose_table(self):
        """NaN rows: the photos have no SfM pose."""
        return np.full((len(self), 2, 8), np.nan, np.float32)

    def __getitem__(self, index):
        raise NotImplementedError('PhotoFolder: photos have no pose or keypoints; use to_device() and eval_batches()')
