"""PASCAL3D+ (reference: cmr_data/p3d.py), one class (default 'car').  The photos are the public PASCAL3D+ release 1.1
under datasets/p3d/PASCAL3D+_release1.1/Images."""
import os.path as osp

import scipy.io as sio

from . import base as base_data


class P3dDataset(base_data.BaseDataset):
    def __init__(self, split, is_train, img_size, p3d_class='car', root=''):
        """split: 'train' or 'val'.  root: the directory holding datasets/ (default: the working directory)."""
        super().__init__(is_train, img_size)
        anno_dir = osp.join(root, 'datasets', 'p3d')
        self.img_dir = osp.join(anno_dir, 'PASCAL3D+_release1.1', 'Images')
        self.kp_path = osp.join(anno_dir, 'data', '{}_kps.mat'.format(p3d_class))
        self.anno_path = osp.join(anno_dir, 'data', '{}_{}.mat'.format(p3d_class, split))
        self.anno_sfm_path = osp.join(anno_dir, 'sfm', '{}_{}.mat'.format(p3d_class, split))
        self.anno = sio.loadmat(self.anno_path, struct_as_record=False, squeeze_me=True)['images']
        self.anno_sfm = sio.loadmat(self.anno_sfm_path, struct_as_record=False, squeeze_me=True)['sfm_anno']
        self.kp_perm = sio.loadmat(self.kp_path, struct_as_record=False, squeeze_me=True)['kp_perm_inds'] - 1
        self.num_kps = len(self.kp_perm)
        self.num_imgs = len(self.anno)
