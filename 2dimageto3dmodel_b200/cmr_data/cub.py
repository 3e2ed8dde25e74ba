"""CUB-200-2011 (reference: cmr_data/cub.py).  5964 training and 5771 test / validation images remain after the
annotation's cleaning; the photos are the public CUB-200-2011 release under datasets/cub/CUB_200_2011/images."""
import os.path as osp

import numpy as np
import scipy.io as sio

from . import base as base_data


class CUBDataset(base_data.BaseDataset):
    def __init__(self, split, is_train, img_size, root=''):
        """split: 'train' or 'testval'.  root: the directory holding datasets/ (default: the working directory)."""
        super().__init__(is_train, img_size)
        cache_path = osp.join(root, 'datasets', 'cub')
        self.data_cache_dir = cache_path
        self.data_dir = osp.join(cache_path, 'CUB_200_2011')
        self.img_dir = osp.join(self.data_dir, 'images')
        self.anno_path = osp.join(self.data_cache_dir, 'data', '%s_cub_cleaned.mat' % split)
        self.anno_sfm_path = osp.join(self.data_cache_dir, 'sfm', 'anno_%s.mat' % split)
        if not osp.exists(self.anno_path):
            raise ValueError('%s doesnt exist!' % self.anno_path)
        self.anno = sio.loadmat(self.anno_path, struct_as_record=False, squeeze_me=True)['images']
        self.anno_sfm = sio.loadmat(self.anno_sfm_path, struct_as_record=False, squeeze_me=True)['sfm_anno']
        self.num_imgs = len(self.anno)
        # keypoint order after a horizontal flip (left and right parts swap)
        self.kp_perm = np.array([1, 2, 3, 4, 5, 6, 11, 12, 13, 10, 7, 8, 9, 14, 15]) - 1
