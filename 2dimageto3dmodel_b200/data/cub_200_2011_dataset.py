"""CUB-200-2011 birds (reference: data/cub_200_2011_dataset.py): pseudo-ground-truth records plus the 200 species labels
(zero-based) read from CUB's images.txt / image_class_labels.txt."""
import os

import numpy as np

from data.abstract_dataset import AbstractDataset


class CubDataset(AbstractDataset):
    def __init__(self, args, **kwargs):
        super().__init__(args, **kwargs)
        self.n_classes = (200,)
        args.n_classes = self.n_classes
        labels = os.path.join(self.root, 'datasets', 'cub', 'CUB_200_2011')
        with open(os.path.join(labels, 'images.txt')) as f:
            image_of_id = dict(line.split(' ') for line in f.readlines())
        with open(os.path.join(labels, 'image_class_labels.txt')) as f:
            class_of_id = dict(line.split(' ') for line in f.readlines())
        self.filename_to_class = {image_of_id[k].strip(): int(v.strip()) - 1 for k, v in class_of_id.items()}
        self.classes = [np.array([self.filename_to_class[p]]) for p in self.data['path']]

    def name(self):
        return 'cub'

    def suggest_truncation_sigma(self):
        return 0.25 if self.args.conditional_class else 1.0

    def suggest_num_discriminators(self):
        return 3 if self.args.texture_resolution >= 512 else 2

    def suggest_mesh_template(self):
        return 'mesh_templates/uvsphere_16rings.obj'
