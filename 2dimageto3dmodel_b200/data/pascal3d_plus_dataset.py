"""Pascal 3D+ cars (reference: data/pascal3d_plus_dataset.py): only the ImageNet part of the pose metadata is used, sample
i reads pseudo-ground-truth file imagenet_indices[i]; labels are [shape, colour 1, colour 2] from datasets/p3d/p3d_labels.csv."""
import os

import numpy as np

from data.abstract_dataset import AbstractDataset


class Pascal3DPlusDataset(AbstractDataset):
    def __init__(self, args, **kwargs):
        super().__init__(args, **kwargs)
        self.imagenet_indices = [i for i, p in enumerate(self.data['path']) if p.startswith('car_imagenet')]
        keep = self.imagenet_indices
        self.data['path'] = [self.data['path'][i] for i in keep]
        for k in ('scale', 'translation', 'rotation'):
            self.data[k] = self.data[k][keep]
        mapping, self.n_classes = Pascal3DPlusDataset.get_p3d_labels(self.root)
        args.n_classes = self.n_classes
        self.classes = [mapping[p.split('/')[-1]] for p in self.data['path']]

    def name(self):
        return 'p3d'

    def suggest_truncation_sigma(self):
        a = self.args
        if a.conditional_class:
            return 0.5 if a.conditional_color else 0.75
        return 1.0

    def suggest_num_discriminators(self):
        return 2

    def suggest_mesh_template(self):
        return 'mesh_templates/uvsphere_31rings.obj'

    def record_index(self, idx):
        return self.imagenet_indices[idx]

    @staticmethod
    def get_p3d_labels(root=''):
        """-> ({filename: int64 [shape, colour 1, colour 2]}, (shapes, colours 1, colours 2)); ids index the sorted names."""
        with open(os.path.join(root, 'datasets', 'p3d', 'p3d_labels.csv')) as f:
            rows = [line.strip().split(',') for line in f.readlines()[1:]]
        names = {col: sorted({r[col] for r in rows}) for col in (1, 2, 3)}      # colour 1, colour 2, shape
        ids = {col: {x: i for i, x in enumerate(v)} for col, v in names.items()}
        mapping = {r[0]: np.array([ids[3][r[3]], ids[1][r[1]], ids[2][r[2]]]) for r in rows}
        return mapping, (len(names[3]), len(names[1]), len(names[2]))
