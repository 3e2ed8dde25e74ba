"""run_reconstruction.py's ImageDataset (:91-133): a CMR dataset item as the network's input tuple."""
import numpy as np
import torch


class ImageDataset(torch.utils.data.Dataset):
    def __init__(self, cmr_dataset, img_size):
        self.cmr_dataset = cmr_dataset
        self.paths = cmr_dataset.get_paths()
        self.extra_img_keys = [f'img_{res}' for res in img_size[1:]] if isinstance(img_size, list) else []

    def __len__(self):
        return len(self.cmr_dataset)

    def __getitem__(self, idx):
        """-> (X [4,R,R] = (masked image in [-1, 1], mask), masked [3,Rk,Rk] per extra size, scale [1],
        translation [3] = (tx, ty, 0), rot [4], ind [1]: idx, plus N when mirrored)."""
        item = self.cmr_dataset[idx]
        img = item['img'].astype('float32') * 2 - 1
        mask = item['mask'].astype('float32')
        img *= mask[np.newaxis, :, :]
        ind = torch.LongTensor([idx])
        if item['mirrored']:
            ind += len(self.cmr_dataset)       # 0 .. N-1 straight, N .. 2N-1 mirrored (DatasetParams)
        pose = item['sfm_pose']
        extra = []
        for k in self.extra_img_keys:
            img_k, mask_k = item[k]
            img_k = img_k.astype('float32') * 2 - 1
            img_k *= mask_k.astype('float32')[np.newaxis, :, :]
            extra.append(torch.FloatTensor(img_k))
        output = torch.cat((torch.FloatTensor(img), torch.FloatTensor(mask).unsqueeze(0)), dim=0)
        return (output, *extra, torch.FloatTensor(pose[:1]), torch.FloatTensor([pose[1], pose[2], 0]),
                torch.FloatTensor(pose[-4:]), ind)
