"""Shared by make_golden_samples.py (reference side) and the sample-export tests (drop-in side): the stand-in dataset the
export draws from, the draw parameters of the golden, and the compact storage of the golden's files."""
import io

import numpy as np
import torch
import torch.nn.functional as F

N, SEED, SIGMA, LATENT = 10, 5, 1.0, 8      # latent 8: wrapper_common.TinyG
RENDER = 512


class PoseSet:
    """What main.py's save_results block reads from train_ds: len(), classes[i] and the poses data['rotation' | 'scale' |
    'translation'] (fp32 [n,4], [n,1], [n,3])."""

    def __init__(self, n=23, seed=17, num_classes=10):
        g = torch.Generator().manual_seed(seed)
        self.data = {'rotation': F.normalize(torch.randn(n, 4, generator=g), dim=1),
                     'scale': 0.6 + 0.3 * torch.rand(n, 1, generator=g),
                     'translation': torch.cat(((torch.rand(n, 2, generator=g) - 0.5) * 0.2, torch.zeros(n, 1)), 1)}
        self.classes = [np.array([(3 * i) % num_classes]) for i in range(n)]

    def __len__(self):
        return len(self.classes)


# ---- the reference's files in samples_reference.npz, stored compactly ----------------------------------------------------
# The .obj files differ only in their `v` lines and in the material name, so the golden holds mesh_0.obj whole and the `v`
# lines of every sample; the grid is held as the PNG file the reference's array encodes to (lossless).  make_golden_samples.py
# checks that unpack_files() gives back every file it captured, byte for byte.

def _v_block(text):
    return "".join(line for line in text.splitlines(keepends=True) if line.startswith("v "))


def pack_files(objs, mtls, grid):
    from PIL import Image
    png = io.BytesIO()
    Image.fromarray(grid).save(png, format="PNG")
    v = [_v_block(t).encode() for t in objs]
    return dict(obj0=np.frombuffer(objs[0].encode(), np.uint8), obj_v=np.frombuffer(b"".join(v), np.uint8),
                obj_v_len=np.array([len(b) for b in v], np.int64), mtl0=np.frombuffer(mtls[0].encode(), np.uint8),
                grid_png=np.frombuffer(png.getvalue(), np.uint8))


def unpack_files(d):
    """-> (obj texts, mtl texts, grid uint8 [H,W,3]) of the reference's export."""
    from PIL import Image
    obj0, mtl0 = d["obj0"].tobytes().decode(), d["mtl0"].tobytes().decode()
    ends = np.cumsum(d["obj_v_len"])
    raw = d["obj_v"].tobytes()
    v = [raw[e - n:e].decode() for e, n in zip(ends, d["obj_v_len"])]
    objs = [obj0.replace(v[0], v[i]).replace("mesh_0", f"mesh_{i}") for i in range(len(v))]
    mtls = [mtl0.replace("mesh_0", f"mesh_{i}") for i in range(len(v))]
    grid = np.asarray(Image.open(io.BytesIO(d["grid_png"].tobytes())))
    return objs, mtls, grid
