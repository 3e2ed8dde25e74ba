"""Timing of the reconstruction training-data path on one GPU.  Prints one JSON line (also written to --out when given):
  1. b3d_image_batch at cfg4 (B 50, R 256) and for a pseudo-GT export batch (B 50, img_size [256, 299, 1024]): CUDA-event
     time per batch against the HBM bound (bytes written, 16 R0^2 + 12 sum(Rk^2) per sample, plus the window bytes read,
     over 3.35 TB/s);
  2. a reference-style host loader (PIL decode + crop + float64 resize per image: ImageDataset over CUBDataset, DataLoader
     with 4 workers and pinned memory, then the copy to the device): images/s;
  3. ReconTrainer.train_epoch at cfg4 fed by train_batches against the same trainer fed by resident tensors, alternated;
  4. to_device packing time of 5964 images (the CUB training split's count).
The photos are synthetic JPEGs at CUB-like sizes (500 x 375) with crop sides drawn from the CUB training split's
distribution (median 312, range 112-550), written to a temporary directory.  The card's name, power limit and SM clock
limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "2dimageto3dmodel_b200"))
sys.path.insert(0, ROOT)

import numpy as np   # noqa: E402
import torch         # noqa: E402

HBM_BYTES_PER_S = 3.35e12     # H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def write_cub_like_tree(root, n, seed=0, hw=(375, 500), ext='jpg', split='train', boxes=None):
    """A CUB-layout tree under root/datasets/cub: n synthetic photos of hw (smooth colour ramps + noise, lossy JPEG or
    lossless PNG), elliptic 0/1 masks, boxes whose padded square side follows the CUB training split (log-normal around
    312, clipped to 112-550; boxes may cross the photo's borders) unless `boxes` lists them (1-based x1, y1, x2, y2),
    random SfM poses.  -> root."""
    import scipy.io as sio
    from PIL import Image
    g = np.random.default_rng(seed)
    top = os.path.join(root, 'datasets', 'cub')
    img_dir = os.path.join(top, 'CUB_200_2011', 'images')
    os.makedirs(os.path.join(img_dir, '001.Synthetic'), exist_ok=True)
    for d in ('data', 'sfm'):
        os.makedirs(os.path.join(top, d), exist_ok=True)
    h, w = hw
    yy, xx = np.mgrid[0:h, 0:w]
    images = np.empty((1, n), dtype=[('rel_path', 'O'), ('bbox', 'O'), ('width', 'O'), ('height', 'O'), ('parts', 'O'),
                                     ('mask', 'O')])
    sfm = np.empty((1, n), dtype=[('rot', 'O'), ('scale', 'O'), ('trans', 'O')])
    for i in range(n):
        side = float(np.clip(np.exp(g.normal(np.log(312), 0.35)), 112, 550)) / 1.1      # box side before the 5 % pad
        bw, bh = (side, side * g.uniform(0.55, 1.0)) if g.random() < 0.5 else (side * g.uniform(0.55, 1.0), side)
        cx, cy = g.uniform(0.3, 0.7) * w, g.uniform(0.3, 0.7) * h
        x1, y1 = int(cx - bw / 2) + 1, int(cy - bh / 2) + 1
        x2, y2 = x1 + int(bw) - 1, y1 + int(bh) - 1
        if boxes is not None:
            x1, y1, x2, y2 = boxes[i]
        base = np.stack([(xx + i) % 256, (yy * 2 + i) % 256, ((xx + yy) // 2) % 256], -1)
        photo = np.clip(base + g.integers(-20, 21, (h, w, 3)), 0, 255).astype(np.uint8)
        rel = f'001.Synthetic/Bird_{i:05d}.{ext}'
        Image.fromarray(photo).save(os.path.join(img_dir, rel), quality=90) if ext == 'jpg' else \
            Image.fromarray(photo).save(os.path.join(img_dir, rel))
        mask = ((((yy - cy) / (bh / 2)) ** 2 + ((xx - cx) / (bw / 2)) ** 2) < 1).astype(np.uint8)
        parts = np.zeros((3, 15), np.uint16)
        q = g.normal(size=4)
        q /= np.linalg.norm(q)
        w_, x_, y_, z_ = q
        rot = np.array([[1 - 2 * (y_ * y_ + z_ * z_), 2 * (x_ * y_ - z_ * w_), 2 * (x_ * z_ + y_ * w_)],
                        [2 * (x_ * y_ + z_ * w_), 1 - 2 * (x_ * x_ + z_ * z_), 2 * (y_ * z_ - x_ * w_)],
                        [2 * (x_ * z_ - y_ * w_), 2 * (y_ * z_ + x_ * w_), 1 - 2 * (x_ * x_ + y_ * y_)]])
        images[0, i] = (rel, {'x1': x1, 'y1': y1, 'x2': x2, 'y2': y2}, w, h, parts, mask)
        sfm[0, i] = (rot, float(side * g.uniform(0.25, 0.35)), np.array([cx, cy]) + g.normal(size=2) * 5)
    sio.savemat(os.path.join(top, 'data', f'{split}_cub_cleaned.mat'), {'images': images})
    sio.savemat(os.path.join(top, 'sfm', f'anno_{split}.mat'), {'sfm_anno': sfm})
    return root


def batch_bytes(ds, idx, sizes):
    """Bytes one batch moves at the least: every output written once, every window read once."""
    win = ds.windows()
    out = len(idx) * (16 * sizes[0] ** 2 + 12 * sum(r * r for r in sizes[1:]))
    return out + 4 * int((win[idx, 0] * win[idx, 1]).sum())


def time_kernel(ds, B, iters=100):
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(0)
    n = len(ds)
    perm = torch.randperm(n, generator=g)
    idx = perm.to(torch.int32).to(dev)
    flip = torch.randint(0, 2, (n,), generator=g, dtype=torch.uint8).to(dev)
    out = ds.batch_outputs(B)
    starts = [(k * B) % (n - B + 1) for k in range(iters)]
    for s in starts[:10]:
        ds.gather(idx[s:s + B], flip[s:s + B], out)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for s in starts:
        ds._gather(idx[s:s + B], flip[s:s + B], out)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / iters
    mean_bytes = np.mean([batch_bytes(ds, perm[s:s + B].numpy(), ds.img_sizes) for s in starts])
    return {"us_per_batch": round(us, 1), "mbytes": round(mean_bytes / 1e6, 1),
            "hbm_bound_us": round(mean_bytes / HBM_BYTES_PER_S * 1e6, 1)}


def host_loader_rate(root, B=50, n_images=300, workers=4):
    from cmr_data.cub import CUBDataset
    from cmr_data.image_dataset import ImageDataset
    ds = ImageDataset(CUBDataset('train', True, 256, root=root), 256)
    sub = torch.utils.data.Subset(ds, range(min(n_images, len(ds))))
    loader = torch.utils.data.DataLoader(sub, batch_size=B, shuffle=True, num_workers=workers, pin_memory=True)
    it = iter(loader)
    next(it)                                                   # workers started
    t0, seen = time.perf_counter(), 0
    for b in it:
        X = b[0].cuda(non_blocking=True)
        seen += X.shape[0]
    torch.cuda.synchronize()
    return round(seen / (time.perf_counter() - t0), 1)


def train_epoch_rates(root, rounds=4, batches=4, B=50):
    from cmr_data.cub import CUBDataset
    from reconstruction_training import ReconTrainer, default_args
    from rendering.mesh_template import MeshTemplate
    from tools.uvsphere import write_uvsphere_obj
    tpl = MeshTemplate(write_uvsphere_obj(os.path.join(tempfile.mkdtemp(), "uvsphere_16rings.obj"), rings=16), device="cuda")
    ds = CUBDataset('train', True, 256, root=root)
    ds.to_device()
    n = batches * B
    ds.num_imgs = n                                            # the epoch covers the first n images
    tr = ReconTrainer(default_args(), tpl, dataset_size=n, device="cuda")
    resident = [tuple(t.clone() for t in b) for b in ds.train_batches(B, 0)]
    tr.train_epoch(resident)                                   # warm-up: every shape
    tr.train_epoch(ds.train_batches(B, 1))
    rates = {"train_batches": [], "resident": []}
    for r in range(rounds):
        for kind in ("train_batches", "resident"):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tr.train_epoch(ds.train_batches(B, 2 + r) if kind == "train_batches" else resident)
            torch.cuda.synchronize()
            rates[kind].append(round(n / (time.perf_counter() - t0), 1))
    return rates


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--images", type=int, default=5964)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_recon_data.py measures on a CUDA device; none is visible")
    from cmr_data.cub import CUBDataset
    res = {"card": card()}
    with tempfile.TemporaryDirectory() as root:
        t0 = time.perf_counter()
        write_cub_like_tree(root, args.images)
        res["write_tree_s"] = round(time.perf_counter() - t0, 1)
        for key, sizes in (("cfg4", 256), ("pseudogt", [256, 299, 1024])):
            ds = CUBDataset('train', True, sizes, root=root)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ds.to_device()
            if key == "cfg4":
                res["to_device_s"] = round(time.perf_counter() - t0, 2)
                res["store_gb"] = round(ds.packed_bytes() / 1e9, 2)
            res[f"kernel_{key}"] = time_kernel(ds, 50)
            del ds
            torch.cuda.empty_cache()
        res["host_loader_img_s"] = host_loader_rate(root)
        res["train_epoch_img_s"] = train_epoch_rates(root)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
