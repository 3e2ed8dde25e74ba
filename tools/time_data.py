"""Timing of the GAN training-data path on one GPU.  Prints one JSON line (also written to --out when given):
  1. b3d_gather_fields at cfg3 (B 32, R 256) and cfg5 (B 8, R 512), device and pinned-host storage: CUDA-event time per
     batch, against the HBM bound (device) and as PCIe read bandwidth (host);
  2. a reference-style host loader (per-sample np.load of the compressed record + mirror_tex, DataLoader with 4 workers and
     pinned memory, then the copy to the device) on a synthetic cache written to local disk: images/s;
  3. GANTrainer.train_epoch at cfg3 fed by train_batches against the same trainer fed by resident tensors, alternated;
  4. to_device packing time of the cache of (2).
The card's name, power limit and SM clock limit are read in the same run."""
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


def gather_bytes(B, R):
    """Bytes one training batch moves: fp16 texture + alpha planes read (2 B) and written as fp32 (4 B), the fp32 mesh
    map read and written, the int64 class row, the int32 index and the flip byte."""
    return B * (4 * R * R * (2 + 4) + 3 * 32 * 32 * (4 + 4) + 8 * 2 + 4 + 1)


def time_gather(B, R, storage, n=256, iters=200):
    from b3d.data import gather_fields
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(0)
    host = storage == "host"

    def store(shape, dtype):
        t = torch.empty(shape, dtype=dtype, pin_memory=host)
        t.copy_((torch.rand(shape, generator=g) * 2 - 1).to(dtype) if dtype != torch.int64 else
                torch.randint(0, 200, shape, generator=g))
        return t if host else t.to(dev)
    st = {"texture": store((n, 3, R, R), torch.float16), "texture_alpha": store((n, 1, R, R), torch.float16),
          "mesh": store((n, 3, 32, 32), torch.float32), "class": store((n, 1), torch.int64)}
    out = {"X_tex": torch.empty(B, 3, R, R, device=dev), "X_alpha": torch.empty(B, 1, R, R, device=dev),
           "X_mesh": torch.empty(B, 3, 32, 32, device=dev), "C": torch.empty(B, 1, dtype=torch.int64, device=dev)}
    fields = [(st["texture"], out["X_tex"], True, 1.0, 0.0), (st["texture_alpha"], out["X_alpha"], True, 1.0, 0.0),
              (st["mesh"], out["X_mesh"], True, 1.0, 0.0), (st["class"], out["C"], False, 1.0, 0.0)]
    perm = torch.randperm(n, generator=g)
    idx = torch.cat([perm, perm]).to(torch.int32).to(dev)            # batches at shifting offsets of a permutation
    flip = torch.randint(0, 2, (2 * n,), generator=g, dtype=torch.uint8).to(dev)
    for k in range(20):
        o = (k * B) % n
        gather_fields(fields, idx[o:o + B], flip[o:o + B])
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for k in range(iters):
        o = (k * B) % n
        gather_fields(fields, idx[o:o + B], flip[o:o + B])
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / iters
    nb = gather_bytes(B, R)
    r = {"B": B, "R": R, "storage": storage, "us_per_batch": round(us, 2), "bytes": nb}
    if host:
        read = B * (4 * R * R * 2 + 3 * 32 * 32 * 4 + 8)
        r["pcie_read_GBps"] = round(read / us / 1e3, 2)
    else:
        r["hbm_bound_us"] = round(nb / HBM_BYTES_PER_S * 1e6, 2)
        r["share_of_hbm_bound"] = round(nb / HBM_BYTES_PER_S * 1e6 / us, 3)
    return r


def write_cache(root, n, R, seed=0):
    """A CUB-layout cache of n records at R^2 (compressed fp16 records, as the exporter writes them)."""
    from data.pseudo_gt import pseudo_gt_dir, save_poses_metadata, save_pseudo_gt
    g = torch.Generator().manual_seed(seed)
    cache = os.path.join(root, "cache", "cub")
    paths = [f"001.Species/Bird_{i:05d}.jpg" for i in range(n)]
    save_poses_metadata(cache, 0.5 + torch.rand(n, 1, generator=g), torch.randn(n, 3, generator=g) * 0.1,
                        torch.nn.functional.normalize(torch.randn(n, 4, generator=g), dim=1), paths)
    d = pseudo_gt_dir(cache, R)
    yy, xx = torch.meshgrid(torch.linspace(-1, 1, R), torch.linspace(-1, 1, R), indexing="ij")
    for i in range(n):
        mask = ((yy * yy + xx * xx) < 0.2 + 0.6 * float(torch.rand(1, generator=g))).float()
        save_pseudo_gt(d, i, {"mesh": torch.randn(3, 32, 32, generator=g) * 0.05,
                              "texture": ((torch.rand(3, R, R, generator=g) * 2 - 1) * mask).half(),
                              "texture_alpha": mask[None].half(),
                              "image": (torch.rand(4, 299, 299, generator=g) * 2 - 1).half()})
    lab = os.path.join(root, "datasets", "cub", "CUB_200_2011")
    os.makedirs(lab, exist_ok=True)
    with open(os.path.join(lab, "images.txt"), "w") as f:
        f.writelines(f"{i + 1} {p}\n" for i, p in enumerate(paths))
    with open(os.path.join(lab, "image_class_labels.txt"), "w") as f:
        f.writelines(f"{i + 1} {i % 200 + 1}\n" for i in range(n))


def cub_args(R, B):
    import bench
    a = bench.gan_args(R, 2)
    a.dataset, a.evaluate, a.batch_size = "cub", False, B
    return a


def host_loader_rate(root, R, B, batches):
    from data.cub_200_2011_dataset import CubDataset
    ds = CubDataset(cub_args(R, B), root=root)
    loader = torch.utils.data.DataLoader(ds, batch_size=B, num_workers=4, pin_memory=True, drop_last=True, shuffle=True)
    n_img, t0, it = 0, None, 0
    while it < batches + 2:
        for data in loader:
            x = [data[k].cuda(non_blocking=True) for k in ("texture", "texture_alpha", "mesh", "class")]
            it += 1
            if it == 2:                                      # worker start-up excluded
                torch.cuda.synchronize()
                t0 = time.perf_counter()
            elif it > 2:
                n_img += B
            if it >= batches + 2:
                break
    torch.cuda.synchronize()
    del x
    return n_img / (time.perf_counter() - t0)


def train_rates(root, B, epochs, rounds):
    from data.cub_200_2011_dataset import CubDataset
    from gan_training import GANTrainer
    args = cub_args(256, B)
    ds = CubDataset(args, root=root).to_device("cuda")
    torch.manual_seed(0)
    tr = GANTrainer(args, device="cuda")
    resident = [{k: v.clone() for k, v in b.items()} for b in ds.train_batches(B, 0)]
    tr.train_epoch(ds.train_batches(B, 0))
    tr.train_epoch(resident)
    out = {"train_batches": [], "resident": []}
    for r in range(rounds):
        for name in ("train_batches", "resident") if r % 2 == 0 else ("resident", "train_batches"):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            n = 0
            for e in range(epochs):
                src = ds.train_batches(B, e + 1) if name == "train_batches" else resident
                n += B * len(tr.train_epoch(src))
            torch.cuda.synchronize()
            out[name].append(n / (time.perf_counter() - t0))
    return {k: {"img_per_s_mean": round(float(np.mean(v)), 1), "runs": [round(x, 1) for x in v]} for k, v in out.items()}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--records", type=int, default=512, help="records in the synthetic on-disk cache (R 256)")
    p.add_argument("--loader-batches", type=int, default=60)
    p.add_argument("--epochs", type=int, default=2)
    p.add_argument("--rounds", type=int, default=4)
    p.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_data: needs a CUDA device")
    res = {"card": card()}
    res["gather"] = [time_gather(32, 256, s) for s in ("device", "host")] + [time_gather(8, 512, s) for s in ("device", "host")]
    print(json.dumps(res["gather"]), flush=True)
    with tempfile.TemporaryDirectory() as root:
        t0 = time.perf_counter()
        write_cache(root, a.records, 256)
        res["cache_write_s"] = round(time.perf_counter() - t0, 1)
        res["host_loader_img_per_s"] = round(host_loader_rate(root, 256, 32, a.loader_batches), 1)
        print(json.dumps(res), flush=True)
        from data.cub_200_2011_dataset import CubDataset
        ds = CubDataset(cub_args(256, 32), root=root)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ds.to_device("cuda")
        res["to_device_s"] = round(time.perf_counter() - t0, 2)
        res["to_device_bytes"] = ds.packed_bytes()
        res["cpu_count"] = os.cpu_count()
        del ds
        res["train_epoch_cfg3"] = train_rates(root, 32, a.epochs, a.rounds)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
