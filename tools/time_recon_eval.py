"""Device timing of the reconstruction validation pass and of the fused RGBA loss kernels on one GPU (development aid).

  * the card's name, power limit and maximum SM clock (read-only nvidia-smi query);
  * ReconTrainer.evaluate at cfg4 shapes — batch 50, the 31-ring (P3D) template, 256 x 256 renders, texture 128,
    --optimize_z0 and deltas: 5 warm-up batches, then 5 windows of 20 timed batches, each one evaluate() call between
    CUDA events (the call ends in its one host sync) -> images/s of the median window;
  * b3d_rgba_{mse,l1}_iou_fwd / b3d_rgba_{mse,l1}_bwd at batch 50 x 256^2, MSE and L1 alternated in the same process
    (5 rounds of 200 launches each, median per launch), each against its HBM lower bound: bytes counted from the shapes
    (forward 32 B per pixel read; backward 32 B read + 16 B written) over the H100 SXM data-sheet 3.35 TB/s."""
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "2dimageto3dmodel_b200"))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
B, R = 50, 256


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else f"{torch.cuda.get_device_name(0)} (nvidia-smi unavailable: no power limit)"


def batch(seed, dev):
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.linspace(-1, 1, R), torch.linspace(-1, 1, R), indexing="ij")
    disk = ((yy * yy + xx * xx) < 0.45).float()
    X = torch.rand(B, 4, R, R, generator=g) * 2 - 1
    X[:, 3] = disk
    X[:, :3] *= disk
    return [t.to(dev) for t in (X, 0.55 + 0.3 * torch.rand(B, 1, generator=g), (torch.rand(B, 3, generator=g) - 0.5) * 0.3,
                                torch.nn.functional.normalize(torch.randn(B, 4, generator=g), dim=-1))]


def events_ms(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def validation_pass(dev):
    from reconstruction_training import ReconTrainer, default_args
    from rendering.mesh_template import MeshTemplate
    from tools.uvsphere import write_uvsphere_obj
    tpl = MeshTemplate(write_uvsphere_obj(os.path.join(tempfile.mkdtemp(), "uvsphere_31rings.obj"), rings=31), device=dev)
    torch.manual_seed(4321)
    tr = ReconTrainer(default_args(optimize_z0=True), tpl, dataset_size=4722, device=dev)
    data = [batch(s, dev) for s in range(4)]
    tr.evaluate([data[i % 4] for i in range(5)])
    n = 20
    ts = [events_ms(lambda: tr.evaluate([data[i % 4] for i in range(n)])) for _ in range(5)]
    ms = statistics.median(ts)
    print(f"validation pass (evaluate), batch {B}, 256^2, texture 128, 31-ring template, 5 x {n} timed batches: "
          f"{ms / n:.2f} ms per batch = {n * B / ms * 1e3:.0f} images/s (median window; windows {min(ts) / n:.2f}-{max(ts) / n:.2f} ms per batch)")


def loss_kernels(dev):
    import b3d
    from b3d import lib, ptr, stream_ptr
    g = torch.Generator(device=dev).manual_seed(1)
    image = torch.rand(B, R, R, 3, device=dev, generator=g) * 2 - 1
    alpha = torch.rand(B, R, R, device=dev, generator=g)
    target = torch.rand(B, 4, R, R, device=dev, generator=g) * 2 - 1
    loss, counts, gloss = torch.empty(1, device=dev), torch.empty(B, 2, device=dev, dtype=torch.int32), torch.ones(1, device=dev)
    d_image, d_alpha = torch.empty_like(image), torch.empty_like(alpha)
    st = stream_ptr(image)
    calls = {
        "mse fwd": lambda: lib.b3d_rgba_mse_iou_fwd(ptr(image), ptr(alpha), ptr(target), B, R, R, ptr(loss), ptr(counts), st),
        "l1 fwd": lambda: lib.b3d_rgba_l1_iou_fwd(ptr(image), ptr(alpha), ptr(target), B, R, R, ptr(loss), ptr(counts), st),
        "mse bwd": lambda: lib.b3d_rgba_mse_bwd(ptr(image), ptr(alpha), ptr(target), B, R, R, ptr(gloss), ptr(d_image), ptr(d_alpha), st),
        "l1 bwd": lambda: lib.b3d_rgba_l1_bwd(ptr(image), ptr(alpha), ptr(target), B, R, R, ptr(gloss), ptr(d_image), ptr(d_alpha), st),
    }
    for fn in calls.values():
        b3d.check(fn())
    launches = 200

    def many(fn):
        for _ in range(launches):
            fn()
    times = {k: [] for k in calls}
    for _ in range(5):
        for k, fn in calls.items():
            times[k].append(events_ms(lambda: many(fn)) / launches * 1e3)
    pix = B * R * R
    for k, ts in times.items():
        nbytes = pix * (32 if "fwd" in k else 48)
        us = statistics.median(ts)
        bound = nbytes / HBM_BYTES_PER_S * 1e6
        print(f"rgba {k}: {us:.1f} us per launch (median of 5 x {launches}; spread {min(ts):.1f}-{max(ts):.1f}), "
              f"{nbytes / 1e6:.0f} MB -> HBM bound {bound:.1f} us = {bound / us:.0%} of 3.35 TB/s")


def main():
    if not torch.cuda.is_available():
        raise SystemExit("time_recon_eval.py needs a CUDA device")
    dev = torch.device("cuda:0")
    print("card (name, power limit, max SM clock):", card())
    validation_pass(dev)
    loss_kernels(dev)


if __name__ == "__main__":
    main()
