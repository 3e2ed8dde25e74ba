"""Weight-gradient timing at cfg3's geometries (batch 32 for the generator's layers, 64 for the discriminator's), and the
discriminator stem (5x5, 8 -> 64 channels at 256^2) both ways: materialised fold + generic kernel, and the raw-input kernel;
its forward both ways too.

    python tools/time_wgrad.py [--ref-lib OTHER/libb3d.so ...] [--reps 7] [--n 20]

--ref-lib (repeatable) loads other builds of libb3d (for instance the previous commit's) and times their
b3d_conv2d_wgrad_tf32 on the same operands, alternating with this tree's library launch window by launch window; a build is
named by its file name.  Each entry is the median over --reps windows of --n launches, CUDA events around each window, and
its spread (slowest - fastest window).  step_ms is one cfg3 step's share: the generator's launches once, the
discriminator's twice (two D steps at batch 64), without D1.c1.khfold, the materialised fold that the raw-input stem
kernel (the stem line, wgrad_raw) replaces."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "2dimageto3dmodel_b200"))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import b3d  # noqa: E402
from b3d.conv import _fprop  # noqa: E402
from b3d.ew import fold_rows  # noqa: E402

B = 32
# name, N, Cin, H, W (x-padded), Cout, k, pad_y, stride — the tensor-core weight-gradient launches of a cfg3 step
CFG3 = [("G.blk1.conv", B, 512, 8, 6, 512, 3, 1, 1), ("G.blk2.conv1", B, 512, 16, 10, 256, 3, 1, 1),
        ("G.blk2.conv2", B, 256, 16, 10, 256, 3, 1, 1), ("G.blk3a.conv", B, 256, 32, 18, 256, 3, 1, 1),
        ("G.blk3_mesh.conv1", B, 256, 32, 18, 64, 3, 1, 1), ("G.blk4.conv1", B, 256, 64, 34, 128, 3, 1, 1),
        ("G.blk4.conv2", B, 128, 64, 34, 128, 3, 1, 1), ("G.blk5.conv", B, 128, 128, 66, 128, 3, 1, 1),
        ("G.blk6.conv1", B, 128, 256, 130, 64, 3, 1, 1), ("G.blk6.conv2", B, 64, 256, 130, 64, 3, 1, 1),
        ("G.blk6.short", B, 128, 256, 128, 64, 1, 0, 1),
        ("D1.c1.khfold", 2 * B, 64, 256, 260, 64, (1, 5), 0, 1), ("D1.conv2", 2 * B, 64, 256, 258, 128, 4, 1, 2),
        ("D1.conv3", 2 * B, 128, 128, 130, 256, 4, 1, 2), ("D1.conv4", 2 * B, 256, 64, 66, 512, 4, 1, 2)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def window(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def windows(fns, reps, n):
    """ms per call of each fn in each of reps windows of n calls, the fns alternated window by window."""
    for f in fns:
        f()
    torch.cuda.synchronize()
    ts = [[] for _ in fns]
    for _ in range(reps):
        for i, f in enumerate(fns):
            ts[i].append(window(f, n))
    return ts


def timed(fns, reps, n):
    """Median ms per call of each fn, the fns alternated window by window."""
    return [sorted(t)[len(t) // 2] for t in windows(fns, reps, n)]


def wgrad_call(lib, dy, x, dw, N, H, W, Cin, Hout, Wout, Cout, kh, kw, pad_y, st, tap_major=1, fold_kh=0):
    vp = lambda t: ctypes.c_void_p(t.data_ptr())
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    return lambda: b3d.check(lib.b3d_conv2d_wgrad_tf32(vp(dy), vp(x), vp(dw), N, H, W, Cin, Hout, Wout, Cout, kh, kw, pad_y, st,
                                                       0, tap_major, fold_kh, 0, stream))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref-lib", action="append", default=[])
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--n", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_wgrad: needs a CUDA device")
    libs = [("this", b3d.lib)]
    for path in a.ref_lib:
        ref = ctypes.CDLL(os.path.abspath(path))
        ref.b3d_last_error.restype = ctypes.c_char_p
        libs.append((os.path.splitext(os.path.basename(path))[0], ref))
    print(json.dumps({"card": card(), "libs": [n for n, _ in libs], "reps": a.reps, "n": a.n}))
    dev = "cuda:0"
    tot = {n: 0.0 for n, _ in libs}
    step = {n: 0.0 for n, _ in libs}
    for name, N, Cin, H, W, Cout, k, py, st in CFG3:
        kh, kw = k if isinstance(k, tuple) else (k, k)
        Hout, Wout = (H + 2 * py - kh) // st + 1, (W - kw) // st + 1
        x = torch.randn(N, H, W, Cin, device=dev)
        dy = torch.randn(N, Hout, Wout, Cout, device=dev)
        dw = torch.zeros(kh * kw, Cout, Cin, device=dev)
        ts = windows([wgrad_call(lib, dy, x, dw, N, H, W, Cin, Hout, Wout, Cout, kh, kw, py, st) for _, lib in libs], a.reps, a.n)
        row = {"layer": name, "gflop": 2.0 * N * Hout * Wout * Cout * Cin * kh * kw / 1e9}
        per_step = 0 if name == "D1.c1.khfold" else 2 if name.startswith("D") else 1
        for (ln, _), t in zip(libs, ts):
            m = sorted(t)[len(t) // 2]
            row[f"ms_{ln}"] = round(m, 4)
            row[f"spread_{ln}"] = round(max(t) - min(t), 4)
            tot[ln] += m
            step[ln] += per_step * m
        print(json.dumps(row), flush=True)
        del x, dy, dw
    print(json.dumps({"total_ms": {k: round(v, 3) for k, v in tot.items()},
                      "step_ms": {k: round(v, 3) for k, v in step.items()}}))

    # the stem of cfg3's D step: raw input [64, 256, 260, 8], 5 rows folded into 64 channels (y padding 2)
    N, H, W, Cout, pad = 2 * B, 256, 260, 64, 2
    Hout, Wout = H, W - 4
    xr = torch.randn(N, H, W, 8, device=dev)
    dy = torch.randn(N, Hout, Wout, Cout, device=dev)
    wf = torch.randn(5, Cout, 64, device=dev) * 0.05
    wf[:, :, 40:] = 0
    dw = torch.zeros(5, Cout, 64, device=dev)
    xf = fold_rows(xr, 5, pad, 64)
    rows = {"fold_rows": lambda: fold_rows(xr, 5, pad, 64),
            "wgrad_on_fold": wgrad_call(b3d.lib, dy, xf, dw, N, H, W, 64, Hout, Wout, Cout, 1, 5, 0, 1),
            "fwd_fold_then_rowwin": lambda: _fprop(fold_rows(xr, 5, pad, 64), wf, None, 1, 5),
            "fwd_on_the_fly": lambda: _fprop(xr, wf, None, 1, 5, fold_kh=5, fold_pad=pad)}
    for ln, lib in libs:
        if lib.b3d_version() >= 350:
            rows[f"wgrad_raw_{ln}"] = wgrad_call(lib, dy, xr, dw, N, H, W, 64, Hout, Wout, Cout, 1, 5, pad, 1, fold_kh=5)
    ts = windows(list(rows.values()), a.reps, a.n)
    out = {"stem": "D1.conv1 cfg3 (N 64, 256x256, 8 -> 64, 5x5)"}
    for k, t in zip(rows, ts):
        out[f"ms_{k}"] = round(sorted(t)[len(t) // 2], 4)
        out[f"spread_{k}"] = round(max(t) - min(t), 4)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
