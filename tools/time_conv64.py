"""Timing of the 64-output-channel forward / input-gradient launches of a cfg3 step (the conv_wgmma<64,8> and
conv_wgmma_rowwin<64,KW,S> instances), at cfg3's geometries: batch 32 for the generator step, 64 for the discriminator's.

    python tools/time_conv64.py [--ref-lib OTHER/libb3d.so] [--reps 7] [--n 20]

--ref-lib loads a second build of libb3d (for instance the previous commit's) and times its b3d_conv2d_tf32 on the same
operands, alternating with this tree's library launch window by launch window.  Each entry is the median over --reps
windows of --n launches, CUDA events around each window, and its spread (slowest - fastest window)."""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "2dimageto3dmodel_b200"))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import b3d  # noqa: E402
import b3d.conv as C  # noqa: E402
from b3d.ew import fold_rows  # noqa: E402
from tools.time_wgrad import card, windows  # noqa: E402

B = 32


def cases(dev):
    """name -> (operands, callable(x...) that launches the layer through b3d.conv's helpers)."""
    g = torch.Generator(device=dev).manual_seed(0)
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g)
    out = {}

    def fwd(name, N, Cin, H, W, k, pad_y, x_crop=0, stats=False):
        x, wt = rnd(N, H, W, Cin), rnd(k * k, 64, Cin) * 0.05
        st = torch.zeros(128, device=dev, dtype=torch.float64) if stats else None
        out[name] = (2.0 * N * H * (W - 2 * x_crop - k + 1) * 64 * Cin * k * k,
                     lambda: C._fprop(x, wt, None, k, k, pad_y, 1, x_crop=x_crop, stats=st))

    def dgrad(name, N, Cout, H, W, k, pad_y, stride, masked, kh=None):
        kh = kh or k
        Hout, Wout = (H + 2 * pad_y - kh) // stride + 1, (W - k) // stride + 1
        gy, wd = rnd(N, Hout, Wout, Cout), rnd(kh * k, 64, Cout) * 0.05
        mask = rnd(N, H, W, 64) if masked else None
        sums = torch.zeros(128, device=dev, dtype=torch.float64) if masked else None
        out[name] = (2.0 * N * Hout * Wout * 64 * Cout * kh * k,
                     lambda: C._dgrad(gy, wd, (H, W), kh, k, pad_y, stride, mask=mask, slope=0.2, sums=sums))

    fwd("G.blk6.conv1.fwd", B, 128, 256, 130, 3, 1, stats=True)
    fwd("G.blk6.conv2.fwd", B, 64, 256, 130, 3, 1, stats=True)
    fwd("G.blk6.short.fwd", B, 128, 256, 130, 1, 0, x_crop=1)
    fwd("G.blk3_mesh.conv1.fwd", B, 256, 32, 18, 3, 1, stats=True)
    dgrad("G.blk6.conv2.dgrad", B, 64, 256, 130, 3, 1, 1, True)
    dgrad("G.conv_final.dgrad", B, 32, 256, 132, 5, 2, 1, False)
    dgrad("D1.conv2.dgrad", 2 * B, 128, 256, 258, 4, 1, 2, True)
    xr = rnd(2 * B, 256, 260, 8)
    xf, wf = fold_rows(xr, 5, 2, 64), rnd(5, 64, 64) * 0.05
    out["D1.stem.fwd.folded"] = (2.0 * 2 * B * 256 * 256 * 64 * 64 * 5, lambda: C._fprop(xf, wf, None, 1, 5))
    out["D1.stem.fwd.on_the_fly"] = (2.0 * 2 * B * 256 * 256 * 64 * 64 * 5,
                                     lambda: C._fprop(xr, wf, None, 1, 5, fold_kh=5, fold_pad=2))
    dgrad("D1.stem.dgrad.folded", B, 64, 256, 260, 5, 0, 1, False, kh=1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref-lib", default=None)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--n", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_conv64: needs a CUDA device")
    libs = [("this", b3d.lib)]
    if a.ref_lib:
        ref = ctypes.CDLL(os.path.abspath(a.ref_lib))
        ref.b3d_last_error.restype = ctypes.c_char_p
        ref.b3d_conv2d_tf32.argtypes = b3d.lib.b3d_conv2d_tf32.argtypes
        ref.b3d_conv2d_tf32.restype = b3d.lib.b3d_conv2d_tf32.restype
        libs.append(("ref", ref))
    print(json.dumps({"card": card(), "libs": [n for n, _ in libs], "reps": a.reps, "n": a.n}))

    def on(lib, fn):
        def run():
            C.lib = lib
            fn()
        return run

    tot = {n: 0.0 for n, _ in libs}
    for name, (flop, fn) in cases("cuda:0").items():
        ts = windows([on(lib, fn) for _, lib in libs], a.reps, a.n)
        C.lib = b3d.lib
        row = {"launch": name, "gflop": round(flop / 1e9, 1)}
        for (ln, _), t in zip(libs, ts):
            m = sorted(t)[len(t) // 2]
            row[f"ms_{ln}"] = round(m, 4)
            row[f"spread_{ln}"] = round(max(t) - min(t), 4)
            row[f"tflops_{ln}"] = round(flop / m / 1e9, 1)
            tot[ln] += m
        print(json.dumps(row), flush=True)
    print(json.dumps({"total_ms": {k: round(v, 3) for k, v in tot.items()}}))


if __name__ == "__main__":
    main()
