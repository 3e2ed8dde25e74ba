"""Timing of the 128- and 256-output-channel forward / input-gradient launches of a cfg3 step (conv_wgmma<128,6>,
conv_wgmma_rowwin<128,KW,S>, conv_wgmma<256,4>), at cfg3's geometries: batch 32 for the generator and the generator step's
discriminator pass, 64 for the discriminator step.  The masked input gradients (the LeakyReLU adjoint fused) run with
and without the bias sums, and unmasked.  Then the cfg4 and cfg5 launches that get 256-wide tiles.

    python tools/time_conv128.py [--ref-lib OTHER/libb3d.so ...] [--reps 7] [--n 20]

--ref-lib (repeatable) loads other builds of libb3d (for instance the previous commit's) and times their
b3d_conv2d_tf32 on the same operands, alternating with this tree's library launch window by launch window.  Each entry is
the median over --reps windows of --n launches, CUDA events around each window, and its spread (slowest - fastest window)."""
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
from tools.time_wgrad import card, windows  # noqa: E402

B = 32


def cases(dev):
    """name -> (FLOP, callable that launches the layer through b3d.conv's helpers)."""
    g = torch.Generator(device=dev).manual_seed(0)
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g)
    out = {}

    def fwd(name, N, Cin, H, W, Cout, k, pad_y, stride=1, x_crop=0, stats=False):
        Hout, Wout = (H + 2 * pad_y - k) // stride + 1, (W - 2 * x_crop - k) // stride + 1
        x, wt = rnd(N, H, W, Cin), rnd(k * k, Cout, Cin) * 0.05
        st = torch.zeros(2 * Cout, device=dev, dtype=torch.float64) if stats else None
        out[name] = (2.0 * N * Hout * Wout * Cout * Cin * k * k,
                     lambda: C._fprop(x, wt, None, k, k, pad_y, stride, x_crop=x_crop, stats=st))

    def dgrad(name, N, Cin, H, W, Cout, k, pad_y, stride=1, x_crop=0, masked=False, sums=False):
        Hout, Wout = (H + 2 * pad_y - k) // stride + 1, (W - 2 * x_crop - k) // stride + 1
        gy, wd = rnd(N, Hout, Wout, Cout), rnd(k * k, Cin, -(-Cout // 32) * 32) * 0.05      # D: K zero-padded to 32
        mask = rnd(N, H, W, Cin) if masked else None
        s = torch.zeros(2 * Cin, device=dev, dtype=torch.float64) if sums else None
        out[name] = (2.0 * N * Hout * Wout * Cout * Cin * k * k,
                     lambda: C._dgrad(gy, wd, (H, W), k, k, pad_y, stride, x_crop, mask=mask, slope=0.2, sums=s))

    # generator (batch 32, BN statistics in the forward epilogue)
    fwd("G.blk1.conv.fwd", B, 512, 8, 6, 512, 3, 1, stats=True)
    fwd("G.blk2.conv1.fwd", B, 512, 16, 10, 256, 3, 1, stats=True)
    fwd("G.blk2.conv2.fwd", B, 256, 16, 10, 256, 3, 1, stats=True)
    fwd("G.blk2.short.fwd", B, 512, 16, 10, 256, 1, 0, x_crop=1)
    fwd("G.blk3a.conv.fwd", B, 256, 32, 18, 256, 3, 1, stats=True)
    fwd("G.blk4.conv1.fwd", B, 256, 64, 34, 128, 3, 1, stats=True)
    fwd("G.blk4.conv2.fwd", B, 128, 64, 34, 128, 3, 1, stats=True)
    fwd("G.blk4.short.fwd", B, 256, 64, 34, 128, 1, 0, x_crop=1)
    fwd("G.blk5.conv.fwd", B, 128, 128, 66, 128, 3, 1, stats=True)
    dgrad("G.blk2.conv2.dgrad", B, 256, 16, 10, 256, 3, 1)
    dgrad("G.blk3a.conv.dgrad", B, 256, 32, 18, 256, 3, 1)
    dgrad("G.blk4.conv1.dgrad", B, 256, 64, 34, 128, 3, 1)
    dgrad("G.blk4.short.dgrad", B, 256, 64, 34, 128, 1, 0, x_crop=1)
    dgrad("G.blk4.conv2.dgrad", B, 128, 64, 34, 128, 3, 1)
    dgrad("G.blk5.conv.dgrad", B, 128, 128, 66, 128, 3, 1)
    dgrad("G.blk6.conv1.dgrad", B, 128, 256, 130, 64, 3, 1)
    # discriminators: forward at 32 (generator step) and 64 (discriminator step), masked input gradients
    for N in (B, 2 * B):
        fwd(f"D1.conv2.fwd.b{N}", N, 64, 256, 258, 128, 4, 1, 2)
        fwd(f"D1.conv3.fwd.b{N}", N, 128, 128, 130, 256, 4, 1, 2)
        fwd(f"D1.conv4.fwd.b{N}", N, 256, 64, 66, 512, 4, 1, 2)
        fwd(f"D2.conv3.fwd.b{N}", N, 128, 16, 18, 256, 4, 1, 2)
    dgrad("D1.conv3.dgrad.b32.masked", B, 128, 128, 130, 256, 4, 1, 2, masked=True)
    dgrad("D1.conv4.dgrad.b32.masked", B, 256, 64, 66, 512, 4, 1, 2, masked=True)
    for name, Cin, H, W, Cout in (("D1.conv3", 128, 128, 130, 256), ("D1.conv4", 256, 64, 66, 512), ("D2.conv3", 128, 16, 18, 256)):
        dgrad(f"{name}.dgrad.b64.masked_sums", 2 * B, Cin, H, W, Cout, 4, 1, 2, masked=True, sums=True)
        dgrad(f"{name}.dgrad.b64.masked", 2 * B, Cin, H, W, Cout, 4, 1, 2, masked=True)
        dgrad(f"{name}.dgrad.b64.unmasked", 2 * B, Cin, H, W, Cout, 4, 1, 2)
    # cfg4 (reconstruction network, batch 50 and 13) and cfg5 (512^2 GAN, batch 8 and 16): the launches the bn256 rule
    # gives 256-wide tiles (tests/conv_plan.py over the tables of tests/test_workload_shapes_gpu.py)
    fwd("cfg4.conv3e.fwd.b50", 50, 128, 64, 66, 256, 3, 1, 2)
    fwd("cfg4.conv4e.fwd.b50", 50, 256, 32, 34, 512, 3, 1, 2)
    for N in (50, 13):
        fwd(f"cfg4.blk4_tex.conv1.fwd.b{N}", N, 256, 64, 34, 256, 3, 1)
        dgrad(f"cfg4.blk4_tex.conv1.dgrad.b{N}", N, 256, 64, 34, 256, 3, 1)
        dgrad(f"cfg4.blk4_tex.conv2.dgrad.b{N}", N, 256, 64, 34, 128, 3, 1)
        dgrad(f"cfg4.blk4_tex.short.dgrad.b{N}", N, 256, 64, 34, 128, 1, 0, x_crop=1)
    fwd("cfg4.blk3b_tex.conv1.fwd.b50", 50, 256, 32, 18, 256, 3, 1)
    dgrad("cfg4.blk3b_tex.conv1.dgrad.b50", 50, 256, 32, 18, 256, 3, 1)
    dgrad("cfg4.blk4_mesh.conv2.dgrad.b50", 50, 256, 32, 18, 64, 3, 1)
    dgrad("cfg4.blk4_mesh.short.dgrad.b50", 50, 256, 32, 18, 64, 1, 0, x_crop=1)
    dgrad("cfg5.G.blk3b.conv1.dgrad.b8", 8, 256, 64, 34, 256, 3, 1)
    dgrad("cfg5.G.blk4.conv1.dgrad.b8", 8, 256, 128, 66, 128, 3, 1)
    dgrad("cfg5.G.blk4.short.dgrad.b8", 8, 256, 128, 66, 128, 1, 0, x_crop=1)
    for N in (8, 16):
        fwd(f"cfg5.d1.conv3.fwd.b{N}", N, 128, 128, 130, 256, 4, 1, 2)
        dgrad(f"cfg5.d1.conv4.dgrad.b{N}.masked", N, 256, 64, 66, 512, 4, 1, 2, masked=True, sums=N == 16)
        dgrad(f"cfg5.d1.conv5.dgrad.b{N}", N, 512, 32, 36, 1, 5, 2)
    fwd("cfg5.d1.conv4.fwd.b16", 16, 256, 64, 66, 512, 4, 1, 2)
    dgrad("cfg5.d3.conv4.dgrad.b16.masked", 16, 256, 32, 34, 512, 4, 1, 2, masked=True, sums=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref-lib", action="append", default=[])
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--n", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_conv128: needs a CUDA device")
    libs = [("this", b3d.lib)]
    for path in a.ref_lib:
        ref = ctypes.CDLL(os.path.abspath(path))
        ref.b3d_last_error.restype = ctypes.c_char_p
        ref.b3d_conv2d_tf32.argtypes = b3d.lib.b3d_conv2d_tf32.argtypes
        ref.b3d_conv2d_tf32.restype = b3d.lib.b3d_conv2d_tf32.restype
        libs.append((os.path.splitext(os.path.basename(path))[0], ref))
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
