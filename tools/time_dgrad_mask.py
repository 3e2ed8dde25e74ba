"""Timing of the input-gradient launches of a cfg3 step that carry the fused LeakyReLU adjoint (b3d_conv_opts.mask: the
discriminators' backward chain, b3d.conv.ActLink), each WITH and WITHOUT the mask on the same operands: the stride-2 4x4
layers of the texture discriminator (d1.conv2 / conv3 / conv4: 64-, 128- and 256-wide tiles) and of the mesh discriminator
(d2.conv2 / conv3), at batch 32 (generator step, no bias sums) and 64 (discriminator step, with them; at batch 64 the
masked launch is also timed without the bias sums, which the unmasked launch does not compute).

    python tools/time_dgrad_mask.py [--ref-lib OTHER/libb3d.so] [--reps 7] [--n 20]

--ref-lib loads a second build of libb3d (for instance the previous commit's), times its b3d_conv2d_tf32 on the same
operands, alternating with this tree's library launch window by launch window, and checks that both builds' masked gx are
bitwise equal.  Each entry is the median over --reps windows of --n launches, CUDA events around each window."""
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
import b3d.conv as C  # noqa: E402
from tools.time_wgrad import card, timed  # noqa: E402

B = 32
# name, layer Cin (= channels of gx and of the mask), H, W (x-padded input), layer Cout; all 4x4, stride 2, pad_y 1
LAYERS = [("d1.conv2", 64, 256, 258, 128), ("d1.conv3", 128, 128, 130, 256), ("d1.conv4", 256, 64, 66, 512),
          ("d2.conv2", 64, 32, 34, 128), ("d2.conv3", 128, 16, 18, 256)]


def sm_clock():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return ""


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref-lib", default=None)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--n", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_dgrad_mask: needs a CUDA device")
    libs = [("this", b3d.lib)]
    if a.ref_lib:
        ref = ctypes.CDLL(os.path.abspath(a.ref_lib))
        ref.b3d_last_error.restype = ctypes.c_char_p
        ref.b3d_conv2d_tf32.argtypes = b3d.lib.b3d_conv2d_tf32.argtypes
        ref.b3d_conv2d_tf32.restype = b3d.lib.b3d_conv2d_tf32.restype
        libs.append(("ref", ref))
    print(json.dumps({"card": card(), "sm_clock_max_now": sm_clock(), "libs": [n for n, _ in libs], "reps": a.reps, "n": a.n}))
    dev = "cuda:0"
    g = torch.Generator(device=dev).manual_seed(0)
    tot = {}
    for name, Cin, H, W, Cout in LAYERS:
        for N in (B, 2 * B):
            Hout, Wout = H // 2, (W - 4) // 2 + 1
            gy = torch.randn(N, Hout, Wout, Cout, device=dev, generator=g)
            wd = torch.randn(16, Cin, Cout, device=dev, generator=g) * 0.05
            mask = torch.randn(N, H, W, Cin, device=dev, generator=g)
            sums = torch.zeros(2 * Cin, device=dev, dtype=torch.float64) if N == 2 * B else None

            def call(lib, m, s=True):
                def run():
                    C.lib = lib
                    try:
                        return C._dgrad(gy, wd, (H, W), 4, 4, 1, 2, mask=mask if m else None, slope=0.2,
                                        sums=sums if m and s else None)
                    finally:
                        C.lib = b3d.lib
                return run

            fns = [(f"{'masked' if m else 'plain'}_{ln}", call(lib, m)) for m in (True, False) for ln, lib in libs]
            if sums is not None:        # the mask without the bias sums: what the mask alone costs over the plain launch
                fns.append(("masked_nosums_this", call(b3d.lib, True, False)))
            row = {"launch": f"{name}.dgrad", "N": N, "gflop": round(2.0 * N * Hout * Wout * Cin * Cout * 16 / 1e9, 1)}
            if a.ref_lib:
                outs = [f() for k, f in fns if k.startswith("masked")]
                row["gx_bitwise_equal"] = bool(torch.equal(outs[0], outs[1]))
                del outs
            ms = timed([f for _, f in fns], a.reps, a.n)
            for (k, _), m in zip(fns, ms):
                row[f"ms_{k}"] = round(m, 4)
                tot[k] = tot.get(k, 0.0) + m
            row["masked_over_plain_this"] = round(row["ms_masked_this"] / row["ms_plain_this"], 3)
            if sums is not None:
                row["masked_nosums_over_plain_this"] = round(row["ms_masked_nosums_this"] / row["ms_plain_this"], 3)
            print(json.dumps(row), flush=True)
            del gy, wd, mask, sums
    print(json.dumps({"total_ms": {k: round(v, 3) for k, v in tot.items()}}))


if __name__ == "__main__":
    main()
