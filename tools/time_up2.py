"""Timing of the generator's upsampled-input layers (conv1 of blk2, blk3a/b, blk4, blk5, blk6 and blk3_mesh, with the block's
1x1 shortcut) the old way and the new way, at their cfg3 (batch 32, 256^2) and cfg5 (batch 8, 512^2) shapes.

  old: the x2-upsampled, x-padded map [N,2H,2W+2,Cin] through b3d.conv's generic helpers: the 3x3 convolution with its
       statistics and the 1x1 shortcut on the upsampled pixels; the two input gradients added as autograd adds them;
  new: the low-resolution padded map [N,H,W+2,Cin] through _up_fprop / _up_dgrad / _up_wgrad (b3d.conv.conv2d_up2_banked),
       the weight gradient including its zeroed dP^T buffer and b3d_up2_fold.

Then the two weight-gradient forms on blk6.conv1 (cfg3 and cfg5), without the shortcut:
  (a) four classes of 2x2-tap weight gradients with Cout as the M operand; the weight-gradient kernel reads dY densely, so
      each class's dY[:, py::2, px::2] is copied out first (the copies are timed with it) and the result is folded the
      same way (one b3d_up2_fold of the same size is timed in its place);
  (b) the 4x4 stride-2 weight gradient with Xp as the M operand (what _up_wgrad runs).
Both are checked against each other before they are timed.

    python tools/time_up2.py [--reps 7] [--n 10]

Each entry is the median over --reps windows of --n calls, CUDA events around each window, the old and new forms
alternated window by window, and the spread (slowest - fastest window).  GFLOP are the multiply-adds the launches execute
(x2), counted from their geometry: zero taps of the pad-column launches included."""
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

# (config, layer, N, low-resolution H, W, Cin, Cout of conv1, Cout of the 1x1 shortcut or 0 = identity)
LAYERS = [
    ("cfg3", "blk2", 32, 8, 4, 512, 256, 256), ("cfg3", "blk3a", 32, 16, 8, 256, 256, 0),
    ("cfg3", "blk3_mesh", 32, 16, 8, 256, 64, 64), ("cfg3", "blk4", 32, 32, 16, 256, 128, 128),
    ("cfg3", "blk5", 32, 64, 32, 128, 128, 0), ("cfg3", "blk6", 32, 128, 64, 128, 64, 64),
    ("cfg5", "blk2", 8, 8, 4, 512, 256, 256), ("cfg5", "blk3a", 8, 16, 8, 256, 256, 0),
    ("cfg5", "blk3b", 8, 32, 16, 256, 256, 0), ("cfg5", "blk3_mesh", 8, 16, 8, 256, 64, 64),
    ("cfg5", "blk4", 8, 64, 32, 256, 128, 128), ("cfg5", "blk5", 8, 128, 64, 128, 128, 0),
    ("cfg5", "blk6", 8, 256, 128, 128, 64, 64),
]
# generator passes per step: forwards (one G step, two D steps), one input gradient, one weight gradient
PASSES = {"fwd": 3, "dgrad": 1, "wgrad": 1}


def layer(dev, N, H, W, Cin, Cout, Csc):
    """direction -> (old GFLOP, new GFLOP, old callable, new callable)."""
    g = torch.Generator(device=dev).manual_seed(H * 7 + Cin)
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g)
    z = lambda *s, dt=torch.float32: torch.zeros(*s, device=dev, dtype=dt)
    H2, W2 = 2 * H, 2 * W
    xu, xp = rnd(N, H2, W2 + 2, Cin), rnd(N, H, W + 2, Cin)
    gy = rnd(N, H2, W2, Cout)
    f9, d9, p16, d4 = rnd(9, Cout, Cin) * .05, rnd(9, Cin, Cout) * .05, rnd(16, Cout, Cin) * .05, rnd(16, Cin, Cout) * .05
    df9, st = z(9, Cout, Cin), z(2 * Cout, dt=torch.float64)
    fsc = dsc = dfsc = gsc_hi = gsc_lo = None
    if Csc:
        fsc, dsc, dfsc = rnd(1, Csc, Cin) * .05, rnd(1, Cin, Csc) * .05, z(1, Csc, Cin)
        gsc_hi, gsc_lo = rnd(N, H2, W2, Csc), rnd(N, H, W, Csc)
    mac9, mac16 = 9 * N * H2 * W2 * Cin * Cout, 16 * N * H * W * Cin * Cout
    sc_hi, sc_lo = N * H2 * W2 * Cin * Csc, N * H * W * Cin * Csc

    def old_fwd():
        C._fprop(xu, f9, None, 3, 3, 1, stats=st)
        if Csc:
            C._fprop(xu, fsc, None, 1, 1, x_crop=1)

    def old_dgrad():
        gx = C._dgrad(gy, d9, (H2, W2 + 2), 3, 3, 1)
        if Csc:
            gx += C._dgrad(gsc_hi, dsc, (H2, W2 + 2), 1, 1, 0, 1, 1)

    def old_wgrad():
        C._wgrad(gy, xu, 3, 3, 1, sink=df9)
        if Csc:
            C._wgrad(gsc_hi, xu, 1, 1, 0, 1, 1, sink=dfsc)

    return {
        "fwd": (2 * (mac9 + sc_hi), 2 * (mac16 + sc_lo), old_fwd, lambda: C._up_fprop(xp, p16, fsc, st)),
        "dgrad": (2 * (9 * N * H2 * (W2 + 2) * Cin * Cout + N * H2 * (W2 + 2) * Cin * Csc),
                  2 * (16 * N * H * (W + 2) * Cin * Cout + N * H * (W + 2) * Cin * Csc), old_dgrad,
                  lambda: C._up_dgrad(gy, d4, gsc_lo, dsc)),
        "wgrad": (2 * (mac9 + sc_hi), 2 * (16 * N * H * (W + 2) * Cin * Cout + sc_lo), old_wgrad,
                  lambda: C._up_wgrad(gy, xp, df9, gsc_lo, dfsc)),
    }


def wgrad_options(dev, N, H, W, Cin, Cout):
    """(a) and (b) on one layer: (GFLOP a, GFLOP b, callable a, callable b); raises if they disagree."""
    g = torch.Generator(device=dev).manual_seed(5)
    xp, gy = torch.randn(N, H, W + 2, Cin, device=dev, generator=g), torch.randn(N, 2 * H, 2 * W, Cout, device=dev, generator=g)
    df9 = torch.zeros(9, Cout, Cin, device=dev)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    vp = lambda t: ctypes.c_void_p(t.data_ptr())

    def option_a(fold=True):
        dp = torch.zeros(4, 4, Cout, Cin, device=dev)             # [class (py, px)][tap (a, b)][Cout][Cin]
        for c, (py, px) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
            gc = gy[:, py::2, px::2].contiguous()
            # dP[py][px][a][b] = sum dY[2i+py, 2j+px] (x) Xp[i + a - (1 - py), j + px + b]: a 2x2 stride-1 weight gradient
            b3d.check(lib.b3d_conv2d_wgrad_tf32(vp(gc), vp(xp), vp(dp[c]), N, H, W + 2, Cin, H, W, Cout, 2, 2, 1 - py, 1, px, 1, 0, 0,
                                                stream))
        if fold:
            b3d.check(lib.b3d_up2_fold(vp(dpt_like), vp(df9), Cout, Cin, stream))
        return dp

    lib = b3d.lib
    dpt_like = torch.zeros(16, Cin, Cout, device=dev)
    # agreement: (b)'s dP^T in D4's tap order against (a)'s dP
    dpa = option_a(fold=False).reshape(16, Cout, Cin)
    dpt = torch.zeros(16, Cin, Cout, device=dev)
    for j0, w, x_off in C.up2_wgrad_columns(W):
        b3d.check(lib.b3d_conv2d_wgrad_tf32(ctypes.c_void_p(xp.data_ptr() + 4 * Cin * j0), vp(gy), vp(dpt), N, 2 * H, 2 * W, Cout, H, w,
                                            Cin, 4, 4, 1, 2, x_off, 1, 0, W + 2, stream))
    for q in range(16):
        py, px, a, b = q >> 3, (q >> 2) & 1, (q >> 1) & 1, q & 1
        ref = dpt[(3 - py - 2 * a) * 4 + 3 - px - 2 * b].t()
        err = float((dpa[q] - ref).abs().max())
        if err > 1e-3 * float(ref.abs().max()):
            raise RuntimeError(f"wgrad options disagree at phase tap {q}: {err}")
    return (2 * 16 * N * H * W * Cin * Cout, 2 * 16 * N * H * (W + 2) * Cin * Cout, option_a,
            lambda: C._up_wgrad(gy, xp, df9))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--n", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_up2: needs a CUDA device")
    print(json.dumps({"card": card(), "reps": a.reps, "n": a.n}))

    def row(name, gf_old, gf_new, fns, labels=("old", "new")):
        ts = windows(fns, a.reps, a.n)
        r = {"launch": name}
        ms = []
        for lab, gf, t in zip(labels, (gf_old, gf_new), ts):
            m = sorted(t)[len(t) // 2]
            ms.append(m)
            r[f"ms_{lab}"], r[f"spread_{lab}"], r[f"gflop_{lab}"] = round(m, 4), round(max(t) - min(t), 4), round(gf / 1e9, 2)
        print(json.dumps(r), flush=True)
        return ms

    per_step = {}
    for cfg, name, N, H, W, Cin, Cout, Csc in LAYERS:
        for d, (gf_old, gf_new, old, new) in layer("cuda:0", N, H, W, Cin, Cout, Csc).items():
            m_old, m_new = row(f"{cfg}.{name}.{d}", gf_old, gf_new, [old, new])
            t = per_step.setdefault(cfg, [0.0, 0.0, 0.0, 0.0])
            t[0] += PASSES[d] * m_old
            t[1] += PASSES[d] * m_new
            t[2] += PASSES[d] * gf_old / 1e9
            t[3] += PASSES[d] * gf_new / 1e9
    for cfg, (mo, mn, go, gn) in per_step.items():
        print(json.dumps({"per_step": cfg, "ms_old": round(mo, 3), "ms_new": round(mn, 3), "gflop_old": round(go, 1),
                          "gflop_new": round(gn, 1)}))
    for cfg, N, H, W in (("cfg3", 32, 128, 64), ("cfg5", 8, 256, 128)):
        gf_a, gf_b, fa, fb = wgrad_options("cuda:0", N, H, W, 128, 64)
        row(f"{cfg}.blk6.conv1.wgrad_options", gf_a, gf_b, [fa, fb], labels=("a", "b"))


if __name__ == "__main__":
    main()
