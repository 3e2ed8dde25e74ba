"""Dense conv2d over libb3d's wgmma implicit-GEMM kernel (NHWC fp32 activations, tf32 tensor cores).

Reference call sites: nn.Conv2d layers of /root/reference/code/models/gan.py (:57-65, :163-177, :294-302,
:359, :364) — 3x3 / 1x1 / 5x5 stride 1 and 4x4 stride 2, zero padding along y only (x padding is explicit:
replicate / circular pads are materialised by the caller exactly as the reference does).

Both entry points, conv2d (a module's own weight) and conv2d_banked (weights from b3d.bank.WeightBank), run one autograd
function over the same three launch helpers; they differ only in where the kernel weight layouts come from."""
import ctypes

import torch

from . import B3DError, check, dev, last_variant, lib, ptr, stream_ptr
from .bank import LayerWeights

VARIANT_LOG = None      # tests set this to a list: every kernel template instance the conv entry points launch is appended


def _conv_call(fn, *args):
    """One convolution entry point of libb3d; records which kernel instances it launched when VARIANT_LOG is a list."""
    rc = fn(*args)
    if VARIANT_LOG is not None and rc == 0:
        VARIANT_LOG.extend(v for v in last_variant().split(";") if v)
    return rc


def _ints(v):
    return (ctypes.c_int * len(v))(*v)


def _pad_last(t, mult):
    c = t.shape[-1]
    return t if c % mult == 0 else torch.nn.functional.pad(t, (0, mult - c % mult))


def taps_layout(weight):
    """[Cout,Cin,kh,kw] -> tap-major K-major rows [kh*kw, Cout, Cin]."""
    co, ci, kh, kw = weight.shape
    return weight.permute(2, 3, 0, 1).reshape(kh * kw, co, ci).contiguous()


def _d_layout(wf):
    """F [T][Cout][Cin] -> D [T][Cin][Cout'], its per-tap transpose with Cout zero-padded to a multiple of 32 (the input
    gradient's operand)."""
    return _pad_last(wf.transpose(1, 2), 32).contiguous()


def _thin(Cout, Cin, kh, kw, stride):
    return Cout <= 4 and Cin % 64 == 0 and kh == 5 and kw == 5 and stride == 1


class _ConvOpts(ctypes.Structure):
    """b3d_conv_opts (include/b3d.h)."""
    _fields_ = [("mask", ctypes.c_void_p), ("mask_slope", ctypes.c_float), ("stats_sum_only", ctypes.c_int),
                ("x_row_pitch", ctypes.c_int), ("nclass", ctypes.c_int), ("class_ooy", ctypes.c_int * 4), ("class_oox", ctypes.c_int * 4)]


# ------------------------------------------------------------------------------------------------------------------
# launch helpers: one per direction
# ------------------------------------------------------------------------------------------------------------------
def _fprop(x, wt, bias, kh, kw, pad_y=0, stride=1, leaky=1.0, pad_out=0, pad_mode=1, x_crop=0, stats=None, fold_kh=0,
           fold_pad=0):
    """conv2d_nhwc on F = wt [kh*kw][Cout][Cin'].  stats: zeroed fp64 [2*Cout] that the epilogue accumulates the output's
    per-channel sum / sum of squares into.  fold_kh > 0: x is the RAW 8-channel stem input whose fold_kh vertical taps (y
    padding fold_pad) the kernel folds into the K dimension on the fly (kh = 1, pad_y = 0)."""
    N, H, W, _ = x.shape
    _, Cout, Cin = wt.shape
    if x_crop and stride != 1:
        raise B3DError("conv2d: x_crop needs stride 1")
    if pad_out and Cout % 4:
        raise B3DError("conv2d: pad_out needs Cout % 4 == 0")
    Hout = (H + 2 * fold_pad - fold_kh + 1) if fold_kh else (H + 2 * pad_y - kh) // stride + 1
    Wout = (W - 2 * x_crop - kw) // stride + 1
    OW = Wout + 2 * pad_out
    out = torch.empty(N, Hout, OW, Cout, device=x.device, dtype=torch.float32)
    optr = ctypes.c_void_p(out.data_ptr() + 4 * pad_out * Cout)          # pixel (n, y, pad_out) of the padded buffer
    b = dev(bias, "bias") if bias is not None else None
    st = stream_ptr(x)
    if _thin(Cout, Cin, kh, kw, stride):
        # 1-4 output channels: fp32 CUDA-core reduction kernel (csrc/thin_kernels.cu), not a 64-wide MMA tile
        check(_conv_call(lib.b3d_conv2d_thin_fwd, ptr(x), ptr(wt), ptr(b), optr, N, H, W, Cin, Hout, Wout, Cout, kh, kw, pad_y,
                         x_crop, OW, Cout, float(leaky), st))
    else:
        if stats is not None and (bias is not None or leaky != 1.0 or stride != 1):
            raise B3DError("conv2d: output statistics are taken before bias / activation (plain stride-1 convs only)")
        dy = [r - pad_y for r in range(kh) for _ in range(kw)]
        dx = [s + x_crop for _ in range(kh) for s in range(kw)]
        check(_conv_call(lib.b3d_conv2d_tf32, ptr(x), ptr(wt), ptr(b), optr, N, H, W, Cin, Hout, Wout, Cout, kh * kw, _ints(dy),
                         _ints(dx), stride, stride, Hout, OW, Cout, 1, 1, 0, 0, float(leaky), None, 0, ptr(stats), fold_kh,
                         fold_pad, None, st))
    if pad_out:
        check(lib.b3d_wrap_x_inplace(ptr(out), N * Hout, Wout, Cout, pad_out, pad_mode, st))
    return out


def stride2_classes(kh, kw, pad_y, H, W):
    """Output-parity decomposition of the input gradient of a stride-2 convolution (pure index arithmetic, unit-tested on
    the CPU): input pixel (y', x') = (2a + cy, 2b + cx) receives dY[a + dy_t, b + dx_t] * W[:, :, r_t, s_t] summed over the
    taps t of its class.  From y' = 2*yo + r - pad_y: only taps with (cy + pad_y - r) even take part, at yo = a + (cy +
    pad_y - r) / 2; likewise along x (no x padding: the input is pre-padded).  Returns one tuple per class:
    (cy, cx, [(r, s)], [dy], [dx], Ha, Wa) with Ha x Wa the number of input pixels of that parity."""
    out = []
    for cy in range(2):
        for cx in range(2):
            rs = [(r, s) for r in range(kh) for s in range(kw) if (cy + pad_y - r) % 2 == 0 and (cx - s) % 2 == 0]
            out.append((cy, cx, rs, [(cy + pad_y - r) // 2 for r, s in rs], [(cx - s) // 2 for r, s in rs],
                        (H - cy + 1) // 2, (W - cx + 1) // 2))
    return out


def _merge_parity_classes(classes):
    """One launch for the four parity classes of a stride-2 input gradient when they have the same extent and tap count
    (even H, W; 4x4 kernels); otherwise one launch per class."""
    return len(classes) == 4 and all(c[2] for c in classes) and len({(len(c[2]), c[5], c[6]) for c in classes}) == 1


def _dgrad(gy, wd, in_hw, kh, kw, pad_y=0, stride=1, x_crop=0, g_pitch=0, mask=None, slope=1.0, sums=None):
    """Gradient w.r.t. the (x-padded) input [N,H,W,Cin'] from gy [N,Hout,Wout,Cout] (zero-padded here to Cout', a multiple
    of 32) and D = wd [kh*kw][Cin'][Cout'].  Stride-2 parity classes address their taps as rows of D (wtap).
    g_pitch > 0: gy is the interior of a padded gradient whose rows are g_pitch pixels apart, read in place.
    mask: the activation this input gradient flows into; the epilogue multiplies by its LeakyReLU'(slope) and, when `sums`
    (zeroed fp64 [2*Cin']) is given, accumulates the per-channel sums of the result into it."""
    gy = _pad_last(gy, 32)                                           # heads with 1 / 3 output channels: zero-pad K
    N, Hout, Wout, Cop = gy.shape
    Cin = wd.shape[1]
    H, W = in_hw
    classes = stride2_classes(kh, kw, pad_y, H, W) if stride == 2 and not x_crop else []
    if stride != 1 and not classes:
        raise B3DError("conv2d_dgrad: stride must be 1 or 2 (x_crop: stride 1 only)")
    merged = _merge_parity_classes(classes)
    opts = None
    if g_pitch or mask is not None or merged:
        opts = _ConvOpts(None, 1.0, 0, g_pitch, 0)
        if mask is not None:
            opts.mask, opts.mask_slope, opts.stats_sum_only = mask.data_ptr(), slope, 1
        if merged:
            opts.nclass = 4
            for i, c in enumerate(classes):
                opts.class_ooy[i], opts.class_oox[i] = c[0], c[1]
    optr = ctypes.cast(ctypes.pointer(opts), ctypes.c_void_p) if opts is not None else None
    gx = torch.empty(N, H, W, Cin, device=gy.device, dtype=torch.float32)
    gptr, st = ctypes.c_void_p(gy.data_ptr()), stream_ptr(gy)      # (a pitched view's data_ptr = its first interior pixel)

    def launch(Ha, Wa, dy, dx, osy, ooy, oox, taps):
        check(_conv_call(lib.b3d_conv2d_tf32, gptr, ptr(wd), None, ptr(gx), N, Hout, Wout, Cop, Ha, Wa, Cin, len(dy), _ints(dy),
                         _ints(dx), 1, 1, H, W, Cin, osy, osy, ooy, oox, 1.0, _ints(taps) if taps else None,
                         kh * kw if taps else 0, ptr(sums), 0, 0, optr, st))

    if stride == 1:
        launch(H, W, [pad_y - r for r in range(kh) for _ in range(kw)], [-s - x_crop for _ in range(kh) for s in range(kw)],
               1, 0, 0, None)
    elif merged:
        launch(classes[0][5], classes[0][6], [v for c in classes for v in c[3]], [v for c in classes for v in c[4]], 2, 0, 0,
               [r * kw + s for c in classes for r, s in c[2]])
    else:
        for cy, cx, rs, dy, dx, Ha, Wa in classes:
            if not rs:
                gx[:, cy::2, cx::2] = 0
                continue
            launch(Ha, Wa, dy, dx, 2, cy, cx, [r * kw + s for r, s in rs])
    return gx


def _wgrad(gy, x, kh, kw, pad_y=0, stride=1, x_crop=0, sink=None, g_pitch=0, fold_kh=0, fold_cin=0):
    """Weight gradient from gy [N,Hout,Wout,Cout] and the (x-padded) input x [N,H,W,Cin].
    sink = None: returns a new [Cout,Cin,kh,kw] tensor (channel counts that are not multiples of 32 are zero-padded here);
    otherwise the gradient is accumulated into sink, the bank's tap-major [kh*kw][Cout][Cin] buffer.
    g_pitch > 0: gy is the interior of a padded gradient whose rows are g_pitch pixels apart, read in place.
    fold_kh > 0: x is the RAW 8-channel stem input whose fold_kh rows (y padding pad_y) fold into fold_cin channels; the
    gradient is the folded layer's (kh = 1), computed from the raw input."""
    N, Hout, Wout, Cout = gy.shape
    _, H, W, Cin = x.shape
    tap_major = int(sink is not None)
    st = stream_ptr(gy)
    if fold_kh:
        dw = sink if tap_major else torch.zeros(Cout, fold_cin, 1, kw, device=gy.device, dtype=torch.float32)
        check(_conv_call(lib.b3d_conv2d_wgrad_tf32, ctypes.c_void_p(gy.data_ptr()), ptr(x), ptr(dw), N, H, W, fold_cin, Hout,
                         Wout, Cout, 1, kw, pad_y, 1, 0, tap_major, fold_kh, g_pitch, st))
        return dw
    if _thin(Cout, Cin, kh, kw, stride):
        dw = sink if tap_major else torch.zeros(Cout, Cin, kh, kw, device=gy.device, dtype=torch.float32)
        check(_conv_call(lib.b3d_conv2d_thin_wgrad, ptr(gy), ptr(x), ptr(dw), N, H, W, Cin, Hout, Wout, Cout, kh, kw, pad_y,
                         x_crop, tap_major, st))
        return dw
    if tap_major:
        if Cout % 32:
            raise B3DError(f"conv2d: tap-major weight gradient needs Cout % 32 == 0 or a thin head (Cout={Cout})")
        dw = sink
    else:
        gy, x = _pad_last(gy, 32), _pad_last(x, 32)
        dw = torch.zeros(gy.shape[3], x.shape[3], kh, kw, device=gy.device, dtype=torch.float32)
    check(_conv_call(lib.b3d_conv2d_wgrad_tf32, ctypes.c_void_p(gy.data_ptr()), ptr(x), ptr(dw), N, H, W, x.shape[3], Hout, Wout,
                     gy.shape[3], kh, kw, pad_y, stride, x_crop, tap_major, 0, g_pitch, st))
    return dw if tap_major else dw[:Cout, :Cin]


# ------------------------------------------------------------------------------------------------------------------
# a 3x3 convolution of a x2 nearest-upsampled input (and the 1x1 shortcut beside it) on the low-resolution map
# ------------------------------------------------------------------------------------------------------------------
# conv3x3(pad_x(up2(X), 1), W, padding=(1, 0)) is the stride-2 transposed convolution of Xp = pad_x(X, 1) (replicate or
# circular alike: the pad columns of the upsampled map are the upsampled pad columns of X):
#   Y[2i + py, 2j + px] = sum_{a, b in {0, 1}} P[q] Xp[i + py + a - 1 (zero outside 0 .. H-1), j + px + b],
#   q = ((py*2 + px)*2 + a)*2 + b,  P[q] = sum_k sum_l A_py[a][k] A_px[b][l] W[k][l],  A_0 = [[1,0,0],[0,1,1]], A_1 = [[1,1,0],[0,0,1]]
# (the bank writes P and its 4x4 transposed layout D4, csrc/sn_kernels.cu): 4 taps per output pixel instead of 9, and the
# upsampled map is never written.  A 1x1 shortcut commutes with the upsample and runs on the low-resolution pixels.
def up2_fprop_taps():
    """(dy, dx, wtap, classes) of the forward's one launch: four parity classes (py, px), output stride 2, class c at output
    offset classes[c], taps (a, b) of class c reading Xp at (i + dy, j + dx) with P[wtap]."""
    cls = [(py, px) for py in range(2) for px in range(2)]
    q = [(py, px, a, b) for py, px in cls for a in range(2) for b in range(2)]
    return ([py + a - 1 for py, px, a, b in q], [px + b for py, px, a, b in q], [((py * 2 + px) * 2 + a) * 2 + b for py, px, a, b in q],
            cls)


def up2_dgrad_taps():
    """(dy, dx) of the input gradient, a 4x4 stride-2 correlation of dY [N,2H,2W,Cout] on D4:
    dXp[i, j'] = sum_{r,s} D4[4r + s] dY[2i + r - 1, 2j' + s - 3] (zero outside dY), for the W + 2 columns j' of Xp.
    Tap (r, s) carries P[q]^T with (r, s) = (3 - py - 2a, 3 - px - 2b)."""
    return [r - 1 for r in range(4) for _ in range(4)], [s - 3 for _ in range(4) for s in range(4)]


def up2_wgrad_columns(W):
    """(first Xp column, columns, x offset) of the three weight-gradient launches that give dP^T [16][Cin][Cout] =
    sum Xp[i, j'] (x) dY[2i + r - 1, 2j' + s - 3] with Xp as the M operand: the interior columns, then each pad column alone
    (of whose taps only s = 3, resp. s = 0 land inside dY), so that no 32-pixel K slice is spent on two pad columns."""
    return [(1, W, -1), (0, 1, -3), (W + 1, 1, 2 * W - 1)]


def _up_fprop(xp, wp, wsc=None, stats=None):
    """xp [N,H,W+2,Cin] (the x-padded low-resolution input), wp = P [16][Cout][Cin] -> y [N,2H,2W,Cout], the 3x3
    convolution of the upsampled map; stats: zeroed fp64 [2*Cout] the epilogue accumulates y's per-channel sum / sum of
    squares into (the four classes tile y).  wsc: the 1x1 shortcut's F [1][Csc][Cin] -> its output [N,H,W,Csc] on the
    interior of xp, else None."""
    N, H, Wp, Cin = xp.shape
    W, Cout = Wp - 2, wp.shape[1]
    st = stream_ptr(xp)
    y = torch.empty(N, 2 * H, 2 * W, Cout, device=xp.device, dtype=torch.float32)
    dy, dx, wtap, cls = up2_fprop_taps()
    opts = _ConvOpts(None, 1.0, 0, 0, 4)
    for i, (py, px) in enumerate(cls):
        opts.class_ooy[i], opts.class_oox[i] = py, px
    check(_conv_call(lib.b3d_conv2d_tf32, ptr(xp), ptr(wp), None, ptr(y), N, H, Wp, Cin, H, W, Cout, 16, _ints(dy), _ints(dx), 1, 1,
                     2 * H, 2 * W, Cout, 2, 2, 0, 0, 1.0, _ints(wtap), 16, ptr(stats), 0, 0,
                     ctypes.cast(ctypes.pointer(opts), ctypes.c_void_p), st))
    sc = None
    if wsc is not None:
        Csc = wsc.shape[1]
        sc = torch.empty(N, H, W, Csc, device=xp.device, dtype=torch.float32)
        check(_conv_call(lib.b3d_conv2d_tf32, ptr(xp), ptr(wsc), None, ptr(sc), N, H, Wp, Cin, H, W, Csc, 1, _ints([0]), _ints([1]), 1,
                         1, H, W, Csc, 1, 1, 0, 0, 1.0, None, 0, None, 0, 0, None, st))
    return y, sc


def _up_dgrad(gy, wd4, gsc=None, wdsc=None):
    """Gradient w.r.t. xp [N,H,W+2,Cin] from gy [N,2H,2W,Cout] on D4 = wd4 [16][Cin][Cout], plus the shortcut's from gsc
    [N,H,W,Csc] on its D = wdsc [1][Cin][Csc] when given."""
    N, H2, W2, Cout = gy.shape
    H, Wp, Cin = H2 // 2, W2 // 2 + 2, wd4.shape[1]
    st = stream_ptr(gy)
    gx = torch.empty(N, H, Wp, Cin, device=gy.device, dtype=torch.float32)
    dy, dx = up2_dgrad_taps()
    check(_conv_call(lib.b3d_conv2d_tf32, ptr(gy), ptr(wd4), None, ptr(gx), N, H2, W2, Cout, H, Wp, Cin, 16, _ints(dy), _ints(dx), 2, 2,
                     H, Wp, Cin, 1, 1, 0, 0, 1.0, None, 0, None, 0, 0, None, st))
    if gsc is not None:
        gs = torch.empty_like(gx)
        check(_conv_call(lib.b3d_conv2d_tf32, ptr(gsc), ptr(wdsc), None, ptr(gs), N, H, Wp - 2, gsc.shape[3], H, Wp, Cin, 1, _ints([0]),
                         _ints([-1]), 1, 1, H, Wp, Cin, 1, 1, 0, 0, 1.0, None, 0, None, 0, 0, None, st))
        gx += gs
    return gx


def _up_wgrad(gy, xp, df, gsc=None, dfsc=None):
    """Weight gradients from gy [N,2H,2W,Cout] and xp [N,H,W+2,Cin]: dP^T [16][Cin][Cout] from the 4x4 stride-2 weight
    gradient with the roles swapped (Xp as the M operand, so that Cin, not Cout, fills the wgmma tile), folded into the
    F-layout sink df [9][Cout][Cin] by b3d_up2_fold; the shortcut's from gsc [N,H,W,Csc] into its sink dfsc."""
    N, H, Wp, Cin = xp.shape
    _, H2, W2, Cout = gy.shape
    st = stream_ptr(gy)
    dpt = torch.zeros(16, Cin, Cout, device=gy.device, dtype=torch.float32)
    for j0, w, x_off in up2_wgrad_columns(Wp - 2):
        check(_conv_call(lib.b3d_conv2d_wgrad_tf32, ctypes.c_void_p(xp.data_ptr() + 4 * Cin * j0), ptr(gy), ptr(dpt), N, H2, W2, Cout,
                         H, w, Cin, 4, 4, 1, 2, x_off, 1, 0, Wp, st))
    check(lib.b3d_up2_fold(ptr(dpt), ptr(df), Cout, Cin, st))
    if gsc is not None:
        check(_conv_call(lib.b3d_conv2d_wgrad_tf32, ptr(gsc), ptr(xp), ptr(dfsc), N, H, Wp, Cin, H, Wp - 2, gsc.shape[3], 1, 1, 0, 1,
                         1, 1, 0, 0, st))


class _UpConv(torch.autograd.Function):
    """conv1 of an upsampling block (and its 1x1 shortcut when lwsc is given) on the low-resolution padded input xp; wf / wfsc
    are the bank outputs autograd differentiates, whose gradients go to the bank's F-layout sinks."""

    @staticmethod
    def forward(ctx, xp, wf, wfsc, lw, lwsc, stats):
        xp = dev(xp.detach(), "x")
        if xp.shape[3] != lw.Cin or lw.wp is None:
            raise B3DError(f"conv2d_up2: input has {xp.shape[3]} channels (layer: {lw.Cin}), or the layer is not an up2 layer")
        y, sc = _up_fprop(xp, dev(lw.wp.detach(), "weight"), dev(lwsc.wf.detach(), "weight") if lwsc is not None else None, stats)
        ctx.save_for_backward(xp)
        ctx.lw, ctx.lwsc = lw, lwsc
        return (y, sc) if sc is not None else y

    @staticmethod
    def backward(ctx, gy, gsc=None):
        xp, = ctx.saved_tensors
        lw, lwsc = ctx.lw, ctx.lwsc
        gy = dev(gy, "grad_output")
        gsc = dev(gsc, "grad_output") if gsc is not None else None
        gx = _up_dgrad(gy, lw.wd, gsc, lwsc.wd if gsc is not None else None) if ctx.needs_input_grad[0] else None
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            if lw.df is None or (gsc is not None and lwsc.df is None):
                raise B3DError("conv2d_up2: weight gradients need the bank's gradient sinks")
            _up_wgrad(gy, xp, lw.df, gsc, lwsc.df if gsc is not None else None)
        return (gx, lw.df if ctx.needs_input_grad[1] else None, lwsc.df if ctx.needs_input_grad[2] else None, None, None, None)


def conv2d_up2_banked(xp_nchw, lw, lw_sc=None, stats=None):
    """conv2d_banked(pad_x(up2(x), 1), lw, pad_y=1, stats=stats) from xp = pad_x(x, 1) alone (lw: a layer the bank registered
    with up2), and the block's 1x1 shortcut conv2d_banked(up2(x), lw_sc) at low resolution, i.e. before its upsample.
    Returns (y, shortcut output or None), logically NCHW."""
    x = xp_nchw.permute(0, 2, 3, 1)
    out = _UpConv.apply(x, lw.wf, lw_sc.wf if lw_sc is not None else None, lw, lw_sc, stats)
    y, sc = out if lw_sc is not None else (out, None)
    return y.permute(0, 3, 1, 2), sc.permute(0, 3, 1, 2) if sc is not None else None


def conv2d_nhwc(x, weight, bias=None, pad_y=0, stride=1, leaky=1.0, wt=None, pad_out=0, pad_mode=1, x_crop=0):
    """x [N,H,W,Cin] (Cin % 32 == 0), weight [Cout,Cin,kh,kw] -> [N,Hout,Wout,Cout]; zero pad along y only.
    pad_out > 0: the result is written into the interior of a [N,Hout,Wout + 2*pad_out,Cout] buffer whose pad columns
    are then filled in place (replicate / circular) — the next convolution's padded input without a copy.
    x_crop > 0 (stride 1): convolve x[:, :, x_crop:W - x_crop] without materialising the slice (taps are shifted)."""
    x = dev(x, "x")
    Cout, Cin_w, kh, kw = weight.shape
    if Cin_w != x.shape[3]:
        raise B3DError(f"conv2d: input has {x.shape[3]} channels, weight expects {Cin_w}")
    wt = dev(wt if wt is not None else taps_layout(weight), "weight")
    return _fprop(x, wt, bias, kh, kw, pad_y, stride, leaky, pad_out, pad_mode, x_crop)


def conv2d_dgrad_nhwc(dy_, weight, in_hw, pad_y=0, stride=1, x_crop=0):
    """Gradient w.r.t. the (x-padded) input [N,H,W,Cin] of conv2d_nhwc, from dy_ [N,Hout,Wout,Cout]."""
    Cout, Cin, kh, kw = weight.shape
    wd = _d_layout(weight.permute(2, 3, 0, 1).reshape(kh * kw, Cout, Cin))
    return _dgrad(dev(dy_, "grad_output"), wd, in_hw, kh, kw, pad_y, stride, x_crop)


def conv2d_wgrad_nhwc(dy_, x, kh, kw, pad_y=0, stride=1, x_crop=0):
    """dW [Cout,Cin,kh,kw] from dy_ [N,Hout,Wout,Cout] and the (x-padded) input x [N,H,W,Cin], both NHWC
    (channel counts that are not multiples of 32 are zero-padded here)."""
    return _wgrad(dev(dy_, "grad_output"), dev(x, "input"), kh, kw, pad_y, stride, x_crop)


# ------------------------------------------------------------------------------------------------------------------
# autograd: y = conv(x, w) + b on NHWC tensors for both entry points
# ------------------------------------------------------------------------------------------------------------------
class ActLink:
    """Hand-over between two chained banked convolutions  conv_L -> bias -> LeakyReLU -> x padding -> conv_L+1  (the
    discriminators, models/gan.py:163-177,294-302) for the backward pass.  The producer (conv_L, `link_out`) records its
    padded output; the consumer (conv_L+1, `link_in`), whose saved input IS that tensor, runs its input-gradient kernels
    with the LeakyReLU adjoint in their epilogue (mask = the activated tensor), folds the pad columns back
    (b3d_wrap_x_bwd_inplace) and leaves the bias gradient here — the producer's backward then reads the interior of the
    padded gradient in place (row-pitch tensor maps) instead of running b3d_pad_leaky_bias_bwd over it.
    Only valid when conv_L+1 is the ONLY consumer of conv_L's output: the caller creates a link exactly then."""
    __slots__ = ("armed", "slope", "pad", "mode", "ptr", "shape", "want_gb", "gb", "done")

    def __init__(self):
        self.armed = self.done = False
        self.gb = None


class _Conv(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, bias, lw, pad_y, stride, leaky, pad_out, pad_mode, x_crop, stats=None, fold_raw=0, link_in=None,
                link_out=None, fold_fwd=False):
        """Runs on lw.wf (F [T'][Cout][Cin']); w is the tensor autograd differentiates: lw.wf itself (bank) or the module weight
        lw.wf was laid out from.  Its gradient is accumulated into lw.df when the bank provides that sink, otherwise returned
        as [Cout,Cin,kh,kw].  The input gradient runs on lw.wd, or on the per-tap transpose of lw.wf when there is none.
        fold_raw = kh > 0: x is the RAW 8-channel stem input [N,H,W,8]; the kernels fold the kh vertical taps into the K
        dimension on the fly (TMA boxes of 4 rows x 8 channels) — the folded tensor is not kept (pad_y = the fold's y padding).
        fold_fwd: the forward alone runs on a folded copy of x (b3d.ew.fold_rows), freed when it returns; the backward still
        reads the raw input."""
        x = dev(x.detach(), "x")
        if lw.wp is not None:               # its wd is D4, not D: only conv2d_up2_banked runs such a layer
            raise B3DError("conv2d: a layer registered with up2 runs through conv2d_up2_banked")
        Cx = x.shape[3]
        fold_pad = 0
        if fold_raw:
            if not lw.fold or Cx != 8 or lw.Cin != 8 or stride != 1 or x_crop:
                raise B3DError("conv2d: on-the-fly fold needs a folded 8-channel stride-1 stem")
            fold_pad = pad_y
        elif Cx != lw.Cinp:
            if lw.fold or Cx != lw.Cin:
                raise B3DError(f"conv2d: input has {Cx} channels, the layer expects {lw.Cinp if lw.fold else lw.Cin}")
            x = _pad_last(x, 32)                                      # thin un-folded inputs (stems): zero-pad K
        kh, kw = (1, lw.kw) if lw.fold else (lw.kh, lw.kw)
        if lw.fold:
            pad_y = 0
        wf, b = dev(lw.wf.detach(), "weight"), bias.detach() if bias is not None else None
        if fold_raw and fold_fwd:
            from .ew import fold_rows
            out = _fprop(fold_rows(x, lw.kh, fold_pad, lw.Cinp), wf, b, kh, kw, 0, stride, leaky, pad_out, pad_mode, x_crop, stats)
        else:
            out = _fprop(x, wf, b, kh, kw, pad_y, stride, leaky, pad_out, pad_mode, x_crop, stats, fold_raw, fold_pad)
        ctx.save_for_backward(x, out if (leaky != 1.0 or pad_out) else None)
        ctx.lw = lw
        ctx.cfg = (pad_y, stride, Cx, bias is not None, leaky, pad_out, pad_mode, x_crop, kh, kw, fold_raw, fold_pad)
        thin = _thin(lw.Cout, lw.Cinp, kh, kw, stride)
        # chained activation adjoint (ActLink): usable as a consumer when x is exactly the producer's padded output
        ctx.link_in = link_in if (link_in is not None and link_in.armed and link_in.ptr == x.data_ptr() and link_in.shape == tuple(x.shape)
                                  and Cx == lw.Cinp and lw.Cinp % 32 == 0 and not fold_raw and not thin) else None
        ctx.link_out = None
        if link_out is not None and pad_out and leaky != 1.0 and lw.Cout % 32 == 0 and not thin:
            link_out.armed, link_out.slope, link_out.pad, link_out.mode = True, float(leaky), int(pad_out), int(pad_mode)
            link_out.ptr, link_out.shape, link_out.done = out.data_ptr(), tuple(out.shape), False
            link_out.want_gb = bias is not None and bool(ctx.needs_input_grad[2])     # frozen discriminator (generator step): no bias sums
            ctx.link_out = link_out
        return out

    @staticmethod
    def backward(ctx, gy):
        x, y = ctx.saved_tensors
        lw = ctx.lw
        pad_y, stride, Cx, has_bias, leaky, pad_out, pad_mode, x_crop, kh, kw, fold_raw, fold_pad = ctx.cfg
        Cout, Cin = lw.Cout, lw.Cinp
        N, H, W, _ = x.shape
        gy = dev(gy, "grad_output")
        st = stream_ptr(gy)
        gb = None
        want_gb = has_bias and ctx.needs_input_grad[2]
        g_pitch = 0                                                    # gy as a window of wider rows (pixels)
        link_out = ctx.link_out
        if link_out is not None and link_out.done:
            # the consumer's input-gradient epilogue already applied LeakyReLU', folded the pad columns and summed the bias
            # gradient: gy is the PADDED gradient [N,Ho,Wo + 2 pad,C]; its interior is read in place
            link_out.done = False
            if tuple(gy.shape) != tuple(y.shape):
                raise B3DError("conv2d: chained gradient has the wrong shape")
            g_pitch = y.shape[2]
            gb = link_out.gb if want_gb else None
            link_out.gb = None
            gy = gy[:, :, pad_out:y.shape[2] - pad_out]                # a view: shapes below are the interior's
        elif pad_out:                     # padding + LeakyReLU + bias gradient in one pass over the padded gradient
            _, Ho, OW, _ = y.shape
            masked = torch.empty(N, Ho, OW - 2 * pad_out, Cout, device=gy.device, dtype=torch.float32)
            gb = torch.zeros(Cout, device=gy.device, dtype=torch.float32) if want_gb else None
            check(lib.b3d_pad_leaky_bias_bwd(ptr(gy), ptr(y), ptr(masked), ptr(gb), N * Ho, OW - 2 * pad_out, Cout, pad_out,
                                             pad_mode, float(leaky), st))
            gy = masked
        elif leaky != 1.0:                # LeakyReLU was fused into the epilogue: mask the incoming gradient by sign(y)
            masked = torch.empty_like(gy)
            check(lib.b3d_leaky_bwd(ptr(gy), ptr(y), ptr(masked), gy.numel(), float(leaky), st))
            gy = masked
        if gb is None and want_gb:
            gb = gy.sum(dim=(0, 1, 2))
        gx = gw = None
        if ctx.needs_input_grad[0]:
            link_in = ctx.link_in             # LeakyReLU adjoint of the PRODUCER of x in this epilogue
            sums = torch.zeros(2 * Cin, device=gy.device, dtype=torch.float64) if link_in is not None and link_in.want_gb else None
            gx = _dgrad(gy, lw.wd if lw.wd is not None else _d_layout(lw.wf.detach()), (gy.shape[1] if fold_raw else H, W), kh,
                        kw, pad_y, stride, x_crop, g_pitch, x if link_in is not None else None,
                        link_in.slope if link_in is not None else 1.0, sums)
            if link_in is not None:
                # gx = LeakyReLU'(x) * d(padded input), pad columns included: fold them back, hand the bias gradient over
                check(lib.b3d_wrap_x_bwd_inplace(ptr(gx), N * H, W - 2 * link_in.pad, Cin, link_in.pad, link_in.mode, st))
                link_in.gb = sums[:Cin].float() if sums is not None else None
                link_in.done = True
            if fold_raw:                                               # adjoint of the fold: back to the raw 8-channel layout
                graw = torch.empty(N, H, W, Cx, device=gy.device, dtype=torch.float32)
                check(lib.b3d_fold_rows_bwd(ptr(gx), ptr(graw), N, H, W, Cx, lw.kh, fold_pad, Cin, st))
                gx = graw
            elif Cx != Cin:
                gx = gx[..., :Cx]
        if ctx.needs_input_grad[1]:
            if fold_raw:
                gw = _wgrad(gy, x, kh, kw, fold_pad, stride, x_crop, lw.df, g_pitch, fold_raw, Cin)
            else:
                gw = _wgrad(gy, x, kh, kw, pad_y, stride, x_crop, lw.df, g_pitch)
            if lw.df is None:
                gw = gw[:, :lw.Cin]                                    # the module weight: drop the zero-padded input channels
        return gx, gw, gb, None, None, None, None, None, None, None, None, None, None, None, None


def fold_kh_weight(weight, cpad=0):
    """[Cout,Cin,kh,kw] -> [Cout, kh*Cin + cpad, 1, kw] matching fold_rows: channel r*Cin + c of the folded input is
    row tap r of input channel c (pure torch; unit-tested on the CPU against the unfolded convolution)."""
    Cout, Cin, kh, kw = weight.shape
    w = weight.permute(0, 2, 1, 3).reshape(Cout, kh * Cin, 1, kw)
    return torch.nn.functional.pad(w, (0, 0, 0, 0, 0, cpad)) if cpad else w


def conv2d(x_nchw, weight, bias=None, pad_y=0, stride=1, leaky=1.0, pad_out=0, pad_mode=1, x_crop=0):
    """Drop-in for F.conv2d(x, w, b, stride, padding=(pad_y, 0)) on logically-NCHW tensors: runs on the wgmma
    kernels over the channels-last storage (a no-copy view when x is already channels_last) and returns a
    logically-NCHW, channels-last tensor.  The weight is laid out per call and used as stored (fp32, no tf32 rounding)."""
    x = x_nchw.permute(0, 2, 3, 1)
    Cout, Cin, kh, kw = weight.shape
    if stride == 1 and kh > 1 and Cin * kh <= 64:
        # thin stems (discriminator conv1: 8 or 11 input channels, 5x5): fold the kh vertical taps into the channel
        # dimension — X'[n,y,x, r*Cin + c] = X[n, y+r-pad_y, x, c] (zero rows = the y padding) — so the tensor cores see
        # kw taps of kh*Cin real channels instead of kh*kw taps of Cin channels zero-padded to 32.  The remaining taps
        # are horizontal: the weight-gradient kernel covers a whole row of taps per CTA (one pass over dY and X').
        from .ew import fold_rows
        cpad = (-kh * Cin) % 32                            # ... and round up to the 32-channel K slice in the same pass
        x = fold_rows(x, kh, pad_y, kh * Cin + cpad)
        weight = fold_kh_weight(weight, cpad)
        Cout, Cin, kh, kw = weight.shape
        pad_y = 0
    lw = LayerWeights(dict(Cout=Cout, Cin=Cin, kh=kh, kw=kw, fold=0, Cinp=-(-Cin // 32) * 32, Coutp=-(-Cout // 32) * 32,
                           Tp=kh * kw))
    lw.wf = _pad_last(taps_layout(weight.detach()), 32)
    y = _Conv.apply(x, weight, bias, lw, int(pad_y), int(stride), float(leaky), int(pad_out), int(pad_mode), int(x_crop))
    return y.permute(0, 3, 1, 2)


def conv2d_banked(x_nchw, lw, pad_y=0, stride=1, leaky=1.0, pad_out=0, pad_mode=1, x_crop=0, stats=None, link_in=None, link_out=None):
    """conv2d for a layer whose weights come from a WeightBank (`lw` = its LayerWeights: F and D normalised and laid out
    for the kernels once per network forward, the weight gradient accumulated straight into the bank's F-layout sink).
    Thin stems registered with fold=True get their kh taps folded into the channels here (b3d.ew.fold_rows), as in conv2d().
    stats: optional zeroed fp64 tensor [2*Cout]; the conv epilogue accumulates the output's per-channel sum / sum of
    squares into it (the following batch norm's statistics without another pass over the tensor)."""
    x = x_nchw.permute(0, 2, 3, 1)
    fold_raw, fold_fwd = 0, False
    if lw.fold:
        Wout = x.shape[2] - lw.kw + 1
        if (lw.Cin == 8 and lw.kw == 5 and lw.Cinp == 64 and stride == 1 and not x_crop and Wout % 128 == 0
                and x.shape[0] * x.shape[1] * (Wout // 128) >= 2 * torch.cuda.get_device_properties(x.device).multi_processor_count):
            # 8-channel stems of wide images: the backward reads the raw input (the weight gradient folds the rows in shared
            # memory), so no folded tensor is kept.  The forward folds the kh rows on the fly (TMA boxes of 4 rows x 8
            # channels) when no weight gradient is taken (generator step); when one is (discriminator step), fold_rows plus the
            # row-window kernel is faster at cfg3's shape (1.68 against 2.13 ms, H100 SXM at 700 W) and its folded copy is
            # freed as the forward returns.
            fold_raw = lw.kh
            fold_fwd = torch.is_grad_enabled() and lw.wf.requires_grad
        else:
            from .ew import fold_rows
            x = fold_rows(x, lw.kh, pad_y, lw.Cinp)
    y = _Conv.apply(x, lw.wf, lw.bias, lw, int(pad_y), int(stride), float(leaky), int(pad_out), int(pad_mode), int(x_crop), stats,
                    fold_raw, link_in, link_out, fold_fwd)
    return y.permute(0, 3, 1, 2)
