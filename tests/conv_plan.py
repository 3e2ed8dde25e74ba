"""The launch plan of libb3d's convolutions, restated in Python: which kernel instances one forward, input-gradient or
weight-gradient call launches, over which output columns, with which pixel tiles, work items, grids and K splits.

It restates the host-side dispatch of b3d_conv2d_tf32 / b3d_conv2d_wgrad_tf32 (csrc/tc_conv.cu) and b3d_conv2d_thin_fwd /
b3d_conv2d_thin_wgrad (csrc/thin_kernels.cu), and the Python layer above them in b3d/conv.py: the thin-head test (_thin),
the stride-2 parity classes and their merge, the zero padding of channel counts to 32, and the folding of thin stems.
Pure arithmetic (no torch, no GPU): the tests compare its instance lists with the ones the library reports for every
launch they make, so it cannot drift from the dispatch unnoticed, and then use it to show which launch geometries their
tables reach.  The SM count is a parameter; tests pass the device's."""
from dataclasses import dataclass
from typing import Optional

BM, BK, MAX_TAPS = 128, 32, 25                  # pixels per work item, channels per K slice (tc_conv.cu)
THIN_NT, THIN_OUTS = 256, 8                     # thin_kernels.cu: threads per block, output pixels per warp
STEM_KW, STEM_STAGES, STEM_NRAW = 5, 4, 3       # tc_conv.cu: raw-input stem weight gradient


@dataclass
class Launch:
    instance: str                 # as b3d_last_variant() spells it
    x0: int = 0                   # output columns [x0, x1) of this launch (a strip launch covers the last few)
    x1: int = 0
    BW: int = 0                   # pixel tile BW x BH x BI (forward / input gradient)
    BH: int = 0
    BI: int = 0
    items: int = 0                # work items (forward / input gradient), CTAs per split (weight gradient)
    grid: int = 0                 # CTAs launched
    N: int = 0                    # images of the launch
    Hout: int = 0                 # rows of the launch's (logical) output
    taps: int = 0                 # filter taps per class
    ncls: int = 1                 # output classes in one launch (merged stride-2 parity classes)
    sy: int = 1                   # input stride of the launch
    BN: int = 0                   # output-channel tile width (forward / input gradient), Cin tile (weight gradient)
    rowwin: int = 0               # taps per filter row of a row-window launch, 0 otherwise
    BWk: Optional[int] = None     # weight gradient: pixel box of one K slice
    BHk: Optional[int] = None
    kslices: Optional[int] = None  # K slices of the whole batch
    splits: Optional[int] = None
    T: Optional[int] = None       # taps per CTA

    @property
    def strip(self):
        """A narrow launch over the remainder columns of a width of "power of two + a few"."""
        return self.x0 > 0

    @property
    def partial_group(self):
        """The last image group of the tiles holds fewer than BI images."""
        return self.BI > 1 and self.N % self.BI != 0


def cdiv(a, b):
    return -(-a // b)


def pow2_floor(v):
    p = 1
    while p * 2 <= v:
        p *= 2
    return p


def r32(c):
    return cdiv(c, 32) * 32


def wgrad_splits(base_ctas, ktotal, sms):
    """K splits of a weight-gradient grid (tc_conv.cu wgrad_splits): the count minimising waves * (K slices per CTA + 16)."""
    smax = min(ktotal // 8, 8 * sms)
    best, best_cost = 1, None
    for s in range(1, smax + 1):
        cost = cdiv(base_ctas * s, sms) * (cdiv(ktotal, s) + 16)
        if best_cost is None or cost < best_cost:
            best, best_cost = s, cost
    return best


# ----------------------------------------------------------------------------------------------------------------------
# b3d_conv2d_tf32
# ----------------------------------------------------------------------------------------------------------------------
def tf32_launches(N, Hout, Wout, Cin, Cout, dy, dx, sy=1, wtap=None, ncls=1, fold_kh=0, sms=132):
    """The launches of one b3d_conv2d_tf32 call: Cin = the K channels, Cout = the output channels, dy / dx / wtap the tap
    lists of all ncls classes."""
    ntaps = len(dy)
    assert 1 <= ntaps <= MAX_TAPS and Cin % BK == 0 and ntaps % ncls == 0
    tpc = ntaps // ncls
    bn256 = Cout % 256 == 0 and N * Hout * Wout // BM * (Cout // 256) * ncls >= sms
    BN = 256 if bn256 else 128 if Cout > 64 else 64
    g_kw = 0
    if sy == 1 and fold_kh == 0:
        kw_ = 1
        while kw_ < tpc and dy[kw_] == dy[0]:
            kw_ += 1
        step = dx[1] - dx[0] if kw_ > 1 else 1
        wstep = wtap[1] - wtap[0] if wtap and kw_ > 1 else 1
        ok = tpc % kw_ == 0 and kw_ in (2, 3, 5) and step in (1, -1) and 1 <= wstep <= 2 and (ncls == 1 or wtap is not None)
        for t in range(ntaps):
            if not ok:
                break
            tc_ = t % tpc
            t0 = t - tc_
            ok = dy[t] == dy[t0 + (tc_ // kw_) * kw_] and dx[t] == dx[0] + (tc_ % kw_) * step
            if wtap:
                ok = ok and wtap[t] == wtap[t0 + (tc_ // kw_) * kw_] + (tc_ % kw_) * wstep
        if ok and BN <= 128:
            g_kw = kw_

    def run(x0, x1):
        wspan = x1 - x0
        BW = pow2_floor(min(wspan, BM))
        BH = pow2_floor(min(Hout, BM // BW))
        BI = BM // (BW * BH)
        tiles = cdiv(wspan, BW) * cdiv(Hout, BH) * cdiv(N, BI)
        work = tiles * cdiv(Cout, BN) * ncls
        rw = g_kw if g_kw and wspan >= BM else 0
        if rw:
            stages = {2: (5, 4), 3: (4, 3), 5: (3, 2)}[rw][0 if BN == 64 else 1]
            inst = f"conv_wgmma_rowwin<{BN},{rw},{stages}>"
        else:
            inst = f"conv_wgmma<{BN},{ {256: 4, 128: 6, 64: 8}[BN]}>"
        return Launch(inst, x0, x1, BW, BH, BI, work, min(work, sms), N, Hout, tpc, ncls, sy, BN, rw)

    bw_full = pow2_floor(min(Wout, BM))
    rem = Wout % bw_full
    if rem != 0 and rem * 8 <= bw_full and Wout > bw_full:
        return [run(0, Wout - rem), run(Wout - rem, Wout)]
    return [run(0, Wout)]


# ----------------------------------------------------------------------------------------------------------------------
# thin heads (1-4 output channels, 5x5, stride 1)
# ----------------------------------------------------------------------------------------------------------------------
def thin(Cout, Cin, kh, kw, stride):
    """b3d.conv._thin: the layers that run on the CUDA-core kernels of thin_kernels.cu."""
    return Cout <= 4 and Cin % 64 == 0 and kh == 5 and kw == 5 and stride == 1


def thin_fwd_launch(N, Hout, Wout, Cin, Cout):
    vec = 4 if Cin % 128 == 0 else 2
    items = N * Hout * cdiv(Wout, THIN_OUTS)
    return Launch(f"conv_thin_fwd<{Cout},{vec}>", 0, Wout, items=items, grid=min(cdiv(items, THIN_NT // 32), 132 * 16), N=N,
                  Hout=Hout, taps=25)


def thin_wgrad_launch(N, Hout, Cin, Cout):
    vec = 4 if Cin % 128 == 0 and Cout == 1 else 2
    cout = max(Cout, 1)
    win = cout * vec <= 6
    chunks = Cin // (32 * vec)
    bpc = min(cdiv(132 * 2, chunks), cdiv(N * Hout, THIN_NT // 32))
    name = "conv_thin_wgrad_win" if win else "conv_thin_wgrad"
    return Launch(f"{name}<{cout},{vec}>", items=bpc * chunks, grid=bpc * chunks, N=N, Hout=Hout, taps=25)


# ----------------------------------------------------------------------------------------------------------------------
# the three launch helpers of b3d/conv.py
# ----------------------------------------------------------------------------------------------------------------------
def fprop(N, H, W, Cin, Cout, kh, kw, pad_y=0, stride=1, x_crop=0, fold_kh=0, fold_pad=0, sms=132):
    """b3d.conv._fprop on x [N,H,W,Cin] and F [kh*kw][Cout][Cin] (Cin as the helper sees it: already padded / folded;
    fold_kh > 0: x is the raw 8-channel stem input, the kernel folds fold_kh rows into 32 * ceil(8 fold_kh / 32) channels)."""
    Hout = (H + 2 * fold_pad - fold_kh + 1) if fold_kh else (H + 2 * pad_y - kh) // stride + 1
    Wout = (W - 2 * x_crop - kw) // stride + 1
    if thin(Cout, Cin, kh, kw, stride):
        return [thin_fwd_launch(N, Hout, Wout, Cin, Cout)]
    K = r32(8 * fold_kh) if fold_kh else Cin
    dy = [r - pad_y for r in range(kh) for _ in range(kw)]
    dx = [s + x_crop for _ in range(kh) for s in range(kw)]
    return tf32_launches(N, Hout, Wout, K, Cout, dy, dx, sy=stride, fold_kh=fold_kh, sms=sms)


def stride2_classes(kh, kw, pad_y, H, W):
    """b3d.conv.stride2_classes: (cy, cx, [(r, s)], [dy], [dx], Ha, Wa) per output parity class."""
    out = []
    for cy in range(2):
        for cx in range(2):
            rs = [(r, s) for r in range(kh) for s in range(kw) if (cy + pad_y - r) % 2 == 0 and (cx - s) % 2 == 0]
            out.append((cy, cx, rs, [(cy + pad_y - r) // 2 for r, s in rs], [(cx - s) // 2 for r, s in rs],
                        (H - cy + 1) // 2, (W - cx + 1) // 2))
    return out


def merge_parity_classes(classes):
    return len(classes) == 4 and all(c[2] for c in classes) and len({(len(c[2]), c[5], c[6]) for c in classes}) == 1


def dgrad(N, H, W, Cin, Cout, kh, kw, pad_y=0, stride=1, x_crop=0, sms=132):
    """b3d.conv._dgrad: the input gradient [N,H,W,Cin] (Cin = rows of D, a multiple of 32) from dY with Cout channels
    (zero-padded to a multiple of 32 for the kernel's K)."""
    K = r32(Cout)
    Hout = (H + 2 * pad_y - kh) // stride + 1
    Wout = (W - 2 * x_crop - kw) // stride + 1
    if stride == 1:
        return tf32_launches(N, H, W, K, Cin, [pad_y - r for r in range(kh) for _ in range(kw)],
                             [-s - x_crop for _ in range(kh) for s in range(kw)], sms=sms)
    assert stride == 2 and not x_crop and Hout > 0 and Wout > 0
    classes = stride2_classes(kh, kw, pad_y, H, W)
    if merge_parity_classes(classes):
        return tf32_launches(N, classes[0][5], classes[0][6], K, Cin, [v for c in classes for v in c[3]],
                             [v for c in classes for v in c[4]], wtap=[r * kw + s for c in classes for r, s in c[2]], ncls=4,
                             sms=sms)
    out = []
    for cy, cx, rs, dy, dx, Ha, Wa in classes:
        if rs:
            out += tf32_launches(N, Ha, Wa, K, Cin, dy, dx, wtap=[r * kw + s for r, s in rs], sms=sms)
    return out


def wgrad(N, H, W, Cin, Cout, kh, kw, pad_y=0, stride=1, x_crop=0, fold_kh=0, fold_cin=0, sms=132):
    """b3d.conv._wgrad: dW from dY [N,Hout,Wout,Cout] and x [N,H,W,Cin] (fold_kh > 0: x is the raw 8-channel stem input
    and the gradient is the folded layer's, fold_cin channels, 1 x kw)."""
    if fold_kh:
        Hout, Wout = H + 2 * pad_y - fold_kh + 1, W - kw + 1
        kx = cdiv(Wout, BK)
        ktotal = N * kx * Hout
        splits = wgrad_splits(Cout // 64, ktotal, sms)
        return [Launch(f"wgrad_stem<{STEM_KW},{STEM_STAGES},{STEM_NRAW}>", 0, Wout, items=Cout // 64, grid=Cout // 64 * splits,
                       N=N, Hout=Hout, taps=kw, BN=64, BWk=BK, BHk=1, kslices=ktotal, splits=splits, T=kw)]
    Hout = (H + 2 * pad_y - kh) // stride + 1
    if thin(Cout, Cin, kh, kw, stride):
        return [thin_wgrad_launch(N, Hout, Cin, Cout)]
    return wgrad_tf32(N, H, W, r32(Cin), r32(Cout), kh, kw, pad_y, stride, x_crop, sms)


def wgrad_tf32(N, H, W, Cin, Cout, kh, kw, pad_y=0, stride=1, x_crop=0, sms=132):
    """b3d_conv2d_wgrad_tf32 on dY [N,Hout,Wout,Cout] and x [N,H,W,Cin] (multiples of 32), x read from column x_crop on."""
    Hout = (H + 2 * pad_y - kh) // stride + 1
    Wout = (W - 2 * x_crop - kw) // stride + 1
    BWk = pow2_floor(min(Wout, BK))
    BHk = BK // BWk
    ktotal = N * cdiv(Wout, BWk) * cdiv(Hout, BHk)
    BN = 128 if Cin > 64 else 64
    T = 1
    if Wout >= BK:
        if stride == 1 and kw == 3 and BN == 64:
            T = 3
        if stride == 2 and kw == 4:
            T = 2
    base = cdiv(Cout, BM) * cdiv(Cin, BN) * kh * (kw // T)
    splits = wgrad_splits(base, ktotal, sms)
    stages, nraw = {(64, 3): (3, 3), (128, 2): (2, 3), (64, 2): (3, 3), (128, 1): (3, 3), (64, 1): (4, 4)}[(BN, T)]
    return [Launch(f"wgrad_wgmma<{BN},{stages},{nraw},{T}>", 0, Wout, items=base, grid=base * splits, N=N, Hout=Hout,
                   taps=kh * kw, BN=BN, BWk=BWk, BHk=BHk, kslices=ktotal, splits=splits, T=T)]


# ----------------------------------------------------------------------------------------------------------------------
# a layer: which helper calls b3d.conv.conv2d / conv2d_banked make
# ----------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Call:
    """One call of a launch helper of b3d/conv.py, with the geometry the helper sees."""
    kind: str           # "fprop", "dgrad" or "wgrad"
    N: int
    H: int
    W: int
    Cin: int            # fprop / wgrad: channels of x as passed; dgrad: rows of D (the input gradient's channels)
    Cout: int           # output channels (dgrad: dY's channels before the zero padding)
    kh: int
    kw: int
    pad_y: int = 0
    stride: int = 1
    x_crop: int = 0
    fold_kh: int = 0    # fprop: raw-input fold on the fly; wgrad: raw-input stem gradient
    fold_pad: int = 0
    masked: bool = False  # dgrad: LeakyReLU adjoint of the producer in the epilogue

    def launches(self, sms=132):
        if self.kind == "fprop":
            return fprop(self.N, self.H, self.W, self.Cin, self.Cout, self.kh, self.kw, self.pad_y, self.stride, self.x_crop,
                         self.fold_kh, self.fold_pad, sms)
        if self.kind == "dgrad":
            return dgrad(self.N, self.H, self.W, self.Cin, self.Cout, self.kh, self.kw, self.pad_y, self.stride, self.x_crop,
                         sms)
        return wgrad(self.N, self.H, self.W, self.Cin, self.Cout, self.kh, self.kw, self.pad_y, self.stride, self.x_crop,
                     self.fold_kh, r32(8 * self.fold_kh) if self.fold_kh else 0, sms)

    def instances(self, sms=132):
        return [l.instance for l in self.launches(sms)]


def layer_calls(N, Cin, H, W, Cout, k, pad_y, stride, x_crop=0, need_dx=True, need_dw=True, masked=False, banked=False,
                sms=132):
    """The helper calls of one convolution forward + backward: b3d.conv.conv2d (a module's weight, banked=False) or
    conv2d_banked with the layer registered in a WeightBank the way MultiScaleDiscriminator registers it (banked=True:
    stride-1 stems with kh * Cin <= 64 folded).  Cin, H, W: the layer's own input (x-padded), before any channel padding."""
    kh = kw = k
    fold = stride == 1 and kh > 1 and Cin * kh <= 64
    calls = []
    if not fold:
        Cx = r32(Cin)                                                   # thin inputs: zero-padded K
        calls.append(Call("fprop", N, H, W, Cx, Cout, kh, kw, pad_y, stride, x_crop))
        if need_dx:
            calls.append(Call("dgrad", N, H, W, Cx, Cout, kh, kw, pad_y, stride, x_crop, masked=masked))
        if need_dw:
            calls.append(Call("wgrad", N, H, W, Cx, Cout, kh, kw, pad_y, stride, x_crop))
        return calls
    Cf = r32(kh * Cin)                                                  # rows folded into the channels
    Hout, Wout = H + 2 * pad_y - kh + 1, W - kw + 1
    fold_raw = (banked and Cin == 8 and kw == 5 and Cf == 64 and not x_crop and Wout % 128 == 0
                and N * H * (Wout // 128) >= 2 * sms)
    if not fold_raw:                                                    # b3d.ew.fold_rows, then a 1 x kw convolution
        calls.append(Call("fprop", N, Hout, W, Cf, Cout, 1, kw))
        if need_dx:
            calls.append(Call("dgrad", N, Hout, W, Cf, Cout, 1, kw, masked=masked))
        if need_dw:
            calls.append(Call("wgrad", N, Hout, W, Cf, Cout, 1, kw))
        return calls
    # raw 8-channel input kept: the forward folds on the fly when no weight gradient is taken, else runs on a folded copy
    if need_dw:
        calls.append(Call("fprop", N, Hout, W, Cf, Cout, 1, kw))
    else:
        calls.append(Call("fprop", N, H, W, Cin, Cout, 1, kw, fold_kh=kh, fold_pad=pad_y))
    if need_dx:
        calls.append(Call("dgrad", N, Hout, W, Cf, Cout, 1, kw, masked=masked))
    if need_dw:
        calls.append(Call("wgrad", N, H, W, Cin, Cout, 1, kw, pad_y, fold_kh=kh))
    return calls
