"""Point-cloud effective-loss ops over libb3d (autograd wrappers; plumbing only).

Reference path: /root/reference/code/utils/effective_loss_function.py:58-81 and the modules it
calls (camera/, quaternions/, utils/trilinear_interpolation.py, utils/smooth_voxels.py).
"""
import ctypes

import torch

from . import B3DError, check, dev, host_floats, lib, mode_id, ptr, stream_ptr

FIELD_OF_VIEW = 1.875          # effective_loss_function.py:69
CAMERA_VIEW_DISTANCE = 2.0     # effective_loss_function.py:70


def smoothing_taps(sigma, kernel_size=21, mode="R"):
    """The 1-D kernel of VoxelsSmooth.separate_kernels (smooth_voxels.py:24-31), on the CPU in fp32
    with the reference's own expression (mode R keeps its positive exponent, SURVEY App. A D4)."""
    a, b = (-kernel_size // 2, kernel_size // 2)
    x = torch.arange(a + 1.0, b + 1.0)
    s = torch.as_tensor(float(sigma), dtype=torch.float32)
    if mode_id(mode) == 0:
        k = torch.exp(pow(-x, 2) / (2 * pow(s, 2)))
    else:
        k = torch.exp(-pow(x, 2) / (2 * pow(s, 2)))
    k = k / k.sum()
    return [float(v) for v in k]


def project(points, quat, V, fov=FIELD_OF_VIEW, cam_dist=CAMERA_VIEW_DISTANCE, want_aux=False, want_bins=False):
    """-> pg [B,N,4] (+ coords [B,N,3], base int32 [B,N,3], inb uint8 [B,N] when want_aux)
    (+ sorted [B,N,4], bin_start [B,nbins+1] when want_bins)."""
    points = dev(points, "point_cloud")
    quat = dev(quat, "rotation")
    B, N, three = points.shape
    if three != 3 or quat.shape != (B, 4):
        raise B3DError(f"bad shapes: point_cloud {tuple(points.shape)}, rotation {tuple(quat.shape)}")
    pg = torch.empty(B, N, 4, device=points.device, dtype=torch.float32)
    coords = base = inb = None
    if want_aux:
        coords = torch.empty(B, N, 3, device=points.device, dtype=torch.float32)
        base = torch.empty(B, N, 3, device=points.device, dtype=torch.int32)
        inb = torch.empty(B, N, device=points.device, dtype=torch.uint8)
    srt = bins = None
    if want_bins:
        srt = torch.empty(B, N, 4, device=points.device, dtype=torch.float32)
        bins = torch.empty(B, lib.b3d_pc_bin_count(V) + 1, device=points.device, dtype=torch.int32)
    check(lib.b3d_pc_project(ptr(points), ptr(quat), B, N, V, fov, cam_dist, ptr(pg), ptr(coords), ptr(base),
                             ptr(inb), ptr(srt), ptr(bins), stream_ptr(points)))
    if want_bins:
        return pg, srt, bins
    return (pg, coords, base, inb) if want_aux else pg


def splat_grid(pg, V, mode="R"):
    """Materialised, clamped occupancy grid [B,V,V,V] (trilinear_interpolation.py:62-74)."""
    pg = dev(pg, "pg")
    B, N, _ = pg.shape
    grid = torch.empty(B, V, V, V, device=pg.device, dtype=torch.float32)
    check(lib.b3d_pc_splat_grid(ptr(pg), B, N, V, mode_id(mode), ptr(grid), stream_ptr(pg)))
    return grid


def _silhouette_fwd(srt, bins, taps, sc, B, N, V, mode, sil, ws, st):
    h = host_floats(taps)
    check(lib.b3d_pc_silhouette_fwd_hosttaps(ptr(srt), ptr(bins), ctypes.cast(h, ctypes.c_void_p), len(taps), ptr(sc), B, N,
                                             V, mode, ptr(sil), ptr(ws), ws.numel() * 4, st))


class _EffectiveLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, points, quat, scale, taps, V, mode, fov, cam_dist):
        points = dev(points.detach(), "point_cloud")
        quat = dev(quat.detach(), "rotation")
        B, N, _ = points.shape
        sc = None
        if scale is not None:
            sc = dev(scale.detach(), "scale").reshape(-1)
            if sc.numel() != B:
                raise B3DError(f"scale must hold one value per sample, got shape {tuple(scale.shape)}")
        pg, srt, bins = project(points, quat, V, fov, cam_dist, want_bins=True)
        sil = torch.empty(B, V, V, device=points.device, dtype=torch.float32)
        # mode P: the splat grid and the occupancy blurred along x and y (2 B V^3 floats), kept for the backward
        nbytes = lib.b3d_pc_silhouette_workspace_bytes(B, V, mode)
        ws = torch.empty(nbytes // 4, device=points.device, dtype=torch.float32)
        _silhouette_fwd(srt, bins, taps, sc, B, N, V, mode, sil, ws, stream_ptr(points))
        ctx.save_for_backward(points, quat, pg, srt, bins, sc if sc is not None else torch.empty(0), ws)
        ctx.cfg = (taps, V, mode, fov, cam_dist, scale.shape if scale is not None else None)
        ctx.ws_spent = False
        return sil

    @staticmethod
    def backward(ctx, dsil):
        points, quat, pg, srt, bins, sc, ws = ctx.saved_tensors
        taps, V, mode, fov, cam_dist, scale_shape = ctx.cfg
        has_scale = scale_shape is not None
        B, N, _ = points.shape
        dsil = dev(dsil, "grad_output")
        dpg = torch.empty_like(pg)
        dscale = torch.empty(B, device=points.device, dtype=torch.float32) if has_scale else None
        h = host_floats(taps)
        st = stream_ptr(points)
        if ctx.ws_spent and ws.numel():
            # a second backward through the same graph (retain_graph=True): the first one overwrote the workspace with
            # its gradients, so the forward refills it
            _silhouette_fwd(srt, bins, taps, sc if has_scale else None, B, N, V, mode, torch.empty_like(dsil), ws, st)
        ctx.ws_spent = True
        check(lib.b3d_pc_silhouette_bwd_hosttaps(ptr(srt), ptr(bins), ctypes.cast(h, ctypes.c_void_p), len(taps),
                                                 ptr(sc) if has_scale else None, ptr(dsil), B, N, V, mode, ptr(dpg),
                                                 ptr(dscale), ptr(ws), ws.numel() * 4, st))
        dpoints = torch.empty_like(points)
        dquat = torch.empty_like(quat)
        check(lib.b3d_pc_project_bwd(ptr(points), ptr(quat), ptr(pg), ptr(dpg), B, N, V, fov, cam_dist, ptr(dpoints),
                                     ptr(dquat), st))
        return (dpoints, dquat, dscale.view(scale_shape) if has_scale else None, None, None, None, None, None)


def effective_loss(points, quat, scale=None, V=64, taps=None, mode="R", fov=FIELD_OF_VIEW,
                   cam_dist=CAMERA_VIEW_DISTANCE):
    """points [B,N,3] (z,y,x), quat [B,4], scale [B,1]|None -> silhouette [B,V,V] (differentiable).

    mode "R": one fused kernel per direction, the grid never leaves shared memory.  mode "P": the x / y blur couples the
    columns, so the grid goes through a workspace of 2 B V^3 floats held from the forward to the backward (four grid
    transfers forward, five backward)."""
    if taps is None:
        taps = smoothing_taps(3.0, 21, mode)
    return _EffectiveLoss.apply(points, quat, scale, list(taps), int(V), mode_id(mode), float(fov), float(cam_dist))


# ------------------------------------------------------------------------------------------------------------------
# dense-grid path: the stand-alone VoxelsSmooth / termination_probs surface, one autograd function per stage
# ------------------------------------------------------------------------------------------------------------------
def _taps_arr(taps):
    h = host_floats(taps)
    return h, ctypes.cast(h, ctypes.c_void_p)


class _BlurAxis(torch.autograd.Function):
    """Zero-padded 1-D cross-correlation of [B,V,V,V] along axis 1 (z), 2 (y) or 3 (x)."""

    @staticmethod
    def forward(ctx, vox, taps, axis):
        v = dev(vox.detach(), "voxels")
        B, V = v.shape[0], v.shape[1]
        out = torch.empty_like(v)
        keep, p = _taps_arr(taps)
        check(lib.b3d_vox_blur_axis(ptr(v), ptr(out), p, len(taps), axis, 0, B, V, stream_ptr(v)))
        ctx.cfg = (list(taps), axis)
        return out

    @staticmethod
    def backward(ctx, g):
        taps, axis = ctx.cfg
        g = dev(g, "grad")
        out = torch.empty_like(g)
        keep, p = _taps_arr(taps)
        check(lib.b3d_vox_blur_axis(ptr(g), ptr(out), p, len(taps), axis, 1, g.shape[0], g.shape[1], stream_ptr(g)))
        return out, None, None


class _ScaleClamp(torch.autograd.Function):
    @staticmethod
    def forward(ctx, vox, scale):
        v, s = dev(vox.detach(), "voxels"), dev(scale.detach(), "scale").reshape(-1)
        out = torch.empty_like(v)
        check(lib.b3d_vox_scale_clamp(ptr(v), ptr(s), ptr(out), v.shape[0], v.shape[1], stream_ptr(v)))
        ctx.save_for_backward(v, s)
        ctx.sshape = scale.shape
        return out

    @staticmethod
    def backward(ctx, g):
        v, s = ctx.saved_tensors
        g = dev(g, "grad")
        gin, ds = torch.empty_like(v), torch.empty_like(s)
        check(lib.b3d_vox_scale_clamp_bwd(ptr(v), ptr(s), ptr(g), ptr(gin), ptr(ds), v.shape[0], v.shape[1], stream_ptr(v)))
        return gin, ds.view(ctx.sshape)


class _Silhouette(torch.autograd.Function):
    @staticmethod
    def forward(ctx, vox, mode):
        v = dev(vox.detach(), "voxels")
        B, V = v.shape[0], v.shape[1]
        sil = torch.empty(B, V, V, device=v.device, dtype=torch.float32)
        check(lib.b3d_vox_termination(ptr(v), B, V, mode, None, ptr(sil), stream_ptr(v)))
        ctx.save_for_backward(v)
        ctx.mode = mode
        return sil

    @staticmethod
    def backward(ctx, g):
        v, = ctx.saved_tensors
        g = dev(g, "grad")
        dv = torch.empty_like(v)
        check(lib.b3d_vox_termination_bwd(ptr(v), ptr(g), v.shape[0], v.shape[1], ctx.mode, ptr(dv), stream_ptr(v)))
        return dv, None


class _SplatSorted(torch.autograd.Function):
    """(points, quat) -> clamped occupancy grid [B,V,V,V]; adjoint = masked corner gather + projection adjoint."""

    @staticmethod
    def forward(ctx, points, quat, V, mode, fov, cam_dist):
        points, quat = dev(points.detach(), "point_cloud"), dev(quat.detach(), "rotation")
        B, N, _ = points.shape
        pg, srt, bins = project(points, quat, V, fov, cam_dist, want_bins=True)
        raw = torch.empty(B, V, V, V, device=points.device, dtype=torch.float32)
        st = stream_ptr(points)
        check(lib.b3d_vox_splat_sorted(ptr(srt), ptr(bins), B, N, V, mode, ptr(raw), st))
        occ = raw.clone()
        check(lib.b3d_vox_clamp01(ptr(occ), occ.numel(), st))
        ctx.save_for_backward(points, quat, pg, srt, bins, raw)
        ctx.cfg = (V, mode, fov, cam_dist)
        return occ

    @staticmethod
    def backward(ctx, g):
        points, quat, pg, srt, bins, raw = ctx.saved_tensors
        V, mode, fov, cam_dist = ctx.cfg
        B, N, _ = points.shape
        d = dev(g, "grad").clone()
        dpg = torch.zeros_like(pg)
        st = stream_ptr(points)
        check(lib.b3d_vox_gather(ptr(srt), ptr(bins), ptr(raw), ptr(d), B, N, V, mode, ptr(dpg), st))
        dpoints, dquat = torch.empty_like(points), torch.empty_like(quat)
        check(lib.b3d_pc_project_bwd(ptr(points), ptr(quat), ptr(pg), ptr(dpg), B, N, V, fov, cam_dist, ptr(dpoints),
                                     ptr(dquat), st))
        return dpoints, dquat, None, None, None, None


def blur_axis(vox, taps, axis):
    return _BlurAxis.apply(vox, [float(t) for t in taps], int(axis))


def scale_clamp(vox, scale):
    return _ScaleClamp.apply(vox, scale)


def silhouette_from_voxels(vox, mode="R"):
    return _Silhouette.apply(vox, mode_id(mode))


def termination_probs(vox, mode="R"):
    """[B,V,V,V] -> [B,V+1,V,V] (effective_loss_function.py:18-56); forward only."""
    v = dev(vox.detach(), "voxels")
    B, V = v.shape[0], v.shape[1]
    probs = torch.empty(B, V + 1, V, V, device=v.device, dtype=torch.float32)
    check(lib.b3d_vox_termination(ptr(v), B, V, mode_id(mode), ptr(probs), None, stream_ptr(v)))
    return probs


def occupancy_grid(points, quat, V, mode="R", fov=FIELD_OF_VIEW, cam_dist=CAMERA_VIEW_DISTANCE):
    return _SplatSorted.apply(points, quat, int(V), mode_id(mode), float(fov), float(cam_dist))


def effective_loss_dense(points, quat, scale=None, V=64, taps=None, mode="P", fov=FIELD_OF_VIEW,
                         cam_dist=CAMERA_VIEW_DISTANCE):
    """The effective loss over a MATERIALISED grid: splat -> clamp -> blur (z only in mode R; x, y, z chained in
    mode P) -> scale/clamp -> ray termination -> silhouette, one stand-alone full-grid kernel per stage.  It is the
    slow twin of `effective_loss` in both modes (the fused entry points) and serves as a cross-check."""
    if taps is None:
        taps = smoothing_taps(3.0, 21, mode)
    occ = occupancy_grid(points, quat, V, mode, fov, cam_dist)
    if mode_id(mode) == 0:
        sm = blur_axis(occ, taps, 1)
    else:
        sm = blur_axis(blur_axis(blur_axis(occ, taps, 3), taps, 2), taps, 1)
    if scale is not None:
        sm = scale_clamp(sm, scale)
    return silhouette_from_voxels(sm, mode)
