"""Bindings of the training-data kernels.
b3d_gather_fields: one launch that assembles a GAN batch from packed per-record stores (gather by index, fp16 -> fp32, UV
mirroring).  The stores may sit in device memory or in pinned host memory (read over PCIe).
b3d_image_batch: one launch that builds a reconstruction batch (crop, cv2-style resize, mirror, poses) from packed photo
windows in device memory.
b3d_pseudogt_pack: one launch that masks, transposes and rounds a batch of pseudo-ground-truth records to fp16.
b3d_sample_pack: one launch that turns a batch of sample renders and textures into the bytes of their PNGs.
b3d_recon_texture_pack: one launch that builds the texture bytes of a batch of exported reconstructions."""
import ctypes

import torch

from . import B3DError, check, lib, ptr, stream_ptr

F32, F16, I64 = 0, 1, 2
MAX_FIELDS = 8
_TYPES = {torch.float32: F32, torch.float16: F16, torch.int64: I64}


class GatherField(ctypes.Structure):
    _fields_ = [("src", ctypes.c_void_p), ("src_type", ctypes.c_int), ("n", ctypes.c_int), ("C_src", ctypes.c_int),
                ("C", ctypes.c_int), ("H", ctypes.c_int), ("W", ctypes.c_int), ("mirror", ctypes.c_int),
                ("scale", ctypes.c_float), ("bias", ctypes.c_float), ("dst", ctypes.c_void_p)]


def _as4(shape):
    """[n, C, H, W] or [n, K] (rows of K, e.g. class labels) -> (n, C, H, W)."""
    if len(shape) == 4:
        return tuple(shape)
    if len(shape) == 2:
        return shape[0], shape[1], 1, 1
    raise B3DError(f"gather: expected a [n,C,H,W] or [n,K] store, got shape {tuple(shape)}")


def gather_fields(fields, idx, flip=None):
    """fields: list of (src, dst, mirror, scale, bias).  src [n,C_src,H,W] fp16 / fp32 (or [n,K] int64), contiguous, on
    the device or in pinned host memory; dst [B,C,H,W] fp32 (int64 [B,K]) on the device, C <= C_src.
    idx: int32 [B] CUDA tensor of record indices; flip: uint8 [B] CUDA tensor or None.
    dst[b,c] = scale * src[idx[b], c] + bias, mirrored in u where mirror and flip[b] are set."""
    if not 1 <= len(fields) <= MAX_FIELDS:
        raise B3DError(f"gather: 1 to {MAX_FIELDS} fields, got {len(fields)}")
    if not (isinstance(idx, torch.Tensor) and idx.is_cuda and idx.dtype == torch.int32 and idx.dim() == 1
            and idx.is_contiguous()):
        raise B3DError("gather: idx must be a contiguous int32 CUDA tensor [B]")
    B = idx.shape[0]
    if flip is not None and not (isinstance(flip, torch.Tensor) and flip.is_cuda and flip.dtype == torch.uint8
                                 and tuple(flip.shape) == (B,) and flip.is_contiguous()):
        raise B3DError("gather: flip must be a contiguous uint8 CUDA tensor [B] or None")
    arr = (GatherField * len(fields))()
    for i, (src, dst, mirror, scale, bias) in enumerate(fields):
        if src.dtype not in _TYPES:
            raise B3DError(f"gather: field {i}: store dtype {src.dtype} (expected float16, float32 or int64)")
        want = torch.int64 if src.dtype == torch.int64 else torch.float32
        if dst.dtype != want or not dst.is_cuda:
            raise B3DError(f"gather: field {i}: output must be a {want} CUDA tensor, got {dst.dtype} on {dst.device}")
        if not (src.is_contiguous() and dst.is_contiguous()):
            raise B3DError(f"gather: field {i}: store and output must be contiguous")
        n, C_src, H, W = _as4(src.shape)
        Bd, C, Hd, Wd = _as4(dst.shape)
        if (Bd, Hd, Wd) != (B, H, W) or C > C_src:
            raise B3DError(f"gather: field {i}: output {tuple(dst.shape)} does not fit store {tuple(src.shape)} and B={B}")
        arr[i] = GatherField(src.data_ptr(), _TYPES[src.dtype], n, C_src, C, H, W, int(bool(mirror)), float(scale),
                             float(bias), dst.data_ptr())
    check(lib.b3d_gather_fields(ctypes.cast(arr, ctypes.c_void_p), len(fields), ptr(idx), ptr(flip), B, stream_ptr(idx)))


MAX_RES = 4          # B3D_IMAGE_MAX_RES
MAX_SIDE = 2048      # B3D_IMAGE_MAX_SIDE


def _cuda(t, dtype, name, dim=None):
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == dtype and t.is_contiguous()
            and (dim is None or t.dim() == dim)):
        raise B3DError(f"image_batch: {name} must be a contiguous {dtype} CUDA tensor"
                       + (f" with {dim} dimensions" if dim is not None else ""))


def image_batch(pixels, offsets, geometry, poses, idx, flip, images, scale, translation, rot, ind):
    """b3d_image_batch: one launch builds a reconstruction batch from packed photo windows.
    Store: pixels int32 [words] (RGBM bytes per word), offsets int64 [n], geometry int32 [n, 5] (ww, wh, wx0, wy0, S),
    poses fp32 [n, 2, 8].  idx int32 [B], flip uint8 [B] or None.  Outputs (fp32 unless noted, on the device):
    images [[B,4,R0,R0], [B,3,R1,R1], ...], scale [B,1], translation [B,3], rot [B,4], ind int64 [B]."""
    _cuda(pixels, torch.int32, 'pixels', 1)
    _cuda(offsets, torch.int64, 'offsets', 1)
    n = offsets.shape[0]
    _cuda(geometry, torch.int32, 'geometry')
    _cuda(poses, torch.float32, 'poses')
    if tuple(geometry.shape) != (n, 5) or tuple(poses.shape) != (n, 2, 8):
        raise B3DError(f"image_batch: geometry {tuple(geometry.shape)} / poses {tuple(poses.shape)} do not fit {n} records")
    _cuda(idx, torch.int32, 'idx', 1)
    B = idx.shape[0]
    if flip is not None:
        _cuda(flip, torch.uint8, 'flip', 1)
        if flip.shape[0] != B:
            raise B3DError(f"image_batch: flip has {flip.shape[0]} entries for {B} samples")
    if not 1 <= len(images) <= MAX_RES:
        raise B3DError(f"image_batch: 1 to {MAX_RES} image outputs, got {len(images)}")
    res = []
    for k, im in enumerate(images):
        _cuda(im, torch.float32, f'image output {k}', 4)
        R = im.shape[-1]
        if tuple(im.shape) != (B, 4 if k == 0 else 3, R, R):
            raise B3DError(f"image_batch: image output {k} has shape {tuple(im.shape)}; expected "
                           f"[{B}, {4 if k == 0 else 3}, R, R]")
        res.append(R)
    for t, name, dt, shape in ((scale, 'scale', torch.float32, (B, 1)), (translation, 'translation', torch.float32, (B, 3)),
                               (rot, 'rot', torch.float32, (B, 4)), (ind, 'ind', torch.int64, (B,))):
        _cuda(t, dt, name)
        if tuple(t.shape) != shape:
            raise B3DError(f"image_batch: {name} has shape {tuple(t.shape)}; expected {list(shape)}")
    res_arr = (ctypes.c_int32 * len(res))(*res)
    img_arr = (ctypes.c_void_p * len(images))(*[im.data_ptr() for im in images])
    check(lib.b3d_image_batch(ptr(pixels), ptr(offsets), ptr(geometry), ptr(poses), n, ptr(idx), ptr(flip), B, len(res),
                              ctypes.cast(res_arr, ctypes.c_void_p), ctypes.cast(img_arr, ctypes.c_void_p), ptr(scale),
                              ptr(translation), ptr(rot), ptr(ind), stream_ptr(idx)))


def pseudogt_pack(vis, tex, alpha, image, tex_out, alpha_out, image_out):
    """b3d_pseudogt_pack: one launch turns a batch of inverse renders into pseudo-ground-truth planes.
    vis uint8 [B,Th,Tw] (texel visibility), tex fp32 [B,R,R,C], alpha fp32 [B,R,R,1], image fp32 [B,Ci,h,w] -> tex_out fp16
    [B,C,R,R], alpha_out fp16 [B,1,R,R], image_out fp16 [B,Ci,h,w]: visibility mask resized to R with F.interpolate's
    bilinear taps (align_corners=False), texture and alpha masked, every plane rounded as .half() rounds.  All tensors
    contiguous on the device."""
    def need(t, dtype, name, dim):
        if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == dtype and t.is_contiguous() and t.dim() == dim):
            raise B3DError(f"pseudogt_pack: {name} must be a contiguous {dtype} CUDA tensor with {dim} dimensions")
    need(vis, torch.uint8, 'vis', 3)
    need(tex, torch.float32, 'tex', 4)
    need(alpha, torch.float32, 'alpha', 4)
    need(image, torch.float32, 'image', 4)
    B, Th, Tw = vis.shape
    R, C = tex.shape[1], tex.shape[3]
    Ci, h, w = image.shape[1:]
    expect = {'tex': (tex, (B, R, R, C)), 'alpha': (alpha, (B, R, R, 1)), 'image': (image, (B, Ci, h, w))}
    for name, (t, shape) in expect.items():
        if tuple(t.shape) != shape:
            raise B3DError(f"pseudogt_pack: {name} has shape {tuple(t.shape)}; expected {list(shape)}")
    for name, t, shape in (('tex_out', tex_out, (B, C, R, R)), ('alpha_out', alpha_out, (B, 1, R, R)),
                           ('image_out', image_out, (B, Ci, h, w))):
        need(t, torch.float16, name, 4)
        if tuple(t.shape) != shape:
            raise B3DError(f"pseudogt_pack: {name} has shape {tuple(t.shape)}; expected {list(shape)}")
    check(lib.b3d_pseudogt_pack(ptr(vis), Th, Tw, ptr(tex), ptr(alpha), B, R, C, ptr(image), Ci, h, w, ptr(tex_out),
                                ptr(alpha_out), ptr(image_out), stream_ptr(vis)))


def sample_pack(image, imidx, tex, tiles_out, tex8_out):
    """b3d_sample_pack: one launch turns a batch of renders and textures into the bytes of the exported PNGs.
    image fp32 [B,H,W,3] (the Renderer output), imidx int32 [B,H,W] (its face-index buffer, 0 = background), tex fp32
    [B,3,T,T] -> tiles_out uint8 [B,H/2,W/2,3] (background 1.0, / 2 + 0.5, 2 x 2 average pool, * 255, clamp, truncate),
    tex8_out uint8 [B,T,T,3] (/ 2 + 0.5, * 255, clamp, truncate), rounded as the torch ops round.  H and W even; all
    tensors contiguous on the device.  Shapes are checked before the device, so a malformed call fails the same way on
    any machine."""
    def need(t, dtype, name, dim):
        if not (isinstance(t, torch.Tensor) and t.dtype == dtype and t.dim() == dim and t.is_contiguous()):
            raise B3DError(f"sample_pack: {name} must be a contiguous {dtype} tensor with {dim} dimensions")
    need(image, torch.float32, 'image', 4)
    need(imidx, torch.int32, 'imidx', 3)
    need(tex, torch.float32, 'tex', 4)
    need(tiles_out, torch.uint8, 'tiles_out', 4)
    need(tex8_out, torch.uint8, 'tex8_out', 4)
    B, H, W = imidx.shape
    T = tex.shape[2]
    if H % 2 or W % 2:
        raise B3DError(f"sample_pack: the render is {H} x {W}; the 2 x 2 pool needs an even height and width")
    for name, t, shape in (('image', image, (B, H, W, 3)), ('tex', tex, (B, 3, T, T)),
                           ('tiles_out', tiles_out, (B, H // 2, W // 2, 3)), ('tex8_out', tex8_out, (B, T, T, 3))):
        if tuple(t.shape) != shape:
            raise B3DError(f"sample_pack: {name} has shape {tuple(t.shape)}; expected {list(shape)}")
    for name, t in (('image', image), ('imidx', imidx), ('tex', tex), ('tiles_out', tiles_out), ('tex8_out', tex8_out)):
        if not t.is_cuda:
            raise B3DError(f"sample_pack: {name} is on {t.device}; libb3d runs on CUDA tensors only, there is no CPU "
                           "fallback")
    check(lib.b3d_sample_pack(ptr(image), ptr(imidx), B, H, W, ptr(tex), T, ptr(tiles_out), ptr(tex8_out),
                              stream_ptr(image)))


def recon_texture_pack(vis, proj, alpha, pred, symmetric, tex8_out, src8_out):
    """b3d_recon_texture_pack: one launch builds the textures of a batch of exported reconstructions.
    vis uint8 [B,Th,Tw] (texel visibility), proj fp32 [B,R,R,3] and alpha fp32 [B,R,R,1] (the photo projected into UV
    space and its hard mask), pred fp32 [B,3,T,T] (the network's texture) -> tex8_out uint8 [B,R,R,3], src8_out uint8
    [B,R,R]: the projection where the pseudo-ground-truth mask keeps it (source 1), with a symmetric template its mirror
    image where only that is kept (source 2), pred bilinearly resampled to R elsewhere (source 0); bytes as sample_pack's
    tex8.  R even; all tensors contiguous on the device.  Shapes are checked before the device."""
    def need(t, dtype, name, dim):
        if not (isinstance(t, torch.Tensor) and t.dtype == dtype and t.dim() == dim and t.is_contiguous()):
            raise B3DError(f"recon_texture_pack: {name} must be a contiguous {dtype} tensor with {dim} dimensions")
    need(vis, torch.uint8, 'vis', 3)
    need(proj, torch.float32, 'proj', 4)
    need(alpha, torch.float32, 'alpha', 4)
    need(pred, torch.float32, 'pred', 4)
    need(tex8_out, torch.uint8, 'tex8_out', 4)
    need(src8_out, torch.uint8, 'src8_out', 3)
    B, Th, Tw = vis.shape
    R, T = proj.shape[1], pred.shape[2]
    if R % 2:
        raise B3DError(f"recon_texture_pack: R {R} is odd; the mirrored column map needs an even resolution")
    for name, t, shape in (('proj', proj, (B, R, R, 3)), ('alpha', alpha, (B, R, R, 1)), ('pred', pred, (B, 3, T, T)),
                           ('tex8_out', tex8_out, (B, R, R, 3)), ('src8_out', src8_out, (B, R, R))):
        if tuple(t.shape) != shape:
            raise B3DError(f"recon_texture_pack: {name} has shape {tuple(t.shape)}; expected {list(shape)}")
    for name, t in (('vis', vis), ('proj', proj), ('alpha', alpha), ('pred', pred), ('tex8_out', tex8_out),
                    ('src8_out', src8_out)):
        if not t.is_cuda:
            raise B3DError(f"recon_texture_pack: {name} is on {t.device}; libb3d runs on CUDA tensors only, there is no "
                           "CPU fallback")
    check(lib.b3d_recon_texture_pack(ptr(vis), Th, Tw, ptr(proj), ptr(alpha), B, R, ptr(pred), T, int(bool(symmetric)),
                                     ptr(tex8_out), ptr(src8_out), stream_ptr(proj)))
