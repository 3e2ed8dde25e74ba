"""Box and image helpers of the CMR loaders (reference: cmr_data/image_utils.py).

`resize_img` is OpenCV's `cv2.resize(..., INTER_LINEAR)` on a float64 image, restated in numpy so the product needs no
OpenCV: per axis, source coordinate fx = (d + 0.5) * scale - 0.5 with scale = 1 / (dst / src), tap sx = floor(fx) and
weights (1 - fx', fx') on (sx, sx + 1), clamped to the edge pixel at both ends; a horizontal pass then a vertical pass, all
in double.  The weights must stay in double: float32 weights move a 500 -> 299 resize by up to 4e-5.  The kernel
b3d_image_batch computes the same taps and the same products (no fused multiply-add), so it agrees with this bit for bit."""
import numpy as np


def peturb_bbox(bbox, pf=0, jf=0):
    """Pad the zero-indexed tight box by pf of its width / height on every side, and jitter each side by up to jf of it
    (the loaders use jf = 0).  The result may reach outside the image."""
    out = list(bbox)
    w, h = bbox[2] - bbox[0] + 1, bbox[3] - bbox[1] + 1
    out[0] -= pf * w + (1 - 2 * np.random.random()) * jf * w
    out[1] -= pf * h + (1 - 2 * np.random.random()) * jf * h
    out[2] += pf * w + (1 - 2 * np.random.random()) * jf * w
    out[3] += pf * h + (1 - 2 * np.random.random()) * jf * h
    return out


def square_bbox(bbox):
    """Round the box to integers (Python's round: .5 goes to the even neighbour) and grow the shorter side to the longer
    one, centred.  -> [x0, y0, x0 + S - 1, y0 + S - 1] with S the side (the last two as floats, as in the reference)."""
    sq = [int(round(c)) for c in bbox]
    w, h = sq[2] - sq[0] + 1, sq[3] - sq[1] + 1
    side = float(max(w, h))
    sq[0] -= int(round((side - w) / 2.0))
    sq[1] -= int(round((side - h) / 2.0))
    sq[2] = sq[0] + side - 1
    sq[3] = sq[1] + side - 1
    return sq


def crop_window(bbox, im_h, im_w):
    """The part of the crop box that lies inside an im_h x im_w image.  -> (x0, y0, wx0, wy0, ww, wh): the box's integer
    origin in the image, the window's origin inside the crop and its size (0 when the box misses the image)."""
    x0, y0, x1, y1 = [int(round(c)) for c in bbox]
    xs, xe = max(0, x0), min(im_w, x1 + 1)
    ys, ye = max(0, y0), min(im_h, y1 + 1)
    return x0, y0, xs - x0, ys - y0, max(0, xe - xs), max(0, ye - ys)


def crop(img, bbox, bgval=0):
    """Crop bbox out of img ([H, W] or [H, W, C]) as float64 [h, w, C]; pixels outside the image are bgval."""
    x0, y0, wx0, wy0, ww, wh = crop_window(bbox, img.shape[0], img.shape[1])
    bw, bh = int(round(bbox[2])) - x0 + 1, int(round(bbox[3])) - y0 + 1
    nc = 1 if img.ndim < 3 else img.shape[2]
    out = np.ones((bh, bw, nc)) * bgval
    if ww and wh:
        src = img[y0 + wy0:y0 + wy0 + wh, x0 + wx0:x0 + wx0 + ww]
        out[wy0:wy0 + wh, wx0:wx0 + ww, :] = src.reshape(wh, ww, nc)
    return out


def linear_taps(src, dst):
    """OpenCV's INTER_LINEAR taps of one axis, src -> dst samples.  -> (s0, s1, w0, w1): int64 [dst] tap indices and
    float64 [dst] weights."""
    scale = 1.0 / (dst / src)
    fx = (np.arange(dst) + 0.5) * scale - 0.5
    s0 = np.floor(fx)
    fx = fx - s0
    s0 = s0.astype(np.int64)
    low, high = s0 < 0, s0 >= src - 1
    fx[low | high] = 0.0
    s0[low] = 0
    s0[high] = src - 1
    return s0, np.minimum(s0 + 1, src - 1), 1.0 - fx, fx


def resize(img, dst_h, dst_w):
    """cv2.resize(img, (dst_w, dst_h)) with INTER_LINEAR on float64 [H, W] or [H, W, C]; a single channel comes back 2-D,
    as from OpenCV."""
    img = np.asarray(img, dtype=np.float64)
    if img.ndim == 3 and img.shape[2] == 1:
        img = img[:, :, 0]
    y0, y1, b0, b1 = linear_taps(img.shape[0], dst_h)
    x0, x1, a0, a1 = linear_taps(img.shape[1], dst_w)
    ex = (slice(None),) + (None,) * (img.ndim - 2)
    rows = img[:, x0] * a0[ex] + img[:, x1] * a1[ex]
    return rows[y0] * b0[(slice(None), None) + ex[1:]] + rows[y1] * b1[(slice(None), None) + ex[1:]]


def resize_img(img, scale_factor):
    """Resize by scale_factor (the new size rounded).  -> (image, [actual y factor, actual x factor])."""
    new_size = np.round(np.array(img.shape[:2]) * scale_factor).astype(int)
    out = resize(img, new_size[0], new_size[1])
    return out, [new_size[0] / float(img.shape[0]), new_size[1] / float(img.shape[1])]
