"""CPU oracle for the textured-mesh render path (pipeline A): template deformation, pose transform,
DIB-R rasterisation, fragment shading and the reconstruction / smoothness losses.

TEST INFRASTRUCTURE ONLY (see oracle/pointcloud.py header for who may import it).

Parity status
  * PINNED (against the reference's own Python, imported in the authoring container by
    tests/golden/make_golden_mesh.py): qrot / circpad / fragment shader / loss_flat / face adjacency
    `ff` / mean_iou / transform_vertices.
  * PINNED: MeshTemplate (mesh_template.py:14-170: index sets, topology / tangent maps, get_vertex_positions,
    deform, adjust_uv_and_texture, compute_normals).  The reference's class imports kaolin for ONE call
    (TriangleMesh.from_obj) and hard-codes .cuda(); tests/golden/make_golden_template.py supplies a stand-in for
    exactly those two things and runs the class UNMODIFIED on the CPU (-> tests/golden/template_reference.npz;
    tests/test_template_reference.py: this restatement and the drop-in equal it on 16 / 31-ring spheres, symmetric
    and not, and on the shipped OBJ templates).  kaolin's OBJ parser itself is the one piece not exercised.
  * PINNED: `render` / `ortho_projection` / `forward_renderer` — everything AROUND the rasteriser: the reference's
    Renderer.forward (renderer.py:39-77) is run unmodified with this file's `rasterize` standing in for kaolin's
    (tests/golden/make_golden_renderer.py -> renderer_reference.npz) and `render` must reproduce it exactly.
  * PARITY UNPINNED: `rasterize` restates kaolin @ e7e5131 `linear_rasterizer` from SURVEY.md App. B
    (kaolin is not in the container and not installable); it is validated for self-consistency
    only (coverage = point-in-triangle, z order, barycentrics sum to 1, autograd = finite differences).

Restates (all under /root/reference/code):
  rendering/renderer.py:9-77          ortho_projection, Renderer.forward
  rendering/fragment_shader.py:6-37   texinterpolation, fragmentshader
  rendering/mesh_template.py:14-186   MeshTemplate
  rendering/utils.py:29-46            circpad, qrot
  rendering/monkey_patches.py:8-156   face adjacency `ff`
  run_reconstruction.py:225-252       mean_iou, transform_vertices
  utils/losses.py:5-17                loss_flat
  models/reconstruction.py:151-180    DatasetParams (z0 = 1 + exp(theta))
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

# kaolin defaults the reference relies on (renderer.py:60-67 passes none), SURVEY App. B
EXPAND = 0.02
KNUM = 30
MULTIPLIER = 1000.0
DELTA = 7000.0
DEPTH_INIT = -1000.0
BARY_EPS = 1e-10
NORMAL_EPS = 1e-8
SEG_EPS = 1e-10


# ---------------------------------------------------------------------------------------------
# template geometry
# ---------------------------------------------------------------------------------------------
def load_obj(path):
    """Triangle OBJ with v / vt / f v/vt lines -> dict of tensors (what kal.rep.TriangleMesh.from_obj
    gives the reference: vertices, faces, uvs, face_textures; mesh_template.py:18)."""
    v, vt, f, ft = [], [], [], []
    with open(path) as fh:
        for line in fh:
            t = line.split()
            if not t:
                continue
            if t[0] == "v":
                v.append([float(x) for x in t[1:4]])
            elif t[0] == "vt":
                vt.append([float(x) for x in t[1:3]])
            elif t[0] == "f":
                f.append([int(x.split("/")[0]) - 1 for x in t[1:4]])
                ft.append([int(x.split("/")[1]) - 1 for x in t[1:4]])
    return dict(vertices=torch.tensor(v, dtype=torch.float32), faces=torch.tensor(f, dtype=torch.long),
                uvs=torch.tensor(vt, dtype=torch.float32), face_textures=torch.tensor(ft, dtype=torch.long))


def face_adjacency(faces):
    """`ff` of monkey_patches.py:96-106: per face, the faces sharing an edge, sorted descending,
    padded with -1."""
    faces = faces.cpu().numpy()
    edge_faces = {}
    for fi, tri in enumerate(faces):
        for a, b in ((0, 1), (1, 2), (2, 0)):
            e = (min(tri[a], tri[b]), max(tri[a], tri[b]))
            edge_faces.setdefault(e, []).append(fi)
    nbrs = [set() for _ in faces]
    for fl in edge_faces.values():
        for a in fl:
            for b in fl:
                if a != b:
                    nbrs[a].add(b)
    width = max(len(n) for n in nbrs)
    ff = np.full((len(faces), width), -1, dtype=np.int64)
    for fi, n in enumerate(nbrs):
        s = sorted(n, reverse=True)
        ff[fi, : len(s)] = s
    return torch.from_numpy(ff)


class TemplateData:
    """Everything MeshTemplate.__init__ derives from the OBJ (mesh_template.py:14-104)."""

    def __init__(self, mesh, mesh_path="", is_symmetric=True, device="cpu"):
        V = mesh["vertices"]
        self.vertices, self.faces = V, mesh["faces"]
        self.uvs, self.face_textures = mesh["uvs"], mesh["face_textures"]
        self.ff = face_adjacency(self.faces)
        poles = [int(V[:, 1].argmax()), int(V[:, 1].argmin())]
        neg = torch.nonzero(V[:, 0] < -1e-4)[:, 0]
        zero = torch.nonzero(V[:, 0].abs() < 1e-4)[:, 0]
        pos = []
        for idx in neg.tolist():                                    # :33-39
            opp = V[idx].clone()
            opp[0] *= -1
            d = (V - opp).norm(dim=-1)
            mv, mi = torch.min(d, dim=0)
            assert mv < 1e-4
            pos.append(int(mi))
        assert len(set(pos)) == len(pos)
        pos = torch.tensor(pos, dtype=torch.long)
        self.pos_indices, self.neg_indices, self.zero_indices = pos, neg, zero
        self.nonneg_indices = torch.cat([pos, zero])
        assert len(pos) + len(neg) + len(zero) == len(V)
        segments, rings = 32, (31 if "31rings" in mesh_path else 16)
        occ = {}
        for ftri, vtri in zip(self.face_textures.tolist(), self.faces.tolist()):   # :57-64
            for t, v in zip(ftri, vtri):
                res = self.uvs[t].numpy() * [segments, rings]
                if math.isclose(res[0], segments, abs_tol=1e-4):
                    res[0] = 0
                occ.setdefault(v, []).append(res)
        topo = torch.zeros(V.shape[0], 2)
        for idx, data in occ.items():
            topo[idx] = torch.tensor(np.mean(np.array(data, dtype=np.float32), axis=0) / [segments, rings],
                                     dtype=torch.float32)
        topo = (topo * 2 - 1) * torch.tensor([1.0, -1.0])           # :71-73
        self.topo_map = topo
        self.nonneg_topo_map = topo[self.nonneg_indices]
        sm = torch.ones_like(V).unsqueeze(0)
        sm[:, zero, 0] = 0
        self.symmetry_mask = sm
        n = F.normalize(V, dim=1)                                    # :82-91
        up = torch.tensor([[0.0, 1.0, 0.0]]).expand_as(n)
        t = F.normalize(torch.cross(n, up, dim=1), dim=1)
        b = torch.cross(n, t, dim=1)
        for p in poles:
            t[p] = 0
            b[p] = 0
        self.tangent_map = torch.stack((n, t, b), dim=1)
        self.nonneg_tangent_map = self.tangent_map[self.nonneg_indices]
        self.is_symmetric = is_symmetric
        for k, v in list(self.__dict__.items()):
            if isinstance(v, torch.Tensor):
                setattr(self, k, v.to(device))


def circpad(x, amount=1):
    """rendering/utils.py:29-33."""
    return torch.cat((x[:, :, :, -amount:], x, x[:, :, :, :amount]), dim=3)


def qrot(q, v):
    """rendering/utils.py:36-46."""
    qvec = q[:, 1:].unsqueeze(1).expand(-1, v.shape[1], -1)
    uv = torch.cross(qvec, v, dim=2)
    uuv = torch.cross(qvec, uv, dim=2)
    return v + 2 * (q[:, :1].unsqueeze(1) * uv + uuv)


def adjust_uv_and_texture(T, texture):
    """mesh_template.py:151-170."""
    if T.is_symmetric:
        delta = 1 / (2 * texture.shape[3])
        expansion = (texture.shape[3] + 1) / texture.shape[3]
        uvs = T.uvs.clone()
        uvs[:, 0] = (uvs[:, 0] + delta) / expansion
        return uvs.expand(texture.shape[0], -1, -1), circpad(texture, 1)
    return T.uvs.expand(texture.shape[0], -1, -1), torch.cat((texture, texture[:, :, :, :1]), dim=3)


def get_vertex_positions(T, displacement_map):
    """mesh_template.py:125-149."""
    topo = T.nonneg_topo_map if T.is_symmetric else T.topo_map
    _, padded = adjust_uv_and_texture(T, displacement_map)
    if T.is_symmetric:
        delta = 1 / (2 * displacement_map.shape[3])
        expansion = (displacement_map.shape[3] + 1) / displacement_map.shape[3]
        topo = topo.clone()
        topo[:, 0] = (topo[:, 0] + 1 + 2 * delta - expansion) / expansion
    B = displacement_map.shape[0]
    grid = topo.to(displacement_map.dtype).unsqueeze(0).unsqueeze(-2).expand(B, -1, -1, -1)
    local = F.grid_sample(padded, grid, mode="bilinear", align_corners=True).squeeze(-1).permute(0, 2, 1)
    tgm = (T.nonneg_tangent_map if T.is_symmetric else T.tangent_map).to(displacement_map.dtype)
    deltas = (local.unsqueeze(-2) @ tgm.expand(B, -1, -1, -1)).squeeze(-2)          # deform :106-111
    if T.is_symmetric:
        vtx = deltas.new_zeros(B, T.topo_map.shape[0], 3)
        vtx[:, T.nonneg_indices] = deltas
        vtx2 = vtx.clone()
        vtx2[:, T.neg_indices] = vtx[:, T.pos_indices] * deltas.new_tensor([-1.0, 1.0, 1.0])
        deltas = vtx2 * T.symmetry_mask.to(deltas.dtype)
    return T.vertices.to(deltas.dtype).unsqueeze(0) + deltas


def compute_normals(T, vertex_positions):
    """mesh_template.py:113-123."""
    a = vertex_positions[:, T.faces[:, 0]]
    b = vertex_positions[:, T.faces[:, 1]]
    c = vertex_positions[:, T.faces[:, 2]]
    return F.normalize(torch.cross(b - a, c - a, dim=2), dim=2)


def loss_flat(ff, n_faces, norms):
    """utils/losses.py:5-17."""
    loss = 0.0
    for i in range(3):
        cos = torch.sum(norms * norms[:, ff[:, i]], dim=-1)
        loss = loss + torch.mean((cos - 1) ** 2)
    return loss * (n_faces / 2.0)


def transform_vertices(vtx, scale, translation, rot, z0=None, scale_delta=0, translation_delta=0):
    """run_reconstruction.py:237-252 (z0 given = --optimize_z0)."""
    vtx = qrot(rot, (scale + scale_delta).unsqueeze(-1) * vtx) + (translation + translation_delta).unsqueeze(1)
    vtx = vtx * vtx.new_tensor([1.0, -1.0, -1.0])
    if z0 is not None:
        z0 = z0.view(-1, 1, 1)
        z = vtx[:, :, 2:]
        factor = (z0 + z / 2) / (z0 - z / 2)
        vtx = torch.cat((vtx[:, :, :2] * factor, z), dim=2)
    return vtx


def mean_iou(alpha_pred, alpha_real):
    """run_reconstruction.py:225-231."""
    p, r = alpha_pred > 0.5, alpha_real > 0.5
    inter = (p & r).float().sum(dim=[1, 2])
    union = (p | r).float().sum(dim=[1, 2])
    return torch.mean(inter / union)


# ---------------------------------------------------------------------------------------------
# renderer
# ---------------------------------------------------------------------------------------------
def ortho_projection(points, faces):
    """renderer.py:9-28."""
    pf = [points[:, faces[:, i], :] for i in range(3)]
    p3d = torch.cat(pf, dim=2)
    p2d = torch.cat([p[:, :, :2] for p in pf], dim=2)
    normal = torch.cross(pf[1] - pf[0], pf[2] - pf[0], dim=2)
    return p3d, p2d, normal


def datanormalize(x, axis):
    """kaolin dib_renderer.utils.datanormalize [UNVERIFIED eps]: x / (||x|| + 1e-8)."""
    return x / (x.norm(dim=axis, keepdim=True) + NORMAL_EPS)


def _seg_dist2(px, py, ax, ay, bx, by):
    """squared distance from (px,py) to segment a-b (all broadcastable)."""
    ex, ey = bx - ax, by - ay
    dx, dy = px - ax, py - ay
    t = ((dx * ex + dy * ey) / (ex * ex + ey * ey + SEG_EPS)).clamp(0, 1)
    rx, ry = dx - t * ex, dy - t * ey
    return rx * rx + ry * ry


def pixel_centres(H, W, dtype, device):
    """SURVEY App. B step 2: x0 = m/W (2x+1-W), y0 = m/H (H-2y-1); row 0 is the top."""
    xs = torch.arange(W, dtype=dtype, device=device)
    ys = torch.arange(H, dtype=dtype, device=device)
    x0 = MULTIPLIER / W * (2 * xs + 1 - W)
    y0 = MULTIPLIER / H * (H - 2 * ys - 1)
    return x0.view(1, 1, W), y0.view(1, H, 1)


def _window(lo, hi, n, size, flip):
    """Conservative pixel index range [i0, i1) whose centres can fall inside [lo, hi) (+-1 pixel)."""
    # centre(i) = m/size * (2i + 1 - size)  (x)   or   m/size * (size - 2i - 1)  (y, flip)
    a = (lo * size / MULTIPLIER + size - 1) / 2
    b = (hi * size / MULTIPLIER + size - 1) / 2
    if flip:
        a, b = (size - 1) - b, (size - 1) - a
    i0 = max(0, int(math.floor(a)) - 1)
    i1 = min(n, int(math.ceil(b)) + 2)
    return i0, max(i0, i1)


def rasterize(p3d, p2d, normalz, attr, H, W, expand=EXPAND, knum=KNUM, multiplier=MULTIPLIER, delta=DELTA,
              record=None):
    """kaolin linear_rasterizer restated from SURVEY.md App. B (PARITY UNPINNED).

    p3d [B,F,9], p2d [B,F,6], normalz [B,F,1], attr [B,F,3d] ->
      imfeat [B,H,W,d], improb [B,H,W,1], imidx [B,H,W] int32 (face+1, 0 = background), imwei [B,H,W,3].
    Differentiable w.r.t. p2d and attr (not p3d / normalz), like kaolin's backward.
    The loops run face by face in face order, like kaolin's per-pixel loops; per face only the pixel
    window that can pass its (expanded) bounding-box test is touched (an exact restriction).

    record: an optional dict that receives every discrete decision behind each pixel (see `_Record`); the outputs
    are the same with or without it."""
    rec = _Record(B=p2d.shape[0], H=H, W=W, dev=p2d.device, multiplier=multiplier, knum=knum) \
        if record is not None else None
    assert multiplier == MULTIPLIER
    B, Fn, _ = p2d.shape
    d = attr.shape[2] // 3
    dt, dev = p2d.dtype, p2d.device
    x0, y0 = pixel_centres(H, W, dt, dev)
    P = (multiplier * p2d).detach()
    Z = p3d.detach()[:, :, 2::3]
    xmin = torch.minimum(torch.minimum(P[..., 0], P[..., 2]), P[..., 4])
    xmax = torch.maximum(torch.maximum(P[..., 0], P[..., 2]), P[..., 4])
    ymin = torch.minimum(torch.minimum(P[..., 1], P[..., 3]), P[..., 5])
    ymax = torch.maximum(torch.maximum(P[..., 1], P[..., 3]), P[..., 5])
    bb = torch.stack([xmin, xmax, ymin, ymax], dim=-1).double().cpu().numpy()
    front_np = (normalz[:, :, 0] >= 0).cpu().numpy()

    def bary(Pf, xs, ys):
        ax, ay, bx, by, cx, cy = [Pf[..., i] for i in range(6)]
        m, p = bx - ax, by - ay
        n, q = cx - ax, cy - ay
        s, t = xs - ax, ys - ay
        k3 = m * q - n * p
        w1 = (s * q - n * t) / (k3 + BARY_EPS)
        w2 = (m * t - s * p) / (k3 + BARY_EPS)
        return 1 - w1 - w2, w1, w2

    imidx = torch.zeros(B, H, W, dtype=torch.int32, device=dev)
    imdep = torch.full((B, H, W), DEPTH_INIT, dtype=dt, device=dev)
    for b in range(B):
        for f in range(Fn):
            if not front_np[b, f]:
                continue
            c0, c1 = _window(bb[b, f, 0], bb[b, f, 1], W, W, False)
            r0, r1 = _window(bb[b, f, 2], bb[b, f, 3], H, H, True)
            if c0 >= c1 or r0 >= r1:
                continue
            xs, ys = x0[0, :, c0:c1], y0[0, r0:r1, :]
            inbox = (xs >= xmin[b, f]) & (xs < xmax[b, f]) & (ys >= ymin[b, f]) & (ys < ymax[b, f])
            w0, w1, w2 = bary(P[b, f], xs, ys)
            inside = (w0 >= 0) & (w1 >= 0) & (w2 >= 0)
            z = w0 * Z[b, f, 0] + w1 * Z[b, f, 1] + w2 * Z[b, f, 2]
            dep = imdep[b, r0:r1, c0:c1]
            upd = inbox & inside & (z > dep)
            imidx[b, r0:r1, c0:c1] = torch.where(upd, torch.full_like(imidx[b, r0:r1, c0:c1], f + 1),
                                                 imidx[b, r0:r1, c0:c1])
            imdep[b, r0:r1, c0:c1] = torch.where(upd, z, dep)

    covered = imidx > 0
    # differentiable barycentrics of the winning face
    sel = (imidx.long() - 1).clamp_min(0).view(B, H * W)
    Pd = (multiplier * p2d).gather(1, sel.unsqueeze(-1).expand(-1, -1, 6)).view(B, H, W, 6)
    w0, w1, w2 = bary(Pd, x0, y0)
    cov = covered.to(dt)
    imwei = torch.stack([w0, w1, w2], dim=-1) * cov.unsqueeze(-1)
    A = attr.gather(1, sel.unsqueeze(-1).expand(-1, -1, 3 * d)).view(B, H, W, 3, d)
    imfeat = (imwei.unsqueeze(-1) * A).sum(dim=3)

    # soft silhouette for uncovered pixels: first `knum` faces (face order) whose expanded box holds the pixel
    e = expand * multiplier
    count = torch.zeros(B, H, W, dtype=torch.int32, device=dev)
    Pm = multiplier * p2d
    pieces = []        # (b, r0, r1, c0, c1, log(1 - p_k) masked)  — summed below, differentiably
    for b in range(B):
        if bool(covered[b].all()):
            continue
        for f in range(Fn):
            c0, c1 = _window(bb[b, f, 0] - e, bb[b, f, 1] + e, W, W, False)
            r0, r1 = _window(bb[b, f, 2] - e, bb[b, f, 3] + e, H, H, True)
            if c0 >= c1 or r0 >= r1:
                continue
            xs, ys = x0[0, :, c0:c1], y0[0, r0:r1, :]
            near = (xs >= xmin[b, f] - e) & (xs < xmax[b, f] + e) & (ys >= ymin[b, f] - e) & (ys < ymax[b, f] + e)
            cnt = count[b, r0:r1, c0:c1]
            use = near & (~covered[b, r0:r1, c0:c1]) & (cnt < knum)
            if rec is not None:
                bounds = (xmin[b, f] - e, xmax[b, f] + e, ymin[b, f] - e, ymax[b, f] + e)
                rec.face(b, f, r0, r1, c0, c1, xs, ys, Pm[b, f].detach(), bounds, near, use,
                         (~covered[b, r0:r1, c0:c1]) & (cnt < knum), covered[b, r0:r1, c0:c1], delta)
            if not bool(use.any()):
                continue
            a = Pm[b, f]
            d2 = torch.minimum(torch.minimum(_seg_dist2(xs, ys, a[0], a[1], a[2], a[3]),
                                             _seg_dist2(xs, ys, a[2], a[3], a[4], a[5])),
                               _seg_dist2(xs, ys, a[4], a[5], a[0], a[1]))
            pk = torch.exp(-delta * d2 / (multiplier * multiplier))
            lk = torch.where(use, torch.log1p(-pk.clamp(max=1 - 1e-7)), torch.zeros_like(pk))
            pieces.append((b, r0, r1, c0, c1, lk))
            count[b, r0:r1, c0:c1] = cnt + use.to(torch.int32)
    log_keep = _SumWindows.apply((B, H, W), [p[:5] for p in pieces], x0, *[p[5] for p in pieces])
    improb = torch.where(covered, torch.ones_like(log_keep), 1 - torch.exp(log_keep))
    if rec is not None:
        record.update(rec.finish(imidx, count))
    return imfeat, improb.unsqueeze(-1), imidx, imwei


class _SumWindows(torch.autograd.Function):
    """out = zeros(shape); out[b, r0:r1, c0:c1] += piece_i for every window (gradient: the slices)."""

    @staticmethod
    def forward(ctx, shape, wins, like, *pieces):
        out = like.new_zeros(shape)
        for (b, r0, r1, c0, c1), pc in zip(wins, pieces):
            out[b, r0:r1, c0:c1] += pc
        ctx.wins = wins
        return out

    @staticmethod
    def backward(ctx, g):
        return (None, None, None) + tuple(g[b, r0:r1, c0:c1] for (b, r0, r1, c0, c1) in ctx.wins)


# ---------------------------------------------------------------------------------------------
# the rasteriser's discrete decisions (rasterize(record=...)) and the pixels where they are stable
# ---------------------------------------------------------------------------------------------
# An fp32 kernel and the fp64 oracle agree to rounding only where both take the same discrete decisions.  stable_pixels
# keeps the pixels where the fp32 and fp64 oracle runs take identical decisions AND every decision is further from its
# switch point than the margins below, so that the kernel (whose soft-path and shading arithmetic is not rounding-exact)
# takes them too.  The face-index buffer is left out of the margins: the kernel reproduces the fp32 oracle's bit for bit.
#   EDGE_TIE_REL  closest edge: the next edge with a different closest point is further by more than this factor of
#                 d^2 + EDGE_TIE_SCALE * multiplier * d.  rx, ry are differences of coordinates up to ~multiplier,
#                 rounded to ~1e-7 multiplier in fp32, so d^2 carries ~2.4e-7 * multiplier * d: the second term keeps
#                 the margin ~8x that rounding for pixels close to the edge, the first is 1e-4 relative far from it.
#                 Two edges that both clamp to their shared vertex have the same closest point and the same adjoint,
#                 so that tie is not a decision.
#   T_MARGIN      segment clamp: the arg-min edge's unclamped foot parameter t is this far from 0 and from 1.
#   TEXEL_MARGIN  texel floor (bilinear, bicubic) or round (nearest): the fractional texel coordinate is this far from
#                 0 and 1, or from 0.5; u, v carry ~1 ulp and textures here are < 300 texels, i.e. < 2e-5 texel.
#   BOX_MARGIN    expanded-box tests, in multiplier units: pixel centres and box bounds (|x| <~ 1) round to ~1e-7.
#   PK_MAX        the soft-silhouette clamp p_k < 1 - 1e-7: p_k stays below this; 1 - p_k then keeps >= 3 significant
#                 digits in fp32.
EDGE_TIE_REL = 1e-4
EDGE_TIE_SCALE = 0.02
T_MARGIN = 1e-4
TEXEL_MARGIN = 1e-4
BOX_MARGIN = 1e-6
PK_MAX = 1 - 1e-4
_SIG_MOD, _SIG_MUL = 2147483647, 1000003


class _Record:
    """Per-pixel decisions of one rasterize call.  Filled face by face by the soft-silhouette loop; `finish` returns:
      imidx      [B,H,W] the coverage / depth winner (face + 1)
      soft_n     [B,H,W] faces that shaped the soft silhouette (<= knum), cand [B,H,W] faces whose expanded box holds
                 the uncovered pixel (cand > soft_n: knum cut the list)
      soft_sig   [B,H,W] hash of the ordered (face, closest point) list
      edge_gap   [B,H,W] min over those faces of (d2 of the next edge with another closest point - d2)
                 / (d2 + EDGE_TIE_SCALE * multiplier * d)
      t_gap      [B,H,W] min over those faces of the arg-min edge's distance of unclamped t from {0, 1}
      box_gap    [B,H,W] min over the faces tested before the knum cap of the distance (multiplier units) of the
                 expanded-box decision from its switch point
      pk_max     [B,H,W] max p_k over those faces
      soft       list of (b, f, r0, c0, use [h,w], edge [h,w], gap [h,w], t [h,w]) per face window, in face order
      tiles      {(b, ty, tx): [faces whose expanded box holds a pixel of the 16x16 tile, in face order]}"""

    def __init__(self, B, H, W, dev, multiplier, knum):
        z = dict(device=dev)
        self.m, self.knum = float(multiplier), knum
        inf = float("inf")
        self.cand = torch.zeros(B, H, W, dtype=torch.int32, **z)
        self.sig = torch.zeros(B, H, W, dtype=torch.int64, **z)
        self.edge_gap = torch.full((B, H, W), inf, dtype=torch.float64, **z)
        self.t_gap = torch.full((B, H, W), inf, dtype=torch.float64, **z)
        self.box_gap = torch.full((B, H, W), inf, dtype=torch.float64, **z)
        self.pk_max = torch.zeros(B, H, W, dtype=torch.float64, **z)
        self.soft, self.tiles = [], {}

    def face(self, b, f, r0, r1, c0, c1, xs, ys, a, bounds, near, use, consider, covered, delta):
        shape = (r1 - r0, c1 - c0)
        xs, ys = xs.expand(shape), ys.expand(shape)
        win = (b, slice(r0, r1), slice(c0, c1))
        rc = near.nonzero()
        for ty, tx in torch.unique(torch.stack([(rc[:, 0] + r0) // 16, (rc[:, 1] + c0) // 16], 1), dim=0).tolist():
            self.tiles.setdefault((b, ty, tx), []).append(f)
        self.cand[win] += (near & ~covered).to(torch.int32)
        # expanded box: all four tests pass -> the nearest bound decides; else all failing tests must flip
        lo_x, hi_x, lo_y, hi_y = bounds
        s = torch.stack([(xs - lo_x).abs(), (hi_x - xs).abs(), (ys - lo_y).abs(), (hi_y - ys).abs()]).double()
        ok = torch.stack([xs >= lo_x, xs < hi_x, ys >= lo_y, ys < hi_y])
        gap = torch.where(near, s.min(0).values, torch.where(ok, torch.zeros_like(s), s).max(0).values) / self.m
        self.box_gap[win] = torch.minimum(self.box_gap[win], torch.where(consider, gap, torch.full_like(gap, math.inf)))
        if not bool(use.any()):
            return
        d2s, ts, feats = [], [], []
        for k in range(3):
            k1 = (k + 1) % 3
            ax, ay, bx, by = a[2 * k], a[2 * k + 1], a[2 * k1], a[2 * k1 + 1]
            ex, ey = bx - ax, by - ay
            traw = ((xs - ax) * ex + (ys - ay) * ey) / (ex * ex + ey * ey + SEG_EPS)
            tc = traw.clamp(0, 1)
            d2s.append(_seg_dist2(xs, ys, ax, ay, bx, by))
            ts.append(traw)
            # closest point: interior of edge k (k), or vertex k / k+1 (3 + vertex) where t clamps
            feats.append(torch.where(tc <= 0, 3 + k, torch.where(tc >= 1, 3 + k1, k)))
        d2, t, feat = torch.stack(d2s), torch.stack(ts), torch.stack(feats)
        e = torch.zeros(shape, dtype=torch.long, device=xs.device)
        dm = d2[0]
        for k in (1, 2):                               # the kernel's arg-min: strict <, first edge wins ties
            less = d2[k] < dm
            e, dm = torch.where(less, k, e), torch.where(less, d2[k], dm)
        fe = feat.gather(0, e.unsqueeze(0))[0]
        second = torch.where(feat != fe, d2, torch.full_like(d2, math.inf)).min(0).values
        dmd = dm.double()
        scale = dmd + EDGE_TIE_SCALE * self.m * dmd.sqrt()
        egap = torch.where(dmd > 0, (second.double() - dmd) / scale.clamp_min(1e-300), torch.zeros_like(dmd))
        te = t.gather(0, e.unsqueeze(0))[0].double()
        tgap = torch.minimum(te.abs(), (te - 1).abs())
        pk = torch.exp(-delta * dmd / (self.m * self.m))
        inf = torch.full_like(egap, math.inf)
        self.edge_gap[win] = torch.minimum(self.edge_gap[win], torch.where(use, egap, inf))
        self.t_gap[win] = torch.minimum(self.t_gap[win], torch.where(use, tgap, inf))
        self.pk_max[win] = torch.maximum(self.pk_max[win], torch.where(use, pk, torch.zeros_like(pk)))
        code = f * 8 + fe + 1
        self.sig[win] = torch.where(use, (self.sig[win] * _SIG_MUL + code) % _SIG_MOD, self.sig[win])
        self.soft.append((b, f, r0, c0, use, e, egap, te))

    def finish(self, imidx, count):
        return dict(imidx=imidx.clone(), soft_n=count.clone(), cand=self.cand, soft_sig=self.sig,
                    edge_gap=self.edge_gap, t_gap=self.t_gap, box_gap=self.box_gap, pk_max=self.pk_max,
                    soft=self.soft, tiles=self.tiles, multiplier=self.m, knum=self.knum)


def pixel_faces(rec, b, y, x):
    """The ordered soft-silhouette list of one pixel: [(face, arg-min edge, edge gap, unclamped t)]."""
    out = []
    for bb, f, r0, c0, use, e, gap, t in rec["soft"]:
        r, c = y - r0, x - c0
        if bb == b and 0 <= r < use.shape[0] and 0 <= c < use.shape[1] and bool(use[r, c]):
            out.append((f, int(e[r, c]), float(gap[r, c]), float(t[r, c])))
    return out


def texel_coords(uv, Th, Tw, filtering):
    """Unnormalised texel coordinates (ix, iy) at which the shader samples (u, v): grid_sample's with the shader's
    (u * 2 - 1, -(v * 2 - 1)) grid, align_corners=True for bilinear, False for nearest / bicubic."""
    gx, gy = uv[..., 0] * 2 - 1, -(uv[..., 1] * 2 - 1)
    if filtering == "bilinear":
        return (gx + 1) / 2 * (Tw - 1), (gy + 1) / 2 * (Th - 1)
    return (gx + 1) * (Tw / 2) - 0.5, (gy + 1) * (Th / 2) - 0.5


def stable_pixels(rec32, rec64, uv32=None, uv64=None, tex_hw=None, filtering="bilinear"):
    """[B,H,W] bool: pixels whose every decision is identical in the fp32 and fp64 records and further than the
    margins above from its switch point.  uv32 / uv64 [B,H,W,2] (the interpolated texture coordinates of each run) and
    tex_hw = (Th, Tw) add the texel decisions of `filtering` on covered pixels."""
    ok = (rec32["imidx"] == rec64["imidx"]) & (rec32["soft_n"] == rec64["soft_n"]) & \
         (rec32["soft_sig"] == rec64["soft_sig"])
    for r in (rec32, rec64):
        ok &= (r["edge_gap"] > EDGE_TIE_REL) & (r["t_gap"] > T_MARGIN) & (r["box_gap"] > BOX_MARGIN) & \
              (r["pk_max"] < PK_MAX)
    if uv32 is not None:
        Th, Tw = tex_hw
        cov = rec32["imidx"] > 0
        fl = []
        for uv in (uv32, uv64):                     # each run's coordinates in its own precision
            for c in texel_coords(uv.detach(), Th, Tw, filtering):
                fr = (c - c.floor()).double()
                near = (fr - 0.5).abs() < TEXEL_MARGIN if filtering == "nearest" else \
                    (fr < TEXEL_MARGIN) | (fr > 1 - TEXEL_MARGIN)
                ok &= ~(cov & near)
                fl.append(c.floor().double())
        ok &= ~cov | ((fl[0] == fl[2]) & (fl[1] == fl[3]))
    return ok


def bin_faces(p2d, H, W, expand=EXPAND, multiplier=MULTIPLIER, tile=16):
    """The CUDA rasteriser's per-tile face lists restated in fp32: -> pos [B, ceil(H/tile), ceil(W/tile), F] int64, the
    face's position in the tile's list (faces in face order whose expanded bounding box reaches the tile's pixel
    centres), -1 where the face is not listed."""
    f32 = torch.float32
    P = p2d.detach().to(f32) * float(multiplier)
    E = torch.tensor(float(expand) * float(multiplier), dtype=f32)
    X, Y = P[..., 0::2], P[..., 1::2]
    lo_x, hi_x = X.min(-1).values - E, X.max(-1).values + E
    lo_y, hi_y = Y.min(-1).values - E, Y.max(-1).values + E
    sx = torch.tensor(float(multiplier), dtype=f32) / torch.tensor(float(W), dtype=f32)
    sy = torch.tensor(float(multiplier), dtype=f32) / torch.tensor(float(H), dtype=f32)
    tx0 = torch.arange(0, W, tile)
    ty0 = torch.arange(0, H, tile)
    cx = lambda x: sx * (2 * x + 1 - W).to(f32)
    cy = lambda y: sy * (H - 2 * y - 1).to(f32)
    x_lo, x_hi = cx(tx0), cx((tx0 + tile - 1).clamp(max=W - 1))
    y_lo, y_hi = cy((ty0 + tile - 1).clamp(max=H - 1)), cy(ty0)
    flag = (lo_x[:, None, None, :] <= x_hi[None, None, :, None]) & (x_lo[None, None, :, None] < hi_x[:, None, None, :]) \
        & (lo_y[:, None, None, :] <= y_hi[None, :, None, None]) & (y_lo[None, :, None, None] < hi_y[:, None, None, :])
    pos = flag.long().cumsum(-1) - 1
    return torch.where(flag, pos, torch.full_like(pos, -1))


def texinterpolation(uv, texture):
    """fragment_shader.py:6-20 (bilinear, align_corners=True)."""
    g = (uv * 2 - 1) * uv.new_tensor([1.0, -1.0])
    return F.grid_sample(texture, g, mode="bilinear", align_corners=True).permute(0, 2, 3, 1)


def fragmentshader(uv, texture, mask, background_image=None):
    """fragment_shader.py:22-37."""
    col = texinterpolation(uv, texture)
    return col * mask if background_image is None else torch.lerp(background_image, col, mask)


def render(points, faces, uv, texture, ft=None, H=256, W=256, background_image=None, return_hardmask=False):
    """Renderer.forward (renderer.py:39-77) -> (imrender, improb|hardmask, normal1, imidx)."""
    ft = faces if ft is None else ft
    p3d, p2d, normal = ortho_projection(points, faces)
    normalz = normal[:, :, 2:3]
    normal1 = datanormalize(normal, 2)
    c = [uv[:, ft[:, i], :] for i in range(3)]
    one = torch.ones_like(c[0][:, :, :1])
    uv9 = torch.cat((c[0], one, c[1], one, c[2], one), dim=2)
    imfeat, improb, imidx, _ = rasterize(p3d, p2d, normalz, uv9, H, W)
    hard = imfeat[..., 2:3]
    img = fragmentshader(imfeat[..., :2], texture, hard, background_image)
    return img, (hard if return_hardmask else improb), normal1, imidx


def forward_renderer(T, vertex_positions, texture, H=256, W=256, **kw):
    """mesh_template.py:172-186."""
    uvs, tex = adjust_uv_and_texture(T, texture)
    img, alpha, _, imidx = render(vertex_positions, T.faces, uvs.to(texture.dtype), tex, T.face_textures, H, W, **kw)
    return img, alpha, imidx


# ---------------------------------------------------------------------------------------------
# procedural stand-in (generator lives in tools/uvsphere.py: it is input data, shared with bench.py's CUDA arm);
# procedural stand-in for the shipped UV-sphere templates (same construction: 32 segments,
# `rings` rings, u = 1/4 + atan2(x,z)/2pi, v = 1 - polar/pi, one vt per pole triangle)
# ---------------------------------------------------------------------------------------------
from tools.uvsphere import write_uvsphere_obj  # noqa: E402,F401
