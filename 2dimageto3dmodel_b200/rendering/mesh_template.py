"""Drop-in for /root/reference/code/rendering/mesh_template.py without kaolin.

`TriangleMesh` stands in for `kal.rep.TriangleMesh.from_obj(path, enable_adjacency=True)` (reference :18)
and carries the attributes the reference reads: vertices, faces, uvs, face_textures and the face-face
adjacency `ff` (kaolin's compute_adjacency_info, patched copy in rendering/monkey_patches.py:96-106).
`MeshTemplate` keeps the reference's attributes and methods (:12-237); its render call goes to the
libb3d rasteriser through rendering.renderer.Renderer.
"""
import math
import os

import numpy as np
import torch
import torch.nn.functional as F

from .utils import circpad, grid_sample_bilinear

SEGMENTS = 32


class TriangleMesh:
    def __init__(self, vertices, faces, uvs, face_textures):
        self.vertices, self.faces, self.uvs, self.face_textures = vertices, faces, uvs, face_textures
        self.ff = self.face_adjacency(faces)

    @classmethod
    def from_obj(cls, path, enable_adjacency=True):
        pos, tex, tri, tri_t = [], [], [], []
        with open(path) as fh:
            for line in fh:
                tok = line.split()
                if not tok or tok[0].startswith('#'):
                    continue
                if tok[0] == 'v':
                    pos.append([float(t) for t in tok[1:4]])
                elif tok[0] == 'vt':
                    tex.append([float(t) for t in tok[1:3]])
                elif tok[0] == 'f':
                    if len(tok) != 4:
                        raise ValueError(f"{path}: only triangle meshes are supported")
                    parts = [t.split('/') for t in tok[1:4]]
                    tri.append([int(p[0]) - 1 for p in parts])
                    tri_t.append([int(p[1]) - 1 if len(p) > 1 and p[1] else int(p[0]) - 1 for p in parts])
        return cls(torch.tensor(pos, dtype=torch.float32), torch.tensor(tri, dtype=torch.long),
                   torch.tensor(tex, dtype=torch.float32), torch.tensor(tri_t, dtype=torch.long))

    @staticmethod
    def face_adjacency(faces):
        """[F, max_neighbours] ids of the faces sharing an edge with each face, largest id first, -1 padded."""
        f = faces.cpu().numpy()
        n = f.shape[0]
        e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), axis=1)
        owner = np.tile(np.arange(n), 3)
        key = e[:, 0].astype(np.int64) * (f.max() + 1) + e[:, 1]
        order = np.argsort(key, kind='stable')
        key, owner = key[order], owner[order]
        groups = np.split(owner, np.nonzero(np.diff(key))[0] + 1)
        nb = [set() for _ in range(n)]
        for grp in groups:
            for a in grp:
                nb[a].update(int(b) for b in grp if b != a)
        width = max((len(s) for s in nb), default=0)
        out = np.full((n, width), -1, dtype=np.int64)
        for i, s in enumerate(nb):
            out[i, :len(s)] = sorted(s, reverse=True)
        return torch.from_numpy(out)

    def to(self, device):
        for k in ('vertices', 'faces', 'uvs', 'face_textures', 'ff'):
            setattr(self, k, getattr(self, k).to(device))
        return self

    def cuda(self):
        return self.to('cuda')


class MeshTemplate:
    def __init__(self, mesh_path, is_symmetric=True, device=None):
        if device is None:
            device = 'cuda' if torch.cuda.is_available() else 'cpu'
        mesh = TriangleMesh.from_obj(mesh_path, enable_adjacency=True)
        V = mesh.vertices
        north, south = int(V[:, 1].argmax()), int(V[:, 1].argmin())

        # mirror pairs across x = 0 (reference :24-47)
        tol = 1e-4
        neg = torch.nonzero(V[:, 0] < -tol).flatten()
        zero = torch.nonzero(V[:, 0].abs() < tol).flatten()
        mirrored = V[neg] * torch.tensor([-1.0, 1.0, 1.0])
        dist = (mirrored[:, None, :] - V[None, :, :]).norm(dim=-1)    # exact differences (cdist uses a GEMM identity)
        gap, pos = dist.min(dim=1)
        if len(neg) and float(gap.max()) >= tol:
            raise ValueError("mesh template is not symmetric about x = 0")
        if len(set(pos.tolist())) != len(pos):
            raise ValueError("mesh template has ambiguous mirror vertices")
        if len(pos) + len(neg) + len(zero) != len(V):
            raise ValueError("vertex partition into -x / +x / x=0 is incomplete")
        nonneg = torch.cat([pos, zero])

        # per-vertex position in the UV map = mean of its texture coordinates, seam wrapped (reference :52-73)
        rings = 31 if '31rings' in mesh_path else 16
        grid = np.array([SEGMENTS, rings], dtype=np.float64)
        samples = [[] for _ in range(len(V))]
        for tcs, vs in zip(mesh.face_textures.tolist(), mesh.faces.tolist()):
            for tc, v in zip(tcs, vs):
                cell = mesh.uvs[tc].numpy() * grid
                if math.isclose(cell[0], SEGMENTS, abs_tol=1e-4):
                    cell[0] = 0
                samples[v].append(cell)
        topo = torch.zeros(len(V), 2)
        for v, cells in enumerate(samples):
            if cells:
                topo[v] = torch.tensor(np.mean(np.array(cells, dtype=np.float32), axis=0) / grid, dtype=torch.float32)
        topo = (topo * 2 - 1) * torch.tensor([1.0, -1.0])

        sym_mask = torch.ones(1, len(V), 3)
        sym_mask[:, zero, 0] = 0          # vertices on the symmetry plane may not leave it

        # tangent frame per vertex: (normal, tangent, bitangent); undefined at the poles (reference :82-94)
        n = F.normalize(V, dim=1)
        t = F.normalize(torch.cross(n, torch.tensor([[0.0, 1.0, 0.0]]).expand_as(n), dim=1), dim=1)
        b = torch.cross(n, t, dim=1)
        for pole in (north, south):
            t[pole] = 0
            b[pole] = 0
        frames = torch.stack((n, t, b), dim=1)

        self.mesh = mesh.to(device)
        self.topo_map = topo.to(device)
        self.nonneg_topo_map = topo[nonneg].to(device)
        self.nonneg_indices = nonneg.to(device)
        self.neg_indices = neg.to(device)
        self.pos_indices = pos.to(device)
        self.symmetry_mask = sym_mask.to(device)
        self.tangent_map = frames.to(device)
        self.nonneg_tangent_map = frames[nonneg].to(device)
        self.is_symmetric = is_symmetric
        self._mirror_x = torch.tensor([-1.0, 1.0, 1.0], device=device)
        self._zero_indices = zero.to(device)
        self._records = {}          # (h, w, symmetric) -> per-vertex records of the fused CUDA vertex pipeline

    # ---- deformation ---------------------------------------------------------------------------------
    def deform(self, deltas):
        """Local (normal, tangent, bitangent) displacements -> object space (reference :106-111)."""
        frames = self.nonneg_tangent_map if self.is_symmetric else self.tangent_map
        return torch.einsum('bvk,vkc->bvc', deltas, frames)

    def compute_normals(self, vertex_positions):
        """Unit face normals of the deformed mesh (reference :113-123)."""
        f = self.mesh.faces
        if vertex_positions.is_cuda and vertex_positions.dtype == torch.float32:
            from b3d.mesh import face_normals                   # one launch each way (csrc/loss_kernels.cu)
            return face_normals(vertex_positions, f)
        a, b, c = vertex_positions[:, f[:, 0]], vertex_positions[:, f[:, 1]], vertex_positions[:, f[:, 2]]
        return F.normalize(torch.cross(b - a, c - a, dim=2), dim=2)

    def _symmetric_shift(self, width):
        # even symmetry puts the seam half a texel in: u -> (u + delta) / expansion
        return 1 / (2 * width), (width + 1) / width

    def _vertex_records(self, h, w):
        """Sampling sites of get_vertex_positions resolved once per map size for libb3d's fused vertex kernel: per vertex
        four texel offsets into the UNPADDED map (wrap-around / seam column folded in), bilinear weights, the tangent frame
        of the sampled vertex, the template position and the x factor (-1 mirrored, 0 on the symmetry plane, +1)."""
        key = (h, w, self.is_symmetric)
        hit = self._records.get(key)
        if hit is None:
            from b3d.vertex import pack_records
            V = self.topo_map.shape[0]
            if self.is_symmetric:
                delta, expansion = self._symmetric_shift(w)
                site = self.nonneg_topo_map.clone()
                site[:, 0] = (site[:, 0] + 1 + 2 * delta - expansion) / expansion
                nn_idx, neg, pos, zero = (t.cpu() for t in (self.nonneg_indices, self.neg_indices, self.pos_indices, self._zero_indices))
                src = torch.zeros(V, dtype=torch.long)              # row of `site` / nonneg frames each vertex samples
                src[nn_idx] = torch.arange(len(nn_idx))
                where = {int(v): i for i, v in enumerate(nn_idx.tolist())}
                src[neg] = torch.tensor([where[int(p)] for p in pos.tolist()], dtype=torch.long)
                sign = torch.ones(V)
                sign[neg], sign[zero] = -1.0, 0.0
                rec, sgn = pack_records(site.cpu()[src], w + 2, h, w, lambda xp: (xp - 1) % w,
                                        self.nonneg_tangent_map.cpu()[src], self.mesh.vertices.cpu(), sign)
            else:
                rec, sgn = pack_records(self.topo_map.cpu(), w + 1, h, w, lambda xp: xp % w, self.tangent_map.cpu(),
                                        self.mesh.vertices.cpu(), torch.ones(V))
            dev_ = self.mesh.vertices.device
            hit = self._records[key] = (rec.to(dev_), sgn.to(dev_))
        return hit

    def vertices_and_pose(self, displacement_map, scale=None, translation=None, rot=None, z0=None):
        """get_vertex_positions + transform_vertices (run_reconstruction.py:237-252) in ONE CUDA launch (and one for the
        backward): -> (raw [B,V,3] object-space vertices, vtx [B,V,3] camera-space vertices or None without a pose).
        scale [B,1] (already including any learned delta), translation [B,3], rot [B,4] unit quaternions, z0 [B,1]|None."""
        from b3d.vertex import vertex_pipeline
        rec, sgn = self._vertex_records(displacement_map.shape[2], displacement_map.shape[3])
        return vertex_pipeline(displacement_map, rec, sgn, self.topo_map.shape[0], scale, translation, rot, z0)

    def get_vertex_positions(self, displacement_map):
        """UV displacement map [B,3,h,w] -> vertex positions [B,V,3] (reference :125-149).  CUDA tensors take the fused
        kernel; the torch composition below is the same math for other devices."""
        if displacement_map.is_cuda and displacement_map.dtype == torch.float32 and not getattr(self, 'disable_fused_vertices', False):
            return self.vertices_and_pose(displacement_map)[0]
        B, w = displacement_map.shape[0], displacement_map.shape[3]
        _, padded = self.adjust_uv_and_texture(displacement_map)
        if self.is_symmetric:
            delta, expansion = self._symmetric_shift(w)
            site = self.nonneg_topo_map.clone()
            site[:, 0] = (site[:, 0] + 1 + 2 * delta - expansion) / expansion
        else:
            site = self.topo_map
        local = grid_sample_bilinear(padded, site[None, :, None, :].expand(B, -1, -1, -1))[..., 0].transpose(1, 2)
        moved = self.deform(local)
        if self.is_symmetric:
            full = moved.new_zeros(B, self.topo_map.shape[0], 3)
            full[:, self.nonneg_indices] = moved
            full[:, self.neg_indices] = full[:, self.pos_indices] * self._mirror_x.to(moved.dtype)
            moved = full * self.symmetry_mask
        return self.mesh.vertices.unsqueeze(0) + moved

    def adjust_uv_and_texture(self, texture, return_texture=True):
        """Template UVs + the texture prepared for lookups across the seam (reference :151-170)."""
        B, w = texture.shape[0], texture.shape[3]
        if self.is_symmetric:
            delta, expansion = self._symmetric_shift(w)
            uvs = self.mesh.uvs.clone()
            uvs[:, 0] = (uvs[:, 0] + delta) / expansion
            return uvs.expand(B, -1, -1), circpad(texture, 1)
        return self.mesh.uvs.expand(B, -1, -1), torch.cat((texture, texture[..., :1]), dim=3)

    def forward_renderer(self, renderer, vertex_positions, texture, num_gpus=1, **kwargs):
        """Render the deformed, textured template (reference :172-186) -> (image B×H×W×3, alpha B×H×W×1)."""
        faces, face_tex = self.mesh.faces, self.mesh.face_textures
        if num_gpus > 1:      # nn.DataParallel scatter compatibility of the reference
            faces, face_tex = faces.repeat(num_gpus, 1), face_tex.repeat(num_gpus, 1)
        uvs, tex = self.adjust_uv_and_texture(texture)
        image, alpha, _ = renderer(points=[vertex_positions, faces], uv_bxpx2=uvs, texture_bx3xthxtw=tex,
                                   ft_fx3=face_tex, **kwargs)
        return image, alpha

    def export_obj(self, path_prefix, vertex_positions, texture):
        """Write <prefix>.obj/.mtl (+ .png when imageio is installed) — reference :188-219."""
        if vertex_positions.dim() != 2:
            raise ValueError("export_obj takes one mesh: vertex_positions [V,3]")
        name = os.path.basename(path_prefix)
        with open(path_prefix + '.obj', 'w') as fh:
            fh.write(f'mtllib {name}.mtl\n')
            fh.writelines('v {:.5f} {:.5f} {:.5f}\n'.format(*v) for v in vertex_positions.tolist())
            fh.writelines('vt {:.5f} {:.5f}\n'.format(*t) for t in self.mesh.uvs.tolist())
            fh.write(f'usemtl {name}\n')
            for f, t in zip(self.mesh.faces.tolist(), self.mesh.face_textures.tolist()):
                fh.write('f ' + ' '.join(f'{a + 1}/{b + 1}' for a, b in zip(f, t)) + '\n')
        with open(path_prefix + '.mtl', 'w') as fh:
            fh.write(f'newmtl {name}\nKa 1.000 1.000 1.000\nKd 1.000 1.000 1.000\nKs 0.000 0.000 0.000\n'
                     f'd 1.0\nillum 1\nmap_Ka {name}.png\nmap_Kd {name}.png\n')
        try:
            import imageio
        except ImportError:
            return
        imageio.imwrite(path_prefix + '.png', (texture.permute(1, 2, 0) * 255).clamp(0, 255).byte().cpu().numpy())
