"""Textured 3-D models of photos from a trained reconstruction network: for every image, an OBJ mesh with its texture and
a sheet of renders.

Per batch, on the GPU:
    pred_tex, mesh_map = generator(X_256)                         eval mode
    raw, vtx = vertices_and_pose(mesh_map, scale, t, rot, z0)     training split: DatasetParams[ind] (as the pseudo-GT
                                                                  export); validation split: the dataset means (as the
                                                                  validation pass); photos without a pose: raw only
  with a pose:
    unshaded render at renderer_resolution(R), texel visibility   as the pseudo-ground-truth export
    the high-resolution photo projected into UV space at R        rendering.inverse_renderer.InverseRenderer
  texture bytes and per-texel source                              b3d_recon_texture_pack: the projection where the
                                                                  pseudo-GT mask keeps it, its mirror image (symmetric
                                                                  template), else pred_tex resampled to R
  B x 8 turntable views (+ B views at the input pose), one render at 512^2 with the exported texture, pooled to 256^2
  tiles by b3d_sample_pack; everything into one device staging buffer (staging.Staging)
then on the host, for every image:
    <name>.obj / .mtl / .png      rendering.mesh_template.ObjWriter, vertices with Y and Z swapped (Y up), as the sample
                                  export writes them
    <name>_views.png              512 x 1280: column 0 the input crop over the render at the input pose (white without
                                  one), columns 1-4 the eight turntable views in two rows"""
import os

import numpy as np
import torch
from PIL import Image

import b3d
from b3d.data import recon_texture_pack, sample_pack
from b3d.mesh import render_indices, texel_visibility
from pseudo_gt_export import renderer_resolution, resize_texture
from reconstruction_training import turntable_rotations, turntable_vertices
from rendering.inverse_renderer import InverseRenderer
from rendering.mesh_template import ObjWriter
from rendering.renderer import Renderer
from staging import Staging, byte_layout, views

VIEW_RES = 512            # render side of the views; their tiles are half of it
TILE = VIEW_RES // 2
TURNTABLE = 8
SOURCES = ('predicted', 'projected', 'mirrored')


def input_tile_bytes(X):
    """The network input X [B,4,TILE,TILE] (masked image in [-1, 1], mask) as uint8 [B,TILE,TILE,3]: background white,
    x / 2 + 0.5, * 255, clamp, truncation (the bytes of b3d_sample_pack's tiles)."""
    img = torch.where(X[:, 3:] > 0, X[:, :3], torch.ones_like(X[:, :3]))
    return ((img / 2 + 0.5) * 255).clamp(0, 255).byte().permute(0, 2, 3, 1)


def views_sheet(input_tile, posed_tile, turntable):
    """uint8 [2 TILE, 5 TILE, 3]: column 0 input_tile over posed_tile (None: white), columns 1-4 the eight turntable
    tiles [8,TILE,TILE,3] in rows of four."""
    t = input_tile.shape[0]
    sheet = np.full((2 * t, 5 * t, 3), 255, np.uint8)
    sheet[:t, :t] = input_tile
    if posed_tile is not None:
        sheet[t:, :t] = posed_tile
    for k in range(TURNTABLE):
        r, c = divmod(k, 4)
        sheet[r * t:(r + 1) * t, (c + 1) * t:(c + 2) * t] = turntable[k]
    return sheet


def write_views(path, sheet):
    Image.fromarray(sheet).save(path)


class ReconstructionExporter:
    """trainer: a ReconTrainer after load_checkpoint(path, 'evaluate'), or any object with its `generator`,
    `dataset_params` and `args` (optimize_deltas, optimize_z0); mesh_template: rendering.mesh_template.MeshTemplate;
    export_resolution: the side R of the exported textures (even).  CUDA only."""

    def __init__(self, trainer, mesh_template, export_resolution=512):
        if not torch.cuda.is_available():
            raise b3d.B3DError('ReconstructionExporter: the export runs on CUDA kernels and needs a CUDA device; there '
                               'is no CPU fallback')
        self.device = next(trainer.generator.parameters()).device
        if self.device.type != 'cuda':
            raise b3d.B3DError(f'ReconstructionExporter: the network is on {self.device}; move it to a CUDA device')
        self.R = int(export_resolution)
        if self.R < 2 or self.R % 2:
            raise ValueError(f'ReconstructionExporter: export_resolution {self.R} must be even and at least 2')
        self.trainer, self.tpl = trainer, mesh_template
        self.renderer_res = renderer_resolution(self.R)
        self.inverse_renderer = InverseRenderer(mesh_template.mesh, self.R, self.R)
        self.view_renderer = Renderer(VIEW_RES, VIEW_RES)
        self.obj = ObjWriter(mesh_template.mesh)
        self.turntable = turntable_rotations(self.device)

    # ------------------------------------------------------------------------------------------------ one batch
    def _pose(self, mesh_map, scale, translation, rot, ind, per_index):
        """(raw, vtx): per_index poses with DatasetParams[ind] (PseudoGTExporter._pose), else with the dataset means
        (ReconTrainer.evaluate)."""
        a, dp = self.trainer.args, self.trainer.dataset_params
        B, z0 = mesh_map.shape[0], None
        sel = ind if per_index else None
        if a.optimize_deltas:
            translation_delta, scale_delta = dp(sel, 'deltas')
            scale, translation = scale + scale_delta, translation + translation_delta
        if a.optimize_z0:
            z0 = dp(sel, 'z0').expand(B, 1)
        return self.tpl.vertices_and_pose(mesh_map, scale, translation, rot, z0)

    def _projection(self, vtx, pred_tex, hd):
        """Texel visibility of the posed mesh and the photo projected into UV space (the pseudo-GT export's steps)."""
        tex_r = resize_texture(pred_tex, self.renderer_res)
        uvs, padded = self.tpl.adjust_uv_and_texture(tex_r)
        H = self.renderer_res
        imidx, imwei, fuv = render_indices(vtx, self.tpl.mesh.faces, uvs, self.tpl.mesh.face_textures, H, H)
        vis = texel_visibility(imidx, imwei, fuv, padded.shape[2], padded.shape[3], self.tpl.is_symmetric)
        proj, alpha = self.inverse_renderer(vtx, hd)
        return vis, proj.contiguous(), alpha.contiguous()

    def _no_projection(self, B):
        """Inputs of the pack that select no projected texel (every texel from pred_tex)."""
        if getattr(self, '_empty', None) is None or self._empty[1].shape[0] < B:
            R, d = self.R, self.device
            self._empty = (torch.zeros(B, 1, 1, dtype=torch.uint8, device=d), torch.zeros(B, R, R, 3, device=d),
                           torch.zeros(B, R, R, 1, device=d))
        return tuple(t[:B] for t in self._empty)

    @torch.no_grad()
    def _device_batch(self, batch, posed, per_index):
        if posed:
            X, hd, scale, translation, rot, ind = (t.to(self.device) for t in batch)
        else:
            X, ind = batch[0].to(self.device), batch[-1].to(self.device)
        ind = ind.reshape(-1)
        B = X.shape[0]
        if tuple(X.shape[1:]) != (4, TILE, TILE):
            raise ValueError(f'export: the network input is {tuple(X.shape[1:])}; expected (4, {TILE}, {TILE})')
        pred_tex, mesh_map = self.trainer.generator(X)
        if posed:
            raw, vtx = self._pose(mesh_map, scale, translation, rot, ind, per_index)
            vis, proj, alpha = self._projection(vtx, pred_tex, hd)
        else:
            raw, vtx = self.tpl.vertices_and_pose(mesh_map)[0], None
            vis, proj, alpha = self._no_projection(B)
        R, V = self.R, raw.shape[1]
        nv = TURNTABLE + (1 if posed else 0)
        lay, nbytes = byte_layout((('vertices', torch.float32, (B, V, 3)), ('tex8', torch.uint8, (B, R, R, 3)),
                                   ('src8', torch.uint8, (B, R, R)), ('views', torch.uint8, (B * nv, TILE, TILE, 3)),
                                   ('input', torch.uint8, (B, TILE, TILE, 3)), ('ind', torch.int64, (B,))))
        v = views(self._staging.device_buffer(nbytes, B), lay)
        recon_texture_pack(vis, proj, alpha, pred_tex.contiguous(), self.tpl.is_symmetric, v['tex8'], v['src8'])

        # the views show the exported texture: its bytes back in [-1, 1]
        tex = v['tex8'].permute(0, 3, 1, 2).float() * (2 / 255) - 1
        rot = self.turntable.repeat(B, 1)
        vtx_views = turntable_vertices(rot, raw.repeat_interleave(TURNTABLE, 0))
        tex_views = tex.repeat_interleave(TURNTABLE, 0)
        if posed:
            vtx_views, tex_views = torch.cat((vtx_views, vtx)), torch.cat((tex_views, tex))
        image, _ = self.tpl.forward_renderer(self.view_renderer, vtx_views.contiguous(), tex_views.contiguous())
        n = image.shape[0]
        # b3d_sample_pack also quantises a texture; a 1 x 1 one keeps that part to one texel per view
        sample_pack(image, self.view_renderer.last_face_index, torch.zeros(n, 3, 1, 1, device=self.device), v['views'],
                    torch.empty(n, 1, 1, 3, dtype=torch.uint8, device=self.device))
        v['input'].copy_(input_tile_bytes(X))
        v['vertices'].copy_(raw[..., [0, 2, 1]])               # Y and Z swapped (Y up), as the sample export
        v['ind'].copy_(ind)
        return lay, nbytes

    # ------------------------------------------------------------------------------------------------ the loop
    def export(self, batches, names, out_dir, posed=True, writers=8, per_index=False):
        """batches: with posed, the eval batches (X_256, img_hd, scale, translation, rot, ind) of a CMR dataset with
        img_size [256, renderer_resolution(R)]; without, batches (X_256, ..., ind) whose pose is not used (PhotoFolder's
        eval_batches).  names: per-index output names (names[ind]); out_dir: where the files go; per_index: pose with the
        per-image DatasetParams (images of the training split), else with their means; writers: threads that compress
        and write the files.  Every batch but the last must have the first batch's size.
        -> dict(names: the names written, in batch order; sources: int64 [N,3] texels per source (predicted, projected,
        mirrored) of each)."""
        self.trainer.generator.eval()
        os.makedirs(out_dir, exist_ok=True)
        self._staging = Staging(self.device, 'reconstruction export')
        written, counts = [], []

        def device_batch(batch):
            lay, nbytes = self._device_batch(batch, posed, per_index)
            return lay, nbytes, 2 * lay['ind'][2][0]

        def drain(host, lay, submit):
            """Host side of one staged batch: the source counts, then two writes per image."""
            v = views(host, lay)
            ind = v['ind'].tolist()
            tiles = v['views'].numpy()                     # B x 8 turntable views, then B views at the input pose
            turntable = tiles[:TURNTABLE * len(ind)].reshape(len(ind), TURNTABLE, TILE, TILE, 3)
            for i, idx in enumerate(ind):
                name = names[idx]
                prefix = os.path.join(out_dir, name)
                written.append(name)
                counts.append(np.bincount(v['src8'][i].numpy().reshape(-1), minlength=3)[:3])
                submit(self.obj.write, prefix, v['vertices'][i].numpy().copy(), v['tex8'][i].numpy().copy())
                sheet = views_sheet(v['input'][i].numpy(), tiles[TURNTABLE * len(ind) + i] if posed else None,
                                    turntable[i])
                submit(write_views, prefix + '_views.png', sheet)

        self._staging.run(batches, device_batch, drain, writers)
        if not written:
            raise ValueError('export: no batches')
        return dict(names=written, sources=np.stack(counts).astype(np.int64))
