"""The sample export of the reference's main.py (`--save_results`, :836-897) as an importable class: textured meshes and
one anti-aliased render grid from a trained generator.

    indices = np.random.choice(len(ds), N, replace=False); classes ds.classes[i] (conditional generators);
    truncated noise                                             the reference's draws, in its order, once for all N
    per batch of B, on the GPU:
      pred_tex, mesh_map = generator(noise, c)                  eval mode
      raw, vtx = vertices_and_pose(mesh_map, scale, t, rot)     ONE launch: object-space and posed ([1, -1, -1]) vertices
      render at 512^2                                           MeshTemplate.forward_renderer, Renderer(512, 512)
      tiles and texture bytes                                   b3d_sample_pack, into one device staging buffer
      raw vertices with Y and Z swapped                         into the same buffer
    one copy to a pinned host slot per batch (staging.Staging), files written by a thread pool:
      out_dir/mesh_{i}.obj / .mtl / .png                        rendering.mesh_template.ObjWriter
      grid_path                                                 the 256^2 tiles as make_grid(nrow=8, padding=0) places them

Exporting N samples in batches of B writes the files the reference writes for `--batch_size N`.  The generator sees
batches of B instead of N, which changes nothing for a generator whose output for a sample depends only on its own noise
and class (the running-average generator in eval mode)."""
import math
import os

import numpy as np
import torch
from PIL import Image

import b3d
from b3d.data import sample_pack
from fid_evaluation import truncated_noise
from rendering.mesh_template import ObjWriter
from rendering.renderer import Renderer
from staging import Staging, byte_layout, views

RENDER_RES = 512          # main.py:158, "For exporting images: higher resolution"
GRID_COLUMNS = 8          # make_grid(nrow=8)


def grid_shape(n, tile_h, tile_w, nrow=GRID_COLUMNS, padding=0):
    """torchvision.utils.make_grid's layout: min(nrow, n) columns, ceil(n / columns) rows, `padding` pixels before every
    row and column and after the last ones."""
    cols = min(nrow, n)
    rows = math.ceil(n / cols)
    return (rows * (tile_h + padding) + padding, cols * (tile_w + padding) + padding, 3), cols


def place_tiles(grid, cols, k0, tiles, padding=0):
    """Tiles k0, k0 + 1, ... ([k, h, w, 3], numpy or torch like grid) into their grid cells, row-major over `cols`
    columns."""
    h, w = tiles.shape[1], tiles.shape[2]
    for i in range(tiles.shape[0]):
        r, c = divmod(k0 + i, cols)
        y, x = r * (h + padding) + padding, c * (w + padding) + padding
        grid[y:y + h, x:x + w] = tiles[i]


def assemble_grid(tiles, nrow=GRID_COLUMNS):
    """uint8 tiles [N,h,w,3] -> the grid image [rows*h, cols*w, 3]; cells after the last tile stay 0."""
    shape, cols = grid_shape(tiles.shape[0], tiles.shape[1], tiles.shape[2], nrow)
    grid = np.zeros(shape, dtype=np.uint8)
    place_tiles(grid, cols, 0, tiles)
    return grid


def sample_draws(ds, num_samples, latent_dim, sigma, conditional, seed=None):
    """main.py:839-863 for --batch_size num_samples: (indices int64 [N] numpy, classes int64 [N,K] or None, noise fp32
    [N,latent_dim]).  classes are ds.classes[i] when the generator is conditional.  seed: a RandomState and a CPU
    torch.Generator seeded with it, the streams of np.random.seed(seed) / torch.manual_seed(seed); None draws from the
    global generators, as the reference does.  More samples than len(ds) raise, as np.random.choice does."""
    rng = np.random.RandomState(seed) if seed is not None else np.random
    gen = torch.Generator().manual_seed(seed) if seed is not None else None
    indices = rng.choice(len(ds), size=num_samples, replace=False)
    classes = None
    if conditional:
        classes = torch.as_tensor(np.stack([np.asarray(ds.classes[i]) for i in indices]), dtype=torch.int64)
    noise = truncated_noise(num_samples, latent_dim, sigma, gen)
    return indices, classes, noise


def write_png(path, pixels):
    Image.fromarray(pixels).save(path)


class SampleExporter:
    """generator: the running-average Generator (models.gan) with a mesh head, called as generator(noise, c, None,
    return_attention=True), e.g. GANTrainer.trainer.generator_running_avg after load_checkpoint(path, 'evaluate');
    mesh_template: rendering.mesh_template.MeshTemplate; dataset: a data.abstract_dataset.AbstractDataset (its poses
    `data['scale' | 'translation' | 'rotation']` and, for a conditional generator, `classes`); truncation_sigma: the
    noise truncation (ds.suggest_truncation_sigma() is the reference's default).  CUDA only."""

    def __init__(self, generator, mesh_template, dataset, truncation_sigma, latent_dim=64):
        if not getattr(generator, 'mesh_head', True):
            raise ValueError('SampleExporter: the generator has no mesh head (texture_only); there is no mesh to export')
        if not torch.cuda.is_available():
            raise b3d.B3DError('SampleExporter: the export runs on CUDA kernels and needs a CUDA device; there is no CPU '
                               'fallback')
        self.device = next(generator.parameters()).device
        if self.device.type != 'cuda':
            raise b3d.B3DError(f'SampleExporter: the network is on {self.device}; move it to a CUDA device')
        self.generator, self.tpl, self.ds = generator, mesh_template, dataset
        self.sigma, self.latent_dim = truncation_sigma, int(latent_dim)
        args = getattr(generator, 'args', None)
        self.conditional = bool(getattr(args, 'conditional_class', False))
        self.renderer = Renderer(RENDER_RES, RENDER_RES)
        self.obj = ObjWriter(mesh_template.mesh)

    # ------------------------------------------------------------------------------------------------ one batch
    @torch.no_grad()
    def _device_batch(self, noise, c, scale, translation, rotation):
        """GPU work of one batch (every input already on the device): fills the staging buffer, returns its layout."""
        B = noise.shape[0]
        pred_tex, mesh_map, _ = self.generator(noise, c, None, return_attention=True)
        raw, vtx = self.tpl.vertices_and_pose(mesh_map, scale, translation, rotation)
        image, _ = self.tpl.forward_renderer(self.renderer, vtx, pred_tex)
        T, V = pred_tex.shape[2], raw.shape[1]
        H, W = image.shape[1], image.shape[2]
        lay, nbytes = byte_layout((('tiles', torch.uint8, (B, H // 2, W // 2, 3)), ('tex8', torch.uint8, (B, T, T, 3)),
                                   ('vertices', torch.float32, (B, V, 3))))
        v = views(self._staging.device_buffer(nbytes, B), lay)
        sample_pack(image, self.renderer.last_face_index, pred_tex.contiguous(), v['tiles'], v['tex8'])
        v['vertices'].copy_(raw[..., [0, 2, 1]])              # main.py:870, Y and Z swapped (Y up)
        return lay, nbytes

    # ------------------------------------------------------------------------------------------------ the loop
    def export(self, out_dir, grid_path, num_samples, batch_size, seed=None, writers=8):
        """Writes out_dir/mesh_{i}.obj / .mtl / .png for i < num_samples and the render grid at grid_path, in batches of
        batch_size (the last one may be smaller).  seed: see sample_draws().  writers: threads that compress and write the files.
        -> dict(indices, noise, classes, grid_shape)."""
        num_samples, batch_size = int(num_samples), int(batch_size)
        if num_samples < 1 or batch_size < 1:
            raise ValueError(f'export: num_samples {num_samples} and batch_size {batch_size} must be positive')
        indices, classes, noise = sample_draws(self.ds, num_samples, self.latent_dim, self.sigma, self.conditional, seed)
        d = self.device
        sel = torch.as_tensor(indices, dtype=torch.int64)
        # every draw and pose goes to the device once, so that no batch waits on a host-to-device copy
        scale = self.ds.data['scale'][sel].reshape(-1, 1).float().to(d)
        translation = self.ds.data['translation'][sel].float().to(d)
        rotation = self.ds.data['rotation'][sel].float().to(d)
        noise_d = noise.to(d)
        classes_d = classes.to(d) if classes is not None else None
        os.makedirs(out_dir, exist_ok=True)
        grid, cols = None, None
        self.generator.eval()
        self._staging = Staging(d, 'sample export')

        def device_batch(k0):
            s = slice(k0, min(k0 + batch_size, num_samples))
            lay, nbytes = self._device_batch(noise_d[s], classes_d[s] if classes_d is not None else None, scale[s],
                                             translation[s], rotation[s])
            return (k0, lay), nbytes, lay['tex8'][2][0]

        def drain(host, meta, submit):
            """Host side of one staged batch: the tiles into the grid, one write per sample."""
            nonlocal grid, cols
            k0, lay = meta
            v = views(host, lay)
            tiles = v['tiles'].numpy()
            if grid is None:
                shape, cols = grid_shape(num_samples, tiles.shape[1], tiles.shape[2])
                grid = np.zeros(shape, dtype=np.uint8)
            place_tiles(grid, cols, k0, tiles)
            for i in range(tiles.shape[0]):
                submit(self.obj.write, os.path.join(out_dir, f'mesh_{k0 + i}'), v['vertices'][i].numpy().copy(),
                       v['tex8'][i].numpy().copy())

        self._staging.run(range(0, num_samples, batch_size), device_batch, drain, writers)
        grid_dir = os.path.dirname(grid_path)
        if grid_dir:
            os.makedirs(grid_dir, exist_ok=True)
        write_png(grid_path, grid)
        return dict(indices=indices, noise=noise, classes=classes, grid_shape=grid.shape)
