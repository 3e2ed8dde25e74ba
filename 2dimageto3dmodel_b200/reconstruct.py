"""Command line of the reconstruction export: textured 3-D models of photos from a trained reconstruction checkpoint.

    python reconstruct.py --name <name> --dataset cub|p3d [--split train|testval|val] [--indices i ...] [--num_images N]
    python reconstruct.py --name <name> --dataset cub --photos DIR

Reads checkpoints_recon/<name>/checkpoint_<which_epoch>.pth (run_reconstruction.py's) and writes, for every image,
<name>.obj / .mtl / .png and <name>_views.png under --output (default results_recon/<name>).  Dataset images are posed
with their SfM annotation and textured from the photo where the mesh sees it; photos from a folder (RGBA PNGs, or images
with a <stem>_mask.png) have no pose and take the network's texture.  Run it from the directory that holds
checkpoints_recon/, datasets/ and mesh_templates/.  The model-shape flags must match the training run's.  `main()` parses
sys.argv (or argv) and runs; importing does nothing."""
import argparse
import os
import re

SPLITS = {'cub': ('train', 'testval'), 'p3d': ('train', 'val')}
NETWORK_RES = 256


def build_parser():
    p = argparse.ArgumentParser(description='Export textured OBJ meshes of photos from a reconstruction checkpoint.')
    p.add_argument('--name', type=str, required=True)
    p.add_argument('--dataset', type=str, required=True, help='(p3d|cub)')
    p.add_argument('--mesh_path', type=str, default='autodetect')
    p.add_argument('--symmetric', type=bool, default=True)
    p.add_argument('--texture_resolution', type=int, default=128)
    p.add_argument('--mesh_resolution', type=int, default=32)
    p.add_argument('--optimize_deltas', type=bool, default=True)
    p.add_argument('--optimize_z0', action='store_true')
    p.add_argument('--which_epoch', type=str, default='latest')
    p.add_argument('--split', type=str, default=None,
                   help='dataset split to export (cub: train|testval, p3d: train|val; default the validation split)')
    p.add_argument('--indices', type=int, nargs='+', default=None, help='export only these images of the split / folder')
    p.add_argument('--num_images', type=int, default=None, help='export only the first N images')
    p.add_argument('--photos', type=str, default=None, help='export a folder of photos instead of a dataset split')
    p.add_argument('--export_resolution', type=int, default=512)
    p.add_argument('--batch_size', type=int, default=16)
    p.add_argument('--writers', type=int, default=8)
    p.add_argument('--output', type=str, default=None, help='default: results_recon/<name>')
    return p


def parse_args(argv=None):
    """Parsed and checked flags: --split defaults to the dataset's validation split, --mesh_path autodetect resolves,
    --output defaults to results_recon/<name>.  Inconsistent flags exit with argparse's usage error."""
    from run_reconstruction import MESH_PATHS
    p = build_parser()
    args = p.parse_args(argv)
    if args.dataset not in SPLITS:
        p.error(f"--dataset {args.dataset}: expected 'cub' or 'p3d'")
    if args.photos is not None:
        if args.split is not None:
            p.error('--split selects dataset images; --photos exports a folder instead')
        if not os.path.isdir(args.photos):
            p.error(f'--photos {args.photos}: not a directory')
    else:
        if args.split is None:
            args.split = SPLITS[args.dataset][1]
        if args.split not in SPLITS[args.dataset]:
            p.error(f"--split {args.split}: {args.dataset} has {' and '.join(SPLITS[args.dataset])}")
    if args.export_resolution < 2 or args.export_resolution % 2:
        p.error(f'--export_resolution {args.export_resolution}: must be even and at least 2')
    for flag in ('batch_size', 'writers', 'num_images'):
        value = getattr(args, flag)
        if value is not None and value < 1:
            p.error(f'--{flag} {value}: must be positive')
    if args.indices is not None and min(args.indices) < 0:
        p.error(f'--indices: {min(args.indices)} is negative')
    if args.mesh_path == 'autodetect':
        args.mesh_path = MESH_PATHS[args.dataset]
    if args.output is None:
        args.output = os.path.join('results_recon', args.name)
    return args


def output_name(path):
    """A dataset image's relative path as a file name: directories joined with '_', the extension dropped."""
    stem = os.path.splitext(path.replace('\\', '/'))[0]
    return re.sub(r'[^\w.-]+', '_', stem.replace('/', '_'))


def select(n, indices, num_images):
    """The item indices to export out of n: --indices (in the order given) or all, then the first --num_images."""
    sel = list(range(n)) if indices is None else list(indices)
    bad = [i for i in sel if not 0 <= i < n]
    if bad:
        raise SystemExit(f'error: --indices {bad[0]} outside the {n} images')
    return sel[:num_images] if num_images is not None else sel


def checkpoint_dataset_size(chk):
    """Rows of the checkpoint's DatasetParams (the training split's size), 1 without them."""
    dp = chk.get('dataset_params')
    return next(iter(dp.values())).shape[0] if dp else 1


def batches_of(ds, sel, batch_size, device):
    """Device batches of items sel, in order: one b3d_image_batch launch each."""
    import torch
    idx = torch.tensor(sel, dtype=torch.int32, device=device)
    for a in range(0, len(sel), batch_size):
        yield ds.gather(idx[a:a + batch_size])


def run(args, root=''):
    """Loads the checkpoint and the images and exports them.  -> ReconstructionExporter.export's dict."""
    import torch
    import checkpoint_io
    from pseudo_gt_export import renderer_resolution
    from reconstruction_export import ReconstructionExporter
    from reconstruction_training import ReconTrainer, default_args
    from rendering.mesh_template import MeshTemplate

    if not torch.cuda.is_available():
        raise SystemExit('error: the reconstruction export runs on CUDA kernels and needs a CUDA device')
    device = torch.device('cuda', torch.cuda.current_device())
    path = os.path.join(root, 'checkpoints_recon', args.name, f'checkpoint_{args.which_epoch}.pth')
    if not os.path.exists(path):
        raise SystemExit(f'error: {path} does not exist')
    opts = default_args(symmetric=args.symmetric, texture_resolution=args.texture_resolution,
                        mesh_resolution=args.mesh_resolution, optimize_deltas=args.optimize_deltas,
                        optimize_z0=args.optimize_z0)
    tpl = MeshTemplate(os.path.join(root, args.mesh_path), is_symmetric=args.symmetric, device=device)
    rec = ReconTrainer(opts, tpl, checkpoint_dataset_size(checkpoint_io.load(path, 'cpu')), device=device)
    rec.load_checkpoint(path, 'evaluate')
    print(f'Exporting epoch {rec.epoch} of {args.name}')

    if args.photos is not None:
        from cmr_data.photos import PhotoFolder
        ds = PhotoFolder(args.photos, NETWORK_RES)
        names, posed = ds.names, False
    else:
        size = [NETWORK_RES, renderer_resolution(args.export_resolution)]
        if args.dataset == 'cub':
            from cmr_data.cub import CUBDataset
            ds = CUBDataset(args.split, False, size, root=root)
        else:
            from cmr_data.p3d import P3dDataset
            ds = P3dDataset(args.split, False, size, root=root)
        names, posed = [output_name(p) for p in ds.get_paths()], True
    sel = select(len(ds), args.indices, args.num_images)
    ds.to_device(device)
    exp = ReconstructionExporter(rec, tpl, args.export_resolution)
    out = exp.export(batches_of(ds, sel, args.batch_size, device), names, args.output, posed=posed,
                     writers=args.writers, per_index=posed and args.split == 'train')
    src = out['sources'].sum(axis=0)
    print(f"Wrote {len(out['names'])} models to {args.output} (texels: {src[1]} projected, {src[2]} mirrored, "
          f"{src[0]} predicted)")
    return out


def main(argv=None):
    return run(parse_args(argv))


if __name__ == '__main__':
    main()
