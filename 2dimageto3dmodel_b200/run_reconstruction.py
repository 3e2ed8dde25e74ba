"""Command line of the reconstruction stage, with the flags, files and log lines of the reference's run_reconstruction.py:

    python run_reconstruction.py --name <name> --dataset cub|p3d [...]         train (--continue_train resumes)
    python run_reconstruction.py --name <name> --dataset cub --evaluate        '[TEST]' line on the validation split
    python run_reconstruction.py --name <name> --dataset cub --generate_pseudogt   the GAN stage's data into cache/<dataset>

Run it from the directory that holds cache/, datasets/ and mesh_templates/.  Each mode calls the existing classes:
CUBDataset / P3dDataset (device batches), ReconTrainer and PseudoGTExporter.  Several GPUs: one process per GPU under
torchrun.  `main()` parses sys.argv (or argv) and runs; importing does nothing."""
import argparse
import os
import sys
import time

SCRIPT = 'run_reconstruction.py'
# validation images shown in TensorBoard (run_reconstruction.py:161, :172)
DEBUG_IDS = {'p3d': [6, 9, 16, 23, 34, 39, 40, 54, 60, 61, 64, 66, 67, 75, 77, 84],
             'cub': [0, 1, 12, 18, 20, 42, 72, 100, 101, 115, 123, 125, 142, 158, 188, 203]}
INCEPTION_RES = 299
# --mesh_path autodetect (run_reconstruction.py:70-76)
MESH_PATHS = {'p3d': 'mesh_templates/uvsphere_31rings.obj', 'cub': 'mesh_templates/uvsphere_16rings.obj'}


def build_parser():
    p = argparse.ArgumentParser()
    p.add_argument('--name', type=str, required=True)
    p.add_argument('--dataset', type=str, required=True, help='(p3d|cub)')
    p.add_argument('--mesh_path', type=str, default='autodetect')
    p.add_argument('--batch_size', type=int, default=50)
    p.add_argument('--image_resolution', type=int, default=256)
    p.add_argument('--symmetric', type=bool, default=True)
    p.add_argument('--texture_resolution', type=int, default=128)
    p.add_argument('--mesh_resolution', type=int, default=32)
    p.add_argument('--loss', type=str, default='mse', help='(mse|l1)')
    p.add_argument('--checkpoint_freq', type=int, default=100)
    p.add_argument('--evaluate_freq', type=int, default=10)
    p.add_argument('--save_freq', type=int, default=10)
    p.add_argument('--tensorboard', action='store_true')
    p.add_argument('--image_freq', type=int, default=10)
    p.add_argument('--no_augmentation', action='store_true')
    p.add_argument('--optimize_deltas', type=bool, default=True)
    p.add_argument('--optimize_z0', action='store_true')
    p.add_argument('--generate_pseudogt', action='store_true')
    p.add_argument('--pseudogt_resolution', type=int, default=512)
    p.add_argument('--evaluate', action='store_true')
    p.add_argument('--continue_train', action='store_true')
    p.add_argument('--which_epoch', type=str, default='latest')
    p.add_argument('--mesh_regularization', type=float, default=0.00005)
    p.add_argument('--epochs', type=int, default=1000)
    p.add_argument('--lr', type=float, default=0.0001)
    p.add_argument('--lr_dataset', type=float, default=0.0001)
    p.add_argument('--lr_decay_every', type=int, default=250)
    p.add_argument('--num_workers', type=int, default=4, help='accepted; the device data path has no loader workers')
    return p


def derive_settings(args):
    """run_reconstruction.py:70-86, :139-148: the autodetected mesh template, the render resolution, the loaders'
    resolutions and whether the training split is augmented.  -> dict(renderer_res, train_res, val_res, is_train)."""
    if args.mesh_path == 'autodetect':
        if args.dataset not in ('cub', 'p3d'):
            raise ValueError('Invalid dataset')
        args.mesh_path = MESH_PATHS[args.dataset]
        print('Using autodetected mesh', args.mesh_path)
    if args.generate_pseudogt:
        renderer_res = max(1024, 2 * args.pseudogt_resolution)
        train_res, val_res = [args.image_resolution, INCEPTION_RES, renderer_res], INCEPTION_RES
    else:
        renderer_res = args.image_resolution
        train_res = val_res = args.image_resolution
    return dict(renderer_res=renderer_res, train_res=train_res, val_res=val_res,
                is_train=not (args.no_augmentation or args.evaluate or args.generate_pseudogt))


def make_datasets(args, s, root=''):
    """:149-175: (training split, validation split or None: P3D has none while exporting pseudo-ground-truth)."""
    if args.dataset == 'p3d':
        from cmr_data.p3d import P3dDataset
        train = P3dDataset('train', s['is_train'], s['train_res'], root=root)
        return train, (None if args.generate_pseudogt else P3dDataset('val', False, s['val_res'], root=root))
    if args.dataset == 'cub':
        from cmr_data.cub import CUBDataset
        return CUBDataset('train', s['is_train'], s['train_res'], root=root), CUBDataset('testval', False, s['val_res'], root=root)
    raise ValueError('Invalid dataset')


def evaluate_all(args, rec, val, batch, log, writer, it, rank, world):
    """evaluate_all (:255-319): the '[TEST]' line, and with a writer the validation scalars and images."""
    import command_line as cl
    import torch
    from data.abstract_dataset import eval_shard
    samples = None
    if args.tensorboard and not (args.evaluate or args.generate_pseudogt):
        start, end = eval_shard(len(val), rank, world)
        samples = [i - start for i in DEBUG_IDS[args.dataset] if start <= i < end]
    stats = rec.evaluate(val.eval_batches(batch, rank, world), distributed=world > 1, samples=samples)
    log(cl.test_line(stats))
    if samples is None:
        return stats
    s = stats['samples']
    if world > 1:
        parts = cl.gather_to_rank0({k: (v.cpu() if torch.is_tensor(v) else v) for k, v in s.items()}, world)
        if parts is None:
            return stats
        s = {k: torch.cat([p[k] for p in parts if p[k] is not None]) for k in ('real', 'fake')}
        s['render'] = [t for p in parts for t in p['render']][:4]
    if writer is None:
        return stats
    cl.write_scalars(writer, [(args.loss + '/val', stats['recon_loss'], it), ('flat/val', stats['flat_loss'], it),
                              ('iou/val', stats['miou'], it)])
    cl.add_image(writer, 'image_val/real', cl.to_grid(s['real']), it)
    cl.add_image(writer, 'image_val/fake', cl.to_grid(s['fake']), it)
    render = torch.stack([torch.as_tensor(t) for t in s['render']]).permute(0, 3, 1, 2)
    cl.add_image(writer, 'image_val/render', cl.make_grid(render, nrow=1), it)
    return stats


def main(argv=None):
    args = build_parser().parse_args(argv)
    import command_line as cl
    inception = cl.load_inception() if args.generate_pseudogt else None
    s = derive_settings(args)
    train, val = make_datasets(args, s)

    import torch
    from reconstruction_training import ReconTrainer
    from rendering.mesh_template import MeshTemplate

    # the reference has no --gpu_ids here: one GPU, or one process per GPU under torchrun
    rank, world, device = cl.init_devices('0', SCRIPT, sys.argv[1:] if argv is None else argv)
    batch = cl.per_rank_batch(args.batch_size, world)
    tpl = MeshTemplate(args.mesh_path, is_symmetric=args.symmetric, device=device)
    rec = ReconTrainer(args, tpl, len(train), device=device)
    rec.keep_last_images = args.tensorboard

    checkpoint_dir = os.path.join('checkpoints_recon', args.name)
    training = not (args.evaluate or args.generate_pseudogt)
    if not training or args.continue_train:
        # --continue_train on its own resumes (the reference restarts from scratch there)
        rec.load_checkpoint(os.path.join(checkpoint_dir, f'checkpoint_{args.which_epoch}.pth'),
                            'resume' if training else 'evaluate')
        if rank == 0:
            print(f'Resuming from epoch {rec.epoch}' if training else f'Evaluating epoch {rec.epoch}')
        if not training:
            args.epochs = -1

    writer = None
    if args.tensorboard and training:
        writer = cl.summary_writer(os.path.join('tensorboard_recon', args.name), not args.continue_train, rank)
    if training:
        os.makedirs(checkpoint_dir, exist_ok=True)
        log = cl.Log(os.path.join(checkpoint_dir, 'log.txt'), args.continue_train, cl.command_line(SCRIPT, argv), rank)
    else:
        log = cl.Log(rank=rank)

    if not args.evaluate:
        train.to_device(device)
    if val is not None:
        val.to_device(device)

    def save(which):
        rec.save_checkpoint(os.path.join(checkpoint_dir, f'checkpoint_{which}.pth'))

    try:
        while rec.epoch < args.epochs:
            start = time.time()
            it0, epoch = rec.total_it, rec.epoch
            outs = rec.train_epoch(train.train_batches(batch, epoch, seed=0, rank=rank, world=world))
            values = torch.stack([torch.stack(o) for o in outs]).tolist()
            lines, scalars = cl.recon_epoch_records(it0, epoch, len(outs), args.loss, values)
            for line in lines:
                log(line)
            log(cl.TIME_LINE.format(time.time() - start))
            cl.write_scalars(writer, scalars)
            if rec.epoch % args.save_freq == 0:
                save('latest')
            if rec.epoch % args.checkpoint_freq == 0:
                save(str(rec.epoch))
            if writer is not None and rec.epoch % args.image_freq == 0:
                X_real, image, alpha = rec.last_images
                cl.add_image(writer, 'image_train/real', cl.to_grid(X_real), rec.total_it)
                cl.add_image(writer, 'image_train/fake', cl.to_grid(image.permute(0, 3, 1, 2)), rec.total_it)
            if rec.epoch % args.evaluate_freq == 0:
                evaluate_all(args, rec, val, batch, log, writer, rec.total_it, rank, world)
    except KeyboardInterrupt:
        print('Aborted.')

    if training:
        save('latest')
    elif args.evaluate:
        evaluate_all(args, rec, val, batch, log, writer, rec.total_it, rank, world)
    elif rank == 0:
        from pseudo_gt_export import PseudoGTExporter
        exp = PseudoGTExporter(rec, tpl, args.pseudogt_resolution, inception)
        print('Exporting pseudo-ground-truth data...')
        exp.export(train.eval_batches(args.batch_size), train.get_paths(), os.path.join('cache', args.dataset),
                   args.dataset, val_batches=val.eval_batches(args.batch_size) if args.dataset == 'cub' else None)
        print('Done.')
    if writer is not None:
        writer.close()
    log.close()
    torch.cuda.synchronize(device)
    cl.shutdown(world)


if __name__ == '__main__':
    main()
