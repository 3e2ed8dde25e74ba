"""Command line of the GAN stage, with the flags, files and log lines of the reference's main.py:

    python main.py --weights <name> --dataset cub|p3d [...]            train (--continue_train resumes)
    python main.py --weights <name> --dataset cub --evaluate [--which_epoch N|latest|best]
    python main.py --weights <name> --dataset cub --save_results       textured meshes and a render grid

Run it from the directory that holds cache/, datasets/ and mesh_templates/.  Each mode calls the existing classes:
CubDataset / Pascal3DPlusDataset (device batches), GANTrainer, FIDEvaluator / select_best_checkpoint and SampleExporter.
Several GPUs: one process per GPU under torchrun.  `main()` parses sys.argv (or argv) and runs; importing does nothing."""
import argparse
import os
import sys
import time

import numpy as np

SCRIPT = 'main.py'


def build_parser():
    p = argparse.ArgumentParser()
    # model
    p.add_argument('--texture_resolution', type=int, default=512)
    p.add_argument('--mesh_resolution', type=int, default=32)
    p.add_argument('--symmetric_g', type=bool, default=True)
    p.add_argument('--texture_only', action='store_true')
    p.add_argument('--conditional_class', default='--conditional_class', action='store_true',
                   help='condition the model on class labels')
    p.add_argument('--conditional_color', action='store_true', help='condition the model on colors (p3d only)')
    p.add_argument('--conditional_text', action='store_true', help='condition the model on captions (cub only)')
    p.add_argument('--norm_g', type=str, default='syncbatch', help='(syncbatch|batch|instance|none)')
    p.add_argument('--latent_dim', type=int, default=64, help='dimensionality of the random vector z')
    p.add_argument('--mesh_path', type=str, default='autodetect', help='path to the .obj mesh template')
    p.add_argument('--text_max_length', type=int, default=18)
    p.add_argument('--text_pretrained_encoder', type=str, default='cache/cub/text_encoder200.pth')
    p.add_argument('--text_train_encoder', action='store_true')
    p.add_argument('--text_attention', type=bool, default=True)
    p.add_argument('--text_embedding_dim', type=int, default=256)
    # training
    p.add_argument('--epochs', type=int, default=600)
    p.add_argument('--norm_d', type=str, default='none', help='(instance|none)')
    p.add_argument('--mesh_regularization', type=float, default=0.0001, help='strength of the smoothness regularizer')
    p.add_argument('--lr_g', type=float, default=0.0001)
    p.add_argument('--lr_d', type=float, default=0.0004)
    p.add_argument('--d_steps_per_g', type=int, default=2)
    p.add_argument('--g_running_average_alpha', type=float, default=0.999)
    p.add_argument('--lr_decay_after', type=int, default=1000)
    p.add_argument('--loss', type=str, default='hinge', help='(hinge|ls|original)')
    p.add_argument('--mask_output', type=bool, default=True)
    p.add_argument('--num_discriminators', type=int, default=-1)
    # session
    p.add_argument('--weights', type=str, required=True)
    p.add_argument('--dataset', type=str, required=True, help='(p3d|cub)')
    p.add_argument('--checkpoint_freq', type=int, default=20, help='save checkpoint every N epochs')
    p.add_argument('--save_freq', type=int, default=5, help='save latest checkpoint every N epochs')
    p.add_argument('--evaluate_freq', type=int, default=20, help='evaluate FID every N epochs')
    p.add_argument('--tensorboard', action='store_true')
    p.add_argument('--gpu_ids', type=str, default='0', help='comma-separated; more than one id: run under torchrun')
    p.add_argument('--continue_train', action='store_true', help='resume training from checkpoint')
    p.add_argument('--evaluate', action='store_true', help='evaluate FID, do not train')
    p.add_argument('--save_results', action='store_true', help='export image/mesh samples, do not train')
    p.add_argument('--which_epoch', type=str, default='latest', help='(N|latest|best)')
    p.add_argument('--batch_size', type=int, default=32)
    p.add_argument('--num_workers', type=int, default=4, help='accepted; the device data path has no loader workers')
    p.add_argument('--truncation_sigma', type=float, default=-1, help='-1 = autodetect; set to a large value to disable')
    return p


def make_dataset(args, root=''):
    """main.py:93-100: the training set of --dataset (a dataset error, e.g. --conditional_text, ends the program)."""
    if args.dataset not in ('cub', 'p3d'):
        raise ValueError('Invalid dataset')
    try:
        if args.dataset == 'p3d':
            from data.pascal3d_plus_dataset import Pascal3DPlusDataset
            return Pascal3DPlusDataset(args, root=root)
        from data.cub_200_2011_dataset import CubDataset
        return CubDataset(args, root=root)
    except ValueError as e:
        raise SystemExit(f'error: {e}')


def derive_settings(args, ds):
    """main.py:102-121: the mesh template, number of discriminators and truncation sigma the dataset suggests where the
    flags ask for autodetection, then the reference's safety checks (AssertionError)."""
    if args.mesh_path == 'autodetect':
        args.mesh_path = ds.suggest_mesh_template()
    if args.num_discriminators == -1:
        args.num_discriminators = ds.suggest_num_discriminators()
    if args.truncation_sigma < 0:
        args.truncation_sigma = ds.suggest_truncation_sigma()
    if args.num_discriminators >= 3:
        assert args.texture_resolution >= 512
    if args.dataset == 'cub':
        assert not args.conditional_color, 'Not supported'
        assert not (args.conditional_class and args.conditional_text), 'Not supported'
    elif args.dataset == 'p3d':
        assert not args.conditional_text, 'Not supported'
    return args


class EvalBatches:
    """The evaluation loader: iterable any number of times (the best-epoch search walks it once per checkpoint)."""

    def __init__(self, ds, batch_size, rank, world):
        self.ds, self.batch_size, self.rank, self.world = ds, batch_size, rank, world

    def __iter__(self):
        return self.ds.eval_batches(self.batch_size, self.rank, self.world)


def last_batch_indices(n, epoch, batch_size, world):
    """The dataset indices of an epoch's last training batch over all ranks (main.py:777 visualises them)."""
    from data.abstract_dataset import epoch_order
    orders = [epoch_order(n, epoch, 0, r, world) for r in range(world)]
    k = len(orders[0]) // batch_size
    return np.concatenate([o[(k - 1) * batch_size:k * batch_size].numpy() for o in orders])


def evaluate_fid(args, evaluator, batches, log, writer, it, world, samples=None, seed=None):
    """main.py's evaluate_fid: the scores, their log lines and, with a writer, the FID scalars and the sample grids."""
    import command_line as cl
    scores = evaluator.evaluate(batches, seed=seed, distributed=world > 1, samples=samples)
    for line in cl.fid_lines(scores):
        log(line)
    if samples is None:
        return scores
    s = scores['samples']
    if world > 1:
        # each rank found the samples of its shard: rank 0 puts them together in the order of `samples`
        parts = cl.gather_to_rank0({k: v.cpu() for k, v in s.items()}, world)
        if parts is None:
            return scores
        s = {k: v.to(evaluator.device) for k, v in cl.merge_samples(parts, samples).items()}
    if writer is None:
        return scores
    if 'real_tex' in s:
        cl.add_image(writer, 'image/real_tex', cl.to_grid_tex(s['real_tex']), it)
    cl.add_image(writer, 'image/fake_tex', cl.to_grid_tex(s['fake_tex']), it)
    cl.add_image(writer, 'image/fake_mesh', cl.to_grid_mesh(s['fake_mesh']), it)
    for tag, k in (('render/fake', 'fake'), ('render/fake_texture', 'fake_texture_only'),
                   ('render/fake_mesh', 'fake_mesh_only'), ('render/real', 'real')):
        if k in s:
            cl.add_image(writer, tag, cl.make_grid(s[k], nrow=4), it)
    writer.add_scalar('fid/combined', scores['fid'], it)
    if 'fid_val' in scores:
        writer.add_scalar('fid/combined_val', scores['fid_val'], it)
    if 'fid_texture_only' in scores:
        writer.add_scalar('fid/texture_only', scores['fid_texture_only'], it)
        writer.add_scalar('fid/mesh_only', scores['fid_mesh_only'], it)
    return scores


def make_evaluator(args, ds, generator, mesh_template, inception, device):
    """main.py:149-185: the FID evaluator of the running-average generator with the real-image statistics of
    cache/<dataset> (and, for CUB, those of the test/validation split)."""
    from fid_evaluation import FIDEvaluator, load_real_statistics
    cache_dir = os.path.join(ds.root, 'cache', args.dataset)
    ev = FIDEvaluator(generator, mesh_template, inception, latent_dim=args.latent_dim,
                      truncation_sigma=args.truncation_sigma, device=device)
    m, s, _ = load_real_statistics(os.path.join(cache_dir, 'precomputed_fid_299x299_train.npz'), 299, len(ds))
    ev.set_real_statistics(m, s)
    if args.dataset == 'cub':
        m, s, n_val = load_real_statistics(os.path.join(cache_dir, 'precomputed_fid_299x299_testval.npz'), 299)
        ev.set_real_statistics(m, s, validation=True, num_images=n_val)
    return ev


def search_lines(best):
    """main.py:803-828's console lines of the best-epoch search, from select_best_checkpoint's result."""
    import command_line as cl
    lines = ['Enumerating checkpoints:'] + [f'Epoch {e}: {best["paths"][e]}' for e in best['fast_fid']]
    best_fid, best_path = float('inf'), None
    for e, fid in best['fast_fid'].items():
        if fid < best_fid:
            best_fid, best_path = fid, best['paths'][e]
        lines += [f'--- Evaluating epoch {e} ---'] + cl.fid_lines(dict(fid=fid)) + [f'Best FID so far: {best_fid} at {best_path}']
    return lines + [f'--- Running final evaluation using {best["best_path"]} ---']


def main(argv=None):
    args = build_parser().parse_args(argv)
    import command_line as cl
    if args.save_results:
        args.evaluate = True
    if len(args.gpu_ids.split(',')) > 1 and int(os.environ.get('WORLD_SIZE', '1')) == 1:
        cl.init_devices(args.gpu_ids, SCRIPT, sys.argv[1:] if argv is None else argv)     # exits with the torchrun command
    fid_needed = not args.texture_only and not args.save_results and (args.evaluate or args.evaluate_freq <= args.epochs)
    inception = cl.load_inception() if fid_needed else None
    ds = make_dataset(args)
    derive_settings(args, ds)

    import torch
    from fid_evaluation import select_best_checkpoint
    from gan_training import GANTrainer
    from rendering.mesh_template import MeshTemplate

    rank, world, device = cl.init_devices(args.gpu_ids, SCRIPT, sys.argv[1:] if argv is None else argv)
    batch = cl.per_rank_batch(args.batch_size, world)
    tpl = None if args.texture_only else MeshTemplate(args.mesh_path, is_symmetric=args.symmetric_g, device=device)
    gan = GANTrainer(args, mesh_template=tpl, device=device)

    evaluator = None
    if fid_needed:
        evaluator = make_evaluator(args, ds, gan.trainer.generator_running_avg, tpl, inception, device)

    checkpoint_dir = os.path.join('gan_weights', args.weights)
    if args.continue_train or args.evaluate:
        which = 'latest' if args.which_epoch == 'best' else args.which_epoch
        resume = args.continue_train and not args.evaluate
        gan.load_checkpoint(os.path.join(checkpoint_dir, f'checkpoint_{which}.pth'), 'resume' if resume else 'evaluate')
        if rank == 0 and (resume or gan.epoch):
            print(f'Resuming from epoch {gan.epoch}' if resume else f'Evaluating epoch {gan.epoch}')
        if not resume:
            args.epochs = -1

    writer = None
    if args.tensorboard and not args.evaluate:
        writer = cl.summary_writer(os.path.join('tensorboard_gan', args.weights), not args.continue_train, rank)
    if not args.evaluate:
        os.makedirs(checkpoint_dir, exist_ok=True)
        log = cl.Log(os.path.join(checkpoint_dir, 'log.txt'), args.continue_train, cl.command_line(SCRIPT, argv), rank)
    else:
        log = cl.Log(rank=rank)

    if evaluator is not None or args.epochs > gan.epoch:
        ds.to_device(device, include_image=args.tensorboard and not args.evaluate)
    eval_batches = EvalBatches(ds, batch, rank, world)

    def save(which):
        gan.save_checkpoint(os.path.join(checkpoint_dir, f'checkpoint_{which}.pth'))

    try:
        while gan.epoch < args.epochs:
            start = time.time()
            it0, epoch = gan.total_it, gan.epoch
            curves = (gan.g_curve, gan.d_fake_curve, gan.d_real_curve, gan.flat_curve)
            lengths = [len(c) for c in curves]
            gan.train_epoch(ds.train_batches(batch, epoch, seed=0, rank=rank, world=world))
            curves = (gan.g_curve, gan.d_fake_curve, gan.d_real_curve, gan.flat_curve)
            lines, scalars = cl.gan_epoch_records(it0, epoch, gan.total_it - it0, args.d_steps_per_g, args.loss, curves,
                                                  lengths, tpl is not None)
            for line in lines:
                log(line)
            log(cl.TIME_LINE.format(time.time() - start))
            cl.write_scalars(writer, scalars)
            if gan.epoch % args.save_freq == 0:
                save('latest')
            if gan.epoch % args.checkpoint_freq == 0:
                save(str(gan.epoch))
            if gan.epoch % args.evaluate_freq == 0 and not args.texture_only:
                vis = last_batch_indices(len(ds), epoch, batch, world) if args.tensorboard else None
                evaluate_fid(args, evaluator, eval_batches, log, writer, gan.total_it, world, samples=vis)
    except KeyboardInterrupt:
        print('Aborted.')

    if not args.evaluate:
        save('latest')
    elif not args.save_results:
        if args.which_epoch == 'best':
            best = select_best_checkpoint(gan, evaluator, checkpoint_dir, eval_batches, seed=1234, distributed=world > 1)
            if rank == 0:
                # the reference prints these as the search goes; here they follow it
                print('\n'.join(search_lines(best)))
            for line in cl.fid_lines(best['scores']):
                log(line)
        else:
            evaluate_fid(args, evaluator, eval_batches, log, None, gan.total_it, world, seed=1234)
    elif rank == 0:
        from sample_export import SampleExporter
        exp = SampleExporter(gan.trainer.generator_running_avg, tpl, ds, args.truncation_sigma, args.latent_dim)
        exp.export(os.path.join('results', args.weights), os.path.join('results', f'{args.weights}.png'),
                   num_samples=args.batch_size, batch_size=args.batch_size)
        print("\nExport of batch with size '{}' successfully done.\n".format(args.batch_size))
    if writer is not None:
        writer.close()
    log.close()
    torch.cuda.synchronize(device)
    cl.shutdown(world)


if __name__ == '__main__':
    main()
