"""The command-line drivers' host logic against tests/golden/drivers_reference.npz (make_golden_drivers.py: the reference's
parsers, derived settings, loop log lines and scalars, executed from its scripts' syntax trees): the same flags and
namespaces, the same settings and failures, the same log lines from the same per-iteration values; importing a driver
does nothing, and the errors that need no GPU come before any CUDA work."""
import argparse
import json
import os
import shlex
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, PKG


def describe(parser):
    """make_golden_drivers.describe: every flag's option strings, dest, default, type, action class and `required`."""
    out = []
    for a in parser._actions:
        if isinstance(a, argparse._HelpAction):
            continue
        out.append(dict(option_strings=a.option_strings, dest=a.dest, default=repr(a.default),
                        type=getattr(a.type, '__name__', None), action=type(a).__name__, required=a.required))
    return out


def parse(parser, argv):
    """make_golden_drivers.parse: the namespace (values as repr) or 'error' when argparse exits."""
    try:
        with open(os.devnull, 'w') as null:
            old, sys.stderr = sys.stderr, null
            try:
                return {k: repr(v) for k, v in sorted(vars(parser.parse_args(argv)).items())}
            finally:
                sys.stderr = old
    except SystemExit:
        return 'error'


@pytest.fixture(scope='module')
def gold():
    return json.loads(str(np.load(os.path.join(GOLDEN, 'drivers_reference.npz'))['json']))


def parsers():
    import main
    import run_reconstruction
    return {'main': main.build_parser(), 'recon': run_reconstruction.build_parser()}


@pytest.mark.parametrize('name', ['main', 'recon'])
def test_flags_equal_the_reference(gold, name):
    assert describe(parsers()[name]) == gold[f'{name}_flags']


@pytest.mark.parametrize('name', ['main', 'recon'])
def test_namespaces_and_failures_equal_the_reference(gold, name):
    p = parsers()[name]
    for argv, expect in gold[f'{name}_samples']:
        assert parse(p, shlex.split(argv)) == expect, argv


def test_bool_flags_keep_the_quirk():
    p = parsers()['main']
    assert p.parse_args(['--weights', 'w', '--dataset', 'cub', '--symmetric_g', 'False']).symmetric_g is True
    assert p.parse_args(['--weights', 'w', '--dataset', 'cub', '--symmetric_g', '']).symmetric_g is False
    assert p.parse_args(['--weights', 'w', '--dataset', 'cub']).conditional_class == '--conditional_class'


def test_derived_settings_equal_the_reference(gold, tmp_path):
    sys.path.insert(0, GOLDEN)
    import dataset_common as DC
    import main
    DC.write_tree(str(tmp_path), DC.make_inputs())
    p = parsers()['main']
    for argv, expect in gold['derived']:
        args = p.parse_args(shlex.split(argv))
        ds = main.make_dataset(args, root=str(tmp_path))
        try:
            main.derive_settings(args, ds)
            got = dict(mesh_path=args.mesh_path, num_discriminators=args.num_discriminators,
                       truncation_sigma=args.truncation_sigma, error=None)
        except AssertionError as e:
            got = dict(error=f'AssertionError: {e}')
        assert got == expect, argv


def test_recon_derived_settings():
    import run_reconstruction as rr
    p = parsers()['recon']
    a = p.parse_args(['--name', 'r', '--dataset', 'p3d', '--generate_pseudogt', '--pseudogt_resolution', '768'])
    s = rr.derive_settings(a)
    assert a.mesh_path == 'mesh_templates/uvsphere_31rings.obj'
    assert s == dict(renderer_res=1536, train_res=[256, 299, 1536], val_res=299, is_train=False)
    a = p.parse_args(['--name', 'r', '--dataset', 'cub', '--image_resolution', '128'])
    assert rr.derive_settings(a) == dict(renderer_res=128, train_res=128, val_res=128, is_train=True)
    assert a.mesh_path == 'mesh_templates/uvsphere_16rings.obj'


def test_line_formats_equal_the_reference(gold):
    import command_line as cl
    fid = cl.fid_lines(dict(fid=1.0, fid_texture_only=2.0, fid_mesh_only=3.0, fid_val=4.0, fid_texture_only_val=5.0,
                            fid_mesh_only_val=6.0))
    ref = gold['main_formats']
    assert [f.format(v) for f, v in zip([x for x in ref if 'FID' in x], (1.0, 2.0, 3.0, 4.0, 5.0, 6.0))] == fid
    assert cl.GAN_LINE in ref and cl.TIME_LINE in ref
    assert set(gold['recon_formats']) == {cl.TEST_LINE, cl.TIME_LINE, cl.RECON_LINE}
    assert cl.test_line(dict(recon_loss=0.5, flat_loss=1.25, miou=0.75, N=7)) == gold['recon_formats'][0].format(0.5, 1.25, 0.75, 7)


def test_gan_lines_and_scalars_from_the_curves(gold):
    """The reference's loop wrote its lines and scalars as it went; here they are rebuilt at each epoch's end from the
    curves alone, as the driver does after GANTrainer.train_epoch."""
    import command_line as cl
    g = gold['gan_loop']
    by_tag = {}
    for tag, v, k in g['scalars']:
        by_tag.setdefault(tag, []).append(v)
    loss = g['loss']
    curves = ([0] + by_tag[f'gan_{loss}/g'], [0] + by_tag[f'gan_{loss}/d_fake_loss'],
              [0] + by_tag[f'gan_{loss}/d_real_loss'], [0] + by_tag['flat'])
    n, d = g['n_iters'], g['d_steps_per_g']
    lines, scalars = [], []
    for e in range(g['epochs']):
        it0 = e * n
        n_g = sum(1 for k in range(it0) if k % (1 + d) == 0)
        lengths = [1 + n_g, 1 + it0 - n_g, 1 + it0 - n_g, 1 + n_g]
        ln, sc = cl.gan_epoch_records(it0, e, n, d, loss, curves, lengths, True)
        lines += ln
        scalars += sc
    assert lines == [x for x in g['lines'] if not x.startswith('Time per epoch')]
    assert [(t, k) for t, _, k in scalars] == [(t, k) for t, _, k in g['scalars']]
    assert [v for _, v, _ in scalars] == [v for _, v, _ in g['scalars']]


def test_recon_lines_and_scalars_from_the_step_values(gold):
    import command_line as cl
    r = gold['recon_loop']
    sc = r['scalars']
    n, loss = r['n_iters'], r['loss']
    recon = [v for t, v, _ in sc if t == f'{loss}/train']
    flat = [v for t, v, _ in sc if t == 'flat/train']
    iou = [v for t, v, _ in sc if t == 'iou/train']
    lines, scalars = [], []
    for e in range(len(recon) // n):
        s = slice(e * n, (e + 1) * n)
        ln, scl = cl.recon_epoch_records(e * n, e, n, loss, list(zip(r['total'][s], recon[s], flat[s], iou[s])))
        lines += ln
        scalars += scl
    assert lines == [x for x in r['lines'] if not x.startswith('Time per epoch')]
    assert [tuple(x) for x in sc] == scalars


def test_make_grid_layout():
    import command_line as cl
    x = torch.arange(5 * 3 * 2 * 3, dtype=torch.float32).reshape(5, 3, 2, 3) + 1
    g = cl.make_grid(x, nrow=4)
    # torchvision: 4 columns of (3 + 2) and 2 rows of (2 + 2), plus the leading padding
    assert g.shape == (3, 2 * 4 + 2, 4 * 5 + 2)
    assert torch.equal(g[:, 2:4, 2:5], x[0]) and torch.equal(g[:, 2:4, 7:10], x[1])
    assert torch.equal(g[:, 6:8, 2:5], x[4]) and float(g[:, 6:8, 7:].abs().sum()) == 0
    assert float(g[:, :2].abs().sum()) == 0 and torch.equal(cl.make_grid(x[:1], nrow=4), x[0])
    m = cl.to_grid_mesh(torch.randn(2, 3, 4, 4))
    tiles = [m[:, 2:6, 2:6], m[:, 2:6, 8:12]]
    for t in tiles:
        assert torch.allclose(t.amin(dim=(1, 2)), torch.zeros(3)) and torch.allclose(t.amax(dim=(1, 2)), torch.ones(3))


def run_quiet(code, env=None, cwd=None):
    return subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, env=env, cwd=cwd, timeout=600)


def test_importing_a_driver_does_nothing(tmp_path):
    code = ("import sys; sys.path.insert(0, %r); sys.argv = ['x', '--bogus']\n"
            "import main, run_reconstruction, torch\n"
            "assert not torch.cuda.is_initialized(); print('ok')" % PKG)
    r = run_quiet(code, cwd=str(tmp_path))
    assert r.returncode == 0 and r.stdout.strip() == 'ok', r.stderr
    assert os.listdir(tmp_path) == []


def test_several_gpu_ids_outside_torchrun_print_the_torchrun_command(tmp_path):
    code = ("import sys; sys.path.insert(0, %r)\nimport main, torch\n"
            "try:\n    main.main(['--weights', 'w', '--dataset', 'cub', '--gpu_ids', '0,1'])\n"
            "except SystemExit as e:\n    assert not torch.cuda.is_initialized(); print(e)\n" % PKG)
    env = {k: v for k, v in os.environ.items() if k not in ('WORLD_SIZE', 'LOCAL_RANK', 'RANK')}
    r = run_quiet(code, env=env, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    assert 'torchrun --nproc-per-node 2 main.py --weights w --dataset cub --gpu_ids 0,1' in r.stdout


@pytest.mark.parametrize('script,argv', [
    ('main', ['--weights', 'w', '--dataset', 'cub']),
    ('main', ['--weights', 'w', '--dataset', 'cub', '--evaluate']),
    ('run_reconstruction', ['--name', 'r', '--dataset', 'cub', '--generate_pseudogt']),
])
def test_a_missing_inception_file_stops_before_any_work(tmp_path, script, argv):
    code = ("import sys; sys.path.insert(0, %r)\nimport %s as m, torch\n"
            "try:\n    m.main(%r)\n"
            "except SystemExit as e:\n    assert not torch.cuda.is_initialized(); print(e)\n" % (PKG, script, argv))
    env = dict(os.environ, B3D_INCEPTION_WEIGHTS=str(tmp_path / 'absent.pth'), TORCH_HOME=str(tmp_path / 'hub'))
    r = run_quiet(code, env=env, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    assert 'B3D_INCEPTION_WEIGHTS' in r.stdout and 'never downloads' in r.stdout


def test_search_lines_equal_the_reference(gold):
    """The best-epoch search's console lines, rebuilt from select_best_checkpoint's result (visit order, paths, choice)."""
    import main
    s = gold['search']
    fast = {e: f for e, f in s['fast_fid']}
    best = dict(fast_fid=fast, paths={e: f'w/checkpoint_{e}.pth' for e in fast}, best_path=s['best_path'])
    assert main.search_lines(best) == s['lines']


def test_merged_samples_follow_the_visualisation_order():
    """Each rank finds the samples of its contiguous shard in dataset order; rank 0 puts them in the order of the
    indices the last training batch drew."""
    import command_line as cl
    samples = [9, 2, 14, 5, 0, 11]
    parts = [{'index': torch.tensor([0, 2, 5]), 'fake': torch.tensor([0., 2., 5.]), 'real': torch.tensor([10., 12., 15.])},
             {'index': torch.tensor([9, 11, 14]), 'fake': torch.tensor([9., 11., 14.]), 'real': torch.tensor([19., 21., 24.])},
             {'index': torch.tensor([], dtype=torch.int64)}]
    m = cl.merge_samples(parts, samples)
    assert m['index'].tolist() == samples
    assert m['fake'].tolist() == [float(i) for i in samples] and m['real'].tolist() == [10. + i for i in samples]
