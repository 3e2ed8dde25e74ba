"""Pins what the CPU tests used to read from a reference checkout at run time, so that they run anywhere:
  * the same-seed parameter state of the reference's ReconstructionNetwork, Generator and Discriminator (per tensor:
    name, shape, fp64 sum and the first 16 values) and its positional encodings,
  * the parameter names / shapes of the shipped generator checkpoint (what a strict load requires),
  * the conv FLOPs of the reference modules (forward hooks) behind bench.py's roofline numerators,
  * what the reference's AbstractDataset reads back from a pseudo-ground-truth record written by data/pseudo_gt.py.
Needs the reference checkout (REFERENCE_CODE=<its code/ directory>); writes reference_pins.npz next to this file.  The shipped OBJ templates
are stored next to it byte for byte, gzip-compressed (uvsphere_16rings.obj.gz, uvsphere_31rings.obj.gz)."""
import gzip
import importlib
import importlib.util
import os
import re
import shutil
import sys
import tempfile
import types

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
PKG = os.path.join(ROOT, "2dimageto3dmodel_b200")
REF = os.environ["REFERENCE_CODE"]        # the reference checkout's code/ directory
TOPS = ("models", "rendering", "utils", "sync_batchnorm", "data")
sys.path.insert(0, HERE)
import gan_common as GC      # noqa: E402
import recon_common as RC    # noqa: E402


def import_reference(name):
    """The reference's module `name`, with the reference tree first on sys.path from here on (its modules import their
    siblings lazily, at construction)."""
    for k in [k for k in sys.modules if k.split('.')[0] in TOPS]:
        del sys.modules[k]
    if PKG in sys.path:
        sys.path.remove(PKG)
    if REF not in sys.path:
        sys.path.insert(0, REF)
    mod = importlib.import_module(name)
    assert mod.__file__.startswith(REF)
    return mod


def pin_state(out, tag, sd):
    out[tag + "_names"] = np.array(list(sd.keys()))
    out[tag + "_shapes"] = np.array([",".join(map(str, v.shape)) for v in sd.values()])
    out[tag + "_sums"] = np.array([float(v.double().sum()) for v in sd.values()])
    out[tag + "_heads"] = np.stack([np.pad(v.detach().double().flatten()[:16].numpy(), (0, max(0, 16 - v.numel()))) for v in sd.values()])


def conv_gflops(module, run):
    tot, hooks = {}, []
    for name, m in module.named_modules():
        if isinstance(m, nn.Conv2d):
            def hook(mod, inp, o, name=name):
                kh, kw = mod.kernel_size
                tot[name] = tot.get(name, 0.0) + 2.0 * o.numel() * mod.in_channels * kh * kw / 1e9
            hooks.append(m.register_forward_hook(hook))
    with torch.no_grad():
        run()
    for h in hooks:
        h.remove()
    return tot


def main():
    out = {}
    sys.path.insert(0, PKG)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_pseudo_gt_format import _record
    from data.pseudo_gt import pseudo_gt_dir, save_pseudo_gt
    spec = importlib.util.spec_from_file_location("ref_abstract_dataset", os.path.join(REF, "data", "abstract_dataset.py"))
    ref_ds = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref_ds)
    with tempfile.TemporaryDirectory() as tmp:
        cache = os.path.join(tmp, "cache", "cub")
        rec = _record(seed=3)
        save_pseudo_gt(pseudo_gt_dir(cache, 32), 0, rec)
        ds = object.__new__(ref_ds.AbstractDataset)
        ds.args = types.SimpleNamespace(texture_resolution=32)
        ds.cache_dir = cache
        theirs = ds.load_pseudo_ground_truth(0)
    out["pgt_keys"] = np.array(sorted(theirs))
    for k, v in theirs.items():
        out["pgt_" + k] = v.numpy()
    out["pgt_mirror_tex"] = ref_ds.AbstractDataset.mirror_tex(theirs["texture"]).numpy()

    ref_recon = import_reference("models.reconstruction")
    pin_state(out, "recon", RC.build(ref_recon).state_dict())
    ref_gan = import_reference("models.gan")
    G, D = GC.build(ref_gan, GC.make_args(256, 2))
    pin_state(out, "gan_G", G.state_dict())
    pin_state(out, "gan_D", D.state_dict())
    for ny, nx in ((32, 32), (32, 16), (256, 128)):
        out[f"pe_{ny}_{nx}"] = np.asarray(ref_gan.positional_encoding(ny, nx), dtype=np.float64)
    ck = torch.load(os.path.join(REF, "gan_weights/pretrained_weights_cub/checkpoint_latest.pth"), map_location="cpu")["generator_running_avg"]
    out["ckpt_names"] = np.array(list(ck.keys()))
    out["ckpt_shapes"] = np.array([",".join(map(str, v.shape)) for v in ck.values()])

    flops = []
    for res, nd in ((256, 2), (512, 3)):
        args = GC.make_args(res, nd)
        G, D = GC.build(ref_gan, args)
        G.eval(); D.eval()
        z, c, alpha, tex, mesh = GC.inputs(args, B=1)
        g = conv_gflops(G, lambda: G(z, c))
        d = conv_gflops(D, lambda: D(torch.cat((tex * alpha, alpha), 1), mesh, c))
        first = sum(v for k, v in d.items() if re.fullmatch(r"d\d\.conv1", k))
        flops += [sum(g.values()), sum(d.values()), first]
    net = RC.build(ref_recon, texture_res=128).eval()
    r = conv_gflops(net, lambda: net(torch.rand(1, 4, 256, 256)))
    flops += [sum(r.values()), r["conv1e"]]
    out["flops_g256_d256_f256_g512_d512_f512_rec_recfirst"] = np.array(flops)

    np.savez_compressed(os.path.join(HERE, "reference_pins.npz"), **out)
    for rings in (16, 31):
        with open(os.path.join(REF, "mesh_templates", f"uvsphere_{rings}rings.obj"), "rb") as src, \
                gzip.GzipFile(os.path.join(HERE, f"uvsphere_{rings}rings.obj.gz"), "wb", compresslevel=9, mtime=0) as dst:
            shutil.copyfileobj(src, dst)


if __name__ == "__main__":
    main()
