"""Host-side checks of the GAN option variants (norm_g instance / none, norm_d instance, the asymmetric generator), no GPU:
the modules build the reference's state dicts (names, shapes and initial values of tests/golden/gan_variants_reference.npz),
a reference-layout state dict loads with strict=True, and the fused glue's wrappers reject bad shapes and channel counts
with B3DError before any CUDA call."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN

sys.path.insert(0, GOLDEN)
import gan_variants_common as GV          # noqa: E402


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(GOLDEN, "gan_variants_reference.npz"))


@pytest.mark.parametrize("name", list(GV.CONFIGS))
def test_modules_build_the_reference_state_dicts(gold, name):
    from models import gan
    _, G, D = GV.build(gan, name)
    for tag, m in (("g", G), ("d", D)):
        names, shapes, sums = GV.state_summary(m)
        assert names == [str(n) for n in gold[f"{name}/{tag}_state_names"]], (name, tag)
        assert shapes == [str(s) for s in gold[f"{name}/{tag}_state_shapes"]], (name, tag)
        ref = gold[f"{name}/{tag}_state_sums"]
        # same seeds, same construction order -> the same initial tensors (sums in fp64 of identical fp32 values)
        np.testing.assert_allclose(sums, ref, rtol=1e-12, atol=1e-12, err_msg=f"{name}/{tag}")


@pytest.mark.parametrize("name", list(GV.CONFIGS))
def test_reference_layout_state_dict_loads_strict(gold, name):
    from models import gan
    _, G, D = GV.build(gan, name)
    for tag, m in (("g", G), ("d", D)):
        names = [str(n) for n in gold[f"{name}/{tag}_state_names"]]
        shapes = [tuple(int(s) for s in str(s).split("x")) if str(s) else () for s in gold[f"{name}/{tag}_state_shapes"]]
        own = m.state_dict()
        sd = {n: torch.full(s, 0.5, dtype=own[n].dtype) for n, s in zip(names, shapes)}
        m.load_state_dict(sd, strict=True)
        assert all(torch.equal(v, sd[k]) for k, v in m.state_dict().items())
    # the instance norms have an affine weight / bias in the discriminators, nothing in the generator, and no buffers
    if GV.CONFIGS[name]["norm_d"] == "instance":
        keys = D.state_dict().keys()
        assert "d1.bn2.weight" in keys and "d1.bn2.bias" in keys and "d1.bn2.running_mean" not in keys
    if GV.CONFIGS[name]["norm_g"] in ("instance", "none"):
        assert not any(".norm1.norm." in k for k in G.state_dict())


def test_generator_takes_the_fused_path_for_every_norm():
    """fusable() accepts the four norm_g values of the reference."""
    from models import gan
    for norm_g in ("syncbatch", "batch", "instance", "none"):
        args = GV.make_args("cfg1")
        args.norm_g = norm_g
        for symmetric in (True, False):
            G = gan.Generator(args, 64, symmetric=symmetric, mesh_head=True)
            assert G.blk1.fusable() and G.blk6.fusable(), (norm_g, symmetric)


def test_unsupported_instance_norm_settings_keep_the_module_path():
    from b3d.ew import identity_norm, norm_kind
    assert norm_kind(torch.nn.InstanceNorm2d(8)) == "instance"
    assert norm_kind(torch.nn.InstanceNorm2d(8, affine=True)) == "instance"
    assert norm_kind(torch.nn.InstanceNorm2d(8, track_running_stats=True)) is None
    assert norm_kind(torch.nn.BatchNorm2d(8)) == "batch"
    assert norm_kind(identity_norm) == "none"
    assert norm_kind(lambda x: x) is None


def _cbn(norm_g, C):
    import types
    from models.gan import ConditionalBatchNorm2d
    return ConditionalBatchNorm2d(types.SimpleNamespace(norm_g=norm_g), C, 16)


@pytest.mark.parametrize("norm_g", ["instance", "none"])
def test_cbn_act_pad_rejects_bad_shapes_before_cuda(norm_g):
    from b3d import B3DError
    from b3d.ew import CIRCULAR, cbn_act_pad
    z = torch.zeros(2, 16)
    with pytest.raises(B3DError, match="4 \\* a divisor"):
        cbn_act_pad(torch.zeros(2, 6, 4, 4), _cbn(norm_g, 6), z)             # C % 4
    with pytest.raises(B3DError, match="4 \\* a divisor"):
        cbn_act_pad(torch.zeros(2, 12, 4, 4), _cbn(norm_g, 12), z)           # 256 % (C / 4)
    with pytest.raises(B3DError, match="norm layer has 32"):
        cbn_act_pad(torch.zeros(2, 16, 4, 4), _cbn(norm_g, 32), z)           # channel count of the norm layer
    with pytest.raises(B3DError, match="does not fit"):
        cbn_act_pad(torch.zeros(2, 16, 4, 2), _cbn(norm_g, 16), z, pad=3, pad_mode=CIRCULAR)    # wraps more than the map
    with pytest.raises(B3DError, match="does not fit"):
        cbn_act_pad(torch.zeros(2, 16, 4, 4), _cbn(norm_g, 16), z, pad_mode=7)
    with pytest.raises(B3DError, match="4-D"):
        cbn_act_pad(torch.zeros(16, 4, 4), _cbn(norm_g, 16), z)
    with pytest.raises(B3DError, match="CUDA"):                              # well-formed, but on the host
        cbn_act_pad(torch.zeros(2, 16, 4, 4), _cbn(norm_g, 16), z, pad_mode=CIRCULAR)


def test_in_act_pad_rejects_bad_shapes_before_cuda():
    from b3d import B3DError
    from b3d.ew import in_act_pad
    norm = torch.nn.InstanceNorm2d(16, affine=True)
    with pytest.raises(B3DError, match="norm layer has 16"):
        in_act_pad(torch.zeros(2, 32, 4, 4), norm, 1)
    with pytest.raises(B3DError, match="4 \\* a divisor"):
        in_act_pad(torch.zeros(2, 20, 4, 4), torch.nn.InstanceNorm2d(20, affine=True), 1)
    with pytest.raises(B3DError, match="does not fit"):
        in_act_pad(torch.zeros(2, 16, 4, 1), norm, 2)
    with pytest.raises(B3DError, match="affine InstanceNorm2d"):
        in_act_pad(torch.zeros(2, 16, 4, 4), torch.nn.InstanceNorm2d(16), 1)
    with pytest.raises(B3DError, match="affine InstanceNorm2d"):
        in_act_pad(torch.zeros(2, 16, 4, 4), torch.nn.InstanceNorm2d(16, affine=True, track_running_stats=True), 1)
    with pytest.raises(B3DError, match="CUDA"):
        in_act_pad(torch.zeros(2, 16, 4, 4), norm, 1)


def test_glue_entry_points_validate_arguments_without_gpu():
    """The C entry points check their arguments before any CUDA call (error code, message, no launch)."""
    import b3d
    lib = b3d.lib
    assert lib.b3d_version() >= 340
    assert lib.b3d_bn_sums_per_sample(None, 2, 32, 12, None, None) != 0
    assert b"4 * a divisor" in lib.b3d_last_error()
    assert lib.b3d_bn_sums_per_sample(None, 0, 32, 16, None, None) != 0
    assert lib.b3d_cbn_act_fwd(None, None, None, None, 0, 0, None, 2, 4, 2, 16, 1, 3, 1, 0.2, 0, None) != 0
    assert b"pad mode" in lib.b3d_last_error()
    assert lib.b3d_cbn_act_bwd1(None, None, None, None, None, 0, 0, None, None, 8, None, None, 0, 0, None, None, 16, 2, 4, 4,
                                16, 1, 1, 1, 0.2, 0, None) != 0
    assert b"statistics pitch" in lib.b3d_last_error()
    assert lib.b3d_cbn_act_bwd2(None, None, None, None, None, 16, None, None, 6, 0.5, 2, 4, 4, 16, None) != 0
    assert b"statistics pitch" in lib.b3d_last_error()
    assert lib.b3d_cbn_prepare(None, 0, 0, 0, None, 0.0, 1e-5, 0.1, 5, None, None, None, None, None, None, None, None, 2, 16,
                               None) != 0
