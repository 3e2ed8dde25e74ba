"""H100-native hot path of NikolaZubic/2dimageto3dmodel.

This directory plays the role of the reference's `code/` directory: put it on sys.path (or run the
reference's drivers with it as the working directory) and the reference's imports resolve to the
CUDA-backed modules here —
    from utils.effective_loss_function import EffectiveLossFunction
    from rendering.renderer import Renderer
    from rendering.mesh_template import MeshTemplate
    from utils.losses import loss_flat, GANLoss
    from models.gan import Generator, MultiScaleDiscriminator
`b3d/` holds the ctypes binding of libb3d.so (C ABI: include/b3d.h), `csrc/` the sm_90a kernels.
"""
