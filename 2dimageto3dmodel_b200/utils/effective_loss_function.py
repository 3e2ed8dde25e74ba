"""Drop-in for /root/reference/code/utils/effective_loss_function.py (class EffectiveLossFunction,
:10-81): points + quaternion (+ scale) -> soft silhouette [B,V,V], computed by the fused sm_90a
kernels of libb3d (csrc/pc_kernels.cu) instead of ~60 ATen launches and nine dense V^3 temporaries.

`semantics="R"` (default) reproduces the reference as written once its execution defects are patched
(SURVEY.md App. A, P1-P3); `semantics="P"` is the paper-intended math.
`PointCloudRender` is the name BASELINE.json's north star uses for this module.
"""
import torch
import torch.nn as nn

from b3d import B3DError, mode_id
from b3d import pointcloud as _pc
from b3d.pointcloud import CAMERA_VIEW_DISTANCE, FIELD_OF_VIEW, effective_loss, smoothing_taps


class EffectiveLossFunction(nn.Module):
    def __init__(self, voxel_size=64, kernel_size=21, smooth_sigma=3.0, semantics="R"):
        super().__init__()
        self.voxel_size = voxel_size
        self.kernel_size = kernel_size
        self.semantics = semantics
        mode_id(semantics)
        # run-time buffer, re-assigned by the sigma schedule (training_test_shape_net.py:29)
        self.register_buffer("sigma", torch.tensor(smooth_sigma))
        self._taps_key = None
        self._taps = None

    def __setattr__(self, name, value):
        # the schedule assigns a fresh tensor to `sigma` every step (training_test_shape_net.py:29): drop the cached
        # taps on every assignment (keying on id() would be wrong: CPython recycles ids)
        if name == "sigma":
            self.__dict__["_taps_key"] = None
        super().__setattr__(name, value)

    def _current_taps(self):
        s = self.sigma
        key = (s._version, self.kernel_size, self.semantics)
        if self._taps_key is None or key != self._taps_key[:3] or self._taps_key[3] is not s:
            # one host read per sigma change (the schedule changes it once per step at most)
            self._taps = smoothing_taps(float(s), self.kernel_size, self.semantics)
            self._taps_key = key + (s,)
        return self._taps

    def forward(self, point_cloud, rotation, scale=None):
        """point_cloud [B,N,3] with columns (z,y,x); rotation [B,4] quaternion (w,x,y,z), normalised
        inside; scale [B,1] or None.  Returns the projection [B,V,V] (differentiable)."""
        if point_cloud.dim() != 3 or point_cloud.size(-1) != 3:
            raise B3DError(f"point_cloud must be [B,N,3], got {tuple(point_cloud.shape)}")
        return effective_loss(point_cloud, rotation, scale, V=self.voxel_size, taps=self._current_taps(),
                              mode=self.semantics, fov=FIELD_OF_VIEW, cam_dist=CAMERA_VIEW_DISTANCE)

    def termination_probs(self, voxels, epsilon=1e-5):
        """Smoothed occupancies [B,V,V,V] -> ray-termination probabilities [B,V+1,V,V] (reference :18-56)."""
        if epsilon != 1e-5:
            raise B3DError("termination_probs: the kernels are built for the reference's epsilon = 1e-5")
        return _pc.termination_probs(voxels, self.semantics)


PointCloudRender = EffectiveLossFunction
