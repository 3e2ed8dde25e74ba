"""Drop-in for /root/reference/code/utils/fid.py (init_inception :9-19, forward_inception_batch :21-25,
calculate_stats :27-30, calculate_frechet_distance :33-82) — SURVEY §8f rank 4.

* The Inception network is utils/inception.py here: its convolutions run on libb3d's wgmma kernels, pools and the
  input transform on csrc/fid_kernels.cu.  CUDA only, like everything behind libb3d.
* `FIDStatistics` keeps the running sums of the pool features ON THE GPU (b3d_fid_accumulate: sum x and sum x x^T in
  fp64) so an evaluation over thousands of renders never copies activations to the host; `calculate_stats` keeps the
  reference's numpy signature for activation arrays.
* `calculate_frechet_distance` evaluates Tr sqrt(S1 S2) through symmetric eigendecompositions,
  Tr sqrt(S1 S2) = sum_i sqrt(lambda_i(S1^1/2 S2 S1^1/2)), instead of scipy.linalg.sqrtm of the non-symmetric product
  (utils/fid.py:67; `sqrtm(..., disp=False)` no longer exists in SciPy >= 1.16): same value for positive semi-definite
  inputs, real by construction, about 20x cheaper at 2048 dimensions.  Pinned against the reference's function on
  full-rank, rank-deficient and the shipped real-image CUB statistics (tests/golden/fid_reference.npz)."""
import warnings

import numpy as np
import torch

from .inception import InceptionV3


def init_inception(weights="pretrained"):
    """utils/fid.py:9-19: the 2048-d final-average-pool block.  `weights`: see InceptionV3."""
    block_idx = InceptionV3.BLOCK_INDEX_BY_DIM[2048]
    return InceptionV3([block_idx], weights=weights)


def forward_inception_features(inception_model, images):
    """[B,3,H,W] images in (0,1) on the GPU -> [B,D] pool features, still on the GPU."""
    pred = inception_model(images)[0]
    if pred.shape[2] != 1 or pred.shape[3] != 1:
        pred = torch.nn.functional.adaptive_avg_pool2d(pred, output_size=(1, 1))
    return pred.reshape(images.shape[0], -1)


def forward_inception_batch(inception_model, images):
    """utils/fid.py:21-25: numpy [B,D]."""
    return forward_inception_features(inception_model, images).detach().cpu().numpy()


def calculate_stats(act):
    """utils/fid.py:27-30.  act: numpy [n,D] (the reference's call) or a CUDA tensor (accumulated on the device)."""
    if isinstance(act, torch.Tensor) and act.is_cuda:
        st = FIDStatistics(act.shape[1], act.device)
        st.update(act)
        return st.finalize()
    act = np.asarray(act)
    return np.mean(act, axis=0), np.cov(act, rowvar=False)


class FIDStatistics:
    """Running mean / covariance of feature batches on the GPU (fp64 sums; np.cov's unbiased normalisation)."""

    def __init__(self, dim=2048, device="cuda"):
        self.dim = int(dim)
        self.n = 0
        self.sum = torch.zeros(self.dim, dtype=torch.float64, device=device)
        self.outer = torch.zeros(self.dim, self.dim, dtype=torch.float64, device=device)

    def update(self, feat):
        from b3d import check, dev, lib, ptr, stream_ptr
        f = dev(feat.detach(), "features")
        if f.dim() != 2 or f.shape[1] != self.dim:
            raise ValueError(f"features must be [n,{self.dim}], got {tuple(f.shape)}")
        check(lib.b3d_fid_accumulate(ptr(f), f.shape[0], self.dim, ptr(self.sum), ptr(self.outer), stream_ptr(f)))
        self.n += int(f.shape[0])

    def all_reduce(self, group=None):
        """One process per GPU, every rank scores its shard of the evaluation set: sum the running sums over the ranks
        (the reference instead scatters every batch over `gpu_ids` inside one process, main.py:163, :254-279).  The sums are
        additive, so the reduced statistics equal the single-process ones up to fp64 summation order."""
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()):
            return self
        n = torch.tensor([float(self.n)], dtype=torch.float64, device=self.sum.device)
        for t in (self.sum, self.outer, n):
            dist.all_reduce(t, group=group)
        self.n = int(round(float(n)))
        return self

    def finalize(self):
        """-> (mu [D], sigma [D,D]) as float64 numpy arrays, the values np.mean / np.cov(rowvar=False) give."""
        if self.n < 2:
            raise ValueError("covariance needs at least two samples")
        mu = self.sum / self.n
        sigma = (self.outer - self.n * torch.outer(mu, mu)) / (self.n - 1)
        return mu.cpu().numpy(), sigma.cpu().numpy()


def _trace_sqrt_product(sigma1, sigma2):
    """Tr sqrt(sigma1 sigma2) for symmetric positive semi-definite inputs, through two symmetric eigendecompositions."""
    w, u = np.linalg.eigh((sigma1 + sigma1.T) * 0.5)
    r = (u * np.sqrt(np.clip(w, 0.0, None))) @ u.T                      # sigma1^(1/2)
    a = r @ sigma2 @ r
    ev = np.linalg.eigvalsh((a + a.T) * 0.5)
    return float(np.sqrt(np.clip(ev, 0.0, None)).sum())


def calculate_frechet_distance(mu1, sigma1, mu2, sigma2, eps=1e-6):
    """d^2 = ||mu1 - mu2||^2 + Tr(C1 + C2 - 2 sqrt(C1 C2))   (utils/fid.py:33-82)."""
    mu1 = np.atleast_1d(np.asarray(mu1, dtype=np.float64))
    mu2 = np.atleast_1d(np.asarray(mu2, dtype=np.float64))
    sigma1 = np.atleast_2d(np.asarray(sigma1, dtype=np.float64))
    sigma2 = np.atleast_2d(np.asarray(sigma2, dtype=np.float64))
    assert mu1.shape == mu2.shape, "Training and test mean vectors have different lengths"
    assert sigma1.shape == sigma2.shape, "Training and test covariances have different dimensions"
    diff = mu1 - mu2
    tr_covmean = _trace_sqrt_product(sigma1, sigma2)
    if not np.isfinite(tr_covmean):
        warnings.warn("fid calculation produces singular product; adding %s to diagonal of cov estimates" % eps)
        offset = np.eye(sigma1.shape[0]) * eps
        tr_covmean = _trace_sqrt_product(sigma1 + offset, sigma2 + offset)
    return diff.dot(diff) + np.trace(sigma1) + np.trace(sigma2) - 2 * tr_covmean
