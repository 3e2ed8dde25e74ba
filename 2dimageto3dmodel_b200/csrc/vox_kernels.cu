// Dense voxel-grid kernels (sm_90a, HBM-bound, one pass each) for the parts of the point-cloud path that need a
// materialised [B,V,V,V] grid: the stand-alone VoxelsSmooth / termination_probs call surface and the paper-intended
// semantics ("mode P": the Gaussian blur runs along x, y AND z, which couples the columns the fused mode-R kernel
// keeps in shared memory).
//   vox_blur_axis     VoxelsSmooth.smooth, one separable kernel   utils/smooth_voxels.py:62-73 (zero padding)
//   vox_scale_clamp   "* scale, clamp(0,1)"                         utils/smooth_voxels.py:80-82   (+ adjoint)
//   vox_termination   termination_probs / silhouette               utils/effective_loss_function.py:18-56,79-81 (+ adjoint)
//   vox_gather        adjoint of the trilinear splat: d/d(grid coords) from the 8 corners of dGrid (also the last step of
//                     the fused mode-P silhouette backward, csrc/pc_kernels.cu)
#include "b3d_common.cuh"

namespace {
using b3d::clamp_nan;
constexpr int NT = 256;
constexpr int MAXT = 63;
constexpr float TERM_EPS = 1e-5f;
struct Taps {
    float w[MAXT + 1];
    int n;
};

// out[b,z,y,x] = sum_k taps[k] * in[.. coordinate(axis) + k - n/2 ..]   (cross-correlation, zero padding)
__global__ void __launch_bounds__(NT)
vox_blur_axis_kernel(const float* __restrict__ in, float* __restrict__ out, const Taps taps, int V, long long total, int axis,
                     int reversed) {
    const long long i = (long long)blockIdx.x * NT + threadIdx.x;
    if (i >= total) return;
    const int x = (int)(i % V), y = (int)((i / V) % V), z = (int)((i / ((long long)V * V)) % V);
    const int c = axis == 1 ? z : (axis == 2 ? y : x);
    const long long stride = axis == 1 ? (long long)V * V : (axis == 2 ? V : 1);
    const int h = taps.n / 2;
    float s = 0.f;
    for (int k = 0; k < taps.n; ++k) {
        const int cc = c + k - h;
        if (cc >= 0 && cc < V) s = fmaf(taps.w[reversed ? taps.n - 1 - k : k], __ldg(in + i + (long long)(cc - c) * stride), s);
    }
    out[i] = s;
}

// fwd: out = clamp(in * scale[b], 0, 1).  bwd: gin = gout * scale[b] * [0 <= in*scale <= 1], dscale[b] += sum gout*mask*in
__global__ void __launch_bounds__(NT)
vox_scale_clamp_kernel(const float* __restrict__ in, const float* __restrict__ scale, float* __restrict__ out, long long per_b) {
    const int b = blockIdx.y;
    const float sc = scale[b];
    for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < per_b; i += (long long)gridDim.x * NT)
        out[b * per_b + i] = clamp_nan(in[b * per_b + i] * sc, 0.f, 1.f);
}
__global__ void __launch_bounds__(NT)
vox_scale_clamp_bwd_kernel(const float* __restrict__ in, const float* __restrict__ scale, const float* __restrict__ gout,
                           float* __restrict__ gin, float* __restrict__ dscale, long long per_b) {
    __shared__ float red[32];
    const int b = blockIdx.y;
    const float sc = scale[b];
    float acc = 0.f;
    for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < per_b; i += (long long)gridDim.x * NT) {
        const float v = in[b * per_b + i], t = v * sc;
        const float g = (t >= 0.f && t <= 1.f) ? gout[b * per_b + i] : 0.f;
        gin[b * per_b + i] = g * sc;
        acc = fmaf(g, v, acc);
    }
    const float tot = b3d::block_sum(acc, red);
    if (threadIdx.x == 0 && tot != 0.f) atomicAdd(dscale + b, tot);
}

// one thread per (b, y, x) column.  probs [B,V+1,V,V] nullable, sil [B,V,V] nullable (flipped along y).
__global__ void __launch_bounds__(NT)
vox_termination_kernel(const float* __restrict__ vox, int V, int mode, float* __restrict__ probs, float* __restrict__ sil,
                       long long ncols) {
    const long long i = (long long)blockIdx.x * NT + threadIdx.x;
    if (i >= ncols) return;
    const int x = (int)(i % V), y = (int)((i / V) % V);
    const long long b = i / ((long long)V * V);
    const float c0 = mode == B3D_MODE_REFERENCE ? expf(TERM_EPS) : 1.f;       // the epsilon pad rows (D10)
    const float* col = vox + b * V * V * V + (long long)y * V + x;
    float T = 1.f, acc = 0.f;
    for (int z = 0; z < V; ++z) {
        const float o = clamp_nan(col[(long long)z * V * V], TERM_EPS, 1.f - TERM_EPS);
        const float t = (z == 0 ? c0 : 1.f) * o * T;
        if (probs) probs[((b * (V + 1) + z) * V + y) * V + x] = t;
        acc += t;
        T *= (1.f - o);
    }
    if (probs) probs[((b * (V + 1) + V) * V + y) * V + x] = T * c0;           // background cell
    if (sil) sil[(b * V + (V - 1 - y)) * V + x] = acc;
}

// dvox from dsil: d sil / d o_z = T_z (1 - Q_{z+1}) (z = 0: c0 - Q_1), through clamp(eps, 1-eps)
__global__ void __launch_bounds__(NT)
vox_termination_bwd_kernel(const float* __restrict__ vox, const float* __restrict__ dsil, int V, int mode,
                           float* __restrict__ dvox, long long ncols) {
    const long long i = (long long)blockIdx.x * NT + threadIdx.x;
    if (i >= ncols) return;
    const int x = (int)(i % V), y = (int)((i / V) % V);
    const long long b = i / ((long long)V * V);
    const float c0 = mode == B3D_MODE_REFERENCE ? expf(TERM_EPS) : 1.f;
    const long long base = b * V * V * V + (long long)y * V + x, zs = (long long)V * V;
    const float g = dsil[(b * V + (V - 1 - y)) * V + x];
    float T = 1.f;
    for (int z = 0; z < V; ++z) {                   // forward sweep: stash T_z
        const float o = clamp_nan(vox[base + z * zs], TERM_EPS, 1.f - TERM_EPS);
        dvox[base + z * zs] = T;
        T *= (1.f - o);
    }
    float Q = 0.f;
    for (int z = V - 1; z >= 0; --z) {
        const float v = vox[base + z * zs];
        const float o = clamp_nan(v, TERM_EPS, 1.f - TERM_EPS);
        const float coef = z == 0 ? (c0 - Q) : dvox[base + z * zs] * (1.f - Q);
        dvox[base + z * zs] = (v >= TERM_EPS && v <= 1.f - TERM_EPS) ? g * coef : 0.f;
        Q = fmaf(1.f - o, Q, o);
    }
}

// dgrid -> d/d(grid coords) of every in-bounds point (sorted list), masked by the splat clamp (0 <= G <= 1 is
// applied by the caller on dgrid).  Writes dpg[original index].
__device__ __forceinline__ void axis_w(float g, float f, int mode, float& w0, float& w1) {
    w1 = g - f;
    w0 = mode == B3D_MODE_REFERENCE ? (1.f - g) - f : 1.f - w1;
}
__global__ void __launch_bounds__(NT)
vox_gather_kernel(const float4* __restrict__ sorted, const int32_t* __restrict__ bin_start, int nbins, int N, int V, int mode,
                  const float* __restrict__ dgrid, float4* __restrict__ dpg) {
    const int b = blockIdx.y;
    const int cnt = bin_start[(size_t)b * (nbins + 1) + nbins];
    const int n = blockIdx.x * NT + threadIdx.x;
    if (n >= cnt) return;
    const float4 g = sorted[(size_t)b * N + n];
    const float fz = floorf(g.x), fy = floorf(g.y), fx = floorf(g.z);
    float wz[2], wy[2], wx[2];
    axis_w(g.x, fz, mode, wz[0], wz[1]);
    axis_w(g.y, fy, mode, wy[0], wy[1]);
    axis_w(g.z, fx, mode, wx[0], wx[1]);
    const float* d = dgrid + (size_t)b * V * V * V;
    float dz = 0.f, dy = 0.f, dx = 0.f;
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const float v = d[((size_t)((int)fz + i) * V + (int)fy + j) * V + (int)fx + k];
                dz += v * (i ? 1.f : -1.f) * wy[j] * wx[k];
                dy += v * wz[i] * (j ? 1.f : -1.f) * wx[k];
                dx += v * wz[i] * wy[j] * (k ? 1.f : -1.f);
            }
    dpg[(size_t)b * N + __float_as_int(g.w)] = make_float4(dz, dy, dx, 0.f);
}

// raw splat (no clamp) from the sorted list; clamp + mask kept separate for the adjoint
__global__ void __launch_bounds__(NT)
vox_splat_sorted_kernel(const float4* __restrict__ sorted, const int32_t* __restrict__ bin_start, int nbins, int N, int V,
                        int mode, float* __restrict__ grid) {
    const int b = blockIdx.y;
    const int cnt = bin_start[(size_t)b * (nbins + 1) + nbins];
    const int n = blockIdx.x * NT + threadIdx.x;
    if (n >= cnt) return;
    const float4 g = sorted[(size_t)b * N + n];
    const float fz = floorf(g.x), fy = floorf(g.y), fx = floorf(g.z);
    float wz[2], wy[2], wx[2];
    axis_w(g.x, fz, mode, wz[0], wz[1]);
    axis_w(g.y, fy, mode, wy[0], wy[1]);
    axis_w(g.z, fx, mode, wx[0], wx[1]);
    float* gb = grid + (size_t)b * V * V * V;
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int k = 0; k < 2; ++k)
                atomicAdd(gb + ((size_t)((int)fz + i) * V + (int)fy + j) * V + (int)fx + k, __fmul_rn(__fmul_rn(wz[i], wy[j]), wx[k]));
}
// in place: g -> clamp(g,0,1);  mask variant: d -> d * [0 <= g <= 1]
__global__ void __launch_bounds__(NT) vox_clamp01_kernel(float* __restrict__ x, long long n) {
    for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < n; i += (long long)gridDim.x * NT) x[i] = clamp_nan(x[i], 0.f, 1.f);
}
__global__ void __launch_bounds__(NT)
vox_mask01_kernel(float* __restrict__ d, const float* __restrict__ raw, long long n) {
    for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < n; i += (long long)gridDim.x * NT) {
        const float g = raw[i];
        d[i] = (g >= 0.f && g <= 1.f) ? d[i] : 0.f;
    }
}

int fill(Taps& t, const float* h, int n) {
    B3D_REQUIRE(h && n >= 1 && n <= MAXT && (n & 1), B3D_EINVAL, "taps: need an odd count <= %d", MAXT);
    for (int i = 0; i < n; ++i) t.w[i] = h[i];
    t.n = n;
    return B3D_OK;
}
inline int blocks(long long n) { return (int)((n + NT - 1) / NT); }
inline int capped(long long n) {
    const long long b = (n + NT - 1) / NT;
    return (int)(b < 132 * 16 ? (b > 0 ? b : 1) : 132 * 16);
}
}  // namespace

namespace b3d {
int vox_gather_launch(const float* sorted, const int32_t* bin_start, const float* dgrid, int B, int N, int V, int mode,
                      float* dpg, cudaStream_t st) {
    vox_gather_kernel<<<dim3(blocks(N), B), NT, 0, st>>>((const float4*)sorted, bin_start, b3d_pc_bin_count(V), N, V, mode, dgrid,
                                                        (float4*)dpg);
    B3D_LAUNCH_OK();
    return B3D_OK;
}
}  // namespace b3d

extern "C" {

int b3d_vox_blur_axis(const float* in, float* out, const float* taps_host, int ktaps, int axis, int reversed, int B, int V,
                      void* stream) {
    B3D_REQUIRE(B >= 0 && V >= 1 && axis >= 1 && axis <= 3, B3D_EINVAL, "b3d_vox_blur_axis: bad arguments");
    Taps t;
    if (int rc = fill(t, taps_host, ktaps)) return rc;
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(in && out && in != out, B3D_EINVAL, "b3d_vox_blur_axis: null or aliased pointers");
    const long long total = (long long)B * V * V * V;
    vox_blur_axis_kernel<<<blocks(total), NT, 0, (cudaStream_t)stream>>>(in, out, t, V, total, axis, reversed);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

int b3d_vox_scale_clamp(const float* in, const float* scale, float* out, int B, int V, void* stream) {
    B3D_REQUIRE(B >= 0 && V >= 1, B3D_EINVAL, "b3d_vox_scale_clamp: bad sizes");
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(in && scale && out, B3D_EINVAL, "b3d_vox_scale_clamp: null pointer");
    const long long per_b = (long long)V * V * V;
    vox_scale_clamp_kernel<<<dim3(capped(per_b), B), NT, 0, (cudaStream_t)stream>>>(in, scale, out, per_b);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

int b3d_vox_scale_clamp_bwd(const float* in, const float* scale, const float* gout, float* gin, float* dscale, int B, int V,
                            void* stream) {
    B3D_REQUIRE(B >= 0 && V >= 1, B3D_EINVAL, "b3d_vox_scale_clamp_bwd: bad sizes");
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(in && scale && gout && gin && dscale, B3D_EINVAL, "b3d_vox_scale_clamp_bwd: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    B3D_CUDA_OK(cudaMemsetAsync(dscale, 0, sizeof(float) * B, st));
    const long long per_b = (long long)V * V * V;
    vox_scale_clamp_bwd_kernel<<<dim3(capped(per_b) < 64 ? capped(per_b) : 64, B), NT, 0, st>>>(in, scale, gout, gin, dscale, per_b);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

int b3d_vox_termination(const float* vox, int B, int V, int mode, float* probs, float* sil, void* stream) {
    B3D_REQUIRE(B >= 0 && V >= 1 && (mode == 0 || mode == 1), B3D_EINVAL, "b3d_vox_termination: bad arguments");
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(vox && (probs || sil), B3D_EINVAL, "b3d_vox_termination: null pointer");
    const long long ncols = (long long)B * V * V;
    vox_termination_kernel<<<blocks(ncols), NT, 0, (cudaStream_t)stream>>>(vox, V, mode, probs, sil, ncols);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

int b3d_vox_termination_bwd(const float* vox, const float* dsil, int B, int V, int mode, float* dvox, void* stream) {
    B3D_REQUIRE(B >= 0 && V >= 1 && (mode == 0 || mode == 1), B3D_EINVAL, "b3d_vox_termination_bwd: bad arguments");
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(vox && dsil && dvox, B3D_EINVAL, "b3d_vox_termination_bwd: null pointer");
    const long long ncols = (long long)B * V * V;
    vox_termination_bwd_kernel<<<blocks(ncols), NT, 0, (cudaStream_t)stream>>>(vox, dsil, V, mode, dvox, ncols);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

// raw (unclamped) occupancy from the bin-sorted points; grid zeroed by the call
int b3d_vox_splat_sorted(const float* sorted, const int32_t* bin_start, int B, int N, int V, int mode, float* grid, void* stream) {
    B3D_REQUIRE(B >= 0 && N >= 0 && V >= 2 && (mode == 0 || mode == 1), B3D_EINVAL, "b3d_vox_splat_sorted: bad arguments");
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(grid && bin_start, B3D_EINVAL, "b3d_vox_splat_sorted: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    B3D_CUDA_OK(cudaMemsetAsync(grid, 0, sizeof(float) * (size_t)B * V * V * V, st));
    if (N == 0) return B3D_OK;
    B3D_REQUIRE(sorted, B3D_EINVAL, "b3d_vox_splat_sorted: null pointer");
    vox_splat_sorted_kernel<<<dim3(blocks(N), B), NT, 0, st>>>((const float4*)sorted, bin_start, b3d_pc_bin_count(V), N, V, mode, grid);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

int b3d_vox_clamp01(float* x, long long n, void* stream) {
    if (n <= 0) return B3D_OK;
    B3D_REQUIRE(x, B3D_EINVAL, "b3d_vox_clamp01: null pointer");
    vox_clamp01_kernel<<<capped(n), NT, 0, (cudaStream_t)stream>>>(x, n);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

// d *= [0 <= raw <= 1]  then  dpg[orig] = corner gather of d  (adjoint of clamp + splat)
int b3d_vox_gather(const float* sorted, const int32_t* bin_start, const float* raw, float* dgrid, int B, int N, int V, int mode,
                   float* dpg, void* stream) {
    B3D_REQUIRE(B >= 0 && N >= 0 && V >= 2 && (mode == 0 || mode == 1), B3D_EINVAL, "b3d_vox_gather: bad arguments");
    if (B == 0 || N == 0) return B3D_OK;
    B3D_REQUIRE(sorted && bin_start && raw && dgrid && dpg, B3D_EINVAL, "b3d_vox_gather: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const long long cells = (long long)B * V * V * V;
    vox_mask01_kernel<<<capped(cells), NT, 0, st>>>(dgrid, raw, cells);
    B3D_LAUNCH_OK();
    return b3d::vox_gather_launch(sorted, bin_start, dgrid, B, N, V, mode, dpg, st);
}
}
