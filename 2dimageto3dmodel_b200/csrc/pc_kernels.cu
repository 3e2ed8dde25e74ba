// Point-cloud "effective loss" path (SURVEY.md §8 rows a1-a5) for sm_90a.
//
//   pc_project_kernel        a1+a2+a3(index part): quaternion rotate, perspective divide, grid coords,
//                            in-bounds mask, floor index buffer.  Uses round-to-nearest intrinsics in the
//                            reference's operation order (no FMA contraction) so that floor(g) — the
//                            reference's int64 index buffer — is reproduced bit for bit.
//   pc_sil_fwd_kernel        a3+a4+a5 fused, mode R: one CTA owns a TY x 16 patch of (y,x) columns over
//                            the whole depth in shared memory; points are splatted with shared-memory
//                            atomics (no global atomics, the V^3 grid never touches HBM), then each thread
//                            walks one column: clamp -> 21-tap z blur (register-blocked, 8 outputs per
//                            window) -> scale/clamp -> ray termination -> silhouette.
//   pc_sil_bwd_kernel        recomputes the patch (+1 halo so every point is owned by exactly one CTA),
//                            runs the ray-march / clamp / blur adjoints column-wise in shared memory and
//                            gathers d/d(grid coords) per point: no dense gradient grid in HBM either.
//   pc_blur_xy_kernel        mode P: clamp + x blur + y blur of one z slice tile with its halo (forward), or the
//                            transposed y, x blur + clamp mask (backward), between the two workspace grids.
//   pc_sil_p_fwd_kernel      mode P: the mode-R forward without its splat (z blur, scale/clamp, ray march) over the
//                            x/y-blurred grid; pc_sil_p_bwd_kernel its column adjoints, written back over that grid.
//   pc_project_bwd_kernel    adjoint of projection + rotation + quaternion normalisation.
//   pc_splat_grid_kernel     materialised occupancy grid (parity tests).
//
// Reference lines restated: quaternions/points_quaternions.py:41-81, quaternions/operations.py:68-136,
// camera/coordinate_system_transformation.py:20-39, utils/trilinear_interpolation.py:17-74,
// utils/smooth_voxels.py:44-84, utils/effective_loss_function.py:18-81 (all under /root/reference/code).
#include "b3d_common.cuh"

namespace {

using b3d::clamp_nan;

constexpr int TX = 16;         // patch width in x (columns are contiguous over x in shared memory)
constexpr int ZB = 8;          // blur outputs produced per register window
constexpr int MAX_TAPS = 63;
constexpr int NTHREADS = 256;
// field_of_view = 1.875 and camera_view_distance = 2.0 are what effective_loss_function.py:69-70 passes
constexpr float TERM_EPS = 1e-5f;      // effective_loss_function.py:18

struct Taps {
    float w[MAX_TAPS + 1];
    int n;
    int finite;     // every tap is finite: blocks of a column whose blur window holds no occupied cell can be skipped (0 * tap = 0)
};

// ----------------------------------------------------------------------------------------------
// exact-order fp32 helpers (mirror torch's separate rounding of every elementwise op)
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }

struct Quat {
    float w, x, y, z;
};

// operations.py:83-86, evaluated left to right like the Python expressions
__device__ __forceinline__ Quat hamilton_exact(const Quat a, const Quat b) {
    Quat r;
    r.w = sub(sub(sub(mul(a.w, b.w), mul(a.x, b.x)), mul(a.y, b.y)), mul(a.z, b.z));
    r.x = sub(add(add(mul(a.w, b.x), mul(a.x, b.w)), mul(a.y, b.z)), mul(a.z, b.y));
    r.y = sub(add(add(mul(a.w, b.y), mul(a.y, b.w)), mul(a.z, b.x)), mul(a.x, b.z));
    r.z = sub(add(add(mul(a.w, b.z), mul(a.z, b.w)), mul(a.x, b.y)), mul(a.y, b.x));
    return r;
}

__device__ __forceinline__ Quat hamilton(const Quat a, const Quat b) {
    Quat r;
    r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
    r.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
    r.y = a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z;
    r.z = a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x;
    return r;
}
__device__ __forceinline__ Quat conj(const Quat a) { return Quat{a.w, -a.x, -a.y, -a.z}; }

// F.normalize(q, dim=-1): q / max(||q||_2, 1e-12)   (points_quaternions.py:53-56)
__device__ __forceinline__ Quat normalize_quat(const float* q, float* norm_out) {
    const float w = q[0], x = q[1], y = q[2], z = q[3];
    float n = __fsqrt_rn(add(add(add(mul(w, w), mul(x, x)), mul(y, y)), mul(z, z)));
    n = n < 1e-12f ? 1e-12f : n;
    if (norm_out) *norm_out = n;
    return Quat{__fdiv_rn(w, n), __fdiv_rn(x, n), __fdiv_rn(y, n), __fdiv_rn(z, n)};
}

// ----------------------------------------------------------------------------------------------
// projection
// ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NTHREADS)
pc_project_kernel(const float* __restrict__ points, const float* __restrict__ quat, int N, int V,
                  float FOV, float CAM_DIST, float4* __restrict__ pg, float* __restrict__ coords, int32_t* __restrict__ base,
                  uint8_t* __restrict__ inb) {
    const int b = blockIdx.y;
    const int n = blockIdx.x * NTHREADS + threadIdx.x;
    if (n >= N) return;
    const Quat q = normalize_quat(quat + 4 * b, nullptr);
    const size_t i = (size_t)b * N + n;
    const float p0 = points[3 * i + 0], p1 = points[3 * i + 1], p2 = points[3 * i + 2];
    const Quat P{0.f, p0, p1, p2};                       // points_quaternions.py:33 (pad scalar 0)
    const Quat r = hamilton_exact(hamilton_exact(q, P), conj(q));   // :72-75 (forward direction)
    // coordinate_system_transformation.py:25-39: columns are (z, y, x)
    const float z = r.x;
    const float den = add(z, CAM_DIST);
    const float y = __fdiv_rn(mul(r.y, FOV), den);
    const float x = __fdiv_rn(mul(r.z, FOV), den);
    // trilinear_interpolation.py:23-25, scalars cast to fp32 as torch does
    const float hi = (float)(0.5 - 1e-6), lo = (float)(-0.5 + 1e-6);
    const bool ok = (z < hi) && (z > lo) && (y < hi) && (y > lo) && (x < hi) && (x > lo);
    // trilinear_interpolation.py:34
    const float vm1 = (float)(V - 1);
    const float gz = mul(vm1, add(z, 0.5f)), gy = mul(vm1, add(y, 0.5f)), gx = mul(vm1, add(x, 0.5f));
    pg[i] = make_float4(gz, gy, gx, ok ? 1.f : 0.f);
    if (coords) {
        coords[3 * i + 0] = z;
        coords[3 * i + 1] = y;
        coords[3 * i + 2] = x;
    }
    if (base) {
        base[3 * i + 0] = (int32_t)floorf(gz);
        base[3 * i + 1] = (int32_t)floorf(gy);
        base[3 * i + 2] = (int32_t)floorf(gx);
    }
    if (inb) inb[i] = ok ? 1 : 0;
}

// trilinear weights of one axis: trilinear_interpolation.py:66 (mode R keeps `1.0 - grid - floor`)
__device__ __forceinline__ void axis_weights(float g, float f, int mode, float& w0, float& w1) {
    w1 = sub(g, f);
    w0 = (mode == B3D_MODE_REFERENCE) ? sub(sub(1.0f, g), f) : sub(1.0f, w1);
}

// ----------------------------------------------------------------------------------------------
// binning: counting sort of the in-bounds points of one sample by the (BY x BX) cell bin of their base
// voxel (y,x).  One CTA per sample; histogram, scan and scatter stay in shared memory.
//   sorted[b, pos] = (gz, gy, gx, bits(original index));   bin_start[b, 0..nbins]
// ----------------------------------------------------------------------------------------------
constexpr int BIN_Y = 8, BIN_X = 16;
constexpr int BIN_THREADS = 512;
constexpr int MAX_BINS = 4096;

__device__ __forceinline__ int bin_of(float gy, float gx, int nbx) {
    return ((int)floorf(gy) / BIN_Y) * nbx + (int)floorf(gx) / BIN_X;
}

__global__ void __launch_bounds__(BIN_THREADS)
pc_bin_kernel(const float4* __restrict__ pg, int N, int nbx, int nbins, float4* __restrict__ sorted,
              int32_t* __restrict__ bin_start) {
    __shared__ int hist[MAX_BINS + 1];
    __shared__ int wsum[BIN_THREADS / 32];
    __shared__ int carry;
    const int b = blockIdx.x, tid = threadIdx.x;
    const float4* p = pg + (size_t)b * N;
    for (int i = tid; i <= nbins; i += BIN_THREADS) hist[i] = 0;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (int n = tid; n < N; n += BIN_THREADS) {
        const float4 g = p[n];
        if (g.w != 0.f) atomicAdd(&hist[bin_of(g.y, g.z, nbx)], 1);
    }
    __syncthreads();
    // exclusive scan of hist[0..nbins) in chunks of BIN_THREADS
    for (int base = 0; base < nbins; base += BIN_THREADS) {
        const int i = base + tid;
        const int v = i < nbins ? hist[i] : 0;
        int x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, x, o);
            if ((tid & 31) >= o) x += y;
        }
        if ((tid & 31) == 31) wsum[tid >> 5] = x;
        __syncthreads();
        int off = carry;
        for (int w = 0; w < (tid >> 5); ++w) off += wsum[w];
        if (i < nbins) hist[i] = off + x - v;
        __syncthreads();
        if (tid == BIN_THREADS - 1) carry = off + x;
        __syncthreads();
    }
    if (tid == 0) hist[nbins] = carry;
    __syncthreads();
    int32_t* bs = bin_start + (size_t)b * (nbins + 1);
    for (int i = tid; i <= nbins; i += BIN_THREADS) bs[i] = hist[i];
    __syncthreads();
    float4* out = sorted + (size_t)b * N;
    for (int n = tid; n < N; n += BIN_THREADS) {
        const float4 g = p[n];
        if (g.w == 0.f) continue;
        const int pos = atomicAdd(&hist[bin_of(g.y, g.z, nbx)], 1);     // hist doubles as the cursor
        out[pos] = make_float4(g.x, g.y, g.z, __int_as_float(n));
    }
}

// ----------------------------------------------------------------------------------------------
// register-blocked 1-D blur along z of one shared-memory column (stride cs between depths).
// out[j] = sum_k taps[k] * |in[zb + j + k - KT/2]|, zero padding (smooth_voxels.py:69-73).  The stored
// occupancy is already clamped to [0,1]; its sign bit carries the clamp mask (backward), hence fabsf.
// ----------------------------------------------------------------------------------------------
template <int KT, bool REVERSED, bool ABS>
__device__ __forceinline__ void blur_window(const float* colp, int cs, int V, int zb, const Taps& taps,
                                            float (&out)[ZB]) {
    if constexpr (KT > 0) {
        constexpr int H = KT / 2, W = ZB + KT - 1;
        float in[W];
        if (zb >= H && zb + ZB + H <= V) {
#pragma unroll
            for (int i = 0; i < W; ++i) in[i] = ABS ? fabsf(colp[(zb - H + i) * cs]) : colp[(zb - H + i) * cs];
        } else {
#pragma unroll
            for (int i = 0; i < W; ++i) {
                const int z = zb - H + i;
                const float v = (z >= 0 && z < V) ? colp[z * cs] : 0.f;
                in[i] = ABS ? fabsf(v) : v;
            }
        }
#pragma unroll
        for (int j = 0; j < ZB; ++j) {
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < KT; ++k) s = fmaf(taps.w[REVERSED ? KT - 1 - k : k], in[j + k], s);
            out[j] = s;
        }
    } else {
        const int kt = taps.n, H = kt / 2;
#pragma unroll
        for (int j = 0; j < ZB; ++j) out[j] = 0.f;
        for (int k = 0; k < kt; ++k) {
            const float t = taps.w[REVERSED ? kt - 1 - k : k];
#pragma unroll
            for (int j = 0; j < ZB; ++j) {
                const int z = zb + j + k - H;
                const float v = (z >= 0 && z < V) ? colp[z * cs] : 0.f;
                out[j] = fmaf(t, ABS ? fabsf(v) : v, out[j]);
            }
        }
    }
}

// occupancy after smooth_voxels.py:80-82 and effective_loss_function.py:33
__device__ __forceinline__ float scaled(float S, bool has_scale, float sc) {
    return has_scale ? clamp_nan(S * sc, 0.f, 1.f) : S;
}

constexpr int TILE_THREADS = 512;

// One sorted record (gz, gy, gx, bits(index)) splatted into a shared patch covering cells [cy0, cy1] x [cx0, cx1]
// (row pitch `pitch`), depth-major.  zlo / zhi [ncol] (initialised to V / -1 by the caller): occupied depth range of every
// column — cells outside it are exactly zero, so their blur, clamp and ray-march terms are constants (the sparsity skip of
// the fwd / bwd kernels).
__device__ __forceinline__ void splat_record(const float4 g, int cy0, int cy1, int cx0, int cx1, int pitch, int ncol,
                                             int mode, float* A, int* zlo, int* zhi) {
    const float fzf = floorf(g.x), fyf = floorf(g.y), fxf = floorf(g.z);
    const int ly = (int)fyf - cy0, lx = (int)fxf - cx0;
    if (ly < -1 || ly > cy1 - cy0 || lx < -1 || lx > cx1 - cx0) return;
    const int fz = (int)fzf;
    float wz[2], wy[2], wx[2];
    axis_weights(g.x, fzf, mode, wz[0], wz[1]);
    axis_weights(g.y, fyf, mode, wy[0], wy[1]);
    axis_weights(g.z, fxf, mode, wx[0], wx[1]);
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        const int cy = ly + j;
        if (cy < 0 || cy > cy1 - cy0) continue;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const int cx = lx + k;
            if (cx < 0 || cx > cx1 - cx0) continue;
            atomicMin(&zlo[cy * pitch + cx], fz);
            atomicMax(&zhi[cy * pitch + cx], fz + 1);
#pragma unroll
            for (int i = 0; i < 2; ++i)     // trilinear_interpolation.py:40-41: (gz_i*gy_j)*gx_k
                atomicAdd(&A[(fz + i) * ncol + cy * pitch + cx], mul(mul(wz[i], wy[j]), wx[k]));
        }
    }
}

// fn(record) for every record of bins [bx_lo, bx_hi] x [by_lo, by_hi], all threads of the CTA taking part
template <typename F>
__device__ __forceinline__ void for_each_record(const float4* __restrict__ sorted, const int32_t* __restrict__ bs, int nbx,
                                                int by_lo, int by_hi, int bx_lo, int bx_hi, F fn) {
    for (int by = by_lo; by <= by_hi; ++by) {
        const int lo = bs[by * nbx + bx_lo], hi = bs[by * nbx + bx_hi + 1];
        for (int n = lo + threadIdx.x; n < hi; n += TILE_THREADS) fn(__ldg(sorted + n));
    }
}

// in place: G -> clamp(G, 0, 1) with the sign bit set where the clamp was active (G outside [0,1])
__device__ __forceinline__ void clamp_patch(float* A, int n) {
    for (int i = threadIdx.x; i < n; i += TILE_THREADS) {
        const float g = A[i];
        const float c = clamp_nan(g, 0.f, 1.f);
        A[i] = (g >= 0.f && g <= 1.f) ? c : -c;
    }
}

// ----------------------------------------------------------------------------------------------
// forward of one patch of TY x TX columns A [V][ncol] (row pitch TX, first column (ty0, tx0)), shared by both modes.
// Work items are (column, block of ZB depths): every item blurs its block along z, turns it into occupancies and
// reduces it to (transmittance of the block, silhouette gathered inside the block); a second, short pass chains the
// blocks of each column.  ABS: A holds clamped occupancies with the clamp mask in the sign bit (mode R); otherwise A
// holds plain values (mode P: the occupancy already blurred along x and y).  zlo / zhi are read only when skip_ok.
// ----------------------------------------------------------------------------------------------
template <int KT, bool ABS>
__device__ __forceinline__ void sil_fwd_columns(const float* A, float* blkP, float* blkS, const int* zlo, const int* zhi,
                                                bool skip_ok, const Taps& taps, bool has_scale, float sc, float c0, int b,
                                                int V, int ncol, int ty0, int tx0, float* __restrict__ sil) {
    const int tid = threadIdx.x, nzb = (V + ZB - 1) / ZB;
    const int HB = (KT > 0 ? KT : taps.n) / 2;
    for (int it = tid; it < nzb * ncol; it += TILE_THREADS) {
        const int col = it % ncol, zb = (it / ncol) * ZB;
        float S[ZB];
        if (skip_ok && (zb + ZB - 1 < zlo[col] - HB || zb > zhi[col] + HB)) {
#pragma unroll
            for (int j = 0; j < ZB; ++j) S[j] = 0.f;             // no occupied cell within the taps' reach: the blur is exactly 0
        } else {
            blur_window<KT, false, ABS>(A + col, ncol, V, zb, taps, S);
        }
        float T = 1.f, acc = 0.f;
#pragma unroll
        for (int j = 0; j < ZB; ++j) {
            if (zb + j < V) {
                const float o = clamp_nan(scaled(S[j], has_scale, sc), TERM_EPS, 1.f - TERM_EPS);
                float term = o * T;                       // o_k * prod_{j<k}(1-o_j)
                if (zb + j == 0) term *= c0;
                acc += term;
                T *= (1.f - o);
            }
        }
        blkP[it] = T;
        blkS[it] = acc;
    }
    __syncthreads();
    for (int col = tid; col < ncol; col += TILE_THREADS) {
        const int y = ty0 + col / TX, x = tx0 + col % TX;
        if (y >= V || x >= V) continue;
        float T = 1.f, acc = 0.f;
        for (int k = 0; k < nzb; ++k) {
            acc = fmaf(T, blkS[k * ncol + col], acc);
            T *= blkP[k * ncol + col];
        }
        sil[((size_t)b * V + (V - 1 - y)) * V + x] = acc;   // flip(1): effective_loss_function.py:81
    }
}

// ----------------------------------------------------------------------------------------------
// forward, mode R: splat into the patch with shared-memory atomics, clamp, then the column work above
// ----------------------------------------------------------------------------------------------
template <int KT>
__global__ void __launch_bounds__(TILE_THREADS)
pc_sil_fwd_kernel(const float4* __restrict__ sorted, const int32_t* __restrict__ bin_start, const Taps taps,
                  const float* __restrict__ scale, int N, int V, int TY, int mode, int nbx, int nby,
                  float* __restrict__ sil) {
    extern __shared__ __align__(128) float sm[];
    const int b = blockIdx.z, ty0 = blockIdx.y * TY, tx0 = blockIdx.x * TX;
    const int ncol = TY * TX, nzb = (V + ZB - 1) / ZB;
    float* A = sm;                       // [V][ncol]
    float* blkP = A + V * ncol;          // [nzb][ncol] transmittance of the block
    float* blkS = blkP + nzb * ncol;     // [nzb][ncol] silhouette collected inside the block
    int* zlo = reinterpret_cast<int*>(blkS + nzb * ncol);    // [ncol] first / last occupied depth of the column
    int* zhi = zlo + ncol;
    const int tid = threadIdx.x;
    const int cy1 = min(ty0 + TY, V) - 1, cx1 = min(tx0 + TX, V) - 1;
    const float4* sp = sorted + (size_t)b * N;
    const int32_t* bs = bin_start + (size_t)b * (nbx * nby + 1);
    for (int i = tid; i < V * ncol; i += TILE_THREADS) A[i] = 0.f;
    for (int i = tid; i < ncol; i += TILE_THREADS) { zlo[i] = V; zhi[i] = -1; }
    __syncthreads();
    // the points of the bins overlapping base cells [ty0-1, cy1] x [tx0-1, cx1]
    for_each_record(sp, bs, nbx, max(ty0 - 1, 0) / BIN_Y, min(cy1 / BIN_Y, nby - 1), max(tx0 - 1, 0) / BIN_X,
                    min(cx1 / BIN_X, nbx - 1),
                    [&](const float4 g) { splat_record(g, ty0, cy1, tx0, cx1, TX, ncol, mode, A, zlo, zhi); });
    __syncthreads();
    clamp_patch(A, V * ncol);
    __syncthreads();

    const bool has_scale = scale != nullptr;
    const float sc = has_scale ? scale[b] : 1.f;
    const float c0 = (mode == B3D_MODE_REFERENCE) ? expf(TERM_EPS) : 1.f;   // D10 pad row
    // sparsity skip: exact only when 0 * tap and 0 * scale are 0 (finite taps / scale; NaN must propagate, SURVEY D4)
    const bool skip_ok = taps.finite && (!has_scale || fabsf(sc) <= 3.0e38f);
    sil_fwd_columns<KT, true>(A, blkP, blkS, zlo, zhi, skip_ok, taps, has_scale, sc, c0, b, V, ncol, ty0, tx0, sil);
}

// ----------------------------------------------------------------------------------------------
// backward of one patch, shared by both modes: A1 [V][ncol] holds the forward's input of the z blur (ABS as in
// sil_fwd_columns), row pitch `pitch`; columns with cy < TY and cx < TX are owned (their terms go into dscale).
// On return A1 holds d(input of the z blur) — masked by the sign bit when ABS — and A2 is scratch.
// ----------------------------------------------------------------------------------------------
template <int KT, bool ABS>
__device__ __forceinline__ void sil_bwd_columns(float* A1, float* A2, float* blkA, float* blkB, float* blkT, const int* zlo,
                                                const int* zhi, bool skip_ok, const Taps& taps, bool has_scale, float sc,
                                                float c0, const float* __restrict__ dsil, int b, int V, int ncol, int pitch,
                                                int TY, int ty0, int tx0, float* red, float* __restrict__ dscale) {
    const int tid = threadIdx.x, nzb = (V + ZB - 1) / ZB;
    const int nitems = nzb * ncol;
    const int HB = (KT > 0 ? KT : taps.n) / 2;

    // pass 1: S = blur_z(O); per block: a = prod(1-o), b = Q at block start for Q = 0 after the block
    for (int it = tid; it < nitems; it += TILE_THREADS) {
        const int col = it % ncol, zb = (it / ncol) * ZB;
        float S[ZB];
        if (skip_ok && (zb + ZB - 1 < zlo[col] - HB || zb > zhi[col] + HB)) {
#pragma unroll
            for (int j = 0; j < ZB; ++j) S[j] = 0.f;
        } else {
            blur_window<KT, false, ABS>(A1 + col, ncol, V, zb, taps, S);
        }
        float a = 1.f, q = 0.f;
#pragma unroll
        for (int j = ZB - 1; j >= 0; --j) {
            if (zb + j < V) {
                A2[(zb + j) * ncol + col] = S[j];
                const float o = clamp_nan(scaled(S[j], has_scale, sc), TERM_EPS, 1.f - TERM_EPS);
                q = fmaf(1.f - o, q, o);            // Q_z = o_z + (1 - o_z) Q_{z+1}
                a *= (1.f - o);
            }
        }
        blkA[it] = a;
        blkB[it] = q;
    }
    __syncthreads();
    // pass 2: chain the blocks of a column: T at the start of each block, Q just after each block
    for (int col = tid; col < ncol; col += TILE_THREADS) {
        float T = 1.f;
        for (int k = 0; k < nzb; ++k) {
            blkT[k * ncol + col] = T;
            T *= blkA[k * ncol + col];
        }
        float Q = 0.f;
        for (int k = nzb - 1; k >= 0; --k) {
            const float bq = blkB[k * ncol + col];
            blkB[k * ncol + col] = Q;               // Q just after block k
            Q = fmaf(blkA[k * ncol + col], Q, bq);
        }
    }
    __syncthreads();
    // pass 3: d sil / d S inside each block
    float dsc = 0.f;
    for (int it = tid; it < nitems; it += TILE_THREADS) {
        const int col = it % ncol, zb = (it / ncol) * ZB;
        const int cy = col / pitch, cx = col % pitch;
        const int y = ty0 + cy, x = tx0 + cx;
        if (y >= V || x >= V) continue;
        if (skip_ok && (zb + ZB - 1 < zlo[col] - HB || zb > zhi[col] + HB)) continue;     // dS == 0 == what A2 already holds
        const bool owned = cy < TY && cx < TX;      // halo columns are owned by the neighbour patch
        const float go = dsil[((size_t)b * V + (V - 1 - y)) * V + x];
        float S[ZB], o[ZB], Tz[ZB];
        float T = blkT[it];
#pragma unroll
        for (int j = 0; j < ZB; ++j) {
            S[j] = (zb + j < V) ? A2[(zb + j) * ncol + col] : 0.f;
            o[j] = clamp_nan(scaled(S[j], has_scale, sc), TERM_EPS, 1.f - TERM_EPS);
            Tz[j] = T;
            T *= (1.f - o[j]);
        }
        float Q = blkB[it];
#pragma unroll
        for (int j = ZB - 1; j >= 0; --j) {
            if (zb + j < V) {
                const float t = has_scale ? S[j] * sc : S[j];
                const float s2 = has_scale ? clamp_nan(t, 0.f, 1.f) : S[j];
                const float coef = (zb + j == 0) ? (c0 - Q) : Tz[j] * (1.f - Q);   // d sil / d o_z
                float d = go * coef;
                d = (s2 >= TERM_EPS && s2 <= 1.f - TERM_EPS) ? d : 0.f;           // clamp(eps, 1-eps) adjoint
                if (has_scale) {
                    d = (t >= 0.f && t <= 1.f) ? d : 0.f;                         // clamp(0, 1) adjoint
                    if (owned) dsc = fmaf(d, S[j], dsc);
                    d *= sc;
                }
                A2[(zb + j) * ncol + col] = d;
                Q = fmaf(1.f - o[j], Q, o[j]);
            }
        }
    }
    if (dscale) {
        const float tot = b3d::block_sum(dsc, red);
        if (tid == 0 && tot != 0.f) atomicAdd(dscale + b, tot);
    }
    __syncthreads();
    // pass 4: dG = mask * blur_z^T(dS)
    for (int it = tid; it < nitems; it += TILE_THREADS) {
        const int col = it % ncol, zb = (it / ncol) * ZB;
        if (skip_ok && (zb + ZB - 1 < zlo[col] - 2 * HB || zb > zhi[col] + 2 * HB)) continue;   // dG == 0 == the empty cells of A1
        float D[ZB];
        blur_window<KT, true, false>(A2 + col, ncol, V, zb, taps, D);
#pragma unroll
        for (int j = 0; j < ZB; ++j) {
            const int z = zb + j;
            if (z < V) A1[z * ncol + col] = (ABS && signbit(A1[z * ncol + col])) ? 0.f : D[j];
        }
    }
    __syncthreads();
}

// ----------------------------------------------------------------------------------------------
// backward, mode R (patch with a +1 halo so that every point is owned by exactly one CTA): splat + clamp as in the
// forward, the column adjoints above, then the gather to the points straight from shared memory
// ----------------------------------------------------------------------------------------------
template <int KT>
__global__ void __launch_bounds__(TILE_THREADS)
pc_sil_bwd_kernel(const float4* __restrict__ sorted, const int32_t* __restrict__ bin_start, const Taps taps,
                  const float* __restrict__ scale, const float* __restrict__ dsil, int N, int V, int TY, int mode,
                  int nbx, int nby, float4* __restrict__ dpg, float* __restrict__ dscale) {
    extern __shared__ __align__(128) float sm[];
    __shared__ float red[32];
    const int b = blockIdx.z, ty0 = blockIdx.y * TY, tx0 = blockIdx.x * TX;
    const int cy1 = min(ty0 + TY, V - 1), cx1 = min(tx0 + TX, V - 1);     // extended patch, clipped to the grid
    const int EX = TX + 1, ncol = (TY + 1) * EX, nzb = (V + ZB - 1) / ZB;
    float* A1 = sm;                      // clamped occupancy (sign = clamp mask) -> dG
    float* A2 = A1 + V * ncol;           // blurred S -> dS
    float* blkA = A2 + V * ncol;         // [nzb][ncol] transmittance of the block
    float* blkB = blkA + nzb * ncol;     // [nzb][ncol] offset of the block's Q recurrence -> Q just after the block
    float* blkT = blkB + nzb * ncol;     // [nzb][ncol] transmittance at the start of the block
    int* zlo = reinterpret_cast<int*>(blkT + nzb * ncol);    // [ncol] first / last occupied depth of the column
    int* zhi = zlo + ncol;
    const int tid = threadIdx.x;
    const float4* sp = sorted + (size_t)b * N;
    const int32_t* bs = bin_start + (size_t)b * (nbx * nby + 1);
    for (int i = tid; i < V * ncol; i += TILE_THREADS) A1[i] = 0.f;
    for (int i = tid; i < ncol; i += TILE_THREADS) { zlo[i] = V; zhi[i] = -1; }
    __syncthreads();
    for_each_record(sp, bs, nbx, max(ty0 - 1, 0) / BIN_Y, min(cy1 / BIN_Y, nby - 1), max(tx0 - 1, 0) / BIN_X,
                    min(cx1 / BIN_X, nbx - 1),
                    [&](const float4 g) { splat_record(g, ty0, cy1, tx0, cx1, EX, ncol, mode, A1, zlo, zhi); });
    __syncthreads();
    const int oy1 = min(ty0 + TY, V) - 1, ox1 = min(tx0 + TX, V) - 1;   // owned base cells (the gather at the end)
    const int gby_lo = ty0 / BIN_Y, gby_hi = min(oy1 / BIN_Y, nby - 1);
    const int gbx_lo = tx0 / BIN_X, gbx_hi = min(ox1 / BIN_X, nbx - 1);
    clamp_patch(A1, V * ncol);
    __syncthreads();

    const bool has_scale = scale != nullptr;
    const float sc = has_scale ? scale[b] : 1.f;
    const float c0 = (mode == B3D_MODE_REFERENCE) ? expf(TERM_EPS) : 1.f;
    // sparsity skip (see the forward kernel): S == 0 exactly outside [zlo - H, zhi + H]; there o = eps is clamped, so
    // d sil / d S == 0 as well, and the transposed blur of dS vanishes outside [zlo - 2H, zhi + 2H]
    const bool skip_ok = taps.finite && (!has_scale || fabsf(sc) <= 3.0e38f);
    sil_bwd_columns<KT, true>(A1, A2, blkA, blkB, blkT, zlo, zhi, skip_ok, taps, has_scale, sc, c0, dsil, b, V, ncol, EX, TY,
                              ty0, tx0, red, dscale);

    // gather: every in-bounds point is owned by the patch holding its base cell
    float4* dp = dpg + (size_t)b * N;
    auto gather = [&](const float4 g) {
        const float fzf = floorf(g.x), fyf = floorf(g.y), fxf = floorf(g.z);
        const int ly = (int)fyf - ty0, lx = (int)fxf - tx0;
        if (ly < 0 || ly >= TY || lx < 0 || lx >= TX) return;
        const int fz = (int)fzf;
        float wz[2], wy[2], wx[2];
        axis_weights(g.x, fzf, mode, wz[0], wz[1]);
        axis_weights(g.y, fyf, mode, wy[0], wy[1]);
        axis_weights(g.z, fxf, mode, wx[0], wx[1]);
        float dz = 0.f, dy = 0.f, dx = 0.f;
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int j = 0; j < 2; ++j)
#pragma unroll
                for (int k = 0; k < 2; ++k) {
                    const float d = A1[(fz + i) * ncol + (ly + j) * EX + lx + k];
                    // d w0/dg = -1, d w1/dg = +1 in both modes (floor has zero gradient)
                    dz += d * (i ? 1.f : -1.f) * wy[j] * wx[k];
                    dy += d * wz[i] * (j ? 1.f : -1.f) * wx[k];
                    dx += d * wz[i] * wy[j] * (k ? 1.f : -1.f);
                }
        dp[__float_as_int(g.w)] = make_float4(dz, dy, dx, 0.f);
    };
    for_each_record(sp, bs, nbx, gby_lo, gby_hi, gbx_lo, gbx_hi, gather);
}

// ----------------------------------------------------------------------------------------------
// mode P.  The blur runs along x, y and z, so the columns are coupled and the grid goes through HBM, in the caller's
// workspace (grid A: raw splat, grid B: clamped occupancy blurred along x and y; both [B,V,V,V], z-major):
//   fwd  b3d_vox_splat_sorted -> A;  pc_blur_xy_kernel<., false>: A -> clamp -> x blur -> y blur -> B;
//        pc_sil_p_fwd_kernel: B -> z blur -> scale / clamp -> ray march -> sil (sil_fwd_columns)
//   bwd  pc_sil_p_bwd_kernel: B -> the column adjoints (sil_bwd_columns) -> dB, in place over B;
//        pc_blur_xy_kernel<., true>: dB -> y^T -> x^T -> mask 0 <= A <= 1 -> dA, in place over A;
//        b3d::vox_gather_launch: dA -> dpg
// ----------------------------------------------------------------------------------------------
constexpr int XY_TX = 64, XY_TY = 32;  // output tile of the x / y blur: one z slice, 64 x 32 cells, halo ktaps/2 around
constexpr int XY_THREADS = 256;

// shared memory of pc_blur_xy_kernel for half-width H: the tile with its halo [RY][P] (P odd: a warp walking down the
// rows hits 32 banks) and the tile after the first blur ([RY][XY_TX + 1] forward, [XY_TY][P] adjoint)
inline size_t xy_tile_floats(int H) {
    const size_t P = XY_TX + 2 * H + 1, RY = XY_TY + 2 * H;
    const size_t mid_f = RY * (XY_TX + 1), mid_a = XY_TY * P;
    return RY * P + (mid_f > mid_a ? mid_f : mid_a);
}

// forward (ADJ false): dst = blur_y(blur_x(clamp(src, 0, 1))).   adjoint (ADJ true): dst = [0 <= raw <= 1] *
// blur_x^T(blur_y^T(src)); raw and dst may be the same buffer (each cell is read and written by one thread).
// Zero padding, taps in the order of vox_blur_axis_kernel.  grid (B*V slices, tiles of the slice).
template <int KT, bool ADJ>
__global__ void __launch_bounds__(XY_THREADS)
pc_blur_xy_kernel(const float* __restrict__ src, const float* raw, float* dst, const Taps taps, int V, int ntx) {
    extern __shared__ __align__(128) float sm[];
    const int H = (KT > 0 ? KT : taps.n) / 2;
    const int W = XY_TX + 2 * H, P = W + 1, RY = XY_TY + 2 * H;
    float* in = sm;
    float* mid = sm + RY * P;
    const size_t slice = (size_t)blockIdx.x * V * V;
    const int ty0 = (blockIdx.y / ntx) * XY_TY, tx0 = (blockIdx.y % ntx) * XY_TX;
    const int tid = threadIdx.x;
    for (int i = tid; i < RY * P; i += XY_THREADS) {
        const int r = i / P, c = i % P, y = ty0 - H + r, x = tx0 - H + c;
        float v = 0.f;
        if (c < W && y >= 0 && y < V && x >= 0 && x < V) {
            v = src[slice + (size_t)y * V + x];
            if (!ADJ) v = clamp_nan(v, 0.f, 1.f);            // trilinear_interpolation.py:74
        }
        in[i] = v;
    }
    __syncthreads();
    float o[ZB];
    if (!ADJ) {
        constexpr int MP = XY_TX + 1;
        for (int it = tid; it < RY * (XY_TX / ZB); it += XY_THREADS) {        // x blur of every row, halo rows included
            const int r = it % RY, xb = (it / RY) * ZB;
            blur_window<KT, false, false>(in + r * P, 1, P, xb + H, taps, o);
#pragma unroll
            for (int j = 0; j < ZB; ++j) mid[r * MP + xb + j] = o[j];
        }
        __syncthreads();
        for (int it = tid; it < XY_TX * (XY_TY / ZB); it += XY_THREADS) {     // y blur
            const int c = it % XY_TX, yb = (it / XY_TX) * ZB, x = tx0 + c;
            if (x >= V) continue;
            blur_window<KT, false, false>(mid + c, MP, RY, yb + H, taps, o);
#pragma unroll
            for (int j = 0; j < ZB; ++j)
                if (ty0 + yb + j < V) dst[slice + (size_t)(ty0 + yb + j) * V + x] = o[j];
        }
    } else {
        for (int it = tid; it < W * (XY_TY / ZB); it += XY_THREADS) {         // y^T of every column, halo columns included
            const int c = it % W, yb = (it / W) * ZB;
            blur_window<KT, true, false>(in + c, P, RY, yb + H, taps, o);
#pragma unroll
            for (int j = 0; j < ZB; ++j) mid[(yb + j) * P + c] = o[j];
        }
        __syncthreads();
        for (int it = tid; it < XY_TY * (XY_TX / ZB); it += XY_THREADS) {     // x^T, then the clamp mask
            const int r = it % XY_TY, xb = (it / XY_TY) * ZB, y = ty0 + r;
            if (y >= V) continue;
            blur_window<KT, true, false>(mid + r * P, 1, P, xb + H, taps, o);
#pragma unroll
            for (int j = 0; j < ZB; ++j) {
                const int x = tx0 + xb + j;
                if (x < V) {
                    const size_t i = slice + (size_t)y * V + x;
                    const float g = raw[i];
                    dst[i] = (g >= 0.f && g <= 1.f) ? o[j] : 0.f;
                }
            }
        }
    }
}

// patch [V][TY * TX] of grid G [B,V,V,V] at (ty0, tx0); cells outside the grid read as 0
__device__ __forceinline__ void load_patch(const float* __restrict__ G, int b, int V, int ty0, int tx0, int ncol, float* A) {
    for (int i = threadIdx.x; i < V * ncol; i += TILE_THREADS) {
        const int z = i / ncol, c = i % ncol, y = ty0 + c / TX, x = tx0 + c % TX;
        A[i] = (y < V && x < V) ? G[(((size_t)b * V + z) * V + y) * V + x] : 0.f;
    }
}

// z blur + scale / clamp + ray march of grid B (mode P): the mode-R forward without its splat
template <int KT>
__global__ void __launch_bounds__(TILE_THREADS)
pc_sil_p_fwd_kernel(const float* __restrict__ G, const Taps taps, const float* __restrict__ scale, int V, int TY,
                    float* __restrict__ sil) {
    extern __shared__ __align__(128) float sm[];
    const int b = blockIdx.z, ty0 = blockIdx.y * TY, tx0 = blockIdx.x * TX;
    const int ncol = TY * TX, nzb = (V + ZB - 1) / ZB;
    float* A = sm;                       // [V][ncol]
    float* blkP = A + V * ncol;          // [nzb][ncol]
    float* blkS = blkP + nzb * ncol;     // [nzb][ncol]
    load_patch(G, b, V, ty0, tx0, ncol, A);
    __syncthreads();
    const bool has_scale = scale != nullptr;
    const float sc = has_scale ? scale[b] : 1.f;
    // no sparsity skip: grid B is dense after the x / y blur, and no occupied-depth ranges are known here
    sil_fwd_columns<KT, false>(A, blkP, blkS, nullptr, nullptr, false, taps, has_scale, sc, 1.f, b, V, ncol, ty0, tx0, sil);
}

// column adjoints of the above: grid B -> d(grid B), in place (the z direction is column-local); dscale accumulated
template <int KT>
__global__ void __launch_bounds__(TILE_THREADS)
pc_sil_p_bwd_kernel(float* __restrict__ G, const Taps taps, const float* __restrict__ scale,
                    const float* __restrict__ dsil, int V, int TY, float* __restrict__ dscale) {
    extern __shared__ __align__(128) float sm[];
    __shared__ float red[32];
    const int b = blockIdx.z, ty0 = blockIdx.y * TY, tx0 = blockIdx.x * TX;
    const int ncol = TY * TX, nzb = (V + ZB - 1) / ZB;
    float* A1 = sm;                      // grid B -> d(grid B)
    float* A2 = A1 + V * ncol;           // S -> dS
    float* blkA = A2 + V * ncol;
    float* blkB = blkA + nzb * ncol;
    float* blkT = blkB + nzb * ncol;
    load_patch(G, b, V, ty0, tx0, ncol, A1);
    __syncthreads();
    const bool has_scale = scale != nullptr;
    const float sc = has_scale ? scale[b] : 1.f;
    sil_bwd_columns<KT, false>(A1, A2, blkA, blkB, blkT, nullptr, nullptr, false, taps, has_scale, sc, 1.f, dsil, b, V, ncol,
                               TX, TY, ty0, tx0, red, dscale);
    for (int i = threadIdx.x; i < V * ncol; i += TILE_THREADS) {
        const int z = i / ncol, c = i % ncol, y = ty0 + c / TX, x = tx0 + c % TX;
        if (y < V && x < V) G[(((size_t)b * V + z) * V + y) * V + x] = A1[i];
    }
}

// ----------------------------------------------------------------------------------------------
// adjoint of pc_project_kernel
// ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NTHREADS)
pc_project_bwd_kernel(const float* __restrict__ points, const float* __restrict__ quat,
                      const float4* __restrict__ pg, const float4* __restrict__ dpg, int N, int V,
                      float FOV, float CAM_DIST, float* __restrict__ dpoints, float* __restrict__ dquat) {
    __shared__ float red[32];
    const int b = blockIdx.y;
    const int n = blockIdx.x * NTHREADS + threadIdx.x;
    float nrm;
    const Quat q = normalize_quat(quat + 4 * b, &nrm);
    Quat dq{0.f, 0.f, 0.f, 0.f};
    if (n < N) {
        const size_t i = (size_t)b * N + n;
        float d0 = 0.f, d1 = 0.f, d2 = 0.f;
        if (pg[i].w != 0.f) {
            const float4 dg = dpg[i];
            const float vm1 = (float)(V - 1);
            const float dc0 = vm1 * dg.x, dc1 = vm1 * dg.y, dc2 = vm1 * dg.z;
            const Quat P{0.f, points[3 * i], points[3 * i + 1], points[3 * i + 2]};
            const Quat u = hamilton(q, P);
            const Quat r = hamilton(u, conj(q));
            const float inv = 1.f / (r.x + CAM_DIST);
            const float c1 = r.y * FOV * inv, c2 = r.z * FOV * inv;
            const Quat Gr{0.f, dc0 - (c1 * dc1 + c2 * dc2) * inv, dc1 * FOV * inv, dc2 * FOV * inv};
            const Quat gu = hamilton(Gr, q);               // d/d(q (x) P)
            const Quat gw = hamilton(conj(u), Gr);         // d/d(q*)
            const Quat a = hamilton(gu, conj(P));
            dq = Quat{a.w + gw.w, a.x - gw.x, a.y - gw.y, a.z - gw.z};
            const Quat dP = hamilton(conj(q), gu);
            d0 = dP.x;
            d1 = dP.y;
            d2 = dP.z;
        }
        dpoints[3 * i + 0] = d0;
        dpoints[3 * i + 1] = d1;
        dpoints[3 * i + 2] = d2;
    }
    const float sw = b3d::block_sum(dq.w, red);
    const float sx = b3d::block_sum(dq.x, red);
    const float sy = b3d::block_sum(dq.y, red);
    const float sz = b3d::block_sum(dq.z, red);
    if (threadIdx.x == 0) {
        // adjoint of q / max(||q||, eps): (I - q^ q^T) / n  (identity / eps in the degenerate branch)
        const float dot = (nrm > 1e-12f) ? (q.w * sw + q.x * sx + q.y * sy + q.z * sz) : 0.f;
        atomicAdd(dquat + 4 * b + 0, (sw - q.w * dot) / nrm);
        atomicAdd(dquat + 4 * b + 1, (sx - q.x * dot) / nrm);
        atomicAdd(dquat + 4 * b + 2, (sy - q.y * dot) / nrm);
        atomicAdd(dquat + 4 * b + 3, (sz - q.z * dot) / nrm);
    }
}

// ----------------------------------------------------------------------------------------------
// materialised grid (tests / mode P)
// ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NTHREADS)
pc_splat_grid_kernel(const float4* __restrict__ pg, int N, int V, int mode, float* __restrict__ grid) {
    const int b = blockIdx.y;
    const int n = blockIdx.x * NTHREADS + threadIdx.x;
    if (n >= N) return;
    const float4 g = pg[(size_t)b * N + n];
    if (g.w == 0.f) return;
    const float fzf = floorf(g.x), fyf = floorf(g.y), fxf = floorf(g.z);
    float wz[2], wy[2], wx[2];
    axis_weights(g.x, fzf, mode, wz[0], wz[1]);
    axis_weights(g.y, fyf, mode, wy[0], wy[1]);
    axis_weights(g.z, fxf, mode, wx[0], wx[1]);
    float* gb = grid + (size_t)b * V * V * V;
    const int fz = (int)fzf, fy = (int)fyf, fx = (int)fxf;
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int k = 0; k < 2; ++k)
                atomicAdd(gb + ((size_t)(fz + i) * V + fy + j) * V + fx + k, mul(mul(wz[i], wy[j]), wx[k]));
}

__global__ void __launch_bounds__(NTHREADS) clamp01_kernel(float* __restrict__ x, size_t n) {
    for (size_t i = (size_t)blockIdx.x * NTHREADS + threadIdx.x; i < n; i += (size_t)gridDim.x * NTHREADS)
        x[i] = clamp_nan(x[i], 0.f, 1.f);
}

// ----------------------------------------------------------------------------------------------
// host side
// ----------------------------------------------------------------------------------------------
constexpr size_t SMEM_BUDGET = 210 * 1024;      // the patch, within the 227 KB a CTA may use

// halo: the mode-R backward's +1 column halo (every point owned by one CTA); the mode-P kernels have none
size_t patch_bytes(int V, int ty, bool bwd, bool halo) {
    const size_t nzb = (V + ZB - 1) / ZB;
    const size_t ncol = halo ? (size_t)(ty + 1) * (TX + 1) : (size_t)ty * TX;
    if (bwd) return 4 * (2 * V * ncol + 3 * nzb * ncol + 2 * ncol);
    return 4 * (V * ncol + 2 * nzb * ncol + 2 * ncol);
}

int pick_ty(int V, bool bwd, bool halo) {
    for (int ty = 16; ty >= 1; ty >>= 1)
        if (patch_bytes(V, ty, bwd, halo) <= SMEM_BUDGET) return ty;
    return 0;
}

inline int bins_x(int V) { return (V + BIN_X - 1) / BIN_X; }
inline int bins_y(int V) { return (V + BIN_Y - 1) / BIN_Y; }

template <typename K>
int set_smem(K kernel, size_t bytes) {
    B3D_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    return B3D_OK;
}

template <int KT>
int launch_sil_fwd(dim3 grid, size_t smem, cudaStream_t st, const float* sorted, const int32_t* bin_start, const Taps& t,
                   const float* scale, int N, int V, int TY, int mode, float* sil) {
    if (int rc = set_smem(pc_sil_fwd_kernel<KT>, smem)) return rc;
    pc_sil_fwd_kernel<KT><<<grid, TILE_THREADS, smem, st>>>((const float4*)sorted, bin_start, t, scale, N, V, TY, mode,
                                                            bins_x(V), bins_y(V), sil);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

int sil_fwd_impl(const float* sorted, const int32_t* bin_start, const Taps& t, const float* scale, int B, int N,
                 int V, int mode, float* sil, cudaStream_t st) {
    const int TY = pick_ty(V, false, false);
    B3D_REQUIRE(TY > 0, B3D_EINVAL, "b3d_pc_silhouette_fwd: V=%d does not fit the shared-memory patch", V);
    const size_t smem = patch_bytes(V, TY, false, false);
    dim3 grid(b3d::ceil_div(V, TX), b3d::ceil_div(V, TY), B);
    if (t.n == 21) return launch_sil_fwd<21>(grid, smem, st, sorted, bin_start, t, scale, N, V, TY, mode, sil);
    return launch_sil_fwd<0>(grid, smem, st, sorted, bin_start, t, scale, N, V, TY, mode, sil);
}

template <int KT>
int launch_sil_bwd(dim3 grid, size_t smem, cudaStream_t st, const float* sorted, const int32_t* bin_start, const Taps& t,
                   const float* scale, const float* dsil, int N, int V, int TY, int mode, float* dpg, float* dscale) {
    if (int rc = set_smem(pc_sil_bwd_kernel<KT>, smem)) return rc;
    pc_sil_bwd_kernel<KT><<<grid, TILE_THREADS, smem, st>>>((const float4*)sorted, bin_start, t, scale, dsil, N, V, TY, mode,
                                                            bins_x(V), bins_y(V), (float4*)dpg, dscale);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

int sil_bwd_impl(const float* sorted, const int32_t* bin_start, const Taps& t, const float* scale,
                 const float* dsil, int B, int N, int V, int mode, float* dpg, float* dscale, cudaStream_t st) {
    const int TY = pick_ty(V, true, true);
    B3D_REQUIRE(TY > 0, B3D_EINVAL, "b3d_pc_silhouette_bwd: V=%d does not fit the shared-memory patch", V);
    const size_t smem = patch_bytes(V, TY, true, true);
    if (dscale) B3D_CUDA_OK(cudaMemsetAsync(dscale, 0, sizeof(float) * B, st));
    dim3 grid(b3d::ceil_div(V, TX), b3d::ceil_div(V, TY), B);
    if (t.n == 21) return launch_sil_bwd<21>(grid, smem, st, sorted, bin_start, t, scale, dsil, N, V, TY, mode, dpg, dscale);
    return launch_sil_bwd<0>(grid, smem, st, sorted, bin_start, t, scale, dsil, N, V, TY, mode, dpg, dscale);
}

// ---- mode P ------------------------------------------------------------------------------------
template <bool ADJ>
int launch_blur_xy(const float* src, const float* raw, float* dst, const Taps& t, int B, int V, cudaStream_t st) {
    const int ntx = b3d::ceil_div(V, XY_TX);
    const dim3 grid((unsigned)B * V, ntx * b3d::ceil_div(V, XY_TY));
    const size_t smem = sizeof(float) * xy_tile_floats(t.n / 2);
    if (t.n == 21) {
        if (int rc = set_smem(pc_blur_xy_kernel<21, ADJ>, smem)) return rc;
        pc_blur_xy_kernel<21, ADJ><<<grid, XY_THREADS, smem, st>>>(src, raw, dst, t, V, ntx);
    } else {
        if (int rc = set_smem(pc_blur_xy_kernel<0, ADJ>, smem)) return rc;
        pc_blur_xy_kernel<0, ADJ><<<grid, XY_THREADS, smem, st>>>(src, raw, dst, t, V, ntx);
    }
    B3D_LAUNCH_OK();
    return B3D_OK;
}

template <int KT>
int launch_sil_p_fwd(dim3 grid, size_t smem, cudaStream_t st, const float* G, const Taps& t, const float* scale, int V,
                     int TY, float* sil) {
    if (int rc = set_smem(pc_sil_p_fwd_kernel<KT>, smem)) return rc;
    pc_sil_p_fwd_kernel<KT><<<grid, TILE_THREADS, smem, st>>>(G, t, scale, V, TY, sil);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

template <int KT>
int launch_sil_p_bwd(dim3 grid, size_t smem, cudaStream_t st, float* G, const Taps& t, const float* scale, const float* dsil,
                     int V, int TY, float* dscale) {
    if (int rc = set_smem(pc_sil_p_bwd_kernel<KT>, smem)) return rc;
    pc_sil_p_bwd_kernel<KT><<<grid, TILE_THREADS, smem, st>>>(G, t, scale, dsil, V, TY, dscale);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

int sil_fwd_paper(const float* sorted, const int32_t* bin_start, const Taps& t, const float* scale, int B, int N, int V,
                  float* sil, float* ws, cudaStream_t st) {
    const int TY = pick_ty(V, false, false);
    B3D_REQUIRE(TY > 0, B3D_EINVAL, "b3d_pc_silhouette_fwd: V=%d does not fit the shared-memory patch", V);
    float* gA = ws;
    float* gB = ws + (size_t)B * V * V * V;
    if (int rc = b3d_vox_splat_sorted(sorted, bin_start, B, N, V, B3D_MODE_PAPER, gA, st)) return rc;
    if (int rc = launch_blur_xy<false>(gA, nullptr, gB, t, B, V, st)) return rc;
    const size_t smem = patch_bytes(V, TY, false, false);
    const dim3 grid(b3d::ceil_div(V, TX), b3d::ceil_div(V, TY), B);
    if (t.n == 21) return launch_sil_p_fwd<21>(grid, smem, st, gB, t, scale, V, TY, sil);
    return launch_sil_p_fwd<0>(grid, smem, st, gB, t, scale, V, TY, sil);
}

int sil_bwd_paper(const float* sorted, const int32_t* bin_start, const Taps& t, const float* scale, const float* dsil, int B,
                  int N, int V, float* dpg, float* dscale, float* ws, cudaStream_t st) {
    const int TY = pick_ty(V, true, false);
    B3D_REQUIRE(TY > 0, B3D_EINVAL, "b3d_pc_silhouette_bwd: V=%d does not fit the shared-memory patch", V);
    float* gA = ws;
    float* gB = ws + (size_t)B * V * V * V;
    if (dscale) B3D_CUDA_OK(cudaMemsetAsync(dscale, 0, sizeof(float) * B, st));
    const size_t smem = patch_bytes(V, TY, true, false);
    const dim3 grid(b3d::ceil_div(V, TX), b3d::ceil_div(V, TY), B);
    const int rc = t.n == 21 ? launch_sil_p_bwd<21>(grid, smem, st, gB, t, scale, dsil, V, TY, dscale)
                             : launch_sil_p_bwd<0>(grid, smem, st, gB, t, scale, dsil, V, TY, dscale);
    if (rc) return rc;
    if (int rc2 = launch_blur_xy<true>(gB, gA, gA, t, B, V, st)) return rc2;
    if (N == 0) return B3D_OK;
    return b3d::vox_gather_launch(sorted, bin_start, gA, B, N, V, B3D_MODE_PAPER, dpg, st);
}

int check_sil_args(const char* who, const void* sorted, const void* bin_start, const void* taps, int ktaps, int B,
                   int N, int V, int mode, const void* workspace, size_t workspace_bytes) {
    B3D_REQUIRE(B >= 0 && N >= 0 && V >= 2, B3D_EINVAL, "%s: bad sizes B=%d N=%d V=%d", who, B, N, V);
    B3D_REQUIRE(ktaps >= 1 && ktaps <= MAX_TAPS && (ktaps & 1), B3D_EINVAL, "%s: ktaps=%d must be odd, <= %d", who,
                ktaps, MAX_TAPS);
    B3D_REQUIRE(mode == B3D_MODE_REFERENCE || mode == B3D_MODE_PAPER, B3D_EINVAL, "%s: unknown mode %d", who, mode);
    B3D_REQUIRE(taps && (B == 0 || (bin_start && (sorted || N == 0))), B3D_EINVAL, "%s: null pointer", who);
    const size_t need = b3d_pc_silhouette_workspace_bytes(B, V, mode);
    B3D_REQUIRE(need == 0 || (workspace && workspace_bytes >= need), B3D_EINVAL,
                "%s: mode %d needs a workspace of %zu bytes (got %s, %zu bytes)", who, mode, need,
                workspace ? "a buffer" : "NULL", workspace_bytes);
    if (need) B3D_CHECK_ALIGNED(workspace);
    return B3D_OK;
}

void fill_taps(Taps& t, const float* host, int n) {
    t.finite = 1;
    for (int i = 0; i < n; ++i) {
        t.w[i] = host[i];
        if (!(fabsf(host[i]) <= 3.0e38f)) t.finite = 0;          // NaN / inf taps must propagate (SURVEY App. A D4)
    }
    t.n = n;
}

}  // namespace

extern "C" {

int b3d_pc_bin_count(int V) { return V >= 2 ? bins_x(V) * bins_y(V) : 0; }

int b3d_pc_project(const float* points, const float* quat, int B, int N, int V, float fov, float cam_dist,
                   float* pg, float* coords, int32_t* base, uint8_t* inb, float* sorted, int32_t* bin_start,
                   void* stream) {
    B3D_REQUIRE(B >= 0 && N >= 0 && V >= 2, B3D_EINVAL, "b3d_pc_project: bad sizes B=%d N=%d V=%d", B, N, V);
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(N == 0 || (sorted == nullptr) == (bin_start == nullptr), B3D_EINVAL,
                "b3d_pc_project: sorted and bin_start go together");
    cudaStream_t st = (cudaStream_t)stream;
    const int nbins = b3d_pc_bin_count(V);
    B3D_REQUIRE(nbins <= MAX_BINS, B3D_EINVAL, "b3d_pc_project: V=%d needs more than %d bins", V, MAX_BINS);
    if (N == 0) {
        if (bin_start) B3D_CUDA_OK(cudaMemsetAsync(bin_start, 0, sizeof(int32_t) * (size_t)B * (nbins + 1), st));
        return B3D_OK;
    }
    B3D_REQUIRE(points && quat && pg, B3D_EINVAL, "b3d_pc_project: null pointer");
    B3D_CHECK_ALIGNED(pg);
    dim3 grid(b3d::ceil_div(N, NTHREADS), B);
    pc_project_kernel<<<grid, NTHREADS, 0, st>>>(points, quat, N, V, fov, cam_dist, (float4*)pg, coords, base, inb);
    B3D_LAUNCH_OK();
    if (sorted) {
        B3D_CHECK_ALIGNED(sorted);
        pc_bin_kernel<<<B, BIN_THREADS, 0, st>>>((const float4*)pg, N, bins_x(V), nbins, (float4*)sorted, bin_start);
        B3D_LAUNCH_OK();
    }
    return B3D_OK;
}

size_t b3d_pc_silhouette_workspace_bytes(int B, int V, int mode) {
    if (mode == B3D_MODE_REFERENCE) return 0;
    return 2ull * (size_t)B * V * V * V * sizeof(float);
}

// taps given in HOST memory (the Python wrapper computes them with the reference's torch expression on
// the CPU, 21 floats) and passed to the kernel by value, so no device->host read is needed.
int b3d_pc_silhouette_fwd_hosttaps(const float* sorted, const int32_t* bin_start, const float* taps_host, int ktaps,
                                   const float* scale, int B, int N, int V, int mode, float* sil, void* workspace,
                                   size_t workspace_bytes, void* stream) {
    if (int rc = check_sil_args("b3d_pc_silhouette_fwd", sorted, bin_start, taps_host, ktaps, B, N, V, mode, workspace,
                                workspace_bytes))
        return rc;
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(sil, B3D_EINVAL, "b3d_pc_silhouette_fwd: null output");
    Taps t;
    fill_taps(t, taps_host, ktaps);
    if (mode == B3D_MODE_PAPER)
        return sil_fwd_paper(sorted, bin_start, t, scale, B, N, V, sil, (float*)workspace, (cudaStream_t)stream);
    return sil_fwd_impl(sorted, bin_start, t, scale, B, N, V, mode, sil, (cudaStream_t)stream);
}

int b3d_pc_silhouette_bwd_hosttaps(const float* sorted, const int32_t* bin_start, const float* taps_host, int ktaps,
                                   const float* scale, const float* dsil, int B, int N, int V, int mode, float* dpg,
                                   float* dscale, void* workspace, size_t workspace_bytes, void* stream) {
    if (int rc = check_sil_args("b3d_pc_silhouette_bwd", sorted, bin_start, taps_host, ktaps, B, N, V, mode, workspace,
                                workspace_bytes))
        return rc;
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(dsil && (dpg || N == 0), B3D_EINVAL, "b3d_pc_silhouette_bwd: null pointer");
    B3D_REQUIRE((scale == nullptr) == (dscale == nullptr), B3D_EINVAL,
                "b3d_pc_silhouette_bwd: scale and dscale must both be given or both be NULL");
    Taps t;
    fill_taps(t, taps_host, ktaps);
    if (mode == B3D_MODE_PAPER)
        return sil_bwd_paper(sorted, bin_start, t, scale, dsil, B, N, V, dpg, dscale, (float*)workspace, (cudaStream_t)stream);
    return sil_bwd_impl(sorted, bin_start, t, scale, dsil, B, N, V, mode, dpg, dscale, (cudaStream_t)stream);
}

int b3d_pc_project_bwd(const float* points, const float* quat, const float* pg, const float* dpg, int B, int N,
                       int V, float fov, float cam_dist, float* dpoints, float* dquat, void* stream) {
    B3D_REQUIRE(B >= 0 && N >= 0 && V >= 2, B3D_EINVAL, "b3d_pc_project_bwd: bad sizes");
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(quat && dquat, B3D_EINVAL, "b3d_pc_project_bwd: null pointer");
    B3D_CUDA_OK(cudaMemsetAsync(dquat, 0, sizeof(float) * 4 * B, (cudaStream_t)stream));
    if (N == 0) return B3D_OK;
    B3D_REQUIRE(points && pg && dpg && dpoints, B3D_EINVAL, "b3d_pc_project_bwd: null pointer");
    dim3 grid(b3d::ceil_div(N, NTHREADS), B);
    pc_project_bwd_kernel<<<grid, NTHREADS, 0, (cudaStream_t)stream>>>(points, quat, (const float4*)pg,
                                                                      (const float4*)dpg, N, V, fov, cam_dist, dpoints,
                                                                      dquat);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

int b3d_pc_splat_grid(const float* pg, int B, int N, int V, int mode, float* grid, void* stream) {
    B3D_REQUIRE(B >= 0 && N >= 0 && V >= 2, B3D_EINVAL, "b3d_pc_splat_grid: bad sizes");
    B3D_REQUIRE(mode == B3D_MODE_REFERENCE || mode == B3D_MODE_PAPER, B3D_EINVAL, "b3d_pc_splat_grid: bad mode");
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(grid, B3D_EINVAL, "b3d_pc_splat_grid: null grid");
    const size_t cells = (size_t)B * V * V * V;
    cudaStream_t st = (cudaStream_t)stream;
    B3D_CUDA_OK(cudaMemsetAsync(grid, 0, cells * sizeof(float), st));
    if (N > 0) {
        B3D_REQUIRE(pg, B3D_EINVAL, "b3d_pc_splat_grid: null pg");
        dim3 g(b3d::ceil_div(N, NTHREADS), B);
        pc_splat_grid_kernel<<<g, NTHREADS, 0, st>>>((const float4*)pg, N, V, mode, grid);
        B3D_LAUNCH_OK();
    }
    const int blocks = (int)((cells + NTHREADS * 8 - 1) / (NTHREADS * 8));
    clamp01_kernel<<<blocks < 132 * 8 ? blocks : 132 * 8, NTHREADS, 0, st>>>(grid, cells);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

}  // extern "C"
