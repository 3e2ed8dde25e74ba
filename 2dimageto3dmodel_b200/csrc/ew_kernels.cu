// HBM-bound helper kernels between the GAN's convolutions (SURVEY.md §2.2: "elementwise / data-movement between
// convs ... each a full HBM round trip -> fuse"), NHWC fp32, 16-byte vector accesses, one pass each.
//   pad_x_*      replicate / circular padding along x (gan.py:329 F.pad replicate; rendering/utils.py:29-33 circpad)
//                forward = gather, backward = gather of the (up to three) output columns that read an input column.
//   leaky_bwd    gradient of the LeakyReLU that the conv epilogue fused (mask from the sign of the OUTPUT).
#include "b3d_common.cuh"

namespace {
constexpr int NT = 256;

// mode 0 = replicate, 1 = circular
__device__ __forceinline__ int src_col(int wo, int a, int W, int mode) {
    const int w = wo - a;
    if (mode == 0) return w < 0 ? 0 : (w >= W ? W - 1 : w);
    return w < 0 ? w + W : (w >= W ? w - W : w);
}

__global__ void __launch_bounds__(NT)
pad_x_fwd_kernel(const float4* __restrict__ x, float4* __restrict__ out, long long rows, int W, int C4, int a, int mode) {
    const int Wo = W + 2 * a;
    const long long total = rows * Wo * C4;
    for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
        const int c = (int)(i % C4);
        const long long t = i / C4;
        const int wo = (int)(t % Wo);
        const long long r = t / Wo;
        out[i] = __ldg(x + (r * W + src_col(wo, a, W, mode)) * C4 + c);
    }
}

__global__ void __launch_bounds__(NT)
pad_x_bwd_kernel(const float4* __restrict__ go, float4* __restrict__ gx, long long rows, int W, int C4, int a, int mode) {
    const int Wo = W + 2 * a;
    const long long total = rows * W * C4;
    for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
        const int c = (int)(i % C4);
        const long long t = i / C4;
        const int w = (int)(t % W);
        const long long r = t / W;
        const float4* g = go + (r * Wo) * C4 + c;
        float4 s = __ldg(g + (long long)(w + a) * C4);
        if (mode == 0) {
            if (w == 0)
                for (int k = 0; k < a; ++k) { const float4 v = __ldg(g + (long long)k * C4); s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w; }
            if (w == W - 1)
                for (int k = 0; k < a; ++k) { const float4 v = __ldg(g + (long long)(W + a + k) * C4); s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w; }
        } else {
            if (w < a) { const float4 v = __ldg(g + (long long)(w + a + W) * C4); s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w; }
            if (w >= W - a) { const float4 v = __ldg(g + (long long)(w + a - W) * C4); s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w; }
        }
        gx[i] = s;
    }
}

__global__ void __launch_bounds__(NT)
leaky_bwd_kernel(const float4* __restrict__ gy, const float4* __restrict__ y, float4* __restrict__ out, long long n4, float slope) {
    for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < n4; i += (long long)gridDim.x * NT) {
        const float4 g = __ldg(gy + i), v = __ldg(y + i);
        out[i] = make_float4(v.x >= 0.f ? g.x : g.x * slope, v.y >= 0.f ? g.y : g.y * slope, v.z >= 0.f ? g.z : g.z * slope,
                             v.w >= 0.f ? g.w : g.w * slope);
    }
}

// In-place wrap fill: buf [rows, W + 2a, 4*C4] whose interior columns a .. a+W-1 were written by a conv epilogue.
__global__ void __launch_bounds__(NT)
wrap_x_kernel(float4* __restrict__ buf, long long rows, int W, int C4, int a, int mode) {
    const int Wo = W + 2 * a;
    const long long total = rows * 2 * a * C4;
    for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
        const int c = (int)(i % C4);
        const long long t = i / C4;
        const int j = (int)(t % (2 * a));
        const long long r = t / (2 * a);
        const int wo = j < a ? j : W + j;                    // pad column: left a, then right a
        buf[(r * Wo + wo) * C4 + c] = buf[(r * Wo + a + src_col(wo, a, W, mode)) * C4 + c];
    }
}

// Discriminator stem input in one pass (models/gan.py:102-111 `_with_positions` + the wrap-around padding in front of conv1,
// :95-96): out[n, y, xo, :] = concat(x[n, :, y, xs], pos[:, y, xs]) with xs = the source column of padded column xo —
// NCHW image planes + NCHW positional planes -> x-padded NHWC, instead of cat -> NCHW-to-NHWC copy -> pad (three passes).
// One thread per output pixel: plane reads are coalesced along x, the pixel's C1 + C2 floats are written as float4s.
template <int CT>
__global__ void __launch_bounds__(NT)
stem_input_fwd_kernel(const float* __restrict__ x, const float* __restrict__ pos, float4* __restrict__ out, int N, int C1, int H,
                      int W, int a, int mode) {
    const int Wo = W + 2 * a;
    const long long total = (long long)N * H * Wo;
    const size_t plane = (size_t)H * W;
    for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
        const int xo = (int)(i % Wo);
        const long long r = i / Wo;
        const int y = (int)(r % H), n = (int)(r / H);
        const int xs = src_col(xo, a, W, mode);
        const float* xp = x + (size_t)n * C1 * plane + (size_t)y * W + xs;
        const float* pp = pos + (size_t)y * W + xs;
        float v[CT];
#pragma unroll
        for (int c = 0; c < CT; ++c) v[c] = c < C1 ? __ldg(xp + (size_t)c * plane) : __ldg(pp + (size_t)(c - C1) * plane);
#pragma unroll
        for (int q = 0; q < CT / 4; ++q) out[i * (CT / 4) + q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
    }
}
// adjoint w.r.t. x: gx[n, c, y, xs] = sum of gout[n, y, xo, c] over the padded columns xo that read xs (c < C1)
template <int CT>
__global__ void __launch_bounds__(NT)
stem_input_bwd_kernel(const float* __restrict__ gout, float* __restrict__ gx, int N, int C1, int H, int W, int a, int mode) {
    const int Wo = W + 2 * a;
    const long long total = (long long)N * H * W;
    const size_t plane = (size_t)H * W;
    for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
        const int xs = (int)(i % W);
        const long long r = i / W;
        const int y = (int)(r % H), n = (int)(r / H);
        const float* g = gout + (size_t)r * Wo * CT;
        float s[CT];
#pragma unroll
        for (int c = 0; c < CT; ++c) s[c] = c < C1 ? g[(size_t)(xs + a) * CT + c] : 0.f;
        if (a > 0) {
            if (mode == 0) {
                if (xs == 0)
                    for (int k = 0; k < a; ++k)
                        for (int c = 0; c < C1; ++c) s[c] += g[(size_t)k * CT + c];
                if (xs == W - 1)
                    for (int k = 0; k < a; ++k)
                        for (int c = 0; c < C1; ++c) s[c] += g[(size_t)(W + a + k) * CT + c];
            } else {
                if (xs < a)
                    for (int c = 0; c < C1; ++c) s[c] += g[(size_t)(xs + a + W) * CT + c];
                if (xs >= W - a)
                    for (int c = 0; c < C1; ++c) s[c] += g[(size_t)(xs + a - W) * CT + c];
            }
        }
        float* o = gx + (size_t)n * C1 * plane + (size_t)y * W + xs;
#pragma unroll
        for (int c = 0; c < CT; ++c)
            if (c < C1) o[(size_t)c * plane] = s[c];
    }
}

// Adjoint of the wrap fill, in place: pad-column gradients are added to the interior columns they were copied from.
// mode 1 (circular): one thread per (row, pad column, channel quad); mode 0 (replicate): one thread per (row, side, quad).
__global__ void __launch_bounds__(NT)
wrap_x_bwd_kernel(float4* __restrict__ g, long long rows, int W, int C4, int a, int mode) {
    const int Wo = W + 2 * a;
    const int per_row = mode ? 2 * a : 2;
    const long long total = rows * per_row * C4;
    for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
        const int c = (int)(i % C4);
        const long long t = i / C4;
        const int j = (int)(t % per_row);
        float4* row = g + (t / per_row) * Wo * C4 + c;
        float4 s;
        int dst;
        if (mode) {
            const int src = j < a ? j : W + j;               // pad column: left a, then right a
            dst = j < a ? W + j : j;                         // left pad j = copy of interior W - a + j; right pad k = copy of interior k
            s = row[(size_t)src * C4];
        } else {
            const int first = j == 0 ? 0 : W + a;
            dst = j == 0 ? a : W + a - 1;
            s = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int k = 0; k < a; ++k) { const float4 v = row[(size_t)(first + k) * C4]; s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w; }
        }
        float4 d = row[(size_t)dst * C4];
        d.x += s.x; d.y += s.y; d.z += s.z; d.w += s.w;
        row[(size_t)dst * C4] = d;
    }
}

// Backward of  conv -> (+bias) -> LeakyReLU -> pad_x  in one pass:  gy = pad_x^T(g_pad) * leaky'(y),  gb += sum gy.
// Thread t owns channel group t % C4 for the pixels t / C4, t / C4 + PPB, ... of its block's slab, so the bias
// partial sums stay in registers; one shared-memory tree + one atomicAdd per (block, channel).
__global__ void __launch_bounds__(NT)
pad_leaky_bias_bwd_kernel(const float4* __restrict__ go, const float4* __restrict__ ypad, float4* __restrict__ gy,
                          float* __restrict__ gb, long long rows, int W, int C4, int a, int mode, float slope,
                          long long pix_per_block) {
    __shared__ float4 red[NT];
    const int Wo = W + 2 * a;
    const int c = threadIdx.x % C4, lane_p = threadIdx.x / C4, PPB = NT / C4;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    constexpr int U = 4;                                   // independent pixels in flight per thread
    // a block walks whole rows (32-bit index math only; `pix_per_block` = rows per block here)
    const long long r0 = (long long)blockIdx.x * pix_per_block;
    const long long r1 = r0 + pix_per_block < rows ? r0 + pix_per_block : rows;
    for (long long r = r0; r < r1; ++r) {
        const float4* g = go + (r * Wo) * C4 + c;
        const float4* yr = ypad + (r * Wo + a) * C4 + c;
        float4* gr = gy + (r * W) * C4 + c;
        for (int wb = lane_p; wb < W; wb += U * PPB) {
            float4 s[U], v[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int w = wb + u * PPB;
                if (w >= W) continue;
                s[u] = __ldg(g + (w + a) * C4);
                v[u] = __ldg(yr + w * C4);
                if (a > 0) {
                    if (mode == 0) {
                        if (w == 0)
                            for (int k = 0; k < a; ++k) { const float4 t = __ldg(g + k * C4); s[u].x += t.x; s[u].y += t.y; s[u].z += t.z; s[u].w += t.w; }
                        if (w == W - 1)
                            for (int k = 0; k < a; ++k) { const float4 t = __ldg(g + (W + a + k) * C4); s[u].x += t.x; s[u].y += t.y; s[u].z += t.z; s[u].w += t.w; }
                    } else {
                        if (w < a) { const float4 t = __ldg(g + (w + a + W) * C4); s[u].x += t.x; s[u].y += t.y; s[u].z += t.z; s[u].w += t.w; }
                        if (w >= W - a) { const float4 t = __ldg(g + (w + a - W) * C4); s[u].x += t.x; s[u].y += t.y; s[u].z += t.z; s[u].w += t.w; }
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int w = wb + u * PPB;
                if (w >= W) continue;
                const float4 m = make_float4(v[u].x >= 0.f ? s[u].x : s[u].x * slope, v[u].y >= 0.f ? s[u].y : s[u].y * slope,
                                             v[u].z >= 0.f ? s[u].z : s[u].z * slope, v[u].w >= 0.f ? s[u].w : s[u].w * slope);
                gr[w * C4] = m;
                acc.x += m.x; acc.y += m.y; acc.z += m.z; acc.w += m.w;
            }
        }
    }
    if (gb == nullptr) return;
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int h = PPB / 2; h >= 1; h >>= 1) {
        if (lane_p < h) {
            const float4 o = red[threadIdx.x + h * C4];
            float4& m = red[threadIdx.x];
            m.x += o.x; m.y += o.y; m.z += o.z; m.w += o.w;
        }
        __syncthreads();
    }
    if (lane_p == 0) {
        const float4 m = red[threadIdx.x];
        atomicAdd(gb + 4 * c + 0, m.x); atomicAdd(gb + 4 * c + 1, m.y); atomicAdd(gb + 4 * c + 2, m.z); atomicAdd(gb + 4 * c + 3, m.w);
    }
}

// Thin-stem fold: out[n, y, x, r*C + c] = x[n, y + r - pad_y, x, c] (zero outside the image, zero for k >= kh*C).
// One block = one output row (n, y); a thread owns one 16-byte channel group k4 for the pixels px, px + PPB, ...: the
// (r, c) decomposition of its four channels is computed once, the inner loop is loads + one float4 store (no divisions).
__global__ void __launch_bounds__(NT)
fold_rows_fwd_kernel(const float* __restrict__ x, float4* __restrict__ out, int N, int H, int W, int C, int Hout, int Cp4,
                     int kh, int pad_y) {
    const int K = kh * C;
    const int k4 = threadIdx.x % Cp4, px0 = threadIdx.x / Cp4, PPB = NT / Cp4;
    if (px0 >= PPB) return;                                  // NT not a multiple of Cp4: the tail threads idle
    for (int row = blockIdx.x; row < N * Hout; row += gridDim.x) {
        const int n = row / Hout, y = row - n * Hout;
        long long src[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int k = 4 * k4 + j;
            const int r = k / C, c = k - r * C;
            const int yy = y + r - pad_y;
            src[j] = (k < K && yy >= 0 && yy < H) ? (((long long)n * H + yy) * W) * C + c : -1;
        }
        float4* orow = out + (long long)row * W * Cp4 + k4;
        constexpr int U = 4;                                 // independent pixels in flight per thread
        if ((C & 3) == 0) {
            // C % 4 == 0: the four channels of a quad come from one image row (same r) -> one 16-byte load per output quad
            for (int xb = px0; xb < W; xb += U * PPB) {
                float4 v[U];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const int xx = xb + u * PPB;
                    v[u] = (xx < W && src[0] >= 0) ? __ldg(reinterpret_cast<const float4*>(x + src[0] + (long long)xx * C))
                                                   : make_float4(0.f, 0.f, 0.f, 0.f);
                }
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const int xx = xb + u * PPB;
                    if (xx < W) orow[(long long)xx * Cp4] = v[u];
                }
            }
            continue;
        }
        for (int xb = px0; xb < W; xb += U * PPB) {
            float v[U][4];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int xx = xb + u * PPB;
#pragma unroll
                for (int j = 0; j < 4; ++j) v[u][j] = (xx < W && src[j] >= 0) ? __ldg(x + src[j] + (long long)xx * C) : 0.f;
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int xx = xb + u * PPB;
                if (xx < W) orow[(long long)xx * Cp4] = make_float4(v[u][0], v[u][1], v[u][2], v[u][3]);
            }
        }
    }
}

__global__ void __launch_bounds__(NT)
fold_rows_bwd_kernel(const float* __restrict__ go, float* __restrict__ gx, int N, int H, int W, int C, int Hout, int Cp,
                     int kh, int pad_y) {
    const long long total = (long long)N * H * W * C;
    for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
        const int c = (int)(i % C);
        long long t = i / C;
        const int xx = (int)(t % W); t /= W;
        const int yy = (int)(t % H);
        const int n = (int)(t / H);
        float s = 0.f;
        for (int r = 0; r < kh; ++r) {
            const int y = yy - r + pad_y;
            if (y >= 0 && y < Hout) s += __ldg(go + (((long long)n * Hout + y) * W + xx) * Cp + r * C + c);
        }
        gx[i] = s;
    }
}

int grid_for(long long n) {
    long long b = (n + NT - 1) / NT;
    const long long cap = 132LL * 16;
    return (int)(b < cap ? (b > 0 ? b : 1) : cap);
}
}  // namespace

extern "C" {
int b3d_pad_x_fwd(const float* x, float* out, long long rows, int W, int C, int amount, int mode, void* stream) {
    B3D_REQUIRE(rows >= 0 && W > 0 && C > 0 && C % 4 == 0 && amount >= 0 && amount <= W && (mode == 0 || mode == 1), B3D_EINVAL,
                "b3d_pad_x_fwd: bad arguments (C=%d must be a multiple of 4, amount=%d <= W=%d)", C, amount, W);
    if (rows == 0) return B3D_OK;
    B3D_REQUIRE(x && out, B3D_EINVAL, "b3d_pad_x_fwd: null pointer");
    B3D_CHECK_ALIGNED(x);
    B3D_CHECK_ALIGNED(out);
    pad_x_fwd_kernel<<<grid_for(rows * (W + 2 * amount) * (C / 4)), NT, 0, (cudaStream_t)stream>>>(
        (const float4*)x, (float4*)out, rows, W, C / 4, amount, mode);
    B3D_LAUNCH_OK();
    return B3D_OK;
}
int b3d_pad_x_bwd(const float* gout, float* gx, long long rows, int W, int C, int amount, int mode, void* stream) {
    B3D_REQUIRE(rows >= 0 && W > 0 && C > 0 && C % 4 == 0 && amount >= 0 && amount <= W && (mode == 0 || mode == 1), B3D_EINVAL,
                "b3d_pad_x_bwd: bad arguments");
    if (rows == 0) return B3D_OK;
    B3D_REQUIRE(gout && gx, B3D_EINVAL, "b3d_pad_x_bwd: null pointer");
    B3D_CHECK_ALIGNED(gout);
    B3D_CHECK_ALIGNED(gx);
    pad_x_bwd_kernel<<<grid_for(rows * W * (C / 4)), NT, 0, (cudaStream_t)stream>>>((const float4*)gout, (float4*)gx, rows, W,
                                                                                C / 4, amount, mode);
    B3D_LAUNCH_OK();
    return B3D_OK;
}
int b3d_fold_rows_fwd(const float* x, float* out, int N, int H, int W, int C, int kh, int pad_y, int Cp, void* stream) {
    B3D_REQUIRE(N >= 0 && H > 0 && W > 0 && C > 0 && kh >= 1 && pad_y >= 0 && H + 2 * pad_y >= kh, B3D_EINVAL, "b3d_fold_rows_fwd: bad sizes");
    B3D_REQUIRE(Cp % 4 == 0 && Cp >= kh * C, B3D_EINVAL, "b3d_fold_rows_fwd: Cp=%d must be a multiple of 4 and >= kh*C=%d", Cp, kh * C);
    if (N == 0) return B3D_OK;
    B3D_REQUIRE(x && out, B3D_EINVAL, "b3d_fold_rows_fwd: null pointer");
    B3D_CHECK_ALIGNED(out);
    const int Hout = H + 2 * pad_y - kh + 1;
    B3D_REQUIRE(Cp / 4 <= NT, B3D_EINVAL, "b3d_fold_rows_fwd: Cp=%d too wide (max %d)", Cp, 4 * NT);
    const int rows = N * Hout;
    fold_rows_fwd_kernel<<<rows < 132 * 16 ? rows : 132 * 16, NT, 0, (cudaStream_t)stream>>>(x, (float4*)out, N, H, W, C, Hout, Cp / 4,
                                                                                       kh, pad_y);
    B3D_LAUNCH_OK();
    return B3D_OK;
}
int b3d_fold_rows_bwd(const float* gout, float* gx, int N, int H, int W, int C, int kh, int pad_y, int Cp, void* stream) {
    B3D_REQUIRE(N >= 0 && H > 0 && W > 0 && C > 0 && kh >= 1 && pad_y >= 0 && H + 2 * pad_y >= kh && Cp >= kh * C, B3D_EINVAL,
                "b3d_fold_rows_bwd: bad sizes");
    if (N == 0) return B3D_OK;
    B3D_REQUIRE(gout && gx, B3D_EINVAL, "b3d_fold_rows_bwd: null pointer");
    const int Hout = H + 2 * pad_y - kh + 1;
    fold_rows_bwd_kernel<<<grid_for((long long)N * H * W * C), NT, 0, (cudaStream_t)stream>>>(gout, gx, N, H, W, C, Hout, Cp, kh, pad_y);
    B3D_LAUNCH_OK();
    return B3D_OK;
}
int b3d_wrap_x_inplace(float* buf, long long rows, int W, int C, int amount, int mode, void* stream) {
    B3D_REQUIRE(rows >= 0 && W > 0 && C > 0 && C % 4 == 0 && amount >= 0 && amount <= W && (mode == 0 || mode == 1), B3D_EINVAL,
                "b3d_wrap_x_inplace: bad arguments (C=%d must be a multiple of 4, amount=%d <= W=%d)", C, amount, W);
    if (rows == 0 || amount == 0) return B3D_OK;
    B3D_REQUIRE(buf, B3D_EINVAL, "b3d_wrap_x_inplace: null pointer");
    B3D_CHECK_ALIGNED(buf);
    wrap_x_kernel<<<grid_for(rows * 2 * amount * (C / 4)), NT, 0, (cudaStream_t)stream>>>((float4*)buf, rows, W, C / 4, amount, mode);
    B3D_LAUNCH_OK();
    return B3D_OK;
}
int b3d_stem_input_fwd(const float* x, const float* pos, float* out, int N, int C1, int C2, int H, int W, int amount, int mode,
                       void* stream) {
    B3D_REQUIRE(N >= 0 && C1 >= 1 && C2 >= 0 && H > 0 && W > 0 && amount >= 0 && amount <= W && (mode == 0 || mode == 1), B3D_EINVAL,
                "b3d_stem_input_fwd: bad arguments");
    B3D_REQUIRE(C1 + C2 == 8 || C1 + C2 == 4, B3D_EINVAL, "b3d_stem_input_fwd: C1 + C2 = %d must be 4 or 8", C1 + C2);
    if (N == 0) return B3D_OK;
    B3D_REQUIRE(x && out && (pos || C2 == 0), B3D_EINVAL, "b3d_stem_input_fwd: null pointer");
    B3D_CHECK_ALIGNED(out);
    const int g = grid_for((long long)N * H * (W + 2 * amount));
    if (C1 + C2 == 8) stem_input_fwd_kernel<8><<<g, NT, 0, (cudaStream_t)stream>>>(x, pos, (float4*)out, N, C1, H, W, amount, mode);
    else stem_input_fwd_kernel<4><<<g, NT, 0, (cudaStream_t)stream>>>(x, pos, (float4*)out, N, C1, H, W, amount, mode);
    B3D_LAUNCH_OK();
    return B3D_OK;
}
int b3d_stem_input_bwd(const float* gout, float* gx, int N, int C1, int C2, int H, int W, int amount, int mode, void* stream) {
    B3D_REQUIRE(N >= 0 && C1 >= 1 && C2 >= 0 && H > 0 && W > 0 && amount >= 0 && amount <= W && (mode == 0 || mode == 1), B3D_EINVAL,
                "b3d_stem_input_bwd: bad arguments");
    B3D_REQUIRE(C1 + C2 == 8 || C1 + C2 == 4, B3D_EINVAL, "b3d_stem_input_bwd: C1 + C2 = %d must be 4 or 8", C1 + C2);
    if (N == 0) return B3D_OK;
    B3D_REQUIRE(gout && gx, B3D_EINVAL, "b3d_stem_input_bwd: null pointer");
    const int g = grid_for((long long)N * H * W);
    if (C1 + C2 == 8) stem_input_bwd_kernel<8><<<g, NT, 0, (cudaStream_t)stream>>>(gout, gx, N, C1, H, W, amount, mode);
    else stem_input_bwd_kernel<4><<<g, NT, 0, (cudaStream_t)stream>>>(gout, gx, N, C1, H, W, amount, mode);
    B3D_LAUNCH_OK();
    return B3D_OK;
}
int b3d_wrap_x_bwd_inplace(float* g, long long rows, int W, int C, int amount, int mode, void* stream) {
    B3D_REQUIRE(rows >= 0 && W >= 2 && C >= 4 && C % 4 == 0 && amount >= 0 && (mode == 0 || mode == 1), B3D_EINVAL,
                "b3d_wrap_x_bwd_inplace: bad arguments");
    B3D_REQUIRE(mode == 0 ? amount <= W : 2 * amount <= W, B3D_EINVAL, "b3d_wrap_x_bwd_inplace: amount=%d too large for W=%d", amount, W);
    if (rows == 0 || amount == 0) return B3D_OK;
    B3D_REQUIRE(g, B3D_EINVAL, "b3d_wrap_x_bwd_inplace: null pointer");
    B3D_CHECK_ALIGNED(g);
    wrap_x_bwd_kernel<<<grid_for(rows * (mode ? 2 * amount : 2) * (C / 4)), NT, 0, (cudaStream_t)stream>>>((float4*)g, rows, W, C / 4, amount, mode);
    B3D_LAUNCH_OK();
    return B3D_OK;
}
int b3d_pad_leaky_bias_bwd(const float* gout_pad, const float* y_pad, float* gy, float* gbias, long long rows, int W, int C,
                           int amount, int mode, float slope, void* stream) {
    B3D_REQUIRE(rows >= 0 && W > 0 && C >= 4 && amount >= 0 && amount <= W && (mode == 0 || mode == 1), B3D_EINVAL,
                "b3d_pad_leaky_bias_bwd: bad arguments");
    B3D_REQUIRE(C % 4 == 0 && NT % (C / 4) == 0, B3D_EINVAL, "b3d_pad_leaky_bias_bwd: C=%d must be 4 * a power of two <= %d", C, 4 * NT);
    if (rows == 0) return B3D_OK;
    B3D_REQUIRE(gout_pad && y_pad && gy, B3D_EINVAL, "b3d_pad_leaky_bias_bwd: null pointer");
    B3D_CHECK_ALIGNED(gout_pad);
    B3D_CHECK_ALIGNED(y_pad);
    B3D_CHECK_ALIGNED(gy);
    long long blocks = rows < 132LL * 16 ? rows : 132LL * 16;
    const long long per = (rows + blocks - 1) / blocks;          // rows per block
    blocks = (rows + per - 1) / per;
    pad_leaky_bias_bwd_kernel<<<(int)blocks, NT, 0, (cudaStream_t)stream>>>((const float4*)gout_pad, (const float4*)y_pad, (float4*)gy,
                                                                          gbias, rows, W, C / 4, amount, mode, slope, per);
    B3D_LAUNCH_OK();
    return B3D_OK;
}
int b3d_leaky_bwd(const float* gy, const float* y, float* out, long long n, float slope, void* stream) {
    B3D_REQUIRE(n >= 0 && n % 4 == 0, B3D_EINVAL, "b3d_leaky_bwd: element count must be a multiple of 4");
    if (n == 0) return B3D_OK;
    B3D_REQUIRE(gy && y && out, B3D_EINVAL, "b3d_leaky_bwd: null pointer");
    leaky_bwd_kernel<<<grid_for(n / 4), NT, 0, (cudaStream_t)stream>>>((const float4*)gy, (const float4*)y, (float4*)out, n / 4, slope);
    B3D_LAUNCH_OK();
    return B3D_OK;
}
}

// ------------------------------------------------------------------------------------------------------------------
// Per-channel fp64 sums and sums of squares of an NHWC activation for the (Sync)BatchNorm layers (models/gan.py:211-232 ->
// F.batch_norm / sync_batchnorm/batchnorm.py:150) in one pass over the tensor.  Threads own a channel quad and stride over
// the pixels (fp32 partial sums of ~50-100 values), a block folds its pixel lanes in shared memory and adds into fp64
// accumulators.  PER_SAMPLE (InstanceNorm2d, models/gan.py:302 / :58): blockIdx.y is the sample, `rows` its pixel count,
// and sample n's sums go to ws + n * 2C — the same pass with the sample index kept.  The pixel loop is bounded by `rows`,
// so a sample smaller than one CTA's pixel range (blk1: 8 x 4 = 32 pixels) leaves the surplus lanes at zero.
// ------------------------------------------------------------------------------------------------------------------
namespace {
template <bool PER_SAMPLE>
__global__ void __launch_bounds__(NT)
bn_sums_kernel(const float4* __restrict__ y, long long rows, int C4, double* __restrict__ ws) {
    if (PER_SAMPLE) {
        y += (long long)blockIdx.y * rows * C4;
        ws += (long long)blockIdx.y * 8 * C4;
    }
    __shared__ float4 rs[NT], rq[NT];
    const int c = threadIdx.x % C4, lane_p = threadIdx.x / C4, PPB = NT / C4;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f), q = s;
    constexpr int U = 4;                                    // independent 16-byte loads in flight per thread
    const long long stride = (long long)gridDim.x * PPB;
    for (long long p = (long long)blockIdx.x * PPB + lane_p; p < rows; p += U * stride) {
        float4 v[U];
#pragma unroll
        for (int u = 0; u < U; ++u) v[u] = p + u * stride < rows ? __ldg(y + (p + u * stride) * C4 + c) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int u = 0; u < U; ++u) {
            s.x += v[u].x; s.y += v[u].y; s.z += v[u].z; s.w += v[u].w;
            q.x = fmaf(v[u].x, v[u].x, q.x); q.y = fmaf(v[u].y, v[u].y, q.y); q.z = fmaf(v[u].z, v[u].z, q.z); q.w = fmaf(v[u].w, v[u].w, q.w);
        }
    }
    rs[threadIdx.x] = s; rq[threadIdx.x] = q;
    __syncthreads();
    for (int h = PPB / 2; h >= 1; h >>= 1) {
        if (lane_p < h) {
            const float4 a = rs[threadIdx.x + h * C4], b = rq[threadIdx.x + h * C4];
            float4& m = rs[threadIdx.x]; float4& n = rq[threadIdx.x];
            m.x += a.x; m.y += a.y; m.z += a.z; m.w += a.w;
            n.x += b.x; n.y += b.y; n.z += b.z; n.w += b.w;
        }
        __syncthreads();
    }
    if (lane_p == 0) {
        const float4 m = rs[threadIdx.x], n = rq[threadIdx.x];
        const int C = 4 * C4;
        atomicAdd(ws + 4 * c + 0, (double)m.x); atomicAdd(ws + 4 * c + 1, (double)m.y);
        atomicAdd(ws + 4 * c + 2, (double)m.z); atomicAdd(ws + 4 * c + 3, (double)m.w);
        atomicAdd(ws + C + 4 * c + 0, (double)n.x); atomicAdd(ws + C + 4 * c + 1, (double)n.y);
        atomicAdd(ws + C + 4 * c + 2, (double)n.z); atomicAdd(ws + C + 4 * c + 3, (double)n.w);
    }
}
}  // namespace

// ------------------------------------------------------------------------------------------------------------------
// Per-layer scalar math of ConditionalBatchNorm2d in ONE launch (was ~15 tiny torch kernels per layer and forward):
// statistics -> mean / inv_std, running-buffer update, and the per-sample affine of the fused pass below,
//   scale[n,c] = inv_std[c] * (1 + gamma[n,c]),   shift[n,c] = beta[n,c] - mean[c] * scale[n,c],   gt[n,c] = 1 + gamma[n,c].
// mode 0: eval (running statistics).  mode 1: batch statistics from fp64 sums [2][C] over `count` values per channel with
// F.batch_norm's formulas (biased variance + eps under the root; running variance unbiased).  mode 2: the reference's
// SyncBN formulas on the (all-reduced) sums: inv_std = clamp(var, eps)^-1/2 (sync_batchnorm/batchnorm.py:133-150).
// mode 3: instance statistics (InstanceNorm2d without running buffers, so in eval mode too): mode 1's formulas on sample n's
// sums [N][2][C] over `count` = H*W values.  mode 4: no normalisation (norm_g 'none'): mean 0, inv_std 1.  Modes 3 and 4
// write mean / inv_std as [N, C] rows and never touch running buffers.
// momentum < 0 selects torch's cumulative average (BatchNorm momentum=None): factor 1 / (num_batches_tracked + 1).
__device__ __forceinline__ void cbn_batch_stats(const double* __restrict__ sums, double count, float eps, int mode, int C, int c,
                                                float& mean, float& invstd, double& var_b) {
    const double m = sums[c] / count;
    var_b = mode == 1 ? sums[C + c] / count - m * m : (sums[C + c] - sums[c] * m) / count;
    if (mode == 1) var_b = var_b > 0.0 ? var_b : 0.0;
    mean = (float)m;
    invstd = mode == 1 ? (float)(1.0 / sqrt(var_b + (double)eps)) : (float)(1.0 / sqrt(var_b > (double)eps ? var_b : (double)eps));
}

__device__ __forceinline__ float cbn_momentum(float momentum, const long long* nbt) {
    return momentum >= 0.f ? momentum : (nbt != nullptr ? (float)(1.0 / (double)(*nbt + 1)) : 0.f);
}

__global__ void __launch_bounds__(NT)
cbn_prepare_kernel(const float* __restrict__ gb, int gb_pitch, int gamma_off, int beta_off, const double* __restrict__ sums,
                   double count, float eps, float momentum, int mode, float* __restrict__ running_mean,
                   float* __restrict__ running_var, long long* __restrict__ nbt, float* __restrict__ mean_out,
                   float* __restrict__ invstd_out, float* __restrict__ scale, float* __restrict__ shift, float* __restrict__ gt,
                   int N, int C) {
    const int i = blockIdx.x * NT + threadIdx.x;
    if (i < N * C) {
        const int n = i / C, c = i - n * C;
        float mean, invstd;
        double var_b;
        if (mode == 0) {
            mean = running_mean[c];
            invstd = rsqrtf(running_var[c] + eps);
        } else if (mode == 3) {                              // instance statistics: sample n's sums, F.batch_norm's formulas
            cbn_batch_stats(sums + (long long)n * 2 * C, count, eps, 1, C, c, mean, invstd, var_b);
        } else if (mode == 4) {                              // no normalisation
            mean = 0.f;
            invstd = 1.f;
        } else {
            cbn_batch_stats(sums, count, eps, mode, C, c, mean, invstd, var_b);
        }
        const float g1 = 1.f + gb[(long long)n * gb_pitch + gamma_off + c];
        const float sc = invstd * g1;
        scale[i] = sc;
        shift[i] = gb[(long long)n * gb_pitch + beta_off + c] - mean * sc;
        gt[i] = g1;
        if (mode >= 3) {                                     // per-sample rows [N, C]
            mean_out[i] = mean;
            invstd_out[i] = invstd;
        } else if (n == 0) {
            mean_out[c] = mean;
            invstd_out[c] = invstd;
        }
    }
    // Running buffers (modes 1, 2; mode 0 is the only one that reads them above): block 0 alone updates every channel, so
    // all its threads read num_batches_tracked (the momentum=None factor) before the barrier and thread 0 increments after it.
    if (blockIdx.x == 0 && (mode == 1 || mode == 2) && running_mean != nullptr) {
        const float f = cbn_momentum(momentum, nbt);
        for (int c = threadIdx.x; c < C; c += NT) {
            float mean, invstd;
            double var_b;
            cbn_batch_stats(sums, count, eps, mode, C, c, mean, invstd, var_b);
            running_mean[c] = (1.f - f) * running_mean[c] + f * mean;
            running_var[c] = (1.f - f) * running_var[c] + f * (float)(var_b * (count / (count > 1.0 ? count - 1.0 : 1.0)));
        }
        __syncthreads();
        if (threadIdx.x == 0 && nbt != nullptr) *nbt += 1;
    }
}

// ------------------------------------------------------------------------------------------------------------------
// SyncBN statistics WITHOUT a separate collective: a one-shot all-reduce over NVLink / NVSwitch peer memory fused into
// the kernel that consumes the sums (SURVEY §5 "one fused SyncBN collective"; VERDICT r1 "weak" #9: 64 latency-bound
// [2,C] NCCL all-reduces per step, each wrapped in ~10 tiny ops).  Every rank owns a symmetric buffer (torch symmetric
// memory: the same allocation mapped into every peer):  data [2 parities][world][SYNC_MAX] doubles + flag [2][world] u32.
// Call k (epoch e = k, parity e & 1) on rank r:  store the local vector into slot [parity][r] of EVERY peer's buffer,
// fence, store e into flag [parity][r] of every peer (release, system scope); spin until the own flags [parity][0..world)
// all read e (acquire); sum the world slots in rank order — bitwise identical on all ranks.  A peer can run at most one
// call ahead (it needs this rank's flag of call k+1 to finish call k+1), and that call uses the other parity, so two
// parities suffice.  A spin that exceeds ~4 s (a dead peer) sets *err and falls through instead of hanging the GPU.
// ------------------------------------------------------------------------------------------------------------------
constexpr int SYNC_MAX = 1024;          // payload doubles per rank (2 * C, C <= 512)
constexpr int SYNC_RANKS = 8;
struct SyncPeers {
    double* data[SYNC_RANKS];           // peer p's buffer (own rank included)
    unsigned* flag[SYNC_RANKS];
};

__device__ __forceinline__ unsigned long long gtimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

// vec: shared-memory vector of n doubles (local contribution in, world total out).  All threads of the CTA call.
__device__ void peer_allreduce(const SyncPeers& P, int rank, int world, unsigned* epoch_ctr, int* err, double* vec, int n) {
    __shared__ unsigned ep_s;
    if (threadIdx.x == 0) ep_s = ++(*epoch_ctr);
    __syncthreads();
    const unsigned e = ep_s, par = e & 1u;
    for (int p = 0; p < world; ++p) {
        double* dst = P.data[p] + ((size_t)par * world + rank) * SYNC_MAX;
        for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = vec[i];
    }
    __threadfence_system();
    __syncthreads();
    if ((int)threadIdx.x < world) {
        unsigned* f = P.flag[threadIdx.x] + par * world + rank;
        asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(f), "r"(e) : "memory");
        const unsigned* mine = P.flag[rank] + par * world + threadIdx.x;
        const unsigned long long t0 = gtimer();
        unsigned v;
        do {
            asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(mine) : "memory");
            if (v != e && gtimer() - t0 > 4000000000ull) { *err = 1; break; }
        } while (v != e);
    }
    __syncthreads();
    const double* src = P.data[rank] + (size_t)par * world * SYNC_MAX;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        double t = 0.0;
        for (int r = 0; r < world; ++r) t += src[(size_t)r * SYNC_MAX + i];
        vec[i] = t;
    }
    __syncthreads();
}

// b3d_cbn_prepare (mode 2: the reference's SyncBN formulas) with the all-reduce of the fp64 sums fused in.  One CTA.
__global__ void __launch_bounds__(512)
cbn_prepare_sync_kernel(SyncPeers P, int rank, int world, unsigned* epoch_ctr, int* err, const float* __restrict__ gb,
                        int gb_pitch, int gamma_off, int beta_off, const double* __restrict__ sums_local, double count, float eps,
                        float momentum, float* __restrict__ running_mean, float* __restrict__ running_var,
                        long long* __restrict__ nbt, float* __restrict__ mean_out, float* __restrict__ invstd_out,
                        float* __restrict__ scale, float* __restrict__ shift, float* __restrict__ gt, int N, int C) {
    __shared__ double tot[SYNC_MAX];
    __shared__ float mean_s[SYNC_MAX / 2], inv_s[SYNC_MAX / 2];
    const float f = cbn_momentum(momentum, nbt);            // read before the barriers in peer_allreduce, incremented after
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) tot[i] = sums_local[i];
    __syncthreads();
    peer_allreduce(P, rank, world, epoch_ctr, err, tot, 2 * C);
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const double m = tot[c] / count;
        const double var_b = (tot[C + c] - tot[c] * m) / count;
        const float mean = (float)m, invstd = (float)(1.0 / sqrt(var_b > (double)eps ? var_b : (double)eps));
        mean_s[c] = mean;
        inv_s[c] = invstd;
        mean_out[c] = mean;
        invstd_out[c] = invstd;
        if (running_mean != nullptr) {
            running_mean[c] = (1.f - f) * running_mean[c] + f * mean;
            running_var[c] = (1.f - f) * running_var[c] + f * (float)(var_b * (count / (count > 1.0 ? count - 1.0 : 1.0)));
            if (c == 0 && nbt != nullptr) *nbt += 1;
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < N * C; i += blockDim.x) {
        const int n = i / C, c = i - n * C;
        const float g1 = 1.f + gb[(long long)n * gb_pitch + gamma_off + c];
        const float sc = inv_s[c] * g1;
        scale[i] = sc;
        shift[i] = gb[(long long)n * gb_pitch + beta_off + c] - mean_s[c] * sc;
        gt[i] = g1;
    }
}

// b3d_cbn_bwd_reduce with the all-reduce of red [2][C] fused in.  One CTA.
__global__ void __launch_bounds__(512)
cbn_bwd_reduce_sync_kernel(SyncPeers P, int rank, int world, unsigned* epoch_ctr, int* err, const float* __restrict__ S1,
                           const float* __restrict__ S2, int s_pitch, const float* __restrict__ gt, float* __restrict__ red, int N,
                           int C) {
    __shared__ double tot[SYNC_MAX];
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float a = 0.f, b = 0.f;
        for (int n = 0; n < N; ++n) {
            const float g = gt[(long long)n * C + c];
            a = fmaf(g, S1[(long long)n * s_pitch + c], a);
            b = fmaf(g, S2[(long long)n * s_pitch + c], b);
        }
        tot[c] = (double)a;
        tot[C + c] = (double)b;
    }
    __syncthreads();
    peer_allreduce(P, rank, world, epoch_ctr, err, tot, 2 * C);
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) red[i] = (float)tot[i];
}

// red[0][c] = sum_n gt[n,c] * S1[n,c],  red[1][c] = sum_n gt[n,c] * S2[n,c]   (batch-norm coupling terms of the backward)
__global__ void __launch_bounds__(NT)
cbn_bwd_reduce_kernel(const float* __restrict__ S1, const float* __restrict__ S2, int s_pitch, const float* __restrict__ gt,
                      float* __restrict__ red, int N, int C) {
    const int c = blockIdx.x * NT + threadIdx.x;
    if (c >= C) return;
    float a = 0.f, b = 0.f;
    for (int n = 0; n < N; ++n) {
        const float g = gt[(long long)n * C + c];
        a = fmaf(g, S1[(long long)n * s_pitch + c], a);
        b = fmaf(g, S2[(long long)n * s_pitch + c], b);
    }
    red[c] = a;
    red[C + c] = b;
}

// Fused generator glue (models/gan.py:282-286 ConditionalBatchNorm2d, :309-311 LeakyReLU + residual, :319 nearest x2
// upsample, :329 replicate pad): one pass from a conv output y [N,H,W,C] to the NEXT conv's padded input
//     out[n, yo, xo, c] = post( leaky(y[n,ys,xs,c] * scale[n,c] + shift[n,c]) + skip[n,ys,xs,c] )
// with (ys, xs) = (yo / up, clamp(xo - pad, 0, up*W - 1) / up), scale = inv_std * (1 + gamma), shift = beta - mean*scale.
// The reference runs ~8 full-tensor kernels for this chain (SURVEY §2.2), each an HBM round trip.
// ------------------------------------------------------------------------------------------------------------------
namespace {
struct CbnGeom {
    int N, H, W, C4;             // input y [N,H,W,4*C4]
    int up, pad;                 // output [N, up*H, up*W + 2*pad, C]
    int skip_pitch, skip_off;    // skip pixel (y,x) lives at row (y*skip_pitch + x + skip_off); pitch 0 = no skip
    int skip_sh;                 // 1: the skip has half y's resolution, pixel (y,x) of y adds skip pixel (y/2, x/2)
    float slope;                 // LeakyReLU slope of the first activation
    int post_leaky;              // apply LeakyReLU again after the residual add (blk6 / mesh head)
};

__device__ __forceinline__ float lk(float v, float s) { return v >= 0.f ? v : v * s; }

// PM: x-padding mode of the output, 0 = replicate (symmetric generator), 1 = circular (asymmetric generator, discriminators;
// the column is wrapped in upsampled coordinates, as circpad applied after F.interpolate).
template <int PM>
__global__ void __launch_bounds__(NT)
cbn_act_fwd_kernel(const float4* __restrict__ y, const float4* __restrict__ scale, const float4* __restrict__ shift,
                   const float4* __restrict__ skip, float4* __restrict__ out, const CbnGeom g) {
    const int Wo = g.up * g.W + 2 * g.pad, Ho = g.up * g.H;
    const long long total = (long long)g.N * Ho * Wo * g.C4;
    for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
        const int c = (int)(i % g.C4);
        long long t = i / g.C4;
        const int xo = (int)(t % Wo);
        t /= Wo;
        const int yo = (int)(t % Ho);
        const int n = (int)(t / Ho);
        int xs = src_col(xo, g.pad, g.up * g.W, PM);
        const int ys = yo / g.up;
        xs /= g.up;
        const float4 v = __ldg(y + (((long long)n * g.H + ys) * g.W + xs) * g.C4 + c);
        const float4 sc = __ldg(scale + (long long)n * g.C4 + c), sh = __ldg(shift + (long long)n * g.C4 + c);
        float4 o = make_float4(lk(fmaf(v.x, sc.x, sh.x), g.slope), lk(fmaf(v.y, sc.y, sh.y), g.slope),
                               lk(fmaf(v.z, sc.z, sh.z), g.slope), lk(fmaf(v.w, sc.w, sh.w), g.slope));
        if (g.skip_pitch) {
            const float4 k = __ldg(skip + (((long long)n * (g.H >> g.skip_sh) + (ys >> g.skip_sh)) * g.skip_pitch + (xs >> g.skip_sh) +
                                           g.skip_off) * g.C4 + c);
            o.x += k.x; o.y += k.y; o.z += k.z; o.w += k.w;
        }
        if (g.post_leaky) o = make_float4(lk(o.x, g.slope), lk(o.y, g.slope), lk(o.z, g.slope), lk(o.w, g.slope));
        out[i] = o;
    }
}

// Same pass with the index arithmetic hoisted: one block walks output rows (n, yo), a thread owns channel quad
// c = tid % C4 for the pixels tid / C4, + NT / C4, ... (needs NT % C4 == 0) — no 64-bit divisions per element, the
// per-sample scale / shift stay in registers along the row.
template <int PM>
__global__ void __launch_bounds__(NT)
cbn_act_fwd_rows_kernel(const float4* __restrict__ y, const float4* __restrict__ scale, const float4* __restrict__ shift,
                        const float4* __restrict__ skip, float4* __restrict__ out, const CbnGeom g) {
    const int Wo = g.up * g.W + 2 * g.pad, Ho = g.up * g.H, Wu = g.up * g.W;
    const int c = threadIdx.x % g.C4, px0 = threadIdx.x / g.C4, PPB = NT / g.C4;
    for (int row = blockIdx.x; row < g.N * Ho; row += gridDim.x) {
        const int n = row / Ho, yo = row - n * Ho;
        const int ys = yo / g.up;
        const float4 sc = __ldg(scale + (long long)n * g.C4 + c), sh = __ldg(shift + (long long)n * g.C4 + c);
        const float4* yrow = y + (((long long)n * g.H + ys) * g.W) * g.C4 + c;
        const float4* srow = g.skip_pitch ? skip + (((long long)n * (g.H >> g.skip_sh) + (ys >> g.skip_sh)) * g.skip_pitch + g.skip_off) * g.C4 + c
                                          : nullptr;
        float4* orow = out + (long long)row * Wo * g.C4 + c;
        constexpr int U = 4;                                 // independent pixels in flight per thread
        for (int xb = px0; xb < Wo; xb += U * PPB) {
            float4 v[U], k[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int xo = xb + u * PPB;
                if (xo >= Wo) continue;
                int xs = src_col(xo, g.pad, Wu, PM);
                xs = g.up == 2 ? xs >> 1 : xs;
                v[u] = __ldg(yrow + (long long)xs * g.C4);
                if (srow) k[u] = __ldg(srow + (long long)(xs >> g.skip_sh) * g.C4);
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int xo = xb + u * PPB;
                if (xo >= Wo) continue;
                float4 o = make_float4(lk(fmaf(v[u].x, sc.x, sh.x), g.slope), lk(fmaf(v[u].y, sc.y, sh.y), g.slope),
                                       lk(fmaf(v[u].z, sc.z, sh.z), g.slope), lk(fmaf(v[u].w, sc.w, sh.w), g.slope));
                if (srow) { o.x += k[u].x; o.y += k[u].y; o.z += k[u].z; o.w += k[u].w; }
                if (g.post_leaky) o = make_float4(lk(o.x, g.slope), lk(o.y, g.slope), lk(o.z, g.slope), lk(o.w, g.slope));
                orow[(long long)xo * g.C4] = o;
            }
        }
    }
}

// Backward pass 1.  Per input pixel: gather the gradient of its up x up children (+ the replicate-pad columns), undo the
// activations, write ga = d/d(pre-activation) and (optionally) gskip; accumulate S1[n,c] = sum ga, S2[n,c] = sum ga * xhat
// with xhat = (y - mean) * inv_std.  One CTA walks `rows_per_cta` image rows of one sample, threads own channel quads.
// PM: the forward's pad mode; with circular padding (1) every pad column is folded back onto the upsampled column it wraps
// from (the order interior, right pad, left pad of b3d_pad_x_bwd).  PS: mean / inv_std are per-sample rows [N, C].
// HS: 1 = the skip has half the resolution (g.skip_sh), 0 = the same as y.
template <int PM, bool PS, int HS>
__global__ void __launch_bounds__(NT)
cbn_act_bwd1_kernel(const float4* __restrict__ gout, const float4* __restrict__ y, const float4* __restrict__ scale,
                    const float4* __restrict__ shift, const float4* __restrict__ skip, const float4* __restrict__ mean,
                    const float4* __restrict__ invstd, float4* __restrict__ ga, float4* __restrict__ gskip, int gskip_pitch,
                    int gskip_off, float* __restrict__ S1, float* __restrict__ S2, int s_pitch, const CbnGeom g, int rows_per_cta) {
    const int n = blockIdx.y;
    const int y0 = blockIdx.x * rows_per_cta, y1 = min(y0 + rows_per_cta, g.H);
    const int Wu = g.up * g.W, Wo = Wu + 2 * g.pad;
    for (int c = threadIdx.x % g.C4, lane_px = threadIdx.x / g.C4, px_step = NT / g.C4; c < g.C4; c += g.C4) {
        const float4 sc = __ldg(scale + (long long)n * g.C4 + c), sh = __ldg(shift + (long long)n * g.C4 + c);
        const long long so = PS ? (long long)n * g.C4 + c : c;
        const float4 mu = __ldg(mean + so), is = __ldg(invstd + so);
        float4 a1 = make_float4(0.f, 0.f, 0.f, 0.f), a2 = a1;
        // a half-resolution skip (skip_sh): one thread walks the 2 x 2 footprint of each skip pixel, so that its gradient is
        // summed in a fixed order; otherwise one pixel per step
        const int Wq = g.W >> HS;
        for (int p = (y0 >> HS) * Wq + lane_px; p < (y1 >> HS) * Wq; p += px_step) {
            float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int e = 0; e < (1 << (2 * HS)); ++e) {
                const int ys = ((p / Wq) << HS) + (e >> 1), xs = ((p % Wq) << HS) + (e & 1);
                float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
                for (int i = 0; i < g.up; ++i) {
                    const float4* row = gout + (((long long)n * g.up * g.H + g.up * ys + i) * Wo) * g.C4 + c;
                    if (PM == 0) {
                        int lo = g.up * xs + g.pad, hi = lo + g.up;      // children columns [lo, hi)
                        if (xs == 0) lo = 0;                              // left pad columns replicate column 0
                        if (xs == g.W - 1) hi = Wo;                       // right pad columns replicate the last column
                        for (int xo = lo; xo < hi; ++xo) {
                            const float4 v = __ldg(row + (long long)xo * g.C4);
                            s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
                        }
                    } else {
                        for (int u = g.up * xs; u < g.up * xs + g.up; ++u) {   // upsampled column u: interior + its copies
                            float4 v = __ldg(row + (long long)(u + g.pad) * g.C4);
                            s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
                            if (u < g.pad) {                              // right pad column Wu + pad + u
                                v = __ldg(row + (long long)(u + g.pad + Wu) * g.C4);
                                s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
                            }
                            if (u >= Wu - g.pad) {                        // left pad column u + pad - Wu
                                v = __ldg(row + (long long)(u + g.pad - Wu) * g.C4);
                                s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
                            }
                        }
                    }
                }
                const long long idx = (((long long)n * g.H + ys) * g.W + xs) * g.C4 + c;
                const float4 v = __ldg(y + idx);
                const float4 pre = make_float4(fmaf(v.x, sc.x, sh.x), fmaf(v.y, sc.y, sh.y), fmaf(v.z, sc.z, sh.z), fmaf(v.w, sc.w, sh.w));
                if (g.post_leaky) {                                       // sign of (leaky(pre) + skip)
                    float4 k = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (g.skip_pitch)
                        k = __ldg(skip + (((long long)n * (g.H >> HS) + (ys >> HS)) * g.skip_pitch + (xs >> HS) + g.skip_off) * g.C4 + c);
                    s.x = (lk(pre.x, g.slope) + k.x) >= 0.f ? s.x : s.x * g.slope;
                    s.y = (lk(pre.y, g.slope) + k.y) >= 0.f ? s.y : s.y * g.slope;
                    s.z = (lk(pre.z, g.slope) + k.z) >= 0.f ? s.z : s.z * g.slope;
                    s.w = (lk(pre.w, g.slope) + k.w) >= 0.f ? s.w : s.w * g.slope;
                }
                t.x += s.x; t.y += s.y; t.z += s.z; t.w += s.w;
                const float4 a = make_float4(pre.x >= 0.f ? s.x : s.x * g.slope, pre.y >= 0.f ? s.y : s.y * g.slope,
                                             pre.z >= 0.f ? s.z : s.z * g.slope, pre.w >= 0.f ? s.w : s.w * g.slope);
                ga[idx] = a;
                a1.x += a.x; a1.y += a.y; a1.z += a.z; a1.w += a.w;
                a2.x = fmaf(a.x, (v.x - mu.x) * is.x, a2.x); a2.y = fmaf(a.y, (v.y - mu.y) * is.y, a2.y);
                a2.z = fmaf(a.z, (v.z - mu.z) * is.z, a2.z); a2.w = fmaf(a.w, (v.w - mu.w) * is.w, a2.w);
            }
            if (gskip) gskip[(((long long)n * (g.H >> HS) + p / Wq) * gskip_pitch + p % Wq + gskip_off) * g.C4 + c] = t;
        }
        float* s1 = S1 + (long long)n * s_pitch + c * 4;
        float* s2 = S2 + (long long)n * s_pitch + c * 4;
        atomicAdd(s1 + 0, a1.x); atomicAdd(s1 + 1, a1.y); atomicAdd(s1 + 2, a1.z); atomicAdd(s1 + 3, a1.w);
        atomicAdd(s2 + 0, a2.x); atomicAdd(s2 + 1, a2.y); atomicAdd(s2 + 2, a2.z); atomicAdd(s2 + 3, a2.w);
    }
}

// Backward pass 2 (in place on ga): dy = inv_std * (ga * gamma_t - m1 - xhat * m2), (m1, m2) = red[0 / 1] * inv_m.
// PS (instance / no normalisation): mean / inv_std are rows [N, C], and the coupling terms are per sample,
// (m1, m2)[n,c] = inv_m * gamma_t[n,c] * (S1, S2)[n,c] read from bwd1's sums at row pitch m4 (float4s) — no reduction
// across samples is needed.  inv_m = 0 drops them (no normalisation).
template <bool PS>
__global__ void __launch_bounds__(NT)
cbn_act_bwd2_kernel(float4* __restrict__ ga, const float4* __restrict__ y, const float4* __restrict__ gamma_t,
                    const float4* __restrict__ mean, const float4* __restrict__ invstd, const float4* __restrict__ m1,
                    const float4* __restrict__ m2, int m4, float inv_m, long long per_n, int C4, long long total) {
    for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < total; i += (long long)gridDim.x * NT) {
        const int c = (int)(i % C4);
        const long long n = i / per_n;
        const float4 a = ga[i], v = __ldg(y + i), gt = __ldg(gamma_t + n * C4 + c);
        const long long so = PS ? n * C4 + c : c;
        const float4 mu = __ldg(mean + so), is = __ldg(invstd + so);
        float4 q1 = __ldg(m1 + (PS ? n * m4 + c : c)), q2 = __ldg(m2 + (PS ? n * m4 + c : c));
        if (PS) {
            q1.x *= gt.x; q1.y *= gt.y; q1.z *= gt.z; q1.w *= gt.w;
            q2.x *= gt.x; q2.y *= gt.y; q2.z *= gt.z; q2.w *= gt.w;
        }
        q1.x *= inv_m; q1.y *= inv_m; q1.z *= inv_m; q1.w *= inv_m;
        q2.x *= inv_m; q2.y *= inv_m; q2.z *= inv_m; q2.w *= inv_m;
        ga[i] = make_float4(is.x * (a.x * gt.x - q1.x - (v.x - mu.x) * is.x * q2.x), is.y * (a.y * gt.y - q1.y - (v.y - mu.y) * is.y * q2.y),
                            is.z * (a.z * gt.z - q1.z - (v.z - mu.z) * is.z * q2.z), is.w * (a.w * gt.w - q1.w - (v.w - mu.w) * is.w * q2.w));
    }
}
}  // namespace

extern "C" {
int b3d_cbn_act_fwd(const float* y, const float* scale, const float* shift, const float* skip, int skip_pitch, int skip_off,
                    float* out, int N, int H, int W, int C, int up, int pad, int pad_mode, float slope, int post_leaky,
                    void* stream) {
    B3D_REQUIRE(N >= 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0 && (up == 1 || up == 2) && pad >= 0, B3D_EINVAL,
                "b3d_cbn_act_fwd: bad arguments");
    B3D_REQUIRE(pad_mode == 0 || (pad_mode == 1 && pad <= up * W), B3D_EINVAL, "b3d_cbn_act_fwd: pad mode %d with pad %d > %d columns",
                pad_mode, pad, up * W);
    const int skip_sh = skip_pitch < 0;
    skip_pitch = skip_sh ? -skip_pitch : skip_pitch;
    B3D_REQUIRE(!skip_sh || (H % 2 == 0 && W % 2 == 0), B3D_EINVAL, "b3d_cbn_act_fwd: a half-resolution skip needs even H, W");
    if (N == 0) return B3D_OK;
    B3D_REQUIRE(y && scale && shift && out && (skip != nullptr) == (skip_pitch != 0), B3D_EINVAL, "b3d_cbn_act_fwd: null pointer");
    CbnGeom g{N, H, W, C / 4, up, pad, skip_pitch, skip_off, skip_sh, slope, post_leaky};
    const long long total = (long long)N * up * H * (up * W + 2 * pad) * (C / 4);
    cudaStream_t st = (cudaStream_t)stream;
    if (g.C4 <= NT && NT % g.C4 == 0 && (up == 1 || up == 2)) {
        const int rows = N * up * H, grid = rows < 132 * 16 ? rows : 132 * 16;
        if (pad_mode == 0)
            cbn_act_fwd_rows_kernel<0><<<grid, NT, 0, st>>>((const float4*)y, (const float4*)scale, (const float4*)shift,
                                                            (const float4*)skip, (float4*)out, g);
        else
            cbn_act_fwd_rows_kernel<1><<<grid, NT, 0, st>>>((const float4*)y, (const float4*)scale, (const float4*)shift,
                                                            (const float4*)skip, (float4*)out, g);
    } else if (pad_mode == 0) {
        cbn_act_fwd_kernel<0><<<grid_for(total), NT, 0, st>>>((const float4*)y, (const float4*)scale, (const float4*)shift,
                                                              (const float4*)skip, (float4*)out, g);
    } else {
        cbn_act_fwd_kernel<1><<<grid_for(total), NT, 0, st>>>((const float4*)y, (const float4*)scale, (const float4*)shift,
                                                              (const float4*)skip, (float4*)out, g);
    }
    B3D_LAUNCH_OK();
    return B3D_OK;
}

// S1, S2 [N,C] are zeroed by the call; gskip (nullable) is written at pixel offset gskip_off with row pitch gskip_pitch
// (its pad columns are NOT touched: the caller zeroes the buffer when gskip_pitch != W).  skip_pitch, gskip_pitch < 0: the
// skip has half the resolution (see b3d_cbn_act_fwd) and gskip receives the sum over each 2 x 2 footprint.  stat_pitch: row pitch of mean /
// inv_std, 0 = one row for all samples (batch statistics), C = per-sample rows (instance / no normalisation).
int b3d_cbn_act_bwd1(const float* gout, const float* y, const float* scale, const float* shift, const float* skip, int skip_pitch,
                     int skip_off, const float* mean, const float* invstd, int stat_pitch, float* ga, float* gskip, int gskip_pitch,
                     int gskip_off, float* S1, float* S2, int s_pitch, int N, int H, int W, int C, int up, int pad, int pad_mode,
                     float slope, int post_leaky, void* stream) {
    B3D_REQUIRE(N >= 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0 && C / 4 <= NT && NT % (C / 4) == 0 && (up == 1 || up == 2), B3D_EINVAL,
                "b3d_cbn_act_bwd1: bad arguments (C/4 must divide %d)", NT);
    B3D_REQUIRE(stat_pitch == 0 || stat_pitch == C, B3D_EINVAL, "b3d_cbn_act_bwd1: statistics pitch %d must be 0 or C=%d", stat_pitch, C);
    B3D_REQUIRE(pad >= 0 && (pad_mode == 0 || (pad_mode == 1 && pad <= up * W)), B3D_EINVAL,
                "b3d_cbn_act_bwd1: pad mode %d with pad %d > %d columns", pad_mode, pad, up * W);
    const int skip_sh = skip_pitch < 0;
    skip_pitch = skip_sh ? -skip_pitch : skip_pitch;
    B3D_REQUIRE(skip_sh == (gskip_pitch < 0) || !gskip, B3D_EINVAL, "b3d_cbn_act_bwd1: skip and its gradient differ in resolution");
    gskip_pitch = gskip_pitch < 0 ? -gskip_pitch : gskip_pitch;
    B3D_REQUIRE(!skip_sh || (H % 2 == 0 && W % 2 == 0), B3D_EINVAL, "b3d_cbn_act_bwd1: a half-resolution skip needs even H, W");
    if (N == 0) return B3D_OK;
    B3D_REQUIRE(gout && y && scale && shift && mean && invstd && ga && S1 && S2, B3D_EINVAL, "b3d_cbn_act_bwd1: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    B3D_REQUIRE(s_pitch >= C && s_pitch % 4 == 0, B3D_EINVAL, "b3d_cbn_act_bwd1: S pitch %d must be >= C and a multiple of 4", s_pitch);
    B3D_CUDA_OK(cudaMemset2DAsync(S1, sizeof(float) * (size_t)s_pitch, 0, sizeof(float) * (size_t)C, (size_t)N, st));
    B3D_CUDA_OK(cudaMemset2DAsync(S2, sizeof(float) * (size_t)s_pitch, 0, sizeof(float) * (size_t)C, (size_t)N, st));
    CbnGeom g{N, H, W, C / 4, up, pad, skip_pitch, skip_off, skip_sh, slope, post_leaky};
    // enough CTAs to fill the GPU a few times, each with >= 1 row
    int rows = (int)(((long long)N * H + 132 * 8 - 1) / (132 * 8));
    rows = rows < 1 ? 1 : rows;
    rows += skip_sh && rows % 2;                          // a CTA owns whole 2 x 2 footprints of a half-resolution skip
    dim3 grid(b3d::ceil_div(H, rows), N);
    auto kernel = skip_sh ? (pad_mode == 0 ? (stat_pitch ? cbn_act_bwd1_kernel<0, true, 1> : cbn_act_bwd1_kernel<0, false, 1>)
                                           : (stat_pitch ? cbn_act_bwd1_kernel<1, true, 1> : cbn_act_bwd1_kernel<1, false, 1>))
                          : (pad_mode == 0 ? (stat_pitch ? cbn_act_bwd1_kernel<0, true, 0> : cbn_act_bwd1_kernel<0, false, 0>)
                                           : (stat_pitch ? cbn_act_bwd1_kernel<1, true, 0> : cbn_act_bwd1_kernel<1, false, 0>));
    kernel<<<grid, NT, 0, st>>>((const float4*)gout, (const float4*)y, (const float4*)scale, (const float4*)shift, (const float4*)skip,
                                (const float4*)mean, (const float4*)invstd, (float4*)ga, (float4*)gskip, gskip_pitch, gskip_off, S1, S2,
                                s_pitch, g, rows);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

// stat_pitch 0: mean / inv_std / m1 / m2 are [C] (batch statistics; m1, m2 = b3d_cbn_bwd_reduce's rows).  stat_pitch C:
// mean / inv_std are [N, C] and m1, m2 are bwd1's per-sample sums S1, S2 at row pitch m_pitch (a multiple of 4).
int b3d_cbn_act_bwd2(float* ga, const float* y, const float* gamma_t, const float* mean, const float* invstd, int stat_pitch,
                     const float* m1, const float* m2, int m_pitch, float inv_m, int N, int H, int W, int C, void* stream) {
    B3D_REQUIRE(N >= 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0, B3D_EINVAL, "b3d_cbn_act_bwd2: bad arguments");
    B3D_REQUIRE(stat_pitch == 0 || (stat_pitch == C && m_pitch >= C && m_pitch % 4 == 0), B3D_EINVAL,
                "b3d_cbn_act_bwd2: statistics pitch %d must be 0 or C=%d (sums pitch %d >= C, a multiple of 4)", stat_pitch, C, m_pitch);
    if (N == 0) return B3D_OK;
    B3D_REQUIRE(ga && y && gamma_t && mean && invstd && m1 && m2, B3D_EINVAL, "b3d_cbn_act_bwd2: null pointer");
    const long long per_n = (long long)H * W * (C / 4), total = per_n * N;
    auto kernel = stat_pitch ? cbn_act_bwd2_kernel<true> : cbn_act_bwd2_kernel<false>;
    kernel<<<grid_for(total), NT, 0, (cudaStream_t)stream>>>((float4*)ga, (const float4*)y, (const float4*)gamma_t, (const float4*)mean,
                                                             (const float4*)invstd, (const float4*)m1, (const float4*)m2, m_pitch / 4,
                                                             inv_m, per_n, C / 4, total);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

// fp64 per-channel sums [2][C] (sum, sum of squares) of y [rows, C], for callers that all-reduce the sums across ranks
// (SyncBN) and finish in b3d_cbn_prepare.  `sums` is zeroed here.
int b3d_bn_sums(const float* y, long long rows, int C, double* sums, void* stream) {
    B3D_REQUIRE(rows > 0 && C >= 4 && C % 4 == 0 && C / 4 <= NT && NT % (C / 4) == 0, B3D_EINVAL,
                "b3d_bn_sums: C=%d must be 4 * a divisor of %d", C, NT);
    B3D_REQUIRE(y && sums, B3D_EINVAL, "b3d_bn_sums: null pointer");
    B3D_CHECK_ALIGNED(y);
    cudaStream_t st = (cudaStream_t)stream;
    B3D_CUDA_OK(cudaMemsetAsync(sums, 0, sizeof(double) * 2 * (size_t)C, st));
    const int ppb = NT / (C / 4);
    long long blocks = (rows + ppb - 1) / ppb;
    if (blocks > 132 * 2) blocks = 132 * 2;                 // few blocks: every block ends with 2C same-address fp64 atomics
    bn_sums_kernel<false><<<(int)blocks, NT, 0, st>>>((const float4*)y, rows, C / 4, sums);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

// fp64 per-(sample, channel) sums [N][2][C] of y [N, HW, C] (InstanceNorm2d statistics, finished by b3d_cbn_prepare mode 3).
// `sums` is zeroed here.  About 264 CTAs in all, split over the samples, at least one per sample.
int b3d_bn_sums_per_sample(const float* y, int N, long long HW, int C, double* sums, void* stream) {
    B3D_REQUIRE(N > 0 && N <= 65535 && HW > 0 && C >= 4 && C % 4 == 0 && C / 4 <= NT && NT % (C / 4) == 0, B3D_EINVAL,
                "b3d_bn_sums_per_sample: N=%d (1..65535), C=%d must be 4 * a divisor of %d", N, C, NT);
    B3D_REQUIRE(y && sums, B3D_EINVAL, "b3d_bn_sums_per_sample: null pointer");
    B3D_CHECK_ALIGNED(y);
    cudaStream_t st = (cudaStream_t)stream;
    B3D_CUDA_OK(cudaMemsetAsync(sums, 0, sizeof(double) * 2 * (size_t)C * N, st));
    const int ppb = NT / (C / 4);
    long long blocks = (HW + ppb - 1) / ppb;
    const long long cap = (132 * 2 + N - 1) / N;
    if (blocks > cap) blocks = cap;
    bn_sums_kernel<true><<<dim3((unsigned)blocks, (unsigned)N), NT, 0, st>>>((const float4*)y, HW, C / 4, sums);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

// ConditionalBatchNorm2d scalar math in one launch (see cbn_prepare_kernel).  gb [N, gb_pitch]: row n holds gamma at
// gamma_off + c and beta at beta_off + c (the batched fc_gamma / fc_beta outputs of all layers).  mode 0 eval, 1 batch
// statistics (F.batch_norm formulas), 2 the reference's SyncBN formulas; sums [2][C] fp64 (modes 1, 2), count = values per
// channel over the (global) batch.  running_mean / running_var / num_batches_tracked (nullable) are updated in modes 1, 2.
// mode 3 instance statistics from sums [N][2][C] (b3d_bn_sums_per_sample), count = H*W; mode 4 no normalisation.
// Outputs: mean, invstd [C] ([N, C] in modes 3, 4); scale, shift, gt [N, C].
int b3d_cbn_prepare(const float* gb, int gb_pitch, int gamma_off, int beta_off, const double* sums, double count, float eps,
                    float momentum, int mode, float* running_mean, float* running_var, long long* num_batches_tracked,
                    float* mean, float* invstd, float* scale, float* shift, float* gt, int N, int C, void* stream) {
    B3D_REQUIRE(N > 0 && C > 0 && gb && mean && invstd && scale && shift && gt, B3D_EINVAL, "b3d_cbn_prepare: bad arguments");
    B3D_REQUIRE(mode >= 0 && mode <= 4, B3D_EINVAL, "b3d_cbn_prepare: unknown mode %d", mode);
    B3D_REQUIRE(mode == 0 ? (running_mean && running_var) : (mode == 4 || (sums != nullptr && count > 0)), B3D_EINVAL,
                "b3d_cbn_prepare: mode %d needs %s", mode, mode == 0 ? "running statistics" : "sums and a count");
    cbn_prepare_kernel<<<(N * C + NT - 1) / NT, NT, 0, (cudaStream_t)stream>>>(gb, gb_pitch, gamma_off, beta_off, sums, count, eps,
                                                                                momentum, mode, running_mean, running_var,
                                                                                num_batches_tracked, mean, invstd, scale, shift, gt, N, C);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

// red [2][C] from the per-sample sums of b3d_cbn_act_bwd1 (row pitch s_pitch) and gt [N,C]
int b3d_cbn_bwd_reduce(const float* S1, const float* S2, int s_pitch, const float* gt, float* red, int N, int C, void* stream) {
    B3D_REQUIRE(N > 0 && C > 0 && S1 && S2 && gt && red, B3D_EINVAL, "b3d_cbn_bwd_reduce: bad arguments");
    cbn_bwd_reduce_kernel<<<(C + NT - 1) / NT, NT, 0, (cudaStream_t)stream>>>(S1, S2, s_pitch, gt, red, N, C);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

// --- SyncBN with the collective fused in (one-shot all-reduce over NVLink peer memory; see peer_allreduce above) ---------
// peer_data / peer_flag: `world` device pointers each (rank order) into every rank's symmetric buffer: data
// [2][world][1024] doubles, flags [2][world] uint32 (zero-initialised once); epoch / err: this rank's own counters (zeroed
// once).  All ranks must issue the same sequence of *_sync calls.  world <= 8, C <= 512.
size_t b3d_sync_buffer_bytes(int world) { return (size_t)2 * world * SYNC_MAX * sizeof(double) + (size_t)2 * world * sizeof(unsigned) + 256; }
size_t b3d_sync_flag_offset(int world) { return (size_t)2 * world * SYNC_MAX * sizeof(double); }

static int fill_peers(SyncPeers& P, const void* const* peer_data, const void* const* peer_flag, int rank, int world, int C) {
    B3D_REQUIRE(world >= 2 && world <= SYNC_RANKS && rank >= 0 && rank < world, B3D_EINVAL, "sync: world=%d rank=%d (2..%d ranks)", world,
                rank, SYNC_RANKS);
    B3D_REQUIRE(C > 0 && 2 * C <= SYNC_MAX, B3D_EINVAL, "sync: C=%d exceeds %d", C, SYNC_MAX / 2);
    B3D_REQUIRE(peer_data && peer_flag, B3D_EINVAL, "sync: null peer tables");
    for (int p = 0; p < SYNC_RANKS; ++p) {
        P.data[p] = p < world ? (double*)const_cast<void*>(peer_data[p]) : nullptr;
        P.flag[p] = p < world ? (unsigned*)const_cast<void*>(peer_flag[p]) : nullptr;
        B3D_REQUIRE(p >= world || (P.data[p] && P.flag[p]), B3D_EINVAL, "sync: null peer pointer %d", p);
    }
    return B3D_OK;
}

int b3d_cbn_prepare_sync(const void* const* peer_data, const void* const* peer_flag, int rank, int world, unsigned* epoch, int* err,
                         const float* gb, int gb_pitch, int gamma_off, int beta_off, const double* sums_local, double count,
                         float eps, float momentum, float* running_mean, float* running_var, long long* num_batches_tracked,
                         float* mean, float* invstd, float* scale, float* shift, float* gt, int N, int C, void* stream) {
    SyncPeers P;
    if (int rc = fill_peers(P, peer_data, peer_flag, rank, world, C)) return rc;
    B3D_REQUIRE(N > 0 && gb && sums_local && count > 0 && mean && invstd && scale && shift && gt && epoch && err, B3D_EINVAL,
                "b3d_cbn_prepare_sync: bad arguments");
    cbn_prepare_sync_kernel<<<1, 512, 0, (cudaStream_t)stream>>>(P, rank, world, epoch, err, gb, gb_pitch, gamma_off, beta_off, sums_local,
                                                                count, eps, momentum, running_mean, running_var, num_batches_tracked,
                                                                mean, invstd, scale, shift, gt, N, C);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

int b3d_cbn_bwd_reduce_sync(const void* const* peer_data, const void* const* peer_flag, int rank, int world, unsigned* epoch, int* err,
                            const float* S1, const float* S2, int s_pitch, const float* gt, float* red, int N, int C, void* stream) {
    SyncPeers P;
    if (int rc = fill_peers(P, peer_data, peer_flag, rank, world, C)) return rc;
    B3D_REQUIRE(N > 0 && S1 && S2 && gt && red && epoch && err, B3D_EINVAL, "b3d_cbn_bwd_reduce_sync: bad arguments");
    cbn_bwd_reduce_sync_kernel<<<1, 512, 0, (cudaStream_t)stream>>>(P, rank, world, epoch, err, S1, S2, s_pitch, gt, red, N, C);
    B3D_LAUNCH_OK();
    return B3D_OK;
}
}
