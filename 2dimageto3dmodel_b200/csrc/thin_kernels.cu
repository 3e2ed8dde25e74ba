// Thin-head convolutions of the GAN: 5x5 layers with 1-4 OUTPUT channels (generator conv_final 64 -> 3, models/gan.py:359;
// discriminator heads 512 -> 1 / 256 -> 1, models/gan.py:177, :302).  On the tensor-core path such a layer pads its
// 1-3 output channels to a 64-wide MMA tile and re-fetches the input once per tap, for 0.3 % of the network's FLOPs.  They are reductions over (tap, ci) with almost no output, so they run
// here on the fp32 CUDA cores with the channel dimension across the lanes of a warp (coalesced NHWC reads, the 25x
// tap reuse served by L1):
//   fwd    one warp = 4 adjacent output pixels of one row; per filter row the 4 + kw - 1 input pixels are loaded once
//          into registers and reused by every (output, s) pair; 4 x COUT warp reductions at the end.
//   wgrad  one warp = a whole output row for one block of 32*VEC input channels; COUT x 25 x VEC accumulators per
//          lane stay in registers along the row, a block folds its warps in shared memory, then one global atomicAdd
//          per weight per block.
// The input gradient of these layers stays on the tensor-core dgrad (N = Cin is wide there).
#include <stdlib.h>

#include "b3d_common.cuh"

namespace {

constexpr int NT = 256, KS = 5;

template <int VEC> struct Vec;
template <> struct Vec<2> { using T = float2; };
template <> struct Vec<4> { using T = float4; };

template <int VEC>
__device__ __forceinline__ void ldv(float (&d)[VEC], const float* p) {
    const typename Vec<VEC>::T v = __ldg(reinterpret_cast<const typename Vec<VEC>::T*>(p));
    if constexpr (VEC == 2) { d[0] = v.x; d[1] = v.y; } else { d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w; }
}

struct ThinGeom {
    int N, H, W, Cin, Hout, Wout, pad_y, xoff;
    int OW, OC;              // output pixel pitch / channel pitch (fwd)
    float leaky;
    int tapmajor;            // wgrad: dW layout 0 = [Cout][Cin][5][5], 1 = tap-major [25][Cout][Cin]
};

// wt [KS][KS][COUT][Cin]
constexpr int OUTS = 8;                       // adjacent output pixels per warp

template <int COUT, int VEC>
__global__ void __launch_bounds__(NT)
conv_thin_fwd_kernel(const float* __restrict__ x, const float* __restrict__ wt, const float* __restrict__ bias,
                     float* __restrict__ out, const ThinGeom g) {
    const int lane = threadIdx.x & 31;
    const int warps_total = gridDim.x * (NT / 32);
    const int xg = (g.Wout + OUTS - 1) / OUTS;
    const long long items = (long long)g.N * g.Hout * xg;
    for (long long it = (long long)blockIdx.x * (NT / 32) + (threadIdx.x >> 5); it < items; it += warps_total) {
        const int x0 = (int)(it % xg) * OUTS;
        const int y = (int)((it / xg) % g.Hout);
        const int n = (int)(it / ((long long)xg * g.Hout));
        float acc[OUTS][COUT];
#pragma unroll
        for (int o = 0; o < OUTS; ++o)
#pragma unroll
            for (int c = 0; c < COUT; ++c) acc[o][c] = 0.f;
        for (int c0 = 0; c0 < g.Cin; c0 += 32 * VEC) {
            const int ci = c0 + lane * VEC;
#pragma unroll 1
            for (int r = 0; r < KS; ++r) {
                // rows outside the image contribute zeros (the y padding): clamp the address, zero the values — no
                // branch between the loads, so a whole row of requests is in flight at once
                const int yy = y + r - g.pad_y;
                const float rv = (yy >= 0 && yy < g.H) ? 1.f : 0.f;
                const int yc = yy < 0 ? 0 : (yy >= g.H ? g.H - 1 : yy);
                const float* row = x + (((long long)n * g.H + yc) * g.W) * g.Cin + ci;
                float px[OUTS + KS - 1][VEC];
#pragma unroll
                for (int j = 0; j < OUTS + KS - 1; ++j) {
                    const int xx = x0 + j + g.xoff;
                    ldv<VEC>(px[j], row + (long long)(xx < g.W ? xx : g.W - 1) * g.Cin);     // columns >= W feed dropped outputs only
#pragma unroll
                    for (int v = 0; v < VEC; ++v) px[j][v] *= rv;
                }
#pragma unroll
                for (int s = 0; s < KS; ++s) {
#pragma unroll
                    for (int c = 0; c < COUT; ++c) {
                        float wv[VEC];
                        ldv<VEC>(wv, wt + ((long long)((r * KS + s) * COUT + c)) * g.Cin + ci);
#pragma unroll
                        for (int o = 0; o < OUTS; ++o)
#pragma unroll
                            for (int v = 0; v < VEC; ++v) acc[o][c] = fmaf(px[o + s][v], wv[v], acc[o][c]);
                    }
                }
            }
        }
        // OUTS x COUT sums over the lanes: butterfly that leaves output o's sums in lane o
#pragma unroll
        for (int c = 0; c < COUT; ++c) {
            float mine = 0.f;
#pragma unroll
            for (int o = 0; o < OUTS; ++o) {
                const float t = b3d::warp_sum(acc[o][c]);
                if (lane == o) mine = t;
            }
            if (lane < OUTS && x0 + lane < g.Wout) {
                float v = mine + (bias ? __ldg(bias + c) : 0.f);
                v = v >= 0.f ? v : v * g.leaky;
                out[(((long long)n * g.Hout + y) * g.OW + x0 + lane) * g.OC + c] = v;
            }
        }
    }
}

// dw [COUT][Cin][KS][KS] += sum_pix gy[pix][co] * x[pix + (r - pad_y, s + xoff)][ci]
template <int COUT, int VEC>
__global__ void __launch_bounds__(NT)
conv_thin_wgrad_kernel(const float* __restrict__ gy, const float* __restrict__ x, float* __restrict__ dw, const ThinGeom g) {
    extern __shared__ float red[];                 // [COUT][KS*KS][32*VEC]
    const int lane = threadIdx.x & 31;
    const int chunks = g.Cin / (32 * VEC);
    const int blocks_per_chunk = gridDim.x / chunks;
    const int chunk = blockIdx.x / blocks_per_chunk, blk = blockIdx.x % blocks_per_chunk;
    const int ci = chunk * 32 * VEC + lane * VEC;
    for (int i = threadIdx.x; i < COUT * KS * KS * 32 * VEC; i += NT) red[i] = 0.f;
    __syncthreads();
    float acc[COUT][KS * KS][VEC];
#pragma unroll
    for (int c = 0; c < COUT; ++c)
#pragma unroll
        for (int t = 0; t < KS * KS; ++t)
#pragma unroll
            for (int v = 0; v < VEC; ++v) acc[c][t][v] = 0.f;
    const int rows = g.N * g.Hout;
    const int wstride = blocks_per_chunk * (NT / 32);
    for (int row = blk * (NT / 32) + (threadIdx.x >> 5); row < rows; row += wstride) {
        const int n = row / g.Hout, y = row % g.Hout;
        const float* gyr = gy + (long long)row * g.Wout * COUT;
#pragma unroll 1
        for (int xo = 0; xo < g.Wout; ++xo) {
            float gv[COUT];
#pragma unroll
            for (int c = 0; c < COUT; ++c) gv[c] = __ldg(gyr + xo * COUT + c);
            // all 25 input pixels of this output pixel are requested before the first FMA (no branches in between:
            // x + s + xoff < W by the geometry check; rows outside the image are clamped and masked)
            float xv[KS * KS][VEC];
#pragma unroll
            for (int r = 0; r < KS; ++r) {
                const int yy = y + r - g.pad_y;
                const int yc = yy < 0 ? 0 : (yy >= g.H ? g.H - 1 : yy);
                const float* xr = x + (((long long)n * g.H + yc) * g.W + xo + g.xoff) * g.Cin + ci;
#pragma unroll
                for (int s = 0; s < KS; ++s) ldv<VEC>(xv[r * KS + s], xr + (long long)s * g.Cin);
            }
#pragma unroll
            for (int r = 0; r < KS; ++r) {
                const int yy = y + r - g.pad_y;
                const float rv = (yy >= 0 && yy < g.H) ? 1.f : 0.f;
#pragma unroll
                for (int c = 0; c < COUT; ++c) {
                    const float gm = gv[c] * rv;
#pragma unroll
                    for (int s = 0; s < KS; ++s)
#pragma unroll
                        for (int v = 0; v < VEC; ++v) acc[c][r * KS + s][v] = fmaf(gm, xv[r * KS + s][v], acc[c][r * KS + s][v]);
                }
            }
        }
    }
#pragma unroll
    for (int c = 0; c < COUT; ++c)
#pragma unroll
        for (int t = 0; t < KS * KS; ++t)
#pragma unroll
            for (int v = 0; v < VEC; ++v) atomicAdd(red + (c * KS * KS + t) * 32 * VEC + lane * VEC + v, acc[c][t][v]);
    __syncthreads();
    for (int i = threadIdx.x; i < COUT * KS * KS * 32 * VEC; i += NT) {
        const int cl = i % (32 * VEC), t = (i / (32 * VEC)) % (KS * KS), c = i / (32 * VEC * KS * KS);
        const int ci = chunk * 32 * VEC + cl;
        atomicAdd(g.tapmajor ? dw + ((long long)t * COUT + c) * g.Cin + ci : dw + ((long long)c * g.Cin + ci) * (KS * KS) + t, red[i]);
    }
}

// Sliding-window variant: along an output row the 5x5 input window moves by one column per pixel, so only its new
// column (5 loads) is fetched per pixel instead of all 25 taps; the window lives in registers (slots rotate mod 5, the
// row loop is unrolled by 5 so every slot index is static) and the new column is requested before the 4/5 of the FMAs
// that do not need it (a 25-loads version leaves the FFMAs waiting on the loads at low occupancy).
template <int COUT, int VEC>
__global__ void __launch_bounds__(NT)
conv_thin_wgrad_win_kernel(const float* __restrict__ gy, const float* __restrict__ x, float* __restrict__ dw, const ThinGeom g) {
    extern __shared__ float red[];                 // [COUT][KS*KS][32*VEC]
    const int lane = threadIdx.x & 31;
    const int chunks = g.Cin / (32 * VEC);
    const int blocks_per_chunk = gridDim.x / chunks;
    const int chunk = blockIdx.x / blocks_per_chunk, blk = blockIdx.x % blocks_per_chunk;
    const int ci = chunk * 32 * VEC + lane * VEC;
    for (int i = threadIdx.x; i < COUT * KS * KS * 32 * VEC; i += NT) red[i] = 0.f;
    __syncthreads();
    float acc[COUT][KS * KS][VEC];
#pragma unroll
    for (int c = 0; c < COUT; ++c)
#pragma unroll
        for (int t = 0; t < KS * KS; ++t)
#pragma unroll
            for (int v = 0; v < VEC; ++v) acc[c][t][v] = 0.f;
    const int rows = g.N * g.Hout;
    const int wstride = blocks_per_chunk * (NT / 32);
    for (int row = blk * (NT / 32) + (threadIdx.x >> 5); row < rows; row += wstride) {
        const int n = row / g.Hout, y = row % g.Hout;
        const float* gyr = gy + (long long)row * g.Wout * COUT;
        const float* xr[KS];
        float rv[KS];
#pragma unroll
        for (int r = 0; r < KS; ++r) {
            const int yy = y + r - g.pad_y;
            rv[r] = (yy >= 0 && yy < g.H) ? 1.f : 0.f;                      // rows outside the image: clamp + mask
            const int yc = yy < 0 ? 0 : (yy >= g.H ? g.H - 1 : yy);
            xr[r] = x + (((long long)n * g.H + yc) * g.W + g.xoff) * g.Cin + ci;
        }
        float win[KS][KS][VEC];                    // win[r][slot]: input column (xo + j) lives in slot (xo + j) % 5
#pragma unroll
        for (int r = 0; r < KS; ++r)
#pragma unroll
            for (int j = 0; j < KS - 1; ++j) {
                ldv<VEC>(win[r][j], xr[r] + (long long)j * g.Cin);
#pragma unroll
                for (int v = 0; v < VEC; ++v) win[r][j][v] *= rv[r];
            }
#pragma unroll 1
        for (int xb = 0; xb < g.Wout; xb += KS) {
#pragma unroll
            for (int u = 0; u < KS; ++u) {
                const int xo = xb + u;
                if (xo < g.Wout) {
                    float nw[KS][VEC];                                      // new column xo + 4: requested first ...
#pragma unroll
                    for (int r = 0; r < KS; ++r) ldv<VEC>(nw[r], xr[r] + (long long)(xo + KS - 1) * g.Cin);
                    float gv[COUT];
#pragma unroll
                    for (int c = 0; c < COUT; ++c) gv[c] = __ldg(gyr + xo * COUT + c);
#pragma unroll
                    for (int s = 0; s < KS - 1; ++s)                        // ... the taps that do not need it run meanwhile
#pragma unroll
                        for (int r = 0; r < KS; ++r)
#pragma unroll
                            for (int c = 0; c < COUT; ++c)
#pragma unroll
                                for (int v = 0; v < VEC; ++v)
                                    acc[c][r * KS + s][v] = fmaf(gv[c], win[r][(u + s) % KS][v], acc[c][r * KS + s][v]);
#pragma unroll
                    for (int r = 0; r < KS; ++r)                            // ... then it enters slot (u + 4) % 5
#pragma unroll
                        for (int v = 0; v < VEC; ++v) {
                            const float m = nw[r][v] * rv[r];
                            win[r][(u + KS - 1) % KS][v] = m;
#pragma unroll
                            for (int c = 0; c < COUT; ++c)
                                acc[c][r * KS + KS - 1][v] = fmaf(gv[c], m, acc[c][r * KS + KS - 1][v]);
                        }
                }
            }
        }
    }
#pragma unroll
    for (int c = 0; c < COUT; ++c)
#pragma unroll
        for (int t = 0; t < KS * KS; ++t)
#pragma unroll
            for (int v = 0; v < VEC; ++v) atomicAdd(red + (c * KS * KS + t) * 32 * VEC + lane * VEC + v, acc[c][t][v]);
    __syncthreads();
    for (int i = threadIdx.x; i < COUT * KS * KS * 32 * VEC; i += NT) {
        const int cl = i % (32 * VEC), t = (i / (32 * VEC)) % (KS * KS), c = i / (32 * VEC * KS * KS);
        const int ci = chunk * 32 * VEC + cl;
        atomicAdd(g.tapmajor ? dw + ((long long)t * COUT + c) * g.Cin + ci : dw + ((long long)c * g.Cin + ci) * (KS * KS) + t, red[i]);
    }
}

template <int COUT, int VEC>
int launch_fwd(const float* x, const float* wt, const float* bias, float* out, const ThinGeom& g, cudaStream_t st) {
    const long long items = (long long)g.N * g.Hout * ((g.Wout + OUTS - 1) / OUTS);
    long long blocks = (items + NT / 32 - 1) / (NT / 32);
    if (blocks > 132 * 16) blocks = 132 * 16;
    conv_thin_fwd_kernel<COUT, VEC><<<(int)blocks, NT, 0, st>>>(x, wt, bias, out, g);
    B3D_LAUNCH_OK();
    b3d::clear_variant();
    b3d::add_variant("conv_thin_fwd<%d,%d>", COUT, VEC);
    return B3D_OK;
}

template <int COUT, int VEC>
int launch_wgrad(const float* gy, const float* x, float* dw, const ThinGeom& g, cudaStream_t st) {
    const int chunks = g.Cin / (32 * VEC);
    int bpc = (132 * 2 + chunks - 1) / chunks;
    const int rows = g.N * g.Hout;
    if (bpc > (rows + NT / 32 - 1) / (NT / 32)) bpc = (rows + NT / 32 - 1) / (NT / 32);
    const size_t smem = (size_t)COUT * KS * KS * 32 * VEC * 4;
    B3D_CUDA_OK(cudaFuncSetAttribute(conv_thin_wgrad_kernel<COUT, VEC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    constexpr bool win = COUT * VEC <= 6;          // window (25 * VEC) + accumulators (COUT * 25 * VEC) fit the register file
    if (win) {
        B3D_CUDA_OK(cudaFuncSetAttribute(conv_thin_wgrad_win_kernel<COUT, VEC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        conv_thin_wgrad_win_kernel<COUT, VEC><<<bpc * chunks, NT, smem, st>>>(gy, x, dw, g);
    } else {
        conv_thin_wgrad_kernel<COUT, VEC><<<bpc * chunks, NT, smem, st>>>(gy, x, dw, g);
    }
    B3D_LAUNCH_OK();
    b3d::clear_variant();
    b3d::add_variant(win ? "conv_thin_wgrad_win<%d,%d>" : "conv_thin_wgrad<%d,%d>", COUT, VEC);
    return B3D_OK;
}

int check_geom(const char* fn, int N, int H, int W, int Cin, int Hout, int Wout, int Cout, int kh, int kw, int pad_y, int x_off) {
    B3D_REQUIRE(N > 0 && H > 0 && W > 0 && Hout > 0 && Wout > 0, B3D_EINVAL, "%s: bad sizes", fn);
    B3D_REQUIRE(kh == KS && kw == KS, B3D_EINVAL, "%s: only 5x5 kernels (got %dx%d)", fn, kh, kw);
    B3D_REQUIRE(Cout >= 1 && Cout <= 4, B3D_EINVAL, "%s: Cout=%d must be 1..4", fn, Cout);
    B3D_REQUIRE(Cin >= 64 && Cin % 64 == 0, B3D_EINVAL, "%s: Cin=%d must be a multiple of 64", fn, Cin);
    B3D_REQUIRE(pad_y >= 0 && x_off >= 0 && Hout == H + 2 * pad_y - kh + 1 && Wout + kw - 1 + x_off <= W, B3D_EINVAL,
                "%s: geometry mismatch (stride 1, zero padding along y only)", fn);
    return B3D_OK;
}

}  // namespace

extern "C" {

int b3d_conv2d_thin_fwd(const float* x, const float* wt, const float* bias, float* out, int N, int H, int W, int Cin, int Hout,
                        int Wout, int Cout, int kh, int kw, int pad_y, int x_off, int OW, int OC, float leaky, void* stream) {
    if (int rc = check_geom("b3d_conv2d_thin_fwd", N, H, W, Cin, Hout, Wout, Cout, kh, kw, pad_y, x_off)) return rc;
    B3D_REQUIRE(x && wt && out, B3D_EINVAL, "b3d_conv2d_thin_fwd: null pointer");
    B3D_REQUIRE(OW >= Wout && OC >= Cout, B3D_EINVAL, "b3d_conv2d_thin_fwd: output pitch smaller than the output");
    B3D_CHECK_ALIGNED(x);
    B3D_CHECK_ALIGNED(wt);
    ThinGeom g{N, H, W, Cin, Hout, Wout, pad_y, x_off, OW, OC, leaky, 0};
    cudaStream_t st = (cudaStream_t)stream;
    const bool v4 = Cin % 128 == 0;
    switch (Cout * 2 + (v4 ? 1 : 0)) {
        case 2: return launch_fwd<1, 2>(x, wt, bias, out, g, st);
        case 3: return launch_fwd<1, 4>(x, wt, bias, out, g, st);
        case 4: return launch_fwd<2, 2>(x, wt, bias, out, g, st);
        case 5: return launch_fwd<2, 4>(x, wt, bias, out, g, st);
        case 6: return launch_fwd<3, 2>(x, wt, bias, out, g, st);
        case 7: return launch_fwd<3, 4>(x, wt, bias, out, g, st);
        case 8: return launch_fwd<4, 2>(x, wt, bias, out, g, st);
        default: return launch_fwd<4, 4>(x, wt, bias, out, g, st);
    }
}

int b3d_conv2d_thin_wgrad(const float* dy, const float* x, float* dw, int N, int H, int W, int Cin, int Hout, int Wout, int Cout,
                          int kh, int kw, int pad_y, int x_off, int tap_major, void* stream) {
    if (int rc = check_geom("b3d_conv2d_thin_wgrad", N, H, W, Cin, Hout, Wout, Cout, kh, kw, pad_y, x_off)) return rc;
    B3D_REQUIRE(dy && x && dw, B3D_EINVAL, "b3d_conv2d_thin_wgrad: null pointer");
    B3D_CHECK_ALIGNED(x);
    ThinGeom g{N, H, W, Cin, Hout, Wout, pad_y, x_off, Wout, Cout, 1.f, tap_major ? 1 : 0};
    cudaStream_t st = (cudaStream_t)stream;
    // 4-wide lanes only where COUT * 25 * 4 accumulators fit the register file (Cout == 1)
    const bool v4 = Cin % 128 == 0 && Cout == 1;
    switch (Cout * 2 + (v4 ? 1 : 0)) {
        case 2: return launch_wgrad<1, 2>(dy, x, dw, g, st);
        case 3: return launch_wgrad<1, 4>(dy, x, dw, g, st);
        case 4: return launch_wgrad<2, 2>(dy, x, dw, g, st);
        case 5: return launch_wgrad<2, 2>(dy, x, dw, g, st);
        case 6: return launch_wgrad<3, 2>(dy, x, dw, g, st);
        default: return launch_wgrad<4, 2>(dy, x, dw, g, st);
    }
}
}
