// FID evaluation path (SURVEY.md §8f rank 4: evaluate_fid, main.py:188-412; utils/fid.py; utils/inception.py) for sm_90a.
// The Inception convolutions run on the wgmma kernels of tc_conv.cu (BatchNorm folded, ReLU in the epilogue, branch
// outputs written straight into their channel slice of the concatenated tensor); this file holds the rest of the network
// and the statistics:
//   inception_input_kernel   utils/inception.py:123-131: bilinear resize to 299 x 299 (align_corners=False), 2x - 1,
//                            NCHW planes -> NHWC with the 3 channels zero-padded to one 32-channel K slice
//   maxpool3x3s2_kernel      nn.MaxPool2d(3, stride 2) / F.max_pool2d(x, 3, 2) on NHWC, optionally into a channel slice
//   mean_hw_kernel           AdaptiveAvgPool2d((1, 1)) -> [N, C]
//   fid_accumulate_kernel    running sums for calculate_stats (utils/fid.py:27-30): sum_k x_k and sum_k x_k x_k^T in fp64
// (3 x 3 average pools never run as such: avg_pool(3, 1, 1, count_include_pad) followed by a 1 x 1 convolution IS a 3 x 3
// convolution with every tap = w / 9, which the host builds once — utils/inception.py here.)
#include "b3d_common.cuh"

namespace {
constexpr int NT = 256;

// torch's upsample_bilinear2d source index, align_corners = False: max((dst + 0.5) * scale - 0.5, 0)
__device__ __forceinline__ void src_index(int dst, float scale, int in, int& i0, int& i1, float& l1) {
    float s = ((float)dst + 0.5f) * scale - 0.5f;
    s = s < 0.f ? 0.f : s;
    i0 = min((int)s, in - 1);
    i1 = min(i0 + 1, in - 1);
    l1 = s - (float)i0;
}

__global__ void __launch_bounds__(NT)
inception_input_kernel(const float* __restrict__ img, int B, int H, int W, int OH, int OW, int OC, int normalize,
                       float* __restrict__ out) {
    const size_t total = (size_t)B * OH * OW;
    const float sh = (float)H / (float)OH, sw = (float)W / (float)OW;
    for (size_t i = (size_t)blockIdx.x * NT + threadIdx.x; i < total; i += (size_t)gridDim.x * NT) {
        const int ox = (int)(i % OW), oy = (int)((i / OW) % OH), b = (int)(i / ((size_t)OW * OH));
        int y0, y1, x0, x1;
        float ly, lx;
        src_index(oy, sh, H, y0, y1, ly);
        src_index(ox, sw, W, x0, x1, lx);
        float v[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float* p = img + ((size_t)b * 3 + c) * H * W;
            const float a = (1.f - lx) * p[(size_t)y0 * W + x0] + lx * p[(size_t)y0 * W + x1];
            const float d = (1.f - lx) * p[(size_t)y1 * W + x0] + lx * p[(size_t)y1 * W + x1];
            const float r = (1.f - ly) * a + ly * d;
            v[c] = normalize ? 2.f * r - 1.f : r;
        }
        float4* o = reinterpret_cast<float4*>(out + i * OC);
        o[0] = make_float4(v[0], v[1], v[2], 0.f);
        for (int j = 1; j < OC / 4; ++j) o[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

// x [N, H, W, C] -> out[n, oy, ox, 0..C) of a tensor with OC channels per pixel (`out` already points at the slice)
__global__ void __launch_bounds__(NT)
maxpool3x3s2_kernel(const float4* __restrict__ x, int N, int H, int W, int C4, int OH, int OW, int OC4,
                    float4* __restrict__ out) {
    const size_t total = (size_t)N * OH * OW * C4;
    for (size_t i = (size_t)blockIdx.x * NT + threadIdx.x; i < total; i += (size_t)gridDim.x * NT) {
        const int c = (int)(i % C4);
        const size_t pix = i / C4;
        const int ox = (int)(pix % OW), oy = (int)((pix / OW) % OH), n = (int)(pix / ((size_t)OW * OH));
        const float4* p = x + (((size_t)n * H + 2 * oy) * W + 2 * ox) * C4 + c;
        float4 m = p[0];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int s = 0; s < 3; ++s) {
                const float4 v = p[((size_t)r * W + s) * C4];
                // torch's max propagates NaN: (v > m) || isnan(v)
                m.x = (v.x > m.x || v.x != v.x) ? v.x : m.x;
                m.y = (v.y > m.y || v.y != v.y) ? v.y : m.y;
                m.z = (v.z > m.z || v.z != v.z) ? v.z : m.z;
                m.w = (v.w > m.w || v.w != v.w) ? v.w : m.w;
            }
        out[pix * OC4 + c] = m;
    }
}

__global__ void __launch_bounds__(NT)
mean_hw_kernel(const float* __restrict__ x, int N, int HW, int C, float* __restrict__ out) {
    const int i = blockIdx.x * NT + threadIdx.x;
    if (i >= N * C) return;
    const int n = i / C, c = i % C;
    const float* p = x + (size_t)n * HW * C + c;
    float s = 0.f;
    for (int k = 0; k < HW; ++k) s += p[(size_t)k * C];
    out[i] = s / (float)HW;
}

// outer[i, j] += sum_k f[k, i] f[k, j] (fp64), sum[i] += sum_k f[k, i]; one 32 x 32 tile of `outer` per CTA
constexpr int FT = 32;
__global__ void __launch_bounds__(NT)
fid_accumulate_kernel(const float* __restrict__ f, int n, int D, double* __restrict__ sum, double* __restrict__ outer) {
    __shared__ float a[FT][FT + 1], b[FT][FT + 1];
    const int i0 = blockIdx.y * FT, j0 = blockIdx.x * FT;
    const int tx = threadIdx.x % FT, ty = threadIdx.x / FT;      // 32 x 8 threads; thread owns rows ty, ty + 8, ... of column tx
    double acc[FT / 8] = {0.0, 0.0, 0.0, 0.0};
    double csum = 0.0;
    for (int k0 = 0; k0 < n; k0 += FT) {
        for (int r = ty; r < FT; r += 8) {
            const int k = k0 + r;
            a[r][tx] = (k < n && i0 + tx < D) ? f[(size_t)k * D + i0 + tx] : 0.f;
            b[r][tx] = (k < n && j0 + tx < D) ? f[(size_t)k * D + j0 + tx] : 0.f;
        }
        __syncthreads();
        for (int r = 0; r < FT; ++r) {
            const double bj = (double)b[r][tx];
#pragma unroll
            for (int q = 0; q < FT / 8; ++q) acc[q] = fma((double)a[r][ty + 8 * q], bj, acc[q]);
            if (blockIdx.y == 0 && ty == 0) csum += bj;
        }
        __syncthreads();
    }
#pragma unroll
    for (int q = 0; q < FT / 8; ++q) {
        const int i = i0 + ty + 8 * q, j = j0 + tx;
        if (i < D && j < D) outer[(size_t)i * D + j] += acc[q];   // tiles are disjoint, launches are stream ordered
    }
    if (blockIdx.y == 0 && ty == 0 && j0 + tx < D) sum[j0 + tx] += csum;
}

inline int grid_for(size_t total) {
    const size_t b = (total + NT - 1) / NT;
    return (int)(b < 132 * 16 ? (b ? b : 1) : 132 * 16);
}

}  // namespace

extern "C" {

int b3d_inception_input(const float* img, int B, int H, int W, int OH, int OW, int OC, int normalize, float* out, void* stream) {
    B3D_REQUIRE(B >= 0 && H > 0 && W > 0 && OH > 0 && OW > 0, B3D_EINVAL, "b3d_inception_input: bad sizes");
    B3D_REQUIRE(OC >= 4 && OC % 4 == 0, B3D_EINVAL, "b3d_inception_input: OC=%d must be a multiple of 4", OC);
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(img && out, B3D_EINVAL, "b3d_inception_input: null pointer");
    B3D_CHECK_ALIGNED(out);
    inception_input_kernel<<<grid_for((size_t)B * OH * OW), NT, 0, (cudaStream_t)stream>>>(img, B, H, W, OH, OW, OC, normalize, out);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

int b3d_maxpool3x3s2_nhwc(const float* x, int N, int H, int W, int C, float* out, int OC, void* stream) {
    B3D_REQUIRE(N >= 0 && H >= 3 && W >= 3 && C > 0, B3D_EINVAL, "b3d_maxpool3x3s2_nhwc: bad sizes");
    B3D_REQUIRE(C % 4 == 0 && OC % 4 == 0 && OC >= C, B3D_EINVAL, "b3d_maxpool3x3s2_nhwc: C=%d, OC=%d must be multiples of 4, OC >= C", C, OC);
    if (N == 0) return B3D_OK;
    B3D_REQUIRE(x && out, B3D_EINVAL, "b3d_maxpool3x3s2_nhwc: null pointer");
    B3D_CHECK_ALIGNED(x);
    B3D_CHECK_ALIGNED(out);
    const int OH = (H - 3) / 2 + 1, OW = (W - 3) / 2 + 1;
    maxpool3x3s2_kernel<<<grid_for((size_t)N * OH * OW * (C / 4)), NT, 0, (cudaStream_t)stream>>>(
        (const float4*)x, N, H, W, C / 4, OH, OW, OC / 4, (float4*)out);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

int b3d_mean_hw_nhwc(const float* x, int N, int HW, int C, float* out, void* stream) {
    B3D_REQUIRE(N >= 0 && HW > 0 && C > 0, B3D_EINVAL, "b3d_mean_hw_nhwc: bad sizes");
    if (N == 0) return B3D_OK;
    B3D_REQUIRE(x && out, B3D_EINVAL, "b3d_mean_hw_nhwc: null pointer");
    mean_hw_kernel<<<b3d::ceil_div(N * C, NT), NT, 0, (cudaStream_t)stream>>>(x, N, HW, C, out);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

int b3d_fid_accumulate(const float* feat, int n, int D, double* sum, double* outer, void* stream) {
    B3D_REQUIRE(n >= 0 && D > 0, B3D_EINVAL, "b3d_fid_accumulate: bad sizes");
    if (n == 0) return B3D_OK;
    B3D_REQUIRE(feat && sum && outer, B3D_EINVAL, "b3d_fid_accumulate: null pointer");
    dim3 grid(b3d::ceil_div(D, FT), b3d::ceil_div(D, FT));
    fid_accumulate_kernel<<<grid, NT, 0, (cudaStream_t)stream>>>(feat, n, D, sum, outer);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

}  // extern "C"
