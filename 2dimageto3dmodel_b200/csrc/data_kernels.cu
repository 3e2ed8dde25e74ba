// GAN training data: batch assembly from packed pseudo-ground-truth stores (data/abstract_dataset.py:68-107,
// main.py:672-690).  One memory-bound launch per batch: gather by index, widen fp16 -> fp32, mirror in UV space.
#include <cuda_fp16.h>

#include "b3d_common.cuh"

namespace {

constexpr int NT = 256;

struct GatherArgs {
    b3d_gather_field f[B3D_GATHER_MAX_FIELDS];
    int vec[B3D_GATHER_MAX_FIELDS];             // output elements per thread (8 fp16, 4 fp32, else 1)
    long long items[B3D_GATHER_MAX_FIELDS];     // threads with work per field
    int block_end[B3D_GATHER_MAX_FIELDS];       // exclusive prefix of the blocks of each field
    const int32_t* idx;
    const uint8_t* flip;
};

__device__ __forceinline__ float affine(float x, float scale, float bias) {
    return (scale == 1.f && bias == 0.f) ? x : __fadd_rn(__fmul_rn(x, scale), bias);
}

template <int VEC>
__device__ __forceinline__ void load_vec(const b3d_gather_field& f, long long off, float* v) {
    if (f.src_type == B3D_GATHER_F16) {
        if constexpr (VEC == 8) {
            const uint4 raw = *reinterpret_cast<const uint4*>(static_cast<const __half*>(f.src) + off);
            const __half2* h = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float2 p = __half22float2(h[k]);
                v[2 * k] = p.x;
                v[2 * k + 1] = p.y;
            }
        } else {
            v[0] = __half2float(static_cast<const __half*>(f.src)[off]);
        }
    } else if constexpr (VEC == 4) {
        const float4 p = *reinterpret_cast<const float4*>(static_cast<const float*>(f.src) + off);
        v[0] = p.x, v[1] = p.y, v[2] = p.z, v[3] = p.w;
    } else {
        v[0] = static_cast<const float*>(f.src)[off];
    }
}

// One thread: VEC consecutive output elements of one row (b, c, y) of field f.
template <int VEC>
__device__ __forceinline__ void gather_run(const b3d_gather_field& f, const GatherArgs& a, long long t) {
    const int wv = f.W / VEC;
    const int x = (int)(t % wv) * VEC;
    long long r = t / wv;
    const int y = (int)(r % f.H);
    r /= f.H;
    const int c = (int)(r % f.C);
    const int b = (int)(r / f.C);
    const long long plane = (long long)f.H * f.W;
    const long long out = ((long long)b * f.C + c) * plane + (long long)y * f.W + x;
    const int s = a.idx[b];
    const bool ok = s >= 0 && s < f.n;
    const long long row = ((long long)s * f.C_src + c) * plane + (long long)y * f.W;

    if (f.src_type == B3D_GATHER_I64) {
        static_cast<long long*>(f.dst)[out] = ok ? static_cast<const long long*>(f.src)[row + x] : -1;
        return;
    }
    float v[VEC];
    if (ok) {
        const bool m = f.mirror && a.flip && a.flip[b];
        // mirrored: the run x .. x+VEC-1 reads columns W-1-((x+W/2) mod W) downwards; VEC divides W/2, so the run does not
        // wrap and starts on a vector boundary
        const int sx = m ? f.W - VEC - (x + f.W / 2) % f.W : x;
        load_vec<VEC>(f, row + sx, v);
        if (m) {
#pragma unroll
            for (int k = 0; k < VEC / 2; ++k) {
                const float tmp = v[k];
                v[k] = v[VEC - 1 - k];
                v[VEC - 1 - k] = tmp;
            }
        }
#pragma unroll
        for (int k = 0; k < VEC; ++k) v[k] = affine(v[k], f.scale, f.bias);
    } else {
#pragma unroll
        for (int k = 0; k < VEC; ++k) v[k] = __int_as_float(0x7fc00000);
    }
    float* dst = static_cast<float*>(f.dst) + out;
    if constexpr (VEC == 1) {
        dst[0] = v[0];
    } else {
#pragma unroll
        for (int k = 0; k < VEC / 4; ++k) reinterpret_cast<float4*>(dst)[k] = make_float4(v[4 * k], v[4 * k + 1], v[4 * k + 2], v[4 * k + 3]);
    }
}

__global__ void __launch_bounds__(NT) gather_fields_kernel(const __grid_constant__ GatherArgs a) {
    int fi = 0;
    while ((int)blockIdx.x >= a.block_end[fi]) ++fi;
    const b3d_gather_field& f = a.f[fi];
    const long long t = (long long)(blockIdx.x - (fi ? a.block_end[fi - 1] : 0)) * NT + threadIdx.x;
    if (t >= a.items[fi]) return;
    switch (a.vec[fi]) {
        case 8: gather_run<8>(f, a, t); break;
        case 4: gather_run<4>(f, a, t); break;
        default: gather_run<1>(f, a, t); break;
    }
}

// device memory, managed memory, or page-locked host memory mapped at the same address (UVA)
int check_accessible(const void* p, const char* what, int field) {
    cudaPointerAttributes at;
    B3D_CUDA_OK(cudaPointerGetAttributes(&at, p));
    const bool ok = at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged ||
                    (at.type == cudaMemoryTypeHost && at.devicePointer == p);
    B3D_REQUIRE(ok, B3D_EINVAL,
                "b3d_gather_fields: %s of field %d is not device-accessible (pageable host memory?): pin it or copy it to "
                "the device",
                what, field);
    return B3D_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Reconstruction training data: crop + cv2-style bilinear resize (double) + mirror of a batch of packed RGBM windows
// (cmr_data/base.py:58-130, run_reconstruction.py:104-133).

constexpr int IMG_NT = 256;
constexpr int IMG_ROWS = 4;   // output rows per CTA

struct ImageArgs {
    const uint32_t* pixels;
    const int64_t* offsets;
    const int32_t* geometry;  // [n, 5]: ww, wh, wx0, wy0, S
    const float* poses;       // [n, 2, 8]
    int n;
    const int32_t* idx;
    const uint8_t* flip;
    int nres;
    int res[B3D_IMAGE_MAX_RES];
    int vec[B3D_IMAGE_MAX_RES];        // 4: float4 stores, 1: scalar
    int block_end[B3D_IMAGE_MAX_RES];  // exclusive prefix of the CTAs of each resolution
    float* images[B3D_IMAGE_MAX_RES];
    float* scale;
    float* translation;
    float* rot;
    int64_t* ind;
};

// cv2 INTER_LINEAR taps of output sample d of an S -> R axis: scale = 1 / (R / S), fx = (d + 0.5) scale - 0.5, clamped to
// the edge.  Every operation rounds on its own (no fused multiply-add), as the numpy restatement does.
__device__ __forceinline__ void linear_tap(int d, int S, double scale, int& s0, double& w1) {
    double fx = __dsub_rn(__dmul_rn((double)d + 0.5, scale), 0.5);
    const double fl = floor(fx);
    fx = __dsub_rn(fx, fl);
    int s = (int)fl;
    if (s < 0) s = 0, fx = 0.0;
    if (s >= S - 1) s = S - 1, fx = 0.0;
    s0 = s;
    w1 = fx;
}

__device__ __forceinline__ double lerp2(double a, double b, double w0, double w1) {
    return __dadd_rn(__dmul_rn(a, w0), __dmul_rn(b, w1));
}

// RGBM word of crop pixel (u, v): the window's word, or the crop background (RGB 255 -> 1.0, mask 0) outside the photo
__device__ __forceinline__ uint32_t crop_word(const uint32_t* win, int ww, int wh, int wx0, int wy0, int u, int v) {
    const unsigned x = (unsigned)(u - wx0), y = (unsigned)(v - wy0);
    return (x < (unsigned)ww && y < (unsigned)wh) ? __ldg(win + (long long)y * ww + x) : 0x00FFFFFFu;
}

struct ImageTile {
    const uint32_t* win;
    int ww, wh, wx0, wy0, S;
    int R, C, y_base, rows;
    bool mirrored;
    float* out;
    long long plane;
};

// The CTA's rows of one sample at one resolution, VEC consecutive output pixels per thread and step.
template <int VEC>
__device__ __forceinline__ void image_rows(const ImageTile& q, const int* col_s0, const double* col_w1, const int* row_s0,
                                           const double* row_w1, const double* lut) {
    const int groups = q.R / VEC;
    for (int t = threadIdx.x; t < q.rows * groups; t += IMG_NT) {
        const int r = t / groups, x_base = (t % groups) * VEC;
        const int v0 = row_s0[r], v1 = min(v0 + 1, q.S - 1);
        const double b1 = row_w1[r], b0 = 1.0 - b1;
        float px[4][VEC];  // [channel][pixel]
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
            const int xr = q.mirrored ? q.R - 1 - (x_base + j) : x_base + j;   // resized column this output column shows
            const int u0 = col_s0[xr], u1 = min(u0 + 1, q.S - 1);
            const double a1 = col_w1[xr], a0 = 1.0 - a1;
            const uint32_t p00 = crop_word(q.win, q.ww, q.wh, q.wx0, q.wy0, u0, v0);
            const uint32_t p01 = crop_word(q.win, q.ww, q.wh, q.wx0, q.wy0, u1, v0);
            const uint32_t p10 = crop_word(q.win, q.ww, q.wh, q.wx0, q.wy0, u0, v1);
            const uint32_t p11 = crop_word(q.win, q.ww, q.wh, q.wx0, q.wy0, u1, v1);
            // mask: the raw annotation value (0 / 1), interpolated like the image
            const double m = lerp2(lerp2((double)(p00 >> 24), (double)(p01 >> 24), a0, a1),
                                   lerp2((double)(p10 >> 24), (double)(p11 >> 24), a0, a1), b0, b1);
            const float mf = __double2float_rn(m);
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const int sh = 8 * c;
                const double v = lerp2(lerp2(lut[(p00 >> sh) & 255u], lut[(p01 >> sh) & 255u], a0, a1),
                                       lerp2(lut[(p10 >> sh) & 255u], lut[(p11 >> sh) & 255u], a0, a1), b0, b1);
                // ImageDataset: float32(img) * 2 - 1, then * float32(mask), each op rounded in fp32
                px[c][j] = __fmul_rn(__fadd_rn(__fmul_rn(__double2float_rn(v), 2.f), -1.f), mf);
            }
            px[3][j] = mf;
        }
        const long long o = (long long)(q.y_base + r) * q.R + x_base;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            if (c == q.C) break;
            float* dst = q.out + c * q.plane + o;
            if constexpr (VEC == 4)
                *reinterpret_cast<float4*>(dst) = make_float4(px[c][0], px[c][1], px[c][2], px[c][3]);
            else
                dst[0] = px[c][0];
        }
    }
}

__global__ void __launch_bounds__(IMG_NT) image_batch_kernel(const __grid_constant__ ImageArgs a) {
    __shared__ int col_s0[B3D_IMAGE_MAX_SIDE];
    __shared__ double col_w1[B3D_IMAGE_MAX_SIDE];
    __shared__ int row_s0[IMG_ROWS];
    __shared__ double row_w1[IMG_ROWS];
    __shared__ double lut[256];  // byte / 255.0, as imread(...) / 255.0

    int k = 0;
    while ((int)blockIdx.x >= a.block_end[k]) ++k;
    const int R = a.res[k];
    const int tiles = (R + IMG_ROWS - 1) / IMG_ROWS;
    const int local = blockIdx.x - (k ? a.block_end[k - 1] : 0);
    const int b = local / tiles, y_base = (local % tiles) * IMG_ROWS;
    const int rows = min(IMG_ROWS, R - y_base);
    const int C = k == 0 ? 4 : 3;
    const long long plane = (long long)R * R;
    float* out = a.images[k] + (long long)b * C * plane;

    const int s = a.idx[b];
    const bool in_range = s >= 0 && s < a.n;
    int ww = 0, wh = 0, wx0 = 0, wy0 = 0, S = 0;
    if (in_range) {
        const int32_t* g = a.geometry + 5LL * s;
        ww = g[0], wh = g[1], wx0 = g[2], wy0 = g[3], S = g[4];
    }
    const bool ok = in_range && S >= 1 && ww >= 0 && wh >= 0;
    const bool mirrored = a.flip && a.flip[b];

    if (k == 0 && y_base == 0 && threadIdx.x < 8) {
        const int f = mirrored ? 1 : 0;
        const float p = ok ? a.poses[(2LL * s + f) * 8 + threadIdx.x] : __int_as_float(0x7fc00000);
        if (threadIdx.x == 0) {
            a.scale[b] = p;
            a.ind[b] = ok ? (int64_t)s + (int64_t)a.n * f : -1;
        } else if (threadIdx.x < 4) {
            a.translation[3LL * b + threadIdx.x - 1] = p;
        } else {
            a.rot[4LL * b + threadIdx.x - 4] = p;
        }
    }
    if (!ok) {
        const float nan = __int_as_float(0x7fc00000);
        for (int c = 0; c < C; ++c)
            for (int t = threadIdx.x; t < rows * R; t += IMG_NT) out[c * plane + (long long)y_base * R + t] = nan;
        return;
    }

    const double scale = __ddiv_rn(1.0, __ddiv_rn((double)R, (double)S));
    for (int d = threadIdx.x; d < R; d += IMG_NT) linear_tap(d, S, scale, col_s0[d], col_w1[d]);
    if (threadIdx.x < rows) linear_tap(y_base + threadIdx.x, S, scale, row_s0[threadIdx.x], row_w1[threadIdx.x]);
    lut[threadIdx.x] = __ddiv_rn((double)threadIdx.x, 255.0);
    __syncthreads();

    const uint32_t* win = a.pixels + a.offsets[s];
    const ImageTile tile{win, ww, wh, wx0, wy0, S, R, C, y_base, rows, mirrored, out, plane};
    if (a.vec[k] == 4)
        image_rows<4>(tile, col_s0, col_w1, row_s0, row_w1, lut);
    else
        image_rows<1>(tile, col_s0, col_w1, row_s0, row_w1, lut);
}

// ---------------------------------------------------------------------------------------------------------------------
// Pseudo-ground-truth records (run_reconstruction.py:571-603): the texel-visibility mask resized to R, the inverse render
// masked with it and moved to NCHW, every plane rounded to fp16 in one launch.

constexpr int PACK_NT = 256;

struct PackArgs {
    const uint8_t* vis;      // [B, Th, Tw] 0 / 1
    int Th, Tw;
    float sy, sx;            // Th / R, Tw / R as F.interpolate(size=R) computes them
    const float* tex;        // [B, R, R, C]
    const float* alpha;      // [B, R, R, 1]
    int R, C;
    const float* image;      // [B, Ci, h, w]
    long long pix_total, image_total;
    int pix_blocks;
    __half* tex_out;         // [B, C, R, R]
    __half* alpha_out;       // [B, 1, R, R]
    __half* image_out;       // [B, Ci, h, w]
};

// upsample_bilinear2d's source taps of output index d (align_corners=False): src = scale (d + 0.5) - 0.5 in fp32 with one
// rounding, clamped at 0; the second tap is the next row / column unless d maps onto the last one, and takes part only
// with a non-zero lambda
__device__ __forceinline__ void mask_taps(int d, int in, float scale, int& i0, int& i1, bool& use1) {
    float src = __fmaf_rn(scale, (float)d + 0.5f, -0.5f);
    if (src < 0.f) src = 0.f;
    i0 = (int)src;
    i1 = i0 + (i0 < in - 1 ? 1 : 0);
    use1 = src - (float)i0 > 0.f;
}

__global__ void __launch_bounds__(PACK_NT) pseudogt_pack_kernel(const __grid_constant__ PackArgs a) {
    if ((int)blockIdx.x < a.pix_blocks) {
        const long long t = (long long)blockIdx.x * PACK_NT + threadIdx.x;
        if (t >= a.pix_total) return;
        const long long plane = (long long)a.R * a.R;
        const long long b = t / plane;
        const int pos = (int)(t - b * plane), y = pos / a.R, x = pos - y * a.R;
        int y0, y1, x0, x1;
        bool uy, ux;
        mask_taps(y, a.Th, a.sy, y0, y1, uy);
        mask_taps(x, a.Tw, a.sx, x0, x1, ux);
        const uint8_t* v = a.vis + b * a.Th * a.Tw;
        const bool seen = v[y0 * a.Tw + x0] || (ux && v[y0 * a.Tw + x1]) ||
                          (uy && (v[y1 * a.Tw + x0] || (ux && v[y1 * a.Tw + x1])));
        const float m = seen ? 1.f : 0.f;
        const float* src = a.tex + t * a.C;
        for (int c = 0; c < a.C; ++c) a.tex_out[(b * a.C + c) * plane + pos] = __float2half_rn(__fmul_rn(src[c], m));
        a.alpha_out[t] = __float2half_rn(__fmul_rn(a.alpha[t], m));
    } else {
        const long long t = (long long)(blockIdx.x - a.pix_blocks) * PACK_NT + threadIdx.x;
        if (t < a.image_total) a.image_out[t] = __float2half_rn(a.image[t]);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Sample export (main.py:874-895): the 2x2 anti-aliased render tiles and the texture images as the bytes written to PNG.

struct SamplePackArgs {
    const float* image;      // [B, H, W, 3]
    const int32_t* imidx;    // [B, H, W] face index + 1, 0 = background
    int H, W;
    const float* tex;        // [B, 3, T, T]
    int T;
    long long tile_total, texel_total;
    int tile_blocks;
    uint8_t* tiles;          // [B, H/2, W/2, 3]
    uint8_t* tex8;           // [B, T, T, 3]
};

// x / 2 + 0.5 as two roundings (halving is exact, so x * 0.5 rounds as x / 2 does)
__device__ __forceinline__ float to_unit(float x) { return __fadd_rn(__fmul_rn(x, 0.5f), 0.5f); }

// (v * 255).clamp(0, 255).byte(): one rounding, then truncation toward zero
__device__ __forceinline__ uint8_t to_byte(float v) {
    v = __fmul_rn(v, 255.f);
    v = v < 0.f ? 0.f : (v > 255.f ? 255.f : v);
    return (uint8_t)__float2uint_rz(v);
}

__global__ void __launch_bounds__(PACK_NT) sample_pack_kernel(const __grid_constant__ SamplePackArgs a) {
    if ((int)blockIdx.x < a.tile_blocks) {
        const long long t = (long long)blockIdx.x * PACK_NT + threadIdx.x;
        if (t >= a.tile_total) return;
        const int Wo = a.W >> 1, Ho = a.H >> 1;
        const long long b = t / ((long long)Ho * Wo);
        const int pos = (int)(t - b * Ho * Wo), yo = pos / Wo, xo = pos - yo * Wo;
        const long long p00 = (b * a.H + 2 * yo) * a.W + 2 * xo;
        const long long p[4] = {p00, p00 + 1, p00 + a.W, p00 + a.W + 1};     // avg_pool2d's window, row by row
        bool bg[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) bg[k] = a.imidx[p[k]] <= 0;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < 4; ++k) s = __fadd_rn(s, to_unit(bg[k] ? 1.f : a.image[p[k] * 3 + c]));
            a.tiles[t * 3 + c] = to_byte(__fmul_rn(s, 0.25f));
        }
    } else {
        const long long t = (long long)(blockIdx.x - a.tile_blocks) * PACK_NT + threadIdx.x;
        if (t >= a.texel_total) return;
        const long long plane = (long long)a.T * a.T;
        const long long b = t / plane, pos = t - b * plane;
#pragma unroll
        for (int c = 0; c < 3; ++c) a.tex8[t * 3 + c] = to_byte(to_unit(a.tex[(b * 3 + c) * plane + pos]));
    }
}

int check_device_ptr(const void* p, const char* what, const char* fn = "b3d_image_batch") {
    cudaPointerAttributes at;
    B3D_CUDA_OK(cudaPointerGetAttributes(&at, p));
    B3D_REQUIRE(at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged, B3D_EINVAL,
                "%s: %s is not device memory", fn, what);
    return B3D_OK;
}

}  // namespace

extern "C" {

int b3d_gather_fields(const b3d_gather_field* fields, int nfields, const int32_t* idx, const uint8_t* flip, int B,
                      void* stream) {
    B3D_REQUIRE(fields && nfields >= 1 && nfields <= B3D_GATHER_MAX_FIELDS && B >= 0, B3D_EINVAL,
                "b3d_gather_fields: bad arguments (nfields %d, B %d)", nfields, B);
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(idx, B3D_EINVAL, "b3d_gather_fields: null idx");
    GatherArgs a = {};
    a.idx = idx;
    a.flip = flip;
    long long blocks = 0;
    for (int i = 0; i < nfields; ++i) {
        const b3d_gather_field& f = fields[i];
        B3D_REQUIRE(f.src && f.dst, B3D_EINVAL, "b3d_gather_fields: null pointer in field %d", i);
        B3D_REQUIRE(f.src_type >= B3D_GATHER_F32 && f.src_type <= B3D_GATHER_I64, B3D_EINVAL,
                    "b3d_gather_fields: field %d has unknown src_type %d", i, f.src_type);
        B3D_REQUIRE(f.n >= 1 && f.C >= 1 && f.C <= f.C_src && f.H >= 1 && f.W >= 1, B3D_EINVAL,
                    "b3d_gather_fields: bad sizes in field %d (n %d, C %d of %d, H %d, W %d)", i, f.n, f.C, f.C_src, f.H, f.W);
        B3D_REQUIRE(!f.mirror || (f.src_type != B3D_GATHER_I64 && f.W % 2 == 0), B3D_EINVAL,
                    "b3d_gather_fields: field %d cannot mirror (int64 rows or odd width %d)", i, f.W);
        a.f[i] = f;
        const uintptr_t al = reinterpret_cast<uintptr_t>(f.src) | reinterpret_cast<uintptr_t>(f.dst);
        int vec = f.src_type == B3D_GATHER_F16 ? 8 : f.src_type == B3D_GATHER_F32 ? 4 : 1;
        if (f.W % (2 * vec) != 0 || (al & 15u) != 0) vec = 1;
        a.vec[i] = vec;
        a.items[i] = (long long)B * f.C * f.H * (f.W / vec);
        blocks += (a.items[i] + NT - 1) / NT;
        B3D_REQUIRE(blocks < (1LL << 31), B3D_EINVAL, "b3d_gather_fields: batch too large");
        a.block_end[i] = (int)blocks;
    }
    for (int i = nfields; i < B3D_GATHER_MAX_FIELDS; ++i) a.block_end[i] = (int)blocks;
    for (int i = 0; i < nfields; ++i) {
        int rc = check_accessible(fields[i].src, "src", i);
        if (rc == B3D_OK) rc = check_accessible(fields[i].dst, "dst", i);
        if (rc != B3D_OK) return rc;
    }
    int rc = check_accessible(idx, "idx", -1);
    if (rc == B3D_OK && flip) rc = check_accessible(flip, "flip", -1);
    if (rc != B3D_OK) return rc;
    gather_fields_kernel<<<(unsigned)blocks, NT, 0, (cudaStream_t)stream>>>(a);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

int b3d_image_batch(const uint32_t* pixels, const int64_t* offsets, const int32_t* geometry, const float* poses, int n,
                    const int32_t* idx, const uint8_t* flip, int B, int nres, const int32_t* res, float* const* images,
                    float* scale, float* translation, float* rot, int64_t* ind, void* stream) {
    static_assert(IMG_NT == 256, "the byte / 255 table is filled one entry per thread");
    B3D_REQUIRE(n >= 1 && B >= 0 && nres >= 1 && nres <= B3D_IMAGE_MAX_RES && res && images, B3D_EINVAL,
                "b3d_image_batch: bad arguments (n %d, B %d, nres %d)", n, B, nres);
    B3D_REQUIRE(pixels && offsets && geometry && poses, B3D_EINVAL, "b3d_image_batch: null store pointer");
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(idx && scale && translation && rot && ind, B3D_EINVAL, "b3d_image_batch: null idx or pose output");
    ImageArgs a = {};
    a.pixels = pixels, a.offsets = offsets, a.geometry = geometry, a.poses = poses, a.n = n;
    a.idx = idx, a.flip = flip, a.nres = nres;
    a.scale = scale, a.translation = translation, a.rot = rot, a.ind = ind;
    long long blocks = 0;
    for (int k = 0; k < nres; ++k) {
        B3D_REQUIRE(images[k], B3D_EINVAL, "b3d_image_batch: null image output %d", k);
        B3D_REQUIRE(res[k] >= 1 && res[k] <= B3D_IMAGE_MAX_SIDE, B3D_EINVAL,
                    "b3d_image_batch: resolution %d of output %d outside [1, %d]", res[k], k, B3D_IMAGE_MAX_SIDE);
        a.res[k] = res[k];
        a.images[k] = images[k];
        a.vec[k] = (res[k] % 4 == 0 && (reinterpret_cast<uintptr_t>(images[k]) & 15u) == 0) ? 4 : 1;
        blocks += (long long)B * ((res[k] + IMG_ROWS - 1) / IMG_ROWS);
        B3D_REQUIRE(blocks < (1LL << 31), B3D_EINVAL, "b3d_image_batch: batch too large");
        a.block_end[k] = (int)blocks;
    }
    for (int k = nres; k < B3D_IMAGE_MAX_RES; ++k) a.block_end[k] = (int)blocks;
    const void* dev[] = {pixels, offsets, geometry, poses, idx, scale, translation, rot, ind};
    const char* names[] = {"pixels", "offsets", "geometry", "poses", "idx", "scale", "translation", "rot", "ind"};
    for (int i = 0; i < 9; ++i) {
        const int rc = check_device_ptr(dev[i], names[i]);
        if (rc != B3D_OK) return rc;
    }
    if (flip) {
        const int rc = check_device_ptr(flip, "flip");
        if (rc != B3D_OK) return rc;
    }
    for (int k = 0; k < nres; ++k) {
        const int rc = check_device_ptr(images[k], "an image output");
        if (rc != B3D_OK) return rc;
    }
    image_batch_kernel<<<(unsigned)blocks, IMG_NT, 0, (cudaStream_t)stream>>>(a);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

int b3d_pseudogt_pack(const uint8_t* vis, int Th, int Tw, const float* tex, const float* alpha, int B, int R, int C,
                      const float* image, int Ci, int h, int w, uint16_t* tex_out, uint16_t* alpha_out,
                      uint16_t* image_out, void* stream) {
    B3D_REQUIRE(B >= 0 && Th >= 1 && Tw >= 1 && R >= 1 && C >= 1 && Ci >= 1 && h >= 1 && w >= 1, B3D_EINVAL,
                "b3d_pseudogt_pack: bad sizes (B %d, texture %d x %d, R %d, C %d, image %d x %d x %d)", B, Th, Tw, R, C,
                Ci, h, w);
    if (B == 0) return B3D_OK;
    PackArgs a = {};
    a.vis = vis, a.Th = Th, a.Tw = Tw;
    a.sy = (float)Th / (float)R, a.sx = (float)Tw / (float)R;
    a.tex = tex, a.alpha = alpha, a.R = R, a.C = C, a.image = image;
    a.pix_total = (long long)B * R * R;
    a.image_total = (long long)B * Ci * h * w;
    a.tex_out = reinterpret_cast<__half*>(tex_out);
    a.alpha_out = reinterpret_cast<__half*>(alpha_out);
    a.image_out = reinterpret_cast<__half*>(image_out);
    const long long pix_blocks = (a.pix_total + PACK_NT - 1) / PACK_NT;
    const long long blocks = pix_blocks + (a.image_total + PACK_NT - 1) / PACK_NT;
    B3D_REQUIRE(blocks < (1LL << 31), B3D_EINVAL, "b3d_pseudogt_pack: batch too large");
    a.pix_blocks = (int)pix_blocks;
    const void* ptrs[] = {vis, tex, alpha, image, tex_out, alpha_out, image_out};
    const char* names[] = {"vis", "tex", "alpha", "image", "tex_out", "alpha_out", "image_out"};
    for (int i = 0; i < 7; ++i) {
        B3D_REQUIRE(ptrs[i], B3D_EINVAL, "b3d_pseudogt_pack: null %s", names[i]);
        const int rc = check_device_ptr(ptrs[i], names[i], "b3d_pseudogt_pack");
        if (rc != B3D_OK) return rc;
    }
    pseudogt_pack_kernel<<<(unsigned)blocks, PACK_NT, 0, (cudaStream_t)stream>>>(a);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

int b3d_sample_pack(const float* image, const int32_t* imidx, int B, int H, int W, const float* tex, int T,
                    uint8_t* tiles, uint8_t* tex8, void* stream) {
    B3D_REQUIRE(B >= 0 && H >= 2 && W >= 2 && T >= 1, B3D_EINVAL,
                "b3d_sample_pack: bad sizes (B %d, render %d x %d, texture %d)", B, H, W, T);
    B3D_REQUIRE(H % 2 == 0 && W % 2 == 0, B3D_EINVAL,
                "b3d_sample_pack: the render is %d x %d; the 2 x 2 pool needs an even height and width", H, W);
    if (B == 0) return B3D_OK;
    SamplePackArgs a = {};
    a.image = image, a.imidx = imidx, a.H = H, a.W = W, a.tex = tex, a.T = T, a.tiles = tiles, a.tex8 = tex8;
    a.tile_total = (long long)B * (H / 2) * (W / 2);
    a.texel_total = (long long)B * T * T;
    const long long tile_blocks = (a.tile_total + PACK_NT - 1) / PACK_NT;
    const long long blocks = tile_blocks + (a.texel_total + PACK_NT - 1) / PACK_NT;
    B3D_REQUIRE(blocks < (1LL << 31), B3D_EINVAL, "b3d_sample_pack: batch too large");
    a.tile_blocks = (int)tile_blocks;
    const void* ptrs[] = {image, imidx, tex, tiles, tex8};
    const char* names[] = {"image", "imidx", "tex", "tiles", "tex8"};
    for (int i = 0; i < 5; ++i) {
        B3D_REQUIRE(ptrs[i], B3D_EINVAL, "b3d_sample_pack: null %s", names[i]);
        const int rc = check_device_ptr(ptrs[i], names[i], "b3d_sample_pack");
        if (rc != B3D_OK) return rc;
    }
    sample_pack_kernel<<<(unsigned)blocks, PACK_NT, 0, (cudaStream_t)stream>>>(a);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

}  // extern "C"
