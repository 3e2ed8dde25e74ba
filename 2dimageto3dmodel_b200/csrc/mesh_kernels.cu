// Textured-mesh render path (SURVEY.md §8 rows a7-a9, a12) for sm_90a: kaolin-free DIB-R.
//
//   mesh_face_setup_kernel   ortho_projection (renderer.py:9-28): gathers by `faces`/`ft`, scales the 2-D
//                            vertices by the rasteriser's multiplier, face normal (FMA pattern of torch.cross),
//                            unit normal (datanormalize, renderer.py:52).
//   mesh_raster_fwd_kernel   kaolin `linear_rasterizer` (renderer.py:60-67; restated from SURVEY App. B) +
//                            fragment shader (fragment_shader.py:6-37) in ONE pass.  kaolin tests every pixel
//                            against every face (H*W*F); here a CTA owns a 16x16 pixel tile, bins the faces
//                            whose expanded bounding box touches the tile with an order-preserving ballot
//                            compaction (face order decides z ties and the knum cap), stages the binned face
//                            records through shared memory and walks only those: ~20 tests per pixel, not 960.
//   mesh_raster_bwd_kernel   adjoint: gradients to the 2-D vertices (barycentrics of the covering face +
//                            soft-silhouette distances), to the per-face UVs / attributes and to the texture.
//                            Per-face gradients are accumulated in shared memory per tile and flushed once; the
//                            knum x 5 per-pixel side buffers kaolin stores are recomputed instead.
//   mesh_face_pack_kernel    the same per-face record from kaolin's own inputs (points3d depths, points2d x
//                            multiplier, normalz) for the stand-alone `linear_rasterizer`.
//
// One rasteriser, five outputs (the MODE template parameter): OUT_UV (interpolated (u, v, hard mask), what
// Renderer's rasteriser call returns), OUT_ATTR (any number d of per-vertex attributes, kaolin's imfeat) and the
// shaded image with grid_sample's bilinear (align_corners=True), nearest or bicubic (align_corners=False) filters.
// The raster parameters (multiplier, expand, delta, knum) are run-time values; the Renderer entry points pass kaolin's
// defaults.
//
// Index buffer (imidx) arithmetic uses round-to-nearest intrinsics in the oracle's operation order so that
// the face-index / visibility buffers are reproduced bit for bit.
#include "b3d_common.cuh"

namespace {

constexpr int TILE = 16;
constexpr int NT = TILE * TILE;
constexpr int CHUNK = 64;          // face records staged per step
constexpr int CAPN = 768;          // per-tile shared-memory accumulators (faces beyond use global atomics)
constexpr float DEPTH_INIT = -1000.f;
constexpr float BARY_EPS = 1e-10f;
constexpr float SEG_EPS = 1e-10f;
constexpr float NORMAL_EPS = 1e-8f;

// kaolin linear_rasterizer's keyword arguments, as the kernels use them
struct RasterParams {
    float mult;      // `multiplier`: 2-D coordinates are scaled by it before every test
    float expand;    // `expand` x multiplier: bounding-box margin of the soft-silhouette faces
    float delta;     // `delta`: sharpness of the soft silhouette
    float mm;        // multiplier^2
    float inv_mm;    // RN(1 / multiplier^2)
    float slope;     // RN(-delta / multiplier^2)
    int knum;        // at most this many faces (in face order) shape an uncovered pixel's soft silhouette
    float sx, sy;    // pixel pitches RN(multiplier / W), RN(multiplier / H)
};
// The kernels take the parameters as scalars (a by-value struct parameter costs the existing instantiations registers
// and spills) and rebuild the struct in registers.
#define RASTER_PARAMS float rp_mult, float rp_expand, float rp_delta, float rp_mm, float rp_inv_mm, float rp_slope, \
                      int rp_knum, float rp_sx, float rp_sy
#define RASTER_PARAMS_LOCAL const RasterParams rp{rp_mult, rp_expand, rp_delta, rp_mm, rp_inv_mm, rp_slope, rp_knum, rp_sx, rp_sy}
#define RASTER_PARAMS_ARGS(p) p.mult, p.expand, p.delta, p.mm, p.inv_mm, p.slope, p.knum, p.sx, p.sy
// kaolin's defaults (renderer.py:60-67 passes none): expand 0.02, knum 30, multiplier 1000, delta 7000
constexpr float DEFAULT_MULT = 1000.f;
RasterParams make_params(float mult, float expand_scaled, float delta, int knum) {
    const float mm = mult * mult;
    return RasterParams{mult, expand_scaled, delta, mm, 1.f / mm, -delta / mm, knum, 0.f, 0.f};
}
RasterParams default_params() { return make_params(DEFAULT_MULT, 0.02f * DEFAULT_MULT, 7000.f, 30); }

// x / multiplier^2, correctly rounded (Markstein: q = RN(x * RN(1/m)), one fma residual step) for the x = -delta * d2 of
// the soft silhouette: the same value as the division, without the division's slow-path call inside the face loops
__device__ __forceinline__ float div_mm(float x, const RasterParams& rp) {
    const float q = __fmul_rn(x, rp.inv_mm);
    return __fmaf_rn(__fmaf_rn(-q, rp.mm, x), rp.inv_mm, q);
}

// what the rasteriser writes to imout
enum : int {
    OUT_UV = 0,          // (u, v, hard mask) from fuv [B,F,6]
    OUT_ATTR = 1,        // d interpolated attributes from attr [B,F,3d]
    OUT_BILINEAR = 2,    // shaded, grid_sample bilinear, align_corners=True (fragment_shader.py's own helper)
    OUT_NEAREST = 3,     // shaded, grid_sample nearest, align_corners=False, zero padding
    OUT_BICUBIC = 4,     // shaded, grid_sample bicubic, align_corners=False, zero padding
};

__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float min3(float a, float b, float c) { return fminf(fminf(a, b), c); }
__device__ __forceinline__ float max3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }

// per-face record: 3 x float4 = (ax,ay,bx,by) (cx,cy,az,bz) (cz,nz,-,-); 2-D coords already x MULT
struct Face {
    float ax, ay, bx, by, cx, cy, az, bz, cz, nz;
};
__device__ __forceinline__ Face unpack(const float4 a, const float4 b, const float4 c) {
    return Face{a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, c.x, c.y};
}

__global__ void __launch_bounds__(NT)
mesh_face_setup_kernel(const float* __restrict__ verts, const int32_t* __restrict__ faces,
                       const float* __restrict__ uv, long long uv_bstride, const int32_t* __restrict__ ft, int P,
                       int F, float4* __restrict__ fgeo, float* __restrict__ fuv, float* __restrict__ normal1) {
    const int b = blockIdx.y;
    const int f = blockIdx.x * NT + threadIdx.x;
    if (f >= F) return;
    float v[3][3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const float* p = verts + ((size_t)b * P + faces[3 * f + i]) * 3;
        v[i][0] = p[0];
        v[i][1] = p[1];
        v[i][2] = p[2];
    }
    const float e1x = sub(v[1][0], v[0][0]), e1y = sub(v[1][1], v[0][1]), e1z = sub(v[1][2], v[0][2]);
    const float e2x = sub(v[2][0], v[0][0]), e2y = sub(v[2][1], v[0][1]), e2z = sub(v[2][2], v[0][2]);
    // torch.cross on CPU evaluates a_i*b_j - a_j*b_i as fma(a_i, b_j, -(a_j*b_i))
    const float nx = __fmaf_rn(e1y, e2z, -mul(e1z, e2y));
    const float ny = __fmaf_rn(e1z, e2x, -mul(e1x, e2z));
    const float nz = __fmaf_rn(e1x, e2y, -mul(e1y, e2x));
    float4* g = fgeo + ((size_t)b * F + f) * 3;
    constexpr float MULT = DEFAULT_MULT;
    g[0] = make_float4(mul(MULT, v[0][0]), mul(MULT, v[0][1]), mul(MULT, v[1][0]), mul(MULT, v[1][1]));
    g[1] = make_float4(mul(MULT, v[2][0]), mul(MULT, v[2][1]), v[0][2], v[1][2]);
    g[2] = make_float4(v[2][2], nz, 0.f, 0.f);
    if (normal1) {
        const float inv = 1.f / (sqrtf(nx * nx + ny * ny + nz * nz) + NORMAL_EPS);
        float* o = normal1 + ((size_t)b * F + f) * 3;
        o[0] = nx * inv;
        o[1] = ny * inv;
        o[2] = nz * inv;
    }
    if (fuv) {
        float* o = fuv + ((size_t)b * F + f) * 6;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const float* p = uv + (size_t)b * uv_bstride + (size_t)ft[3 * f + i] * 2;
            o[2 * i] = p[0];
            o[2 * i + 1] = p[1];
        }
    }
}

// kaolin's inputs as given: points3d [B,F,9] (only the depths are read), points2d [B,F,6], normalz [B,F,1]
__global__ void __launch_bounds__(NT)
mesh_face_pack_kernel(const float* __restrict__ p3d, const float* __restrict__ p2d, const float* __restrict__ normalz,
                      float mult, int F, float4* __restrict__ fgeo) {
    const int b = blockIdx.y;
    const int f = blockIdx.x * NT + threadIdx.x;
    if (f >= F) return;
    const size_t bf = (size_t)b * F + f;
    const float* q = p2d + bf * 6;
    const float* z = p3d + bf * 9;
    float4* g = fgeo + bf * 3;
    g[0] = make_float4(mul(mult, q[0]), mul(mult, q[1]), mul(mult, q[2]), mul(mult, q[3]));
    g[1] = make_float4(mul(mult, q[4]), mul(mult, q[5]), z[2], z[5]);
    g[2] = make_float4(z[8], normalz[bf], 0.f, 0.f);
}

// pixel centres, SURVEY App. B step 2 (row 0 is the top of the image)
// sx = RN(m / W), sy = RN(m / H): the pixel pitches, divided on the host
__device__ __forceinline__ float centre_x(int x, int W, float sx) { return mul(sx, (float)(2 * x + 1 - W)); }
__device__ __forceinline__ float centre_y(int y, int H, float sy) { return mul(sy, (float)(H - 2 * y - 1)); }

struct Bary {
    float w0, w1, w2, k3;
};
__device__ __forceinline__ Bary barycentric(const Face& f, float x0, float y0) {
    const float m = sub(f.bx, f.ax), p = sub(f.by, f.ay);
    const float n = sub(f.cx, f.ax), q = sub(f.cy, f.ay);
    const float s = sub(x0, f.ax), t = sub(y0, f.ay);
    const float k3 = sub(mul(m, q), mul(n, p));
    const float den = add(k3, BARY_EPS);
    const float w1 = __fdiv_rn(sub(mul(s, q), mul(n, t)), den);
    const float w2 = __fdiv_rn(sub(mul(m, t), mul(s, p)), den);
    return Bary{sub(sub(1.f, w1), w2), w1, w2, den};
}

// squared distance to segment a-b and the clamped foot parameter
__device__ __forceinline__ float seg_dist2(float px, float py, float ax, float ay, float bx, float by, float& t,
                                           float& rx, float& ry) {
    const float ex = bx - ax, ey = by - ay, dx = px - ax, dy = py - ay;
    t = (dx * ex + dy * ey) / (ex * ex + ey * ey + SEG_EPS);
    t = fminf(fmaxf(t, 0.f), 1.f);
    rx = dx - t * ex;
    ry = dy - t * ey;
    return rx * rx + ry * ry;
}

struct TileCtx {
    int nlist;
};

// Order-preserving compaction of the faces whose expanded bounding box touches the tile.
// list[] receives face ids in increasing order; posof (optional) maps face -> list position.
__device__ __forceinline__ int bin_faces(const float4* __restrict__ fg, int F, float x0lo, float x0hi, float y0lo,
                                         float y0hi, float EXPAND, int* list, int* posof, int* warp_cnt) {
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    int count = 0;
    for (int base = 0; base < F; base += NT) {
        const int f = base + tid;
        bool flag = false;
        if (f < F) {
            const float4 a = __ldg(fg + (size_t)f * 3), b = __ldg(fg + (size_t)f * 3 + 1);
            const float xmin = min3(a.x, a.z, b.x), xmax = max3(a.x, a.z, b.x);
            const float ymin = min3(a.y, a.w, b.y), ymax = max3(a.y, a.w, b.y);
            flag = (sub(xmin, EXPAND) <= x0hi) && (x0lo < add(xmax, EXPAND)) && (sub(ymin, EXPAND) <= y0hi) &&
                   (y0lo < add(ymax, EXPAND));
            if (posof) posof[f] = -1;
        }
        const unsigned bal = __ballot_sync(0xffffffffu, flag);
        if (lane == 0) warp_cnt[w] = __popc(bal);
        __syncthreads();
        int off = 0, tot = 0;
#pragma unroll
        for (int i = 0; i < NT / 32; ++i) {
            const int c = warp_cnt[i];
            off += (i < w) ? c : 0;
            tot += c;
        }
        if (flag) {
            const int pos = count + off + __popc(bal & ((1u << lane) - 1u));
            list[pos] = f;
            if (posof) posof[f] = pos;
        }
        count += tot;
        __syncthreads();
    }
    return count;
}

__device__ __forceinline__ void stage_faces(const float4* __restrict__ fg, const int* list, int c0, int n,
                                            float4* stage) {
    for (int i = threadIdx.x; i < n * 3; i += NT) stage[i] = __ldg(fg + (size_t)list[c0 + i / 3] * 3 + (i % 3));
}

// bilinear texture fetch, grid_sample(align_corners=True, zeros padding) with uv -> (u*2-1, -(v*2-1))
struct TexTap {
    int x0, y0;
    float wx1, wy1;
};
__device__ __forceinline__ TexTap tex_tap(float u, float v, int Th, int Tw) {
    const float ix = u * (float)(Tw - 1), iy = (1.f - v) * (float)(Th - 1);
    const float fx = floorf(ix), fy = floorf(iy);
    return TexTap{(int)fx, (int)fy, ix - fx, iy - fy};
}
__device__ __forceinline__ float tex_at(const float* __restrict__ t, int y, int x, int Th, int Tw) {
    return (x >= 0 && x < Tw && y >= 0 && y < Th) ? __ldg(t + (size_t)y * Tw + x) : 0.f;
}

// interpolated (u, v) of a covered pixel and the interpolated constant-1 attribute (= hard mask) from the barycentrics
// w0..w2 and the covering face's corner uvs a[6]; shared by the shader, its adjoint and the texel-visibility kernel so
// that all three sample the texture at the same point
struct ShadePoint {
    float u, v, msum;
};
__device__ __forceinline__ ShadePoint shade_point(float w0, float w1, float w2, const float* a) {
    return ShadePoint{w0 * a[0] + w1 * a[2] + w2 * a[4], w0 * a[1] + w1 * a[3] + w2 * a[5], w0 + w1 + w2};
}

// the texture adjoint's contribution g * wx * wy to the four taps (x0,y0), (x0+1,y0), (x0,y0+1), (x0+1,y0+1)
struct TapWeights {
    float w00, w01, w10, w11;
};
__device__ __forceinline__ TapWeights tap_weights(float g, const TexTap& tp) {
    const float wx0 = 1.f - tp.wx1, wy0 = 1.f - tp.wy1;
    return TapWeights{g * wx0 * wy0, g * tp.wx1 * wy0, g * wx0 * tp.wy1, g * tp.wx1 * tp.wy1};
}

// grid_sample with align_corners=False: the unnormalised coordinate ((g + 1) * size - 1) / 2, evaluated as torch's CPU
// kernel does, (g + 1) * (size / 2) - 0.5, on g = u * 2 - 1 (x) or -(v * 2 - 1) (y, the shader's flip)
__device__ __forceinline__ float unnorm_x(float u, int Tw) {
    return __fsub_rn(__fmul_rn(__fadd_rn(__fsub_rn(__fmul_rn(u, 2.f), 1.f), 1.f), 0.5f * (float)Tw), 0.5f);
}
__device__ __forceinline__ float unnorm_y(float v, int Th) {
    return __fsub_rn(__fmul_rn(__fadd_rn(-__fsub_rn(__fmul_rn(v, 2.f), 1.f), 1.f), 0.5f * (float)Th), 0.5f);
}

// grid_sample's cubic convolution weights (A = -0.75) of the taps floor(x) - 1 .. floor(x) + 2 at fraction t, and their
// derivatives d/dt
constexpr float CUBIC_A = -0.75f;
__device__ __forceinline__ float cubic1(float x) { return ((CUBIC_A + 2.f) * x - (CUBIC_A + 3.f)) * x * x + 1.f; }
__device__ __forceinline__ float cubic2(float x) {
    return ((CUBIC_A * x - 5.f * CUBIC_A) * x + 8.f * CUBIC_A) * x - 4.f * CUBIC_A;
}
__device__ __forceinline__ float dcubic1(float x) { return (3.f * (CUBIC_A + 2.f) * x - 2.f * (CUBIC_A + 3.f)) * x; }
__device__ __forceinline__ float dcubic2(float x) { return (3.f * CUBIC_A * x - 10.f * CUBIC_A) * x + 8.f * CUBIC_A; }
__device__ __forceinline__ void cubic_weights(float t, float (&c)[4]) {
    c[0] = cubic2(t + 1.f);
    c[1] = cubic1(t);
    c[2] = cubic1(1.f - t);
    c[3] = cubic2(2.f - t);
}
__device__ __forceinline__ void cubic_dweights(float t, float (&c)[4]) {
    c[0] = dcubic2(t + 1.f);
    c[1] = dcubic1(t);
    c[2] = -dcubic1(1.f - t);
    c[3] = -dcubic2(2.f - t);
}

template <int MODE>
__global__ void __launch_bounds__(NT)
mesh_raster_fwd_kernel(const float4* __restrict__ fgeo, const float* __restrict__ fuv, int d, const float* __restrict__ tex,
                       const float* __restrict__ bg, RASTER_PARAMS, int F, int H, int W, int Th, int Tw,
                       int32_t* __restrict__ imidx, float* __restrict__ imwei, float* __restrict__ imout,
                       float* __restrict__ improb) {
    constexpr bool SHADE = MODE >= OUT_BILINEAR;
    RASTER_PARAMS_LOCAL;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float4* stage = reinterpret_cast<float4*>(smem_raw);
    int* list = reinterpret_cast<int*>(stage + CHUNK * 3);
    __shared__ int warp_cnt[NT / 32];

    const float MULT = rp.mult, EXPAND = rp.expand, DELTA = rp.delta;
    const int b = blockIdx.z, tid = threadIdx.x;
    const int tx0 = blockIdx.x * TILE, ty0 = blockIdx.y * TILE;
    const int px = tx0 + (tid & (TILE - 1)), py = ty0 + (tid >> 4);
    const bool valid = px < W && py < H;
    const float x0 = centre_x(px, W, rp.sx), y0 = centre_y(py, H, rp.sy);
    const float4* fg = fgeo + (size_t)b * F * 3;

    const int nlist = bin_faces(fg, F, centre_x(tx0, W, rp.sx), centre_x(min(tx0 + TILE - 1, W - 1), W, rp.sx),
                                centre_y(min(ty0 + TILE - 1, H - 1), H, rp.sy), centre_y(ty0, H, rp.sy), EXPAND, list,
                                nullptr, warp_cnt);

    // pass A: nearest front-facing face containing the pixel centre
    int best = -1;
    float bz = DEPTH_INIT, bw0 = 0.f, bw1 = 0.f, bw2 = 0.f;
    for (int c0 = 0; c0 < nlist; c0 += CHUNK) {
        const int n = min(CHUNK, nlist - c0);
        stage_faces(fg, list, c0, n, stage);
        __syncthreads();
        if (valid) {
            for (int j = 0; j < n; ++j) {
                const Face f = unpack(stage[3 * j], stage[3 * j + 1], stage[3 * j + 2]);
                if (f.nz < 0.f) continue;
                const float xmin = min3(f.ax, f.bx, f.cx), xmax = max3(f.ax, f.bx, f.cx);
                const float ymin = min3(f.ay, f.by, f.cy), ymax = max3(f.ay, f.by, f.cy);
                if (x0 < xmin || x0 >= xmax || y0 < ymin || y0 >= ymax) continue;
                const Bary w = barycentric(f, x0, y0);
                if (!(w.w0 >= 0.f && w.w1 >= 0.f && w.w2 >= 0.f)) continue;
                const float z = add(add(mul(w.w0, f.az), mul(w.w1, f.bz)), mul(w.w2, f.cz));
                if (z > bz) {
                    bz = z;
                    best = list[c0 + j];
                    bw0 = w.w0;
                    bw1 = w.w1;
                    bw2 = w.w2;
                }
            }
        }
        __syncthreads();
    }

    // pass B: soft silhouette of the uncovered pixels (first knum faces, in face order, whose expanded
    // bounding box contains the pixel)
    float keep = 1.f;
    if (__syncthreads_or(valid && best < 0)) {
        int cnt = 0;
        for (int c0 = 0; c0 < nlist; c0 += CHUNK) {
            const int n = min(CHUNK, nlist - c0);
            stage_faces(fg, list, c0, n, stage);
            __syncthreads();
            if (valid && best < 0) {
                for (int j = 0; j < n && cnt < rp.knum; ++j) {
                    const Face f = unpack(stage[3 * j], stage[3 * j + 1], stage[3 * j + 2]);
                    const float xmin = min3(f.ax, f.bx, f.cx), xmax = max3(f.ax, f.bx, f.cx);
                    const float ymin = min3(f.ay, f.by, f.cy), ymax = max3(f.ay, f.by, f.cy);
                    if (x0 < sub(xmin, EXPAND) || x0 >= add(xmax, EXPAND) || y0 < sub(ymin, EXPAND) ||
                        y0 >= add(ymax, EXPAND))
                        continue;
                    float t, rx, ry;
                    const float d2 = fminf(fminf(seg_dist2(x0, y0, f.ax, f.ay, f.bx, f.by, t, rx, ry),
                                                 seg_dist2(x0, y0, f.bx, f.by, f.cx, f.cy, t, rx, ry)),
                                           seg_dist2(x0, y0, f.cx, f.cy, f.ax, f.ay, t, rx, ry));
                    keep *= 1.f - expf(div_mm(-DELTA * d2, rp));
                    ++cnt;
                }
            }
            __syncthreads();
        }
    }
    if (!valid) return;

    const size_t pix = ((size_t)b * H + py) * W + px;
    imidx[pix] = best + 1;
    imwei[3 * pix + 0] = bw0;
    imwei[3 * pix + 1] = bw1;
    imwei[3 * pix + 2] = bw2;
    improb[pix] = best >= 0 ? 1.f : 1.f - keep;
    if constexpr (MODE == OUT_ATTR) {
        // imfeat = sum_i w_i attr_i[0..d) on covered pixels, 0 on the background
        float* o = imout + pix * d;
        const float* a = fuv + ((size_t)b * F + max(best, 0)) * 3 * d;
        for (int k = 0; k < d; ++k) o[k] = best >= 0 ? bw0 * a[k] + bw1 * a[d + k] + bw2 * a[2 * d + k] : 0.f;
        return;
    }
    float o0 = 0.f, o1 = 0.f, o2 = 0.f;
    if (best >= 0) {
        const ShadePoint sp = shade_point(bw0, bw1, bw2, fuv + ((size_t)b * F + best) * 6);
        const float u = sp.u, v = sp.v, msum = sp.msum;
        if constexpr (SHADE) {
            float col[3];
            if constexpr (MODE == OUT_BILINEAR) {
                const TexTap tp = tex_tap(u, v, Th, Tw);
                const float wx0 = 1.f - tp.wx1, wy0 = 1.f - tp.wy1;
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const float* t = tex + ((size_t)b * 3 + c) * Th * Tw;
                    col[c] = (tex_at(t, tp.y0, tp.x0, Th, Tw) * wx0 + tex_at(t, tp.y0, tp.x0 + 1, Th, Tw) * tp.wx1) * wy0 +
                             (tex_at(t, tp.y0 + 1, tp.x0, Th, Tw) * wx0 + tex_at(t, tp.y0 + 1, tp.x0 + 1, Th, Tw) * tp.wx1) *
                                 tp.wy1;
                }
            } else if constexpr (MODE == OUT_NEAREST) {
                const int xi = __float2int_rn(unnorm_x(u, Tw)), yi = __float2int_rn(unnorm_y(v, Th));  // half to even
#pragma unroll
                for (int c = 0; c < 3; ++c) col[c] = tex_at(tex + ((size_t)b * 3 + c) * Th * Tw, yi, xi, Th, Tw);
            } else {
                const float ix = unnorm_x(u, Tw), iy = unnorm_y(v, Th);
                const float fx = floorf(ix), fy = floorf(iy);
                const int xs = (int)fx - 1, ys = (int)fy - 1;
                float cx[4], cy[4];
                cubic_weights(ix - fx, cx);
                cubic_weights(iy - fy, cy);
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const float* t = tex + ((size_t)b * 3 + c) * Th * Tw;
                    float acc = 0.f;
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        float row = 0.f;
#pragma unroll
                        for (int j = 0; j < 4; ++j) row += cx[j] * tex_at(t, ys + i, xs + j, Th, Tw);
                        acc += cy[i] * row;
                    }
                    col[c] = acc;
                }
            }
            if (bg) {
                const float* g = bg + 3 * pix;
                o0 = g[0] + msum * (col[0] - g[0]);
                o1 = g[1] + msum * (col[1] - g[1]);
                o2 = g[2] + msum * (col[2] - g[2]);
            } else {
                o0 = col[0] * msum;
                o1 = col[1] * msum;
                o2 = col[2] * msum;
            }
        } else {
            o0 = u;
            o1 = v;
            o2 = msum;
        }
    } else if (SHADE && bg) {
        o0 = bg[3 * pix];
        o1 = bg[3 * pix + 1];
        o2 = bg[3 * pix + 2];
    }
    imout[3 * pix + 0] = o0;
    imout[3 * pix + 1] = o1;
    imout[3 * pix + 2] = o2;
}

// Per-face adjoints live in shared memory as NSLOT floats per binned face: slots 0-5 the 2-D vertices, the rest the
// per-vertex uvs (6) or attributes (3d).  Faces past the first `capn` of the tile's list go to global atomics.
__device__ __forceinline__ void acc_add(float* acc, int pos, int k, float v, float* gdst, int nslot, int capn) {
    if (v == 0.f) return;
    if (pos < capn)
        atomicAdd(acc + pos * nslot + k, v);
    else
        atomicAdd(gdst, v);
}

// Warp-level pre-reduction of per-face adjoints (VERDICT r1 "weak" #4: the backward was bound by same-address shared-memory
// fp32 atomics, which compile to CAS loops): the lanes of a warp (2 pixel rows of the tile) that hit the SAME face sum
// their NV values with shuffles and one lane per face does the accumulate.  All 32 lanes call; fidx < 0 = nothing to add.
template <int NV>
__device__ __forceinline__ void warp_face_acc(float* acc, int fidx, int pos, const float (&vals)[NV], int k0, float* gdst6a,
                                              float* gdst6b) {
    const int lane = threadIdx.x & 31;
    unsigned todo = __ballot_sync(0xffffffffu, fidx >= 0);
    while (todo) {
        const int leader = __ffs(todo) - 1;
        const int key = __shfl_sync(0xffffffffu, fidx, leader);
        const bool mine = fidx == key;
        todo &= ~__ballot_sync(0xffffffffu, mine);
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const float v = b3d::warp_sum(mine ? vals[k] : 0.f);
            if (lane == leader) {
                const int kk = k0 + k;
                acc_add(acc, pos, kk, v, kk < 6 ? gdst6a + key * 6 + kk : gdst6b + key * 6 + (kk - 6), 12, CAPN);
            }
        }
    }
}

// The same for the attribute adjoint w_i * g[k] (i < 3, k < d) of OUT_ATTR: slot 6 + i*d + k, global dattr [F,3d].
__device__ __forceinline__ void warp_face_acc_attr(float* acc, int fidx, int pos, const float* g, float w0, float w1,
                                                   float w2, int d, float* gattr, int capn) {
    const int lane = threadIdx.x & 31, nslot = 6 + 3 * d;
    unsigned todo = __ballot_sync(0xffffffffu, fidx >= 0);
    while (todo) {
        const int leader = __ffs(todo) - 1;
        const int key = __shfl_sync(0xffffffffu, fidx, leader);
        const bool mine = fidx == key;
        todo &= ~__ballot_sync(0xffffffffu, mine);
        for (int k = 0; k < d; ++k) {
            const float gk = mine ? g[k] : 0.f;
            const float v0 = b3d::warp_sum(w0 * gk), v1 = b3d::warp_sum(w1 * gk), v2 = b3d::warp_sum(w2 * gk);
            if (lane == leader) {
                float* ga = gattr + (size_t)key * 3 * d + k;
                acc_add(acc, pos, 6 + k, v0, ga, nslot, capn);
                acc_add(acc, pos, 6 + d + k, v1, ga + d, nslot, capn);
                acc_add(acc, pos, 6 + 2 * d + k, v2, ga + 2 * d, nslot, capn);
            }
        }
    }
}

template <int MODE>
__global__ void __launch_bounds__(NT)
mesh_raster_bwd_kernel(const float4* __restrict__ fgeo, const float* __restrict__ fuv, int d, const float* __restrict__ tex,
                       int has_bg, RASTER_PARAMS, int F, int H, int W, int Th, int Tw,
                       const int32_t* __restrict__ imidx, const float* __restrict__ imwei,
                       const float* __restrict__ d_imout, const float* __restrict__ d_improb, float* __restrict__ dfp2d,
                       float* __restrict__ dfuv, float* __restrict__ dtex) {
    constexpr bool SHADE = MODE >= OUT_BILINEAR;
    RASTER_PARAMS_LOCAL;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float4* stage = reinterpret_cast<float4*>(smem_raw);
    float* acc = reinterpret_cast<float*>(stage + CHUNK * 3);
    int* list = reinterpret_cast<int*>(acc + CAPN * 12);
    int* posof = list + F;
    __shared__ int warp_cnt[NT / 32];

    const float MULT = rp.mult, EXPAND = rp.expand, DELTA = rp.delta;
    // per-face slots in `acc`: 12 (2-D vertices + uvs), or 6 + 3d with d attributes (fewer faces fit)
    const int nslot = MODE == OUT_ATTR ? 6 + 3 * d : 12;
    const int capn = MODE == OUT_ATTR ? CAPN * 12 / nslot : CAPN;
    const int b = blockIdx.z, tid = threadIdx.x;
    const int tx0 = blockIdx.x * TILE, ty0 = blockIdx.y * TILE;
    const int px = tx0 + (tid & (TILE - 1)), py = ty0 + (tid >> 4);
    const bool valid = px < W && py < H;
    const float x0 = centre_x(px, W, rp.sx), y0 = centre_y(py, H, rp.sy);
    const float4* fg = fgeo + (size_t)b * F * 3;
    float* gp = dfp2d + (size_t)b * F * 6;
    float* gu = dfuv + (size_t)b * F * (MODE == OUT_ATTR ? 3 * d : 6);

    const int nlist = bin_faces(fg, F, centre_x(tx0, W, rp.sx), centre_x(min(tx0 + TILE - 1, W - 1), W, rp.sx),
                                centre_y(min(ty0 + TILE - 1, H - 1), H, rp.sy), centre_y(ty0, H, rp.sy), EXPAND, list,
                                posof, warp_cnt);
    const int nacc = min(nlist, capn) * nslot;
    for (int i = tid; i < nacc; i += NT) acc[i] = 0.f;
    __syncthreads();

    const size_t pix = ((size_t)b * H + py) * W + px;
    const int fidx = valid ? imidx[pix] - 1 : -1;

    // ---- colour path: covering face -------------------------------------------------------------------
    float cv[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) cv[k] = 0.f;
    bool coord_grad = fidx >= 0;          // nearest filtering: no gradient to the sampling point
    if (fidx >= 0) {
        const float w0 = imwei[3 * pix], w1 = imwei[3 * pix + 1], w2 = imwei[3 * pix + 2];
        const float* a = fuv + ((size_t)b * F + fidx) * (MODE == OUT_ATTR ? 3 * d : 6);
        float du = 0.f, dv = 0.f, dw0, dw1, dw2;
        if constexpr (MODE == OUT_ATTR) {
            // d/dw_i of sum_k g_k (sum_i w_i attr_i[k])
            const float* g = d_imout + pix * d;
            dw0 = 0.f, dw1 = 0.f, dw2 = 0.f;
            for (int k = 0; k < d; ++k) {
                dw0 += g[k] * a[k];
                dw1 += g[k] * a[d + k];
                dw2 += g[k] * a[2 * d + k];
            }
        } else {
            const float g0 = d_imout[3 * pix], g1 = d_imout[3 * pix + 1], g2 = d_imout[3 * pix + 2];
            if constexpr (SHADE) {
                const ShadePoint sp = shade_point(w0, w1, w2, a);
                const float msum = sp.msum;
                const float g[3] = {g0 * msum, g1 * msum, g2 * msum};      // colour = tex * mask (or lerp)
                if constexpr (MODE == OUT_BILINEAR) {
                    const TexTap tp = tex_tap(sp.u, sp.v, Th, Tw);
                    const float wx0 = 1.f - tp.wx1, wy0 = 1.f - tp.wy1;
                    float sx = 0.f, sy = 0.f;
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        const float* t = tex + ((size_t)b * 3 + c) * Th * Tw;
                        float* dt = dtex + ((size_t)b * 3 + c) * Th * Tw;
                        const float t00 = tex_at(t, tp.y0, tp.x0, Th, Tw), t01 = tex_at(t, tp.y0, tp.x0 + 1, Th, Tw);
                        const float t10 = tex_at(t, tp.y0 + 1, tp.x0, Th, Tw), t11 = tex_at(t, tp.y0 + 1, tp.x0 + 1, Th, Tw);
                        sx += g[c] * ((t01 - t00) * wy0 + (t11 - t10) * tp.wy1);
                        sy += g[c] * ((t10 - t00) * wx0 + (t11 - t01) * tp.wx1);
                        if (g[c] != 0.f) {
                            const bool xa = tp.x0 >= 0 && tp.x0 < Tw, xb = tp.x0 + 1 >= 0 && tp.x0 + 1 < Tw;
                            const bool ya = tp.y0 >= 0 && tp.y0 < Th, yb = tp.y0 + 1 >= 0 && tp.y0 + 1 < Th;
                            // the same products as tap_weights (texel_visibility_kernel marks the taps where they are > 0)
                            if (ya && xa) atomicAdd(dt + (size_t)tp.y0 * Tw + tp.x0, g[c] * wx0 * wy0);
                            if (ya && xb) atomicAdd(dt + (size_t)tp.y0 * Tw + tp.x0 + 1, g[c] * tp.wx1 * wy0);
                            if (yb && xa) atomicAdd(dt + (size_t)(tp.y0 + 1) * Tw + tp.x0, g[c] * wx0 * tp.wy1);
                            if (yb && xb) atomicAdd(dt + (size_t)(tp.y0 + 1) * Tw + tp.x0 + 1, g[c] * tp.wx1 * tp.wy1);
                        }
                    }
                    du = sx * (float)(Tw - 1);
                    dv = -sy * (float)(Th - 1);
                } else if constexpr (MODE == OUT_NEAREST) {
                    const int xi = __float2int_rn(unnorm_x(sp.u, Tw)), yi = __float2int_rn(unnorm_y(sp.v, Th));
                    if (xi >= 0 && xi < Tw && yi >= 0 && yi < Th) {
#pragma unroll
                        for (int c = 0; c < 3; ++c)
                            if (g[c] != 0.f) atomicAdd(dtex + ((size_t)b * 3 + c) * Th * Tw + (size_t)yi * Tw + xi, g[c]);
                    }
                    coord_grad = false;
                } else {
                    const float ix = unnorm_x(sp.u, Tw), iy = unnorm_y(sp.v, Th);
                    const float fx = floorf(ix), fy = floorf(iy);
                    const int xs = (int)fx - 1, ys = (int)fy - 1;
                    float cx[4], cy[4], dcx[4], dcy[4];
                    cubic_weights(ix - fx, cx);
                    cubic_weights(iy - fy, cy);
                    cubic_dweights(ix - fx, dcx);
                    cubic_dweights(iy - fy, dcy);
                    float sx = 0.f, sy = 0.f;
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        const float* t = tex + ((size_t)b * 3 + c) * Th * Tw;
                        float* dt = dtex + ((size_t)b * 3 + c) * Th * Tw;
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const int y = ys + i;
                            float rx = 0.f, rdx = 0.f;
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                const int x = xs + j;
                                const float tv = tex_at(t, y, x, Th, Tw);
                                rx += cx[j] * tv;
                                rdx += dcx[j] * tv;
                                if (g[c] != 0.f && x >= 0 && x < Tw && y >= 0 && y < Th)
                                    atomicAdd(dt + (size_t)y * Tw + x, g[c] * cy[i] * cx[j]);
                            }
                            sx += g[c] * cy[i] * rdx;
                            sy += g[c] * dcy[i] * rx;
                        }
                    }
                    // ix = (u * 2 - 1 + 1) * Tw / 2 - 0.5, iy = (-(v * 2 - 1) + 1) * Th / 2 - 0.5
                    du = sx * (float)Tw;
                    dv = -sy * (float)Th;
                }
            } else {
                du = g0;
                dv = g1;
            }
            dw0 = du * a[0] + dv * a[1], dw1 = du * a[2] + dv * a[3], dw2 = du * a[4] + dv * a[5];
            // d/d(per-vertex uv)
            cv[6] = w0 * du; cv[7] = w0 * dv; cv[8] = w1 * du; cv[9] = w1 * dv; cv[10] = w2 * du; cv[11] = w2 * dv;
        }
        if (coord_grad) {
            // d/d(2-D vertices) through the barycentrics
            const Face f = unpack(fg[(size_t)fidx * 3], fg[(size_t)fidx * 3 + 1], fg[(size_t)fidx * 3 + 2]);
            const float m = f.bx - f.ax, p = f.by - f.ay, n = f.cx - f.ax, q = f.cy - f.ay;
            const float s = x0 - f.ax, t = y0 - f.ay;
            const float D = (m * q - n * p) + BARY_EPS;
            const float a1 = (dw1 - dw0) / D, a2 = (dw2 - dw0) / D, a3 = -(a1 * w1 + a2 * w2);
            const float Gs = a1 * q - a2 * p, Gt = -a1 * n + a2 * m, Gm = a2 * t + a3 * q;
            const float Gp = -a2 * s - a3 * n, Gn = -a1 * t - a3 * p, Gq = a1 * s + a3 * m;
            cv[0] = -(Gs + Gm + Gn) * MULT; cv[1] = -(Gt + Gp + Gq) * MULT; cv[2] = Gm * MULT; cv[3] = Gp * MULT;
            cv[4] = Gn * MULT; cv[5] = Gq * MULT;
        }
    }
    if constexpr (MODE == OUT_ATTR) {
        float cp[6];
#pragma unroll
        for (int k = 0; k < 6; ++k) cp[k] = cv[k];
        const int pos = fidx >= 0 ? posof[fidx] : 0;
        warp_face_acc_attr(acc, fidx, pos, d_imout + pix * d, fidx >= 0 ? imwei[3 * pix] : 0.f,
                           fidx >= 0 ? imwei[3 * pix + 1] : 0.f, fidx >= 0 ? imwei[3 * pix + 2] : 0.f, d, gu, capn);
        // 2-D vertex slots of the attribute layout: the same index arithmetic as warp_face_acc's first six
        const int lane = tid & 31;
        unsigned todo = __ballot_sync(0xffffffffu, fidx >= 0);
        while (todo) {
            const int leader = __ffs(todo) - 1;
            const int key = __shfl_sync(0xffffffffu, fidx, leader);
            const bool mine = fidx == key;
            todo &= ~__ballot_sync(0xffffffffu, mine);
#pragma unroll
            for (int k = 0; k < 6; ++k) {
                const float v = b3d::warp_sum(mine ? cp[k] : 0.f);
                if (lane == leader) acc_add(acc, pos, k, v, gp + key * 6 + k, nslot, capn);
            }
        }
    } else if constexpr (MODE != OUT_NEAREST) {      // nearest: the colour path adds nothing to the vertices or uvs
        warp_face_acc<12>(acc, fidx, fidx >= 0 ? posof[fidx] : 0, cv, 0, gp, gu);
    }

    // ---- soft-silhouette path: uncovered pixels ----------------------------------------------------------
    const float gpb = (valid && fidx < 0 && d_improb) ? d_improb[pix] : 0.f;
    const bool soft = gpb != 0.f;
    if (__syncthreads_or(soft)) {
        float keep = 1.f;
        for (int pass = 0; pass < 2; ++pass) {
            int cnt = 0;
            for (int c0 = 0; c0 < nlist; c0 += CHUNK) {
                const int n = min(CHUNK, nlist - c0);
                stage_faces(fg, list, c0, n, stage);
                __syncthreads();
                if (__any_sync(0xffffffffu, soft)) {       // warp-uniform: lanes without a soft pixel carry zeros
                    for (int j = 0; j < n; ++j) {
                        const Face f = unpack(stage[3 * j], stage[3 * j + 1], stage[3 * j + 2]);
                        const float xmin = min3(f.ax, f.bx, f.cx), xmax = max3(f.ax, f.bx, f.cx);
                        const float ymin = min3(f.ay, f.by, f.cy), ymax = max3(f.ay, f.by, f.cy);
                        const bool act = soft && cnt < rp.knum && !(x0 < sub(xmin, EXPAND) || x0 >= add(xmax, EXPAND) ||
                                                                    y0 < sub(ymin, EXPAND) || y0 >= add(ymax, EXPAND));
                        if (!__any_sync(0xffffffffu, act)) continue;
                        float g6[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                        if (act) {
                            ++cnt;
                            float te, rxe, rye, t1, rx1, ry1;
                            float dm = seg_dist2(x0, y0, f.ax, f.ay, f.bx, f.by, te, rxe, rye);
                            int e = 0;
                            const float d1 = seg_dist2(x0, y0, f.bx, f.by, f.cx, f.cy, t1, rx1, ry1);
                            if (d1 < dm) { dm = d1; e = 1; te = t1; rxe = rx1; rye = ry1; }
                            const float d2 = seg_dist2(x0, y0, f.cx, f.cy, f.ax, f.ay, t1, rx1, ry1);
                            if (d2 < dm) { dm = d2; e = 2; te = t1; rxe = rx1; rye = ry1; }
                            const float pk = expf(div_mm(-DELTA * dm, rp));
                            if (pass == 0) {
                                keep *= 1.f - pk;
                            } else if (pk < 1.f - 1e-7f) {
                                // d improb / d p_k = prod_{j != k}(1 - p_j);  d p_k / d d2 = -delta/m^2 p_k
                                const float c = gpb * (keep / (1.f - pk)) * rp.slope * pk;
                                const float ga = -2.f * (1.f - te) * c * MULT, gb = -2.f * te * c * MULT;
                                // edge e joins vertex e and e+1: slots (2e, 2e+1) and (2(e+1)%6, ...)
                                const float va[2] = {ga * rxe, ga * rye}, vb[2] = {gb * rxe, gb * rye};
#pragma unroll
                                for (int q = 0; q < 3; ++q) {
                                    if (e == q) { g6[2 * q] += va[0]; g6[2 * q + 1] += va[1]; }
                                    if ((e + 1) % 3 == q) { g6[2 * q] += vb[0]; g6[2 * q + 1] += vb[1]; }
                                }
                            }
                        }
                        if (pass == 1) {                    // every lane of the warp looks at the SAME face: reduce, one accumulate
                            const int pos = c0 + j, fi = list[pos];
#pragma unroll
                            for (int k = 0; k < 6; ++k) {
                                const float v = b3d::warp_sum(g6[k]);
                                if ((tid & 31) == 0) acc_add(acc, pos, k, v, gp + fi * 6 + k, nslot, capn);
                            }
                        }
                    }
                }
                __syncthreads();
            }
        }
    }
    __syncthreads();
    for (int i = tid; i < nacc; i += NT) {
        const float v = acc[i];
        if (v != 0.f) {
            const int fi = list[i / nslot], k = i % nslot;
            atomicAdd(k < 6 ? gp + fi * 6 + k : gu + (size_t)fi * (nslot - 6) + (k - 6), v);
        }
    }
}

// Texel visibility of a forward render: the texels whose texture gradient under an all-ones upstream gradient is > 0,
// i.e. the taps mesh_raster_bwd_kernel<true> would add a positive weight to, without running the adjoint.  A CTA covers
// VIS_PIX * NT pixels of one sample and marks texels in a per-sample bit mask in shared memory (the padded columns folded
// onto the texels they copy), then ORs its non-zero words into the global words once each.
constexpr int VIS_PIX = 16;

__device__ __forceinline__ void mark_texel(unsigned int* bits, int y, int x, float w, int Th, int Tw, int Tw_out,
                                           int symmetric) {
    if (!(w > 0.f) || x < 0 || x >= Tw || y < 0 || y >= Th) return;
    // symmetric: circpad(tex, 1) put source column Tw_out-1 first and column 0 last; otherwise column 0 was appended
    const int xs = symmetric ? (x == 0 ? Tw_out - 1 : (x == Tw - 1 ? 0 : x - 1)) : (x == Tw_out ? 0 : x);
    const int bit = y * Tw_out + xs;
    const unsigned int m = 1u << (bit & 31);
    if (!(bits[bit >> 5] & m)) atomicOr(bits + (bit >> 5), m);
}

__global__ void __launch_bounds__(NT)
texel_visibility_kernel(const int32_t* __restrict__ imidx, const float* __restrict__ imwei, const float* __restrict__ fuv,
                        int F, long long HW, int Th, int Tw, int Tw_out, int symmetric, int nwords,
                        unsigned int* __restrict__ words) {
    extern __shared__ unsigned int bits[];
    const int b = blockIdx.y;
    for (int i = threadIdx.x; i < nwords; i += NT) bits[i] = 0u;
    __syncthreads();
    const long long p0 = (long long)blockIdx.x * NT * VIS_PIX + threadIdx.x;
    for (int k = 0; k < VIS_PIX; ++k) {
        const long long p = p0 + (long long)k * NT;
        if (p >= HW) break;
        const size_t pix = (size_t)b * HW + p;
        const int fidx = imidx[pix] - 1;
        if (fidx < 0) continue;
        const ShadePoint sp = shade_point(imwei[3 * pix], imwei[3 * pix + 1], imwei[3 * pix + 2],
                                          fuv + ((size_t)b * F + fidx) * 6);
        const float g = 1.f * sp.msum;          // the adjoint's g[c] = d_imout * msum with d_imout = 1
        if (g == 0.f) continue;
        const TexTap tp = tex_tap(sp.u, sp.v, Th, Tw);
        const TapWeights tw = tap_weights(g, tp);
        mark_texel(bits, tp.y0, tp.x0, tw.w00, Th, Tw, Tw_out, symmetric);
        mark_texel(bits, tp.y0, tp.x0 + 1, tw.w01, Th, Tw, Tw_out, symmetric);
        mark_texel(bits, tp.y0 + 1, tp.x0, tw.w10, Th, Tw, Tw_out, symmetric);
        mark_texel(bits, tp.y0 + 1, tp.x0 + 1, tw.w11, Th, Tw, Tw_out, symmetric);
    }
    __syncthreads();
    unsigned int* dst = words + (size_t)b * nwords;
    for (int i = threadIdx.x; i < nwords; i += NT) {
        const unsigned int v = bits[i];
        if (v) atomicOr(dst + i, v);
    }
}

__global__ void __launch_bounds__(NT)
visibility_bytes_kernel(const unsigned int* __restrict__ words, int nbits, int nwords, long long total,
                        uint8_t* __restrict__ vis) {
    const long long t = (long long)blockIdx.x * NT + threadIdx.x;
    if (t >= total) return;
    const long long b = t / nbits;
    const int i = (int)(t - b * nbits);
    vis[t] = (uint8_t)((words[b * nwords + (i >> 5)] >> (i & 31)) & 1u);
}

size_t fwd_smem(int F) { return sizeof(float4) * CHUNK * 3 + sizeof(int) * (size_t)F; }
size_t bwd_smem(int F) { return sizeof(float4) * CHUNK * 3 + sizeof(float) * CAPN * 12 + 2 * sizeof(int) * (size_t)F; }

}  // namespace

extern "C" {

int b3d_mesh_face_setup(const float* verts, const int32_t* faces, const float* uv, int uv_batched,
                        const int32_t* ft, int B, int P, int F, int T, float* fgeo, float* fuv, float* normal1,
                        void* stream) {
    B3D_REQUIRE(B >= 0 && P > 0 && F > 0, B3D_EINVAL, "b3d_mesh_face_setup: bad sizes B=%d P=%d F=%d", B, P, F);
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(verts && faces && fgeo, B3D_EINVAL, "b3d_mesh_face_setup: null pointer");
    B3D_REQUIRE((fuv == nullptr) || (uv && ft && T > 0), B3D_EINVAL, "b3d_mesh_face_setup: fuv needs uv and ft");
    B3D_CHECK_ALIGNED(fgeo);
    dim3 grid(b3d::ceil_div(F, NT), B);
    mesh_face_setup_kernel<<<grid, NT, 0, (cudaStream_t)stream>>>(verts, faces, uv, uv_batched ? (long long)T * 2 : 0,
                                                                 ft, P, F, (float4*)fgeo, fuv, normal1);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

}  // extern "C"

namespace {

// one launch code for every entry point of the rasteriser: `fattr` is fuv [B,F,6] (OUT_UV and the shaded modes) or
// attr [B,F,3d] (OUT_ATTR)
// the pixel pitches of an H x W image, rounded as the in-kernel division __fdiv_rn(multiplier, W) would round them
RasterParams with_pitch(RasterParams rp, int H, int W) {
    rp.sx = rp.mult / (float)W;
    rp.sy = rp.mult / (float)H;
    return rp;
}

template <int MODE>
int launch_fwd(const float* fgeo, const float* fattr, int d, const float* tex, const float* bg, RasterParams rp,
               int B, int F, int H, int W, int Th, int Tw, int32_t* imidx, float* imwei, float* imout, float* improb,
               cudaStream_t st) {
    rp = with_pitch(rp, H, W);
    const size_t smem = fwd_smem(F);
    B3D_REQUIRE(smem <= 200 * 1024, B3D_EINVAL, "mesh raster: F=%d too large for the tile list", F);
    dim3 grid(b3d::ceil_div(W, TILE), b3d::ceil_div(H, TILE), B);
    B3D_CUDA_OK(cudaFuncSetAttribute(mesh_raster_fwd_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    mesh_raster_fwd_kernel<MODE><<<grid, NT, smem, st>>>((const float4*)fgeo, fattr, d, tex, bg, RASTER_PARAMS_ARGS(rp), F, H, W, Th, Tw, imidx,
                                                         imwei, imout, improb);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

template <int MODE>
int launch_bwd(const float* fgeo, const float* fattr, int d, const float* tex, int has_bg, RasterParams rp, int B,
               int F, int H, int W, int Th, int Tw, const int32_t* imidx, const float* imwei, const float* d_imout,
               const float* d_improb, float* dfp2d, float* dfattr, float* dtex, cudaStream_t st) {
    rp = with_pitch(rp, H, W);
    const size_t smem = bwd_smem(F);
    B3D_REQUIRE(smem <= 200 * 1024, B3D_EINVAL, "mesh raster bwd: F=%d too large for the tile list", F);
    const size_t nattr = MODE == OUT_ATTR ? 3 * (size_t)d : 6;
    B3D_CUDA_OK(cudaMemsetAsync(dfp2d, 0, sizeof(float) * 6 * (size_t)B * F, st));
    B3D_CUDA_OK(cudaMemsetAsync(dfattr, 0, sizeof(float) * nattr * (size_t)B * F, st));
    if (dtex) B3D_CUDA_OK(cudaMemsetAsync(dtex, 0, sizeof(float) * 3 * (size_t)B * Th * Tw, st));
    dim3 grid(b3d::ceil_div(W, TILE), b3d::ceil_div(H, TILE), B);
    B3D_CUDA_OK(cudaFuncSetAttribute(mesh_raster_bwd_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    mesh_raster_bwd_kernel<MODE><<<grid, NT, smem, st>>>((const float4*)fgeo, fattr, d, tex, has_bg, RASTER_PARAMS_ARGS(rp), F, H, W, Th, Tw,
                                                         imidx, imwei, d_imout, d_improb, dfp2d, dfattr, dtex);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

// B3D_FILTER_* -> shaded output mode
int filter_mode(int filter) {
    return filter == B3D_FILTER_BILINEAR ? OUT_BILINEAR
         : filter == B3D_FILTER_NEAREST  ? OUT_NEAREST
         : filter == B3D_FILTER_BICUBIC  ? OUT_BICUBIC
                                         : -1;
}

int check_params(const char* fn, int d, float expand, int knum, float multiplier, float delta, RasterParams* rp) {
    B3D_REQUIRE(d >= 1, B3D_EINVAL, "%s: d=%d attributes per vertex, need d >= 1", fn, d);
    B3D_REQUIRE(knum >= 1, B3D_EINVAL, "%s: knum=%d, need knum >= 1", fn, knum);
    B3D_REQUIRE(multiplier > 0.f, B3D_EINVAL, "%s: multiplier=%g, need multiplier > 0", fn, multiplier);
    B3D_REQUIRE(delta > 0.f, B3D_EINVAL, "%s: delta=%g, need delta > 0", fn, delta);
    B3D_REQUIRE(expand >= 0.f, B3D_EINVAL, "%s: expand=%g, need expand >= 0", fn, expand);
    // the box margin and the soft-silhouette scale in multiplier units, as kaolin forms them (in double, then fp32)
    *rp = make_params(multiplier, (float)((double)expand * (double)multiplier), delta, knum);
    return B3D_OK;
}

}  // namespace

extern "C" {

int b3d_mesh_face_pack(const float* points3d, const float* points2d, const float* normalz, float multiplier, int B, int F,
                       float* fgeo, void* stream) {
    B3D_REQUIRE(B >= 0 && F > 0, B3D_EINVAL, "b3d_mesh_face_pack: bad sizes B=%d F=%d", B, F);
    B3D_REQUIRE(multiplier > 0.f, B3D_EINVAL, "b3d_mesh_face_pack: multiplier=%g, need multiplier > 0", multiplier);
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(points3d && points2d && normalz && fgeo, B3D_EINVAL, "b3d_mesh_face_pack: null pointer");
    B3D_REQUIRE(B <= 65535, B3D_EINVAL, "b3d_mesh_face_pack: batch too large");
    B3D_CHECK_ALIGNED(fgeo);
    mesh_face_pack_kernel<<<dim3(b3d::ceil_div(F, NT), B), NT, 0, (cudaStream_t)stream>>>(points3d, points2d, normalz,
                                                                                         multiplier, F, (float4*)fgeo);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

int b3d_mesh_raster_attr_fwd(const float* fgeo, const float* attr, int d, int B, int F, int H, int W, float expand,
                             int knum, float multiplier, float delta, int32_t* imidx, float* imwei, float* imfeat,
                             float* improb, void* stream) {
    RasterParams rp;
    if (int rc = check_params("b3d_mesh_raster_attr_fwd", d, expand, knum, multiplier, delta, &rp)) return rc;
    B3D_REQUIRE(B >= 0 && F > 0 && H > 0 && W > 0, B3D_EINVAL, "b3d_mesh_raster_attr_fwd: bad sizes");
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(fgeo && attr && imidx && imwei && imfeat && improb, B3D_EINVAL, "b3d_mesh_raster_attr_fwd: null pointer");
    B3D_CHECK_ALIGNED(fgeo);
    return launch_fwd<OUT_ATTR>(fgeo, attr, d, nullptr, nullptr, rp, B, F, H, W, 0, 0, imidx, imwei, imfeat, improb,
                                (cudaStream_t)stream);
}

int b3d_mesh_raster_attr_bwd(const float* fgeo, const float* attr, int d, int B, int F, int H, int W, float expand,
                             int knum, float multiplier, float delta, const int32_t* imidx, const float* imwei,
                             const float* d_imfeat, const float* d_improb, float* dp2d, float* dattr, void* stream) {
    RasterParams rp;
    if (int rc = check_params("b3d_mesh_raster_attr_bwd", d, expand, knum, multiplier, delta, &rp)) return rc;
    B3D_REQUIRE(B >= 0 && F > 0 && H > 0 && W > 0, B3D_EINVAL, "b3d_mesh_raster_attr_bwd: bad sizes");
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(fgeo && attr && imidx && imwei && d_imfeat && dp2d && dattr, B3D_EINVAL,
                "b3d_mesh_raster_attr_bwd: null pointer");
    return launch_bwd<OUT_ATTR>(fgeo, attr, d, nullptr, 0, rp, B, F, H, W, 0, 0, imidx, imwei, d_imfeat, d_improb, dp2d,
                                dattr, nullptr, (cudaStream_t)stream);
}

int b3d_mesh_render_filtered_fwd(const float* fgeo, const float* fuv, const float* tex, const float* bg, int B, int F,
                                 int H, int W, int Th, int Tw, int filter, int32_t* imidx, float* imwei, float* imout,
                                 float* improb, void* stream) {
    const int mode = filter_mode(filter);
    B3D_REQUIRE(mode >= 0, B3D_EINVAL, "b3d_mesh_render_filtered_fwd: unknown filter %d", filter);
    B3D_REQUIRE(B >= 0 && F > 0 && H > 0 && W > 0, B3D_EINVAL, "b3d_mesh_render_filtered_fwd: bad sizes");
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(fgeo && fuv && tex && imidx && imwei && imout && improb, B3D_EINVAL,
                "b3d_mesh_render_filtered_fwd: null pointer");
    B3D_REQUIRE(Th > 1 && Tw > 1, B3D_EINVAL, "b3d_mesh_render_filtered_fwd: bad texture size");
    B3D_CHECK_ALIGNED(fgeo);
    const RasterParams rp = default_params();
    cudaStream_t st = (cudaStream_t)stream;
    switch (mode) {
        case OUT_NEAREST:
            return launch_fwd<OUT_NEAREST>(fgeo, fuv, 3, tex, bg, rp, B, F, H, W, Th, Tw, imidx, imwei, imout, improb, st);
        case OUT_BICUBIC:
            return launch_fwd<OUT_BICUBIC>(fgeo, fuv, 3, tex, bg, rp, B, F, H, W, Th, Tw, imidx, imwei, imout, improb, st);
        default:
            return launch_fwd<OUT_BILINEAR>(fgeo, fuv, 3, tex, bg, rp, B, F, H, W, Th, Tw, imidx, imwei, imout, improb, st);
    }
}

int b3d_mesh_render_filtered_bwd(const float* fgeo, const float* fuv, const float* tex, int has_bg, int B, int F, int H,
                                 int W, int Th, int Tw, int filter, const int32_t* imidx, const float* imwei,
                                 const float* d_imout, const float* d_improb, float* dfp2d, float* dfuv, float* dtex,
                                 void* stream) {
    const int mode = filter_mode(filter);
    B3D_REQUIRE(mode >= 0, B3D_EINVAL, "b3d_mesh_render_filtered_bwd: unknown filter %d", filter);
    B3D_REQUIRE(B >= 0 && F > 0 && H > 0 && W > 0, B3D_EINVAL, "b3d_mesh_render_filtered_bwd: bad sizes");
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(fgeo && fuv && tex && imidx && imwei && d_imout && dfp2d && dfuv && dtex, B3D_EINVAL,
                "b3d_mesh_render_filtered_bwd: null pointer");
    const RasterParams rp = default_params();
    cudaStream_t st = (cudaStream_t)stream;
    switch (mode) {
        case OUT_NEAREST:
            return launch_bwd<OUT_NEAREST>(fgeo, fuv, 3, tex, has_bg, rp, B, F, H, W, Th, Tw, imidx, imwei, d_imout,
                                           d_improb, dfp2d, dfuv, dtex, st);
        case OUT_BICUBIC:
            return launch_bwd<OUT_BICUBIC>(fgeo, fuv, 3, tex, has_bg, rp, B, F, H, W, Th, Tw, imidx, imwei, d_imout,
                                           d_improb, dfp2d, dfuv, dtex, st);
        default:
            return launch_bwd<OUT_BILINEAR>(fgeo, fuv, 3, tex, has_bg, rp, B, F, H, W, Th, Tw, imidx, imwei, d_imout,
                                            d_improb, dfp2d, dfuv, dtex, st);
    }
}

int b3d_mesh_render_fwd(const float* fgeo, const float* fuv, const float* tex, const float* bg, int B, int F, int H,
                        int W, int Th, int Tw, int32_t* imidx, float* imwei, float* imout, float* improb,
                        void* stream) {
    B3D_REQUIRE(B >= 0 && F > 0 && H > 0 && W > 0, B3D_EINVAL, "b3d_mesh_render_fwd: bad sizes");
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(fgeo && fuv && imidx && imwei && imout && improb, B3D_EINVAL, "b3d_mesh_render_fwd: null pointer");
    B3D_REQUIRE(tex == nullptr || (Th > 1 && Tw > 1), B3D_EINVAL, "b3d_mesh_render_fwd: bad texture size");
    B3D_CHECK_ALIGNED(fgeo);
    if (tex)
        return b3d_mesh_render_filtered_fwd(fgeo, fuv, tex, bg, B, F, H, W, Th, Tw, B3D_FILTER_BILINEAR, imidx, imwei,
                                            imout, improb, stream);
    return launch_fwd<OUT_UV>(fgeo, fuv, 3, nullptr, nullptr, default_params(), B, F, H, W, 0, 0, imidx, imwei, imout,
                              improb, (cudaStream_t)stream);
}

int b3d_mesh_render_bwd(const float* fgeo, const float* fuv, const float* tex, int has_bg, int B, int F, int H, int W,
                        int Th, int Tw, const int32_t* imidx, const float* imwei, const float* d_imout,
                        const float* d_improb, float* dfp2d, float* dfuv, float* dtex, void* stream) {
    B3D_REQUIRE(B >= 0 && F > 0 && H > 0 && W > 0, B3D_EINVAL, "b3d_mesh_render_bwd: bad sizes");
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(fgeo && fuv && imidx && imwei && d_imout && dfp2d && dfuv, B3D_EINVAL,
                "b3d_mesh_render_bwd: null pointer");
    B3D_REQUIRE((tex == nullptr) == (dtex == nullptr), B3D_EINVAL, "b3d_mesh_render_bwd: tex and dtex go together");
    if (tex)
        return b3d_mesh_render_filtered_bwd(fgeo, fuv, tex, has_bg, B, F, H, W, Th, Tw, B3D_FILTER_BILINEAR, imidx, imwei,
                                            d_imout, d_improb, dfp2d, dfuv, dtex, stream);
    return launch_bwd<OUT_UV>(fgeo, fuv, 3, nullptr, 0, default_params(), B, F, H, W, 0, 0, imidx, imwei, d_imout,
                              d_improb, dfp2d, dfuv, nullptr, (cudaStream_t)stream);
}

int b3d_texel_visibility(const int32_t* imidx, const float* imwei, const float* fuv, int B, int F, int H, int W, int Th,
                         int Tw, int symmetric, uint32_t* words, uint8_t* vis, void* stream) {
    B3D_REQUIRE(B >= 0 && F > 0 && H > 0 && W > 0, B3D_EINVAL, "b3d_texel_visibility: bad sizes");
    const int Tw_out = Tw - (symmetric ? 2 : 1);
    B3D_REQUIRE(Th > 1 && Tw_out >= 1 && (!symmetric || Tw_out >= 2), B3D_EINVAL,
                "b3d_texel_visibility: bad texture size %d x %d (symmetric %d)", Th, Tw, symmetric);
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(imidx && imwei && fuv && words && vis, B3D_EINVAL, "b3d_texel_visibility: null pointer");
    const long long nbits = (long long)Th * Tw_out;
    const int nwords = (int)((nbits + 31) / 32);
    const size_t smem = sizeof(unsigned int) * (size_t)nwords;
    B3D_REQUIRE(smem <= 200 * 1024, B3D_EINVAL, "b3d_texel_visibility: texture %d x %d too large for the bit mask", Th,
                Tw_out);
    const long long HW = (long long)H * W;
    const long long ctas = (HW + (long long)NT * VIS_PIX - 1) / ((long long)NT * VIS_PIX);
    const long long total = (long long)B * nbits;
    B3D_REQUIRE(B <= 65535 && ctas < (1LL << 31) && (total + NT - 1) / NT < (1LL << 31), B3D_EINVAL,
                "b3d_texel_visibility: batch too large");
    cudaStream_t st = (cudaStream_t)stream;
    B3D_CUDA_OK(cudaMemsetAsync(words, 0, sizeof(uint32_t) * (size_t)B * nwords, st));
    B3D_CUDA_OK(cudaFuncSetAttribute(texel_visibility_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    texel_visibility_kernel<<<dim3((unsigned)ctas, B), NT, smem, st>>>(imidx, imwei, fuv, F, HW, Th, Tw, Tw_out,
                                                                       symmetric ? 1 : 0, nwords, words);
    B3D_LAUNCH_OK();
    visibility_bytes_kernel<<<(unsigned)((total + NT - 1) / NT), NT, 0, st>>>(words, (int)nbits, nwords, total, vis);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

}  // extern "C"
