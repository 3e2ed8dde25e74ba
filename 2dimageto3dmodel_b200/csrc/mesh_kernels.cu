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
//                            soft-silhouette distances), to the per-face UVs and to the texture.  Per-face
//                            gradients are accumulated in shared memory per tile and flushed once; the
//                            knum x 5 per-pixel side buffers kaolin stores are recomputed instead.
//
// Index buffer (imidx) arithmetic uses round-to-nearest intrinsics in the oracle's operation order so that
// the face-index / visibility buffers are reproduced bit for bit.
#include "b3d_common.cuh"

namespace {

constexpr int TILE = 16;
constexpr int NT = TILE * TILE;
constexpr int CHUNK = 64;          // face records staged per step
constexpr int CAPN = 768;          // per-tile shared-memory accumulators (faces beyond use global atomics)
constexpr float MULT = 1000.f;     // kaolin default `multiplier`
constexpr float EXPAND = 0.02f * 1000.f;
constexpr float DELTA = 7000.f;
constexpr int KNUM = 30;
constexpr float DEPTH_INIT = -1000.f;
constexpr float BARY_EPS = 1e-10f;
constexpr float SEG_EPS = 1e-10f;
constexpr float NORMAL_EPS = 1e-8f;

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

// pixel centres, SURVEY App. B step 2 (row 0 is the top of the image)
__device__ __forceinline__ float centre_x(int x, int W) { return mul(__fdiv_rn(MULT, (float)W), (float)(2 * x + 1 - W)); }
__device__ __forceinline__ float centre_y(int y, int H) { return mul(__fdiv_rn(MULT, (float)H), (float)(H - 2 * y - 1)); }

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
                                         float y0hi, int* list, int* posof, int* warp_cnt) {
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

template <bool SHADE>
__global__ void __launch_bounds__(NT)
mesh_raster_fwd_kernel(const float4* __restrict__ fgeo, const float* __restrict__ fuv, const float* __restrict__ tex,
                       const float* __restrict__ bg, int F, int H, int W, int Th, int Tw,
                       int32_t* __restrict__ imidx, float* __restrict__ imwei, float* __restrict__ imout,
                       float* __restrict__ improb) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float4* stage = reinterpret_cast<float4*>(smem_raw);
    int* list = reinterpret_cast<int*>(stage + CHUNK * 3);
    __shared__ int warp_cnt[NT / 32];

    const int b = blockIdx.z, tid = threadIdx.x;
    const int tx0 = blockIdx.x * TILE, ty0 = blockIdx.y * TILE;
    const int px = tx0 + (tid & (TILE - 1)), py = ty0 + (tid >> 4);
    const bool valid = px < W && py < H;
    const float x0 = centre_x(px, W), y0 = centre_y(py, H);
    const float4* fg = fgeo + (size_t)b * F * 3;

    const int nlist = bin_faces(fg, F, centre_x(tx0, W), centre_x(min(tx0 + TILE - 1, W - 1), W),
                                centre_y(min(ty0 + TILE - 1, H - 1), H), centre_y(ty0, H), list, nullptr, warp_cnt);

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

    // pass B: soft silhouette of the uncovered pixels (first KNUM faces, in face order, whose expanded
    // bounding box contains the pixel)
    float keep = 1.f;
    if (__syncthreads_or(valid && best < 0)) {
        int cnt = 0;
        for (int c0 = 0; c0 < nlist; c0 += CHUNK) {
            const int n = min(CHUNK, nlist - c0);
            stage_faces(fg, list, c0, n, stage);
            __syncthreads();
            if (valid && best < 0) {
                for (int j = 0; j < n && cnt < KNUM; ++j) {
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
                    keep *= 1.f - expf(-DELTA * d2 / (MULT * MULT));
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
    float o0 = 0.f, o1 = 0.f, o2 = 0.f;
    if (best >= 0) {
        const ShadePoint sp = shade_point(bw0, bw1, bw2, fuv + ((size_t)b * F + best) * 6);
        const float u = sp.u, v = sp.v, msum = sp.msum;
        if (SHADE) {
            const TexTap tp = tex_tap(u, v, Th, Tw);
            const float wx0 = 1.f - tp.wx1, wy0 = 1.f - tp.wy1;
            float col[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float* t = tex + ((size_t)b * 3 + c) * Th * Tw;
                col[c] = (tex_at(t, tp.y0, tp.x0, Th, Tw) * wx0 + tex_at(t, tp.y0, tp.x0 + 1, Th, Tw) * tp.wx1) * wy0 +
                         (tex_at(t, tp.y0 + 1, tp.x0, Th, Tw) * wx0 + tex_at(t, tp.y0 + 1, tp.x0 + 1, Th, Tw) * tp.wx1) *
                             tp.wy1;
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

__device__ __forceinline__ void acc_add(float* acc, int pos, int k, float v, float* gdst) {
    if (v == 0.f) return;
    if (pos < CAPN)
        atomicAdd(acc + pos * 12 + k, v);
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
                acc_add(acc, pos, kk, v, kk < 6 ? gdst6a + key * 6 + kk : gdst6b + key * 6 + (kk - 6));
            }
        }
    }
}

template <bool SHADE>
__global__ void __launch_bounds__(NT)
mesh_raster_bwd_kernel(const float4* __restrict__ fgeo, const float* __restrict__ fuv, const float* __restrict__ tex,
                       int has_bg, int F, int H, int W, int Th, int Tw, const int32_t* __restrict__ imidx,
                       const float* __restrict__ imwei, const float* __restrict__ d_imout,
                       const float* __restrict__ d_improb, float* __restrict__ dfp2d, float* __restrict__ dfuv,
                       float* __restrict__ dtex) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float4* stage = reinterpret_cast<float4*>(smem_raw);
    float* acc = reinterpret_cast<float*>(stage + CHUNK * 3);
    int* list = reinterpret_cast<int*>(acc + CAPN * 12);
    int* posof = list + F;
    __shared__ int warp_cnt[NT / 32];

    const int b = blockIdx.z, tid = threadIdx.x;
    const int tx0 = blockIdx.x * TILE, ty0 = blockIdx.y * TILE;
    const int px = tx0 + (tid & (TILE - 1)), py = ty0 + (tid >> 4);
    const bool valid = px < W && py < H;
    const float x0 = centre_x(px, W), y0 = centre_y(py, H);
    const float4* fg = fgeo + (size_t)b * F * 3;
    float* gp = dfp2d + (size_t)b * F * 6;
    float* gu = dfuv + (size_t)b * F * 6;

    const int nlist = bin_faces(fg, F, centre_x(tx0, W), centre_x(min(tx0 + TILE - 1, W - 1), W),
                                centre_y(min(ty0 + TILE - 1, H - 1), H), centre_y(ty0, H), list, posof, warp_cnt);
    const int nacc = min(nlist, CAPN) * 12;
    for (int i = tid; i < nacc; i += NT) acc[i] = 0.f;
    __syncthreads();

    const size_t pix = ((size_t)b * H + py) * W + px;
    const int fidx = valid ? imidx[pix] - 1 : -1;

    // ---- colour path: covering face -------------------------------------------------------------------
    float cv[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) cv[k] = 0.f;
    if (fidx >= 0) {
        const float g0 = d_imout[3 * pix], g1 = d_imout[3 * pix + 1], g2 = d_imout[3 * pix + 2];
        const float w0 = imwei[3 * pix], w1 = imwei[3 * pix + 1], w2 = imwei[3 * pix + 2];
        const float* a = fuv + ((size_t)b * F + fidx) * 6;
        float du, dv;
        if (SHADE) {
            const ShadePoint sp = shade_point(w0, w1, w2, a);
            const float msum = sp.msum;
            const TexTap tp = tex_tap(sp.u, sp.v, Th, Tw);
            const float wx0 = 1.f - tp.wx1, wy0 = 1.f - tp.wy1;
            const float g[3] = {g0 * msum, g1 * msum, g2 * msum};      // colour = tex * mask (or lerp)
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
        } else {
            du = g0;
            dv = g1;
        }
        // d/d(per-vertex uv)
        cv[6] = w0 * du; cv[7] = w0 * dv; cv[8] = w1 * du; cv[9] = w1 * dv; cv[10] = w2 * du; cv[11] = w2 * dv;
        // d/d(2-D vertices) through the barycentrics
        const float dw0 = du * a[0] + dv * a[1], dw1 = du * a[2] + dv * a[3], dw2 = du * a[4] + dv * a[5];
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
    warp_face_acc<12>(acc, fidx, fidx >= 0 ? posof[fidx] : 0, cv, 0, gp, gu);

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
                        const bool act = soft && cnt < KNUM && !(x0 < sub(xmin, EXPAND) || x0 >= add(xmax, EXPAND) ||
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
                            const float pk = expf(-DELTA * dm / (MULT * MULT));
                            if (pass == 0) {
                                keep *= 1.f - pk;
                            } else if (pk < 1.f - 1e-7f) {
                                // d improb / d p_k = prod_{j != k}(1 - p_j);  d p_k / d d2 = -delta/m^2 p_k
                                const float c = gpb * (keep / (1.f - pk)) * (-DELTA / (MULT * MULT)) * pk;
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
                                if ((tid & 31) == 0) acc_add(acc, pos, k, v, gp + fi * 6 + k);
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
            const int fi = list[i / 12], k = i % 12;
            atomicAdd(k < 6 ? gp + fi * 6 + k : gu + fi * 6 + (k - 6), v);
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

int b3d_mesh_render_fwd(const float* fgeo, const float* fuv, const float* tex, const float* bg, int B, int F, int H,
                        int W, int Th, int Tw, int32_t* imidx, float* imwei, float* imout, float* improb,
                        void* stream) {
    B3D_REQUIRE(B >= 0 && F > 0 && H > 0 && W > 0, B3D_EINVAL, "b3d_mesh_render_fwd: bad sizes");
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(fgeo && fuv && imidx && imwei && imout && improb, B3D_EINVAL, "b3d_mesh_render_fwd: null pointer");
    B3D_REQUIRE(tex == nullptr || (Th > 1 && Tw > 1), B3D_EINVAL, "b3d_mesh_render_fwd: bad texture size");
    B3D_CHECK_ALIGNED(fgeo);
    const size_t smem = fwd_smem(F);
    B3D_REQUIRE(smem <= 200 * 1024, B3D_EINVAL, "b3d_mesh_render_fwd: F=%d too large for the tile list", F);
    dim3 grid(b3d::ceil_div(W, TILE), b3d::ceil_div(H, TILE), B);
    cudaStream_t st = (cudaStream_t)stream;
    if (tex) {
        B3D_CUDA_OK(cudaFuncSetAttribute(mesh_raster_fwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem));
        mesh_raster_fwd_kernel<true><<<grid, NT, smem, st>>>((const float4*)fgeo, fuv, tex, bg, F, H, W, Th, Tw, imidx,
                                                            imwei, imout, improb);
    } else {
        B3D_CUDA_OK(cudaFuncSetAttribute(mesh_raster_fwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem));
        mesh_raster_fwd_kernel<false><<<grid, NT, smem, st>>>((const float4*)fgeo, fuv, nullptr, nullptr, F, H, W, 0, 0,
                                                             imidx, imwei, imout, improb);
    }
    B3D_LAUNCH_OK();
    return B3D_OK;
}

int b3d_mesh_render_bwd(const float* fgeo, const float* fuv, const float* tex, int has_bg, int B, int F, int H, int W,
                        int Th, int Tw, const int32_t* imidx, const float* imwei, const float* d_imout,
                        const float* d_improb, float* dfp2d, float* dfuv, float* dtex, void* stream) {
    B3D_REQUIRE(B >= 0 && F > 0 && H > 0 && W > 0, B3D_EINVAL, "b3d_mesh_render_bwd: bad sizes");
    if (B == 0) return B3D_OK;
    B3D_REQUIRE(fgeo && fuv && imidx && imwei && d_imout && dfp2d && dfuv, B3D_EINVAL,
                "b3d_mesh_render_bwd: null pointer");
    B3D_REQUIRE((tex == nullptr) == (dtex == nullptr), B3D_EINVAL, "b3d_mesh_render_bwd: tex and dtex go together");
    const size_t smem = bwd_smem(F);
    B3D_REQUIRE(smem <= 200 * 1024, B3D_EINVAL, "b3d_mesh_render_bwd: F=%d too large for the tile list", F);
    cudaStream_t st = (cudaStream_t)stream;
    B3D_CUDA_OK(cudaMemsetAsync(dfp2d, 0, sizeof(float) * 6 * (size_t)B * F, st));
    B3D_CUDA_OK(cudaMemsetAsync(dfuv, 0, sizeof(float) * 6 * (size_t)B * F, st));
    if (dtex) B3D_CUDA_OK(cudaMemsetAsync(dtex, 0, sizeof(float) * 3 * (size_t)B * Th * Tw, st));
    dim3 grid(b3d::ceil_div(W, TILE), b3d::ceil_div(H, TILE), B);
    if (tex) {
        B3D_CUDA_OK(cudaFuncSetAttribute(mesh_raster_bwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem));
        mesh_raster_bwd_kernel<true><<<grid, NT, smem, st>>>((const float4*)fgeo, fuv, tex, has_bg, F, H, W, Th, Tw,
                                                            imidx, imwei, d_imout, d_improb, dfp2d, dfuv, dtex);
    } else {
        B3D_CUDA_OK(cudaFuncSetAttribute(mesh_raster_bwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem));
        mesh_raster_bwd_kernel<false><<<grid, NT, smem, st>>>((const float4*)fgeo, fuv, nullptr, 0, F, H, W, 0, 0, imidx,
                                                             imwei, d_imout, d_improb, dfp2d, dfuv, nullptr);
    }
    B3D_LAUNCH_OK();
    return B3D_OK;
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
