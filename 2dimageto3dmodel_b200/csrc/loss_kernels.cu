// Loss kernels of the mesh path (SURVEY.md §8 row a12) for sm_90a.
//   flat_loss_*      loss_flat (utils/losses.py:5-17): neighbour-face normal cosine regulariser
//   rgba_mse_iou_*   nn.MSELoss on cat(image, alpha) vs the RGBA target (run_reconstruction.py:429-431)
//                    fused with mean_iou's counts (run_reconstruction.py:225-231): one pass over the
//                    rendered image instead of cat + permute + sub + square + mean + 4 threshold passes.
#include "b3d_common.cuh"

namespace {
constexpr int NT = 256;

// loss = (F/2) * sum_i mean_{b,f} (n_f . n_{ff[f,i]} - 1)^2
__global__ void __launch_bounds__(NT)
flat_loss_fwd_kernel(const float* __restrict__ norms, const int32_t* __restrict__ ff, int B, int F, int K,
                     float* __restrict__ loss) {
    __shared__ float red[32];
    const int b = blockIdx.y;
    const float* nb = norms + (size_t)b * F * 3;
    float acc = 0.f;
    for (int f = blockIdx.x * NT + threadIdx.x; f < F; f += gridDim.x * NT) {
        const float x = nb[3 * f], y = nb[3 * f + 1], z = nb[3 * f + 2];
        for (int i = 0; i < K; ++i) {
            int g = ff[f * K + i];
            g = g < 0 ? g + F : g;            // torch indexing semantics for the -1 padding
            const float c = x * nb[3 * g] + y * nb[3 * g + 1] + z * nb[3 * g + 2] - 1.f;
            acc = fmaf(c, c, acc);
        }
    }
    const float tot = b3d::block_sum(acc, red);
    if (threadIdx.x == 0) atomicAdd(loss, tot * (0.5f * (float)F) / ((float)B * (float)F));
}

__global__ void __launch_bounds__(NT)
flat_loss_bwd_kernel(const float* __restrict__ norms, const int32_t* __restrict__ ff, int B, int F, int K,
                     const float* __restrict__ gloss, float* __restrict__ dnorms) {
    const int b = blockIdx.y;
    const int f = blockIdx.x * NT + threadIdx.x;
    if (f >= F) return;
    const float coef = gloss[0] * (0.5f * (float)F) / ((float)B * (float)F);
    const float* nb = norms + (size_t)b * F * 3;
    float* db = dnorms + (size_t)b * F * 3;
    const float x = nb[3 * f], y = nb[3 * f + 1], z = nb[3 * f + 2];
    float gx = 0.f, gy = 0.f, gz = 0.f;
    for (int i = 0; i < K; ++i) {
        int g = ff[f * K + i];
        g = g < 0 ? g + F : g;
        const float ox = nb[3 * g], oy = nb[3 * g + 1], oz = nb[3 * g + 2];
        const float k = 2.f * coef * (x * ox + y * oy + z * oz - 1.f);
        gx = fmaf(k, ox, gx);
        gy = fmaf(k, oy, gy);
        gz = fmaf(k, oz, gz);
        atomicAdd(db + 3 * g + 0, k * x);
        atomicAdd(db + 3 * g + 1, k * y);
        atomicAdd(db + 3 * g + 2, k * z);
    }
    atomicAdd(db + 3 * f + 0, gx);
    atomicAdd(db + 3 * f + 1, gy);
    atomicAdd(db + 3 * f + 2, gz);
}

// Unit face normals of a deformed mesh (rendering/mesh_template.py:148-152 = reference :113-123):
// n_f = normalize((v_b - v_a) x (v_c - v_a)), F.normalize semantics (n / max(|n|, 1e-12)).  One thread per (image, face):
// replaces three gathers, two subtractions, cross, norm, clamp and a division (and ~35 launches of their autograd graph,
// three of them sort-based index_put) by one launch each way.
constexpr float NORMALIZE_EPS = 1e-12f;
__global__ void __launch_bounds__(NT)
face_normals_fwd_kernel(const float* __restrict__ verts, const int32_t* __restrict__ faces, int B, int V, int F,
                        float* __restrict__ out) {
    const long long i = (long long)blockIdx.x * NT + threadIdx.x;
    if (i >= (long long)B * F) return;
    const int f = (int)(i % F), b = (int)(i / F);
    const float* vb = verts + (size_t)b * V * 3;
    const int ia = faces[3 * f], ib = faces[3 * f + 1], ic = faces[3 * f + 2];
    const float ax = vb[3 * ia], ay = vb[3 * ia + 1], az = vb[3 * ia + 2];
    const float ux = vb[3 * ib] - ax, uy = vb[3 * ib + 1] - ay, uz = vb[3 * ib + 2] - az;
    const float vx = vb[3 * ic] - ax, vy = vb[3 * ic + 1] - ay, vz = vb[3 * ic + 2] - az;
    const float nx = uy * vz - uz * vy, ny = uz * vx - ux * vz, nz = ux * vy - uy * vx;
    const float inv = 1.f / fmaxf(sqrtf(nx * nx + ny * ny + nz * nz), NORMALIZE_EPS);
    out[3 * i] = nx * inv; out[3 * i + 1] = ny * inv; out[3 * i + 2] = nz * inv;
}
// dverts [B,V,3] (zeroed by the caller) += adjoint; g = d loss / d normals
__global__ void __launch_bounds__(NT)
face_normals_bwd_kernel(const float* __restrict__ verts, const int32_t* __restrict__ faces, const float* __restrict__ g, int B, int V,
                        int F, float* __restrict__ dverts) {
    const long long i = (long long)blockIdx.x * NT + threadIdx.x;
    if (i >= (long long)B * F) return;
    const int f = (int)(i % F), b = (int)(i / F);
    const float* vb = verts + (size_t)b * V * 3;
    float* db = dverts + (size_t)b * V * 3;
    const int ia = faces[3 * f], ib = faces[3 * f + 1], ic = faces[3 * f + 2];
    const float ax = vb[3 * ia], ay = vb[3 * ia + 1], az = vb[3 * ia + 2];
    const float ux = vb[3 * ib] - ax, uy = vb[3 * ib + 1] - ay, uz = vb[3 * ib + 2] - az;
    const float vx = vb[3 * ic] - ax, vy = vb[3 * ic + 1] - ay, vz = vb[3 * ic + 2] - az;
    const float nx = uy * vz - uz * vy, ny = uz * vx - ux * vz, nz = ux * vy - uy * vx;
    const float len = sqrtf(nx * nx + ny * ny + nz * nz);
    float gx = g[3 * i], gy = g[3 * i + 1], gz = g[3 * i + 2];
    if (len > NORMALIZE_EPS) {          // d(n / |n|) = (g - nh (nh . g)) / |n|
        const float inv = 1.f / len;
        const float hx = nx * inv, hy = ny * inv, hz = nz * inv;
        const float d = hx * gx + hy * gy + hz * gz;
        gx = (gx - hx * d) * inv; gy = (gy - hy * d) * inv; gz = (gz - hz * d) * inv;
    } else {                            // clamped denominator: n / eps
        gx /= NORMALIZE_EPS; gy /= NORMALIZE_EPS; gz /= NORMALIZE_EPS;
    }
    // n = u x v:  du = v x g,  dv = g x u
    const float dux = vy * gz - vz * gy, duy = vz * gx - vx * gz, duz = vx * gy - vy * gx;
    const float dvx = gy * uz - gz * uy, dvy = gz * ux - gx * uz, dvz = gx * uy - gy * ux;
    atomicAdd(db + 3 * ib, dux); atomicAdd(db + 3 * ib + 1, duy); atomicAdd(db + 3 * ib + 2, duz);
    atomicAdd(db + 3 * ic, dvx); atomicAdd(db + 3 * ic + 1, dvy); atomicAdd(db + 3 * ic + 2, dvz);
    atomicAdd(db + 3 * ia, -(dux + dvx)); atomicAdd(db + 3 * ia + 1, -(duy + dvy)); atomicAdd(db + 3 * ia + 2, -(duz + dvz));
}

// image [B,H,W,3], alpha [B,H,W], target [B,4,H,W]; sse += sum of squared error; counts[b] = {inter, union}
__global__ void __launch_bounds__(NT)
rgba_mse_iou_fwd_kernel(const float* __restrict__ image, const float* __restrict__ alpha,
                        const float* __restrict__ target, int HW, float inv_n, float* __restrict__ loss,
                        int32_t* __restrict__ counts) {
    __shared__ float red[32];
    const int b = blockIdx.y;
    const float* tb = target + (size_t)b * 4 * HW;
    float acc = 0.f;
    int inter = 0, uni = 0;
    for (int p = blockIdx.x * NT + threadIdx.x; p < HW; p += gridDim.x * NT) {
        const size_t pix = (size_t)b * HW + p;
        const float a = alpha[pix], ta = tb[3 * (size_t)HW + p];
        float d = a - ta;
        acc = fmaf(d, d, acc);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            d = image[3 * pix + c] - tb[(size_t)c * HW + p];
            acc = fmaf(d, d, acc);
        }
        const bool pa = a > 0.5f, pt = ta > 0.5f;
        inter += (pa && pt) ? 1 : 0;
        uni += (pa || pt) ? 1 : 0;
    }
    const float tot = b3d::block_sum(acc, red);
    const float fi = b3d::block_sum((float)inter, red);
    const float fu = b3d::block_sum((float)uni, red);
    if (threadIdx.x == 0) {
        atomicAdd(loss, tot * inv_n);
        if (counts) {
            atomicAdd(counts + 2 * b, (int)fi);
            atomicAdd(counts + 2 * b + 1, (int)fu);
        }
    }
}

__global__ void __launch_bounds__(NT)
rgba_mse_bwd_kernel(const float* __restrict__ image, const float* __restrict__ alpha, const float* __restrict__ target,
                    int HW, float inv_n, const float* __restrict__ gloss, float* __restrict__ d_image,
                    float* __restrict__ d_alpha) {
    const int b = blockIdx.y;
    const float k = 2.f * inv_n * gloss[0];
    const float* tb = target + (size_t)b * 4 * HW;
    for (int p = blockIdx.x * NT + threadIdx.x; p < HW; p += gridDim.x * NT) {
        const size_t pix = (size_t)b * HW + p;
        d_alpha[pix] = k * (alpha[pix] - tb[3 * (size_t)HW + p]);
#pragma unroll
        for (int c = 0; c < 3; ++c) d_image[3 * pix + c] = k * (image[3 * pix + c] - tb[(size_t)c * HW + p]);
    }
}
}  // namespace

extern "C" {

int b3d_flat_loss_fwd(const float* norms, const int32_t* ff, int B, int F, int K, float* loss, void* stream) {
    B3D_REQUIRE(B > 0 && F > 0 && K > 0 && norms && ff && loss, B3D_EINVAL, "b3d_flat_loss_fwd: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    B3D_CUDA_OK(cudaMemsetAsync(loss, 0, sizeof(float), st));
    flat_loss_fwd_kernel<<<dim3(b3d::ceil_div(F, NT), B), NT, 0, st>>>(norms, ff, B, F, K, loss);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

int b3d_flat_loss_bwd(const float* norms, const int32_t* ff, int B, int F, int K, const float* gloss, float* dnorms,
                      void* stream) {
    B3D_REQUIRE(B > 0 && F > 0 && K > 0 && norms && ff && gloss && dnorms, B3D_EINVAL,
                "b3d_flat_loss_bwd: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    B3D_CUDA_OK(cudaMemsetAsync(dnorms, 0, sizeof(float) * 3 * (size_t)B * F, st));
    flat_loss_bwd_kernel<<<dim3(b3d::ceil_div(F, NT), B), NT, 0, st>>>(norms, ff, B, F, K, gloss, dnorms);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

int b3d_face_normals_fwd(const float* verts, const int32_t* faces, int B, int V, int F, float* normals, void* stream) {
    B3D_REQUIRE(B > 0 && V > 0 && F > 0 && verts && faces && normals, B3D_EINVAL, "b3d_face_normals_fwd: bad arguments");
    face_normals_fwd_kernel<<<b3d::ceil_div(B * F, NT), NT, 0, (cudaStream_t)stream>>>(verts, faces, B, V, F, normals);
    B3D_LAUNCH_OK();
    return B3D_OK;
}
int b3d_face_normals_bwd(const float* verts, const int32_t* faces, const float* gnormals, int B, int V, int F, float* dverts,
                         void* stream) {
    B3D_REQUIRE(B > 0 && V > 0 && F > 0 && verts && faces && gnormals && dverts, B3D_EINVAL, "b3d_face_normals_bwd: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    B3D_CUDA_OK(cudaMemsetAsync(dverts, 0, sizeof(float) * 3 * (size_t)B * V, st));
    face_normals_bwd_kernel<<<b3d::ceil_div(B * F, NT), NT, 0, st>>>(verts, faces, gnormals, B, V, F, dverts);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

int b3d_rgba_mse_iou_fwd(const float* image, const float* alpha, const float* target, int B, int H, int W, float* loss,
                         int32_t* counts, void* stream) {
    B3D_REQUIRE(B > 0 && H > 0 && W > 0 && image && alpha && target && loss, B3D_EINVAL,
                "b3d_rgba_mse_iou_fwd: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    B3D_CUDA_OK(cudaMemsetAsync(loss, 0, sizeof(float), st));
    if (counts) B3D_CUDA_OK(cudaMemsetAsync(counts, 0, sizeof(int32_t) * 2 * B, st));
    const int HW = H * W;
    const int gx = min(b3d::ceil_div(HW, NT), 132 * 4);
    rgba_mse_iou_fwd_kernel<<<dim3(gx, B), NT, 0, st>>>(image, alpha, target, HW, 1.f / (4.f * (float)B * (float)HW),
                                                       loss, counts);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

int b3d_rgba_mse_bwd(const float* image, const float* alpha, const float* target, int B, int H, int W,
                     const float* gloss, float* d_image, float* d_alpha, void* stream) {
    B3D_REQUIRE(B > 0 && H > 0 && W > 0 && image && alpha && target && gloss && d_image && d_alpha, B3D_EINVAL,
                "b3d_rgba_mse_bwd: bad arguments");
    const int HW = H * W;
    const int gx = min(b3d::ceil_div(HW, NT), 132 * 4);
    rgba_mse_bwd_kernel<<<dim3(gx, B), NT, 0, (cudaStream_t)stream>>>(image, alpha, target, HW,
                                                                     1.f / (4.f * (float)B * (float)HW), gloss,
                                                                     d_image, d_alpha);
    B3D_LAUNCH_OK();
    return B3D_OK;
}
}  // extern "C"
