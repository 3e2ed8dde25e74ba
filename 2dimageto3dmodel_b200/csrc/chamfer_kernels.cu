// Chamfer / pairwise nearest-neighbour kernel for sm_90a (BASELINE.json north star; the reference's only
// pairwise-NN site is the mirror-vertex argmin of rendering/mesh_template.py:33-39).
//
// Shared-memory blocking over the candidate set: a CTA stages TILE candidates as float4 in shared memory
// (read back as conflict-free broadcasts) and every thread keeps QPT query points in registers, so one
// LDS.128 feeds QPT distance evaluations.  Distances are ((dx*dx + dy*dy) + dz*dz) with round-to-nearest
// intrinsics (no FMA contraction) and candidates are visited in index order with a strict '<', so the
// argmin indices equal the brute-force definition bit for bit.  FLOP-bound (8 NM per direction), not HBM.
#include "b3d_common.cuh"

namespace {
constexpr int NT = 256;
constexpr int QPT = 4;
constexpr int TILE = 1024;

__global__ void __launch_bounds__(NT)
chamfer_nn_kernel(const float* __restrict__ q, const float* __restrict__ c, int N, int M, float* __restrict__ dist,
                  int32_t* __restrict__ idx) {
    __shared__ float4 tile[TILE];
    const int b = blockIdx.y;
    const float* qb = q + (size_t)b * N * 3;
    const float* cb = c + (size_t)b * M * 3;
    float qx[QPT], qy[QPT], qz[QPT], best[QPT];
    int bi[QPT];
#pragma unroll
    for (int u = 0; u < QPT; ++u) {
        const int i = (blockIdx.x * QPT + u) * NT + threadIdx.x;
        const int ii = i < N ? i : 0;
        qx[u] = N > 0 ? qb[3 * ii] : 0.f;
        qy[u] = N > 0 ? qb[3 * ii + 1] : 0.f;
        qz[u] = N > 0 ? qb[3 * ii + 2] : 0.f;
        best[u] = INFINITY;
        bi[u] = 0;
    }
    for (int m0 = 0; m0 < M; m0 += TILE) {
        const int n = min(TILE, M - m0);
        __syncthreads();
        for (int j = threadIdx.x; j < n; j += NT)
            tile[j] = make_float4(cb[3 * (m0 + j)], cb[3 * (m0 + j) + 1], cb[3 * (m0 + j) + 2], 0.f);
        __syncthreads();
#pragma unroll 4
        for (int j = 0; j < n; ++j) {
            const float4 p = tile[j];
#pragma unroll
            for (int u = 0; u < QPT; ++u) {
                const float dx = __fsub_rn(qx[u], p.x), dy = __fsub_rn(qy[u], p.y), dz = __fsub_rn(qz[u], p.z);
                const float d = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
                if (d < best[u]) {
                    best[u] = d;
                    bi[u] = m0 + j;
                }
            }
        }
    }
#pragma unroll
    for (int u = 0; u < QPT; ++u) {
        const int i = (blockIdx.x * QPT + u) * NT + threadIdx.x;
        if (i < N) {
            dist[(size_t)b * N + i] = best[u];
            idx[(size_t)b * N + i] = bi[u];
        }
    }
}

// d(sum_i g_i |q_i - c_{idx_i}|^2): dq_i += 2 g_i (q_i - c_j), dc_j -= 2 g_i (q_i - c_j)
__global__ void __launch_bounds__(NT)
chamfer_bwd_kernel(const float* __restrict__ q, const float* __restrict__ c, const int32_t* __restrict__ idx,
                   const float* __restrict__ g, int N, int M, float* __restrict__ dq, float* __restrict__ dc) {
    const int b = blockIdx.y, i = blockIdx.x * NT + threadIdx.x;
    if (i >= N) return;
    const size_t qi = ((size_t)b * N + i) * 3;
    const size_t cj = ((size_t)b * M + idx[(size_t)b * N + i]) * 3;
    const float k = 2.f * g[(size_t)b * N + i];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const float v = k * (q[qi + d] - c[cj + d]);
        atomicAdd(dq + qi + d, v);
        atomicAdd(dc + cj + d, -v);
    }
}
}  // namespace

extern "C" {
int b3d_chamfer_nn(const float* query, const float* cand, int B, int N, int M, float* dist, int32_t* idx,
                   void* stream) {
    B3D_REQUIRE(B >= 0 && N >= 0 && M > 0, B3D_EINVAL, "b3d_chamfer_nn: bad sizes B=%d N=%d M=%d", B, N, M);
    if (B == 0 || N == 0) return B3D_OK;
    B3D_REQUIRE(query && cand && dist && idx, B3D_EINVAL, "b3d_chamfer_nn: null pointer");
    dim3 grid(b3d::ceil_div(N, NT * QPT), B);
    chamfer_nn_kernel<<<grid, NT, 0, (cudaStream_t)stream>>>(query, cand, N, M, dist, idx);
    B3D_LAUNCH_OK();
    return B3D_OK;
}

int b3d_chamfer_bwd(const float* query, const float* cand, const int32_t* idx, const float* gdist, int B, int N,
                    int M, float* dquery, float* dcand, void* stream) {
    B3D_REQUIRE(B >= 0 && N >= 0 && M > 0, B3D_EINVAL, "b3d_chamfer_bwd: bad sizes");
    if (B == 0 || N == 0) return B3D_OK;
    B3D_REQUIRE(query && cand && idx && gdist && dquery && dcand, B3D_EINVAL, "b3d_chamfer_bwd: null pointer");
    chamfer_bwd_kernel<<<dim3(b3d::ceil_div(N, NT), B), NT, 0, (cudaStream_t)stream>>>(query, cand, idx, gdist, N, M,
                                                                                     dquery, dcand);
    B3D_LAUNCH_OK();
    return B3D_OK;
}
}
