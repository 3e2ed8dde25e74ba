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

}  // extern "C"
