// Implicit-GEMM 2-D convolution on the Hopper tensor cores (sm_90a, wgmma kind tf32): the dense convs of the
// conv-GAN generator / discriminators (models/gan.py:57-65,163-177,294-302,359,364; SURVEY.md §8 a13/a14).
//
//   Y[n, y, x, co] = sum_t sum_ci  X[n, sy*y + dy[t], sx*x + dx[t], ci] * Wt[t, co, ci]      (NHWC, fp32)
//
// "Tap-shifted TMA" formulation: no im2col buffer.  A work item is 128 output pixels (a BW x BH x BI box of the
// output) x BN output channels.  For every filter tap t and every 32-channel slice of Cin the TMA producer issues ONE
// 4-D tiled load of the input box shifted by (dy[t], dx[t]) — out-of-bounds rows and columns are zero-filled by the
// TMA unit, which IS the convolution's zero padding — and one 3-D load of the weight slice; both land in
// 128-byte-swizzled K-major tiles that `wgmma.mma_async ... .tf32` consumes directly (fp32 words, tf32 precision,
// fp32 accumulation in registers).  The same kernel computes
//   * fprop   (dy = r - pad_y, dx = s, Wt[t] = W[:, :, r, s]),
//   * dgrad   (dy = pad_y - r, dx = -s, Wt[t] = W[:, :, r, s]^T)  — the "full" correlation falls out of the
//     TMA zero fill, and strided (4x4 / stride 2) dgrad runs as 4 parity classes with a strided epilogue,
//   * strided fprop (element strides in the tensor map).
// Warp roles (384 threads): warpgroup 0 = TMA producer (one thread issues), warpgroups 1-2 = wgmma with the weights as the
// M operand (64-channel blocks) and the 128-pixel tile as the N operand — on alternate work items with BN <= 128, on one
// 128-channel half of every item with BN = 256 — and the epilogue straight from the accumulator registers (bias /
// LeakyReLU / BN statistics / fused activation adjoint -> global).
// Persistent: a CTA per SM walks the work items; the STAGES-deep mbarrier ring keeps the producer loading the next item
// while the consumers run the epilogue of the current one.  The fused activation adjoint's mask travels through the same
// ring: after an item's K steps the producer loads its mask tile as BN / 32 more stages (one 128-pixel x 32-channel TMA box
// of the mask, which has the output's geometry, each), and the epilogue reads the mask from shared memory.
#include "tc_common.cuh"

namespace {

constexpr int BM = 128;         // output pixels per work item (the N of one m64n128k8 per 64-channel block)
constexpr int BK = 32;          // fp32 channels per K slice = 128 B = one swizzle row
constexpr int MMA_K = 8;        // tf32
constexpr int MAX_TAPS = 25;
constexpr int NTHREADS = 384;   // warpgroup 0: TMA producer, warpgroups 1-2: MMA + epilogue

struct ConvParams {
    int N, Hout, Wout, Cout;          // logical output extent covered by tiles (before the epilogue transform)
    int BW, BH, BI;                   // output box per work item, BW*BH*BI == 128
    int tiles_x, tiles_y;             // tiles along W and H (tiles along N = tiles / (tiles_x*tiles_y))
    int xbase;                        // first output column of this launch (a strip launch covers the last few columns)
    int ntaps, kslices;               // filter taps (per class), Cin / 32
    int sy, sx;                       // input coordinate = s * out + d[t]
    int dy[MAX_TAPS], dx[MAX_TAPS];
    int wtap[MAX_TAPS];               // weight tap (row of the tap-major weight array) read for loop tap t
    // epilogue: out pixel (n, osy*y + cooy[class], osx*x + coox[class]) of a tensor [N, OH, OW, OC], channel offset 0
    int OH, OW, OC, osy, osx;
    float leaky;                      // 1.0 = identity
    double* stats;                    // nullable: [2][Cout] fp64 sum / sum of squares of the (pre-bias) output, accumulated
    int fold;                         // > 0: the A operand is folded on the fly from a raw [N,H,W,8] tensor (thin stems): K slice ks
    int fold_y0;                      //      = image rows y + fold_y0 + 4 ks .. + 3 of the 8 channels (tensor map dims c, x, row, n)
    int mask;                         // 1: acc *= (mask >= 0 ? 1 : mslope) before statistics / bias, the mask (a tensor of the output's
    float mslope;                     //    geometry) read through the third tensor map (LeakyReLU adjoint fused into the input gradient)
    int stats_sum;                    // statistics: sums only (the bias gradient of the fused adjoint)
    int ncls;                         // >= 1 output classes in ONE launch (the stride-2 input gradient's parity classes): class c uses taps
    int cooy[4], coox[4];             //      [c * ntaps, (c + 1) * ntaps) of dy / dx / wtap and the output offset (cooy[c], coox[c])
    uint32_t esn, esy, esx;           // element strides of the output between pixels of a tile one step apart along n / y / x
    int dx0, shift[5];                // row window (KW > 1): window starts at column x + dx0; tap t of a filter row reads it shift[t] rows in
};

// KW == 1: one stage = the 128-pixel A tile of one tap and its weight tile.  KW > 1 (row window): one stage = ONE window of
// 128 + KW - 1 input pixels of a filter row and the KW weight tiles of that row; the consumers feed tap t as the window
// shifted by whole 128-byte rows (the 128-byte swizzle is a function of the absolute shared-memory address, so TMA's write
// pattern and the shifted descriptor agree), i.e. the A operand is loaded once per filter row instead of once per tap.
// A mask stage holds one 32-channel chunk of the item's mask tile in the A region, 128-byte swizzled: see mask_offset.
constexpr int MASK_BYTES = BM * BK * 4;
template <int BN, int STAGES, int KW>
struct CSmem {
    static constexpr int WIN_BYTES = (BM + KW - 1) * BK * 4;                 // what the A box delivers
    static constexpr int A_BYTES = (WIN_BYTES + 1023) / 1024 * 1024;         // B tiles start on a swizzle-atom boundary
    static constexpr int B_BYTES = KW * BN * BK * 4;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int TX_BYTES = WIN_BYTES + B_BYTES;
    static constexpr int TOTAL = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
    static_assert(A_BYTES >= MASK_BYTES, "a mask chunk does not fit the A region of a stage");
};

// Byte offset of mask element (pixel px of the tile, channel ch of the 32-channel chunk) in a mask stage: TMA writes the
// box's 128-byte pixel rows with the 128-byte swizzle (16-byte chunk index XOR px % 8; stages are 1024-byte aligned).
__device__ __forceinline__ uint32_t mask_offset(int px, int ch) { return px * 128 + ((((ch >> 2) ^ px) & 7) << 4) + (ch & 3) * 4; }

// Every tile width swaps the operands: the BN x 32 weight tile is the M operand, in 64-channel blocks, and the whole
// 128-pixel tile the N operand of one m64n128k8 per block and K step (6 KB of shared memory read per 65 536 MACs).  A
// consumer warpgroup holds at most 128 channels x 128 pixels (128 accumulator registers per thread).  With BN <= 128 each
// warpgroup owns whole work items (item k of the CTA goes to warpgroup k % 2), so one warpgroup's epilogue overlaps the
// other's main loop.  With BN == 256 (kCoop) both warpgroups work on every item, warpgroup h on channels 128 h .. 128 h + 127.
template <int BN>
constexpr bool kCoop = BN > 128;
template <int BN>
constexpr int kBlocks = (kCoop<BN> ? BN / 2 : BN) / 64;       // 64-channel M blocks per consumer warpgroup
// Arrivals that hand a stage back to the producer: every consumer warp that waits on the stage's full barrier takes part,
// the 4 warps of the item's owner (8 with kCoop).  An operand stage, read by wgmma, gets 4 from the leader of each
// warpgroup that read it once the wgmma group has retired; a mask stage gets one from each warp once the warp's loads of
// its block are done, whether or not it read that stage.  So no stage is refilled before every warp that waits on it has
// seen the fill: phase bits never skip a phase, and no wait can see a barrier two phases on.
template <int BN>
constexpr int kEmptyArrivals = kCoop<BN> ? 8 : 4;
template <int BN>
constexpr int kLeaderArrivals = kEmptyArrivals<BN> / (kCoop<BN> ? 2 : 1);     // per warpgroup leader, for an operand stage
static_assert(kLeaderArrivals<64> == 4 && kLeaderArrivals<128> == 4 && kLeaderArrivals<256> == 4,
              "a leader stands for the 4 warps of its warpgroup");
// Mask stages per 64-channel block of an item: the two 32-channel chunks of the block of each warpgroup on the item.  Item
// mask stage i holds the chunk of block i / G, warpgroup (i % G) / 2, channels c0 + 128 ((i % G) / 2) + 64 (i / G) + 32 (i % 2):
// the chunks that the warpgroups read at the same time are in the ring at the same time (G <= STAGES), and a block's
// stages are handed back before the next block's are waited on.
template <int BN>
constexpr int kMaskGroup = kCoop<BN> ? 4 : 2;
__host__ __device__ constexpr int mask_chunk_channel(int i, int G) { return 128 * ((i % G) / 2) + 64 * (i / G) + 32 * (i % 2); }

// The K loop of one work item for one consumer warpgroup: its kBlocks 64 x 128 (channel x pixel) accumulators, channels
// cb .. of the item's weight tile.  `full` is the warpgroup's row of full barriers and `phase` holds the parity of its next
// wait on each of them: with BN <= 128 a warpgroup skips the other's stages, so it cannot derive the parity from git.  A
// stage is handed back to the producer once the wgmma group that read it has retired (kEmptyArrivals).
template <int BN, int STAGES, int KW, bool FOLD>
__device__ __forceinline__ void mainloop(float (&acc)[kBlocks<BN>][BM / 2], unsigned char* base, uint64_t* full, uint64_t* empty,
                                         int KI, uint32_t& git, uint32_t& phase, int cb, bool leader, const int* shift) {
    constexpr int A_BYTES = CSmem<BN, STAGES, KW>::A_BYTES, STAGE = CSmem<BN, STAGES, KW>::STAGE_BYTES;
    for (int it = 0; it < KI; ++it, ++git) {
        const int s = git % STAGES;
        tc::mbar_wait(full + s, (phase >> s) & 1);
        phase ^= 1u << s;
        const uint32_t a = tc::smem_u32(base + s * STAGE), b = a + A_BYTES + cb * 128;
        tc::wgmma_fence();
#pragma unroll
        for (int t = 0; t < KW; ++t) {
            const uint32_t shifted = a + (KW > 1 ? shift[t] * 128 : 0);
#pragma unroll
            for (int k = 0; k < BK / MMA_K; ++k) {
                const uint32_t acc_flag = (it | t | k) ? 1u : 0u;
                // on-the-fly fold: K step k = image row k of the 4-row box, a [128 px][32 B] tile of its own (32-byte swizzle)
                const uint64_t dp = FOLD ? tc::desc_k32(a + k * (BM * 32)) : tc::desc_k128(shifted + k * MMA_K * 4);
#pragma unroll
                for (int m = 0; m < kBlocks<BN>; ++m)
                    tc::Wgmma<BM>::mma(acc[m], tc::desc_k128(b + t * (BN * 128) + m * (64 * 128) + k * MMA_K * 4), dp, acc_flag);
            }
        }
        tc::wgmma_commit();
        tc::wgmma_wait<1>();
        if (it > 0 && leader) tc::mbar_arrive(empty + (git - 1) % STAGES, kLeaderArrivals<BN>);
    }
    tc::wgmma_wait<0>();
    if (KI > 0 && leader) tc::mbar_arrive(empty + (git - 1) % STAGES, kLeaderArrivals<BN>);
}

// Where a work item's 128-pixel tile lies in the output tensor (and in the mask, which has the output's geometry): pixel
// px = (bi, by, bx) of the BI x BH x BW box is output pixel (n0 + bi, y0 + by, x0 + bx) of the launch's logical extent, and
// its channel 0 is element  base + bi esn + by esy + bx esx  (the part after base fits 32 bits: checked by the host).
struct TileAt {
    int n0, y0, x0;
    size_t base;
    int lbw, lbwh;                    // log2 BW, log2 (BW * BH): both are powers of two
};
__device__ __forceinline__ void tile_origin(const ConvParams& p, TileAt& t, int tile, int cls) {
    t.x0 = p.xbase + (tile % p.tiles_x) * p.BW;
    t.y0 = (tile / p.tiles_x) % p.tiles_y * p.BH;
    t.n0 = tile / (p.tiles_x * p.tiles_y) * p.BI;
    t.base = (((size_t)t.n0 * p.OH + (size_t)(p.osy * t.y0 + p.cooy[cls])) * p.OW + (size_t)(p.osx * t.x0 + p.coox[cls])) * p.OC;
}
// false when pixel px (0 .. 127) of the tile lies outside the launch's extent (`rel` is then not to be used)
__device__ __forceinline__ bool tile_pixel(const ConvParams& p, const TileAt& t, int px, uint32_t& rel) {
    const int bi = px >> t.lbwh, by = (px >> t.lbw) & (p.BH - 1), bx = px & (p.BW - 1);
    rel = bi * p.esn + by * p.esy + bx * p.esx;
    return t.n0 + bi < p.N && t.y0 + by < p.Hout && t.x0 + bx < p.Wout;
}

// The mask of one 64-channel block as sign bits: this thread's 64 values (channels cw, cw + 8 of the warp's 32-channel
// chunk, whose mask stage starts at shared address `mstage`; pixels 8 j + 2 (lane % 4) + {0, 1}) become bit 4 j' + 2 e2 + e1
// of neg[j / 8] (j' = j % 8), set where !(m >= 0): the slope rule of pad_leaky_bias_bwd_kernel, NaN included.  The
// warp then hands back all G mask stages of the block (ring positions g0 .. g0 + G - 1, see kEmptyArrivals) before any
// epilogue arithmetic, so an item's mask stages leave the ring as soon as they are read.  Across the warp the loads of
// one (j, e1, e2) cover 8 chunk indices x 4 words: conflict-free.
template <int G, int STAGES>
__device__ __forceinline__ void mask_bits(uint32_t (&neg)[2], uint32_t mstage, int cw, int lane, uint64_t* empty, uint32_t g0) {
    int q;                                                                // a zero the compiler cannot see through, as below
    asm volatile("mov.u32 %0, 0;" : "=r"(q));
    q += 2 * (lane & 3);
    // mask element [e2][e1] of pixel q + e1 and chunk channel (cw + 8 e2) % 32; pixel 8 j further is 1024 j bytes further
    uint32_t mb[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) mb[i] = mstage + mask_offset(q + (i & 1), (cw + 8 * (i >> 1)) & 31);
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
        uint32_t bits = 0;
#pragma unroll
        for (int j = 0; j < BM / 16; ++j)
#pragma unroll
            for (int i = 0; i < 4; ++i) bits |= (tc::lds_f32(mb[i] + 1024 * (j + 8 * hf)) >= 0.f ? 0u : 1u) << (4 * j + i);
        neg[hf] = bits;
    }
    __syncwarp();
    if (lane == 0)
#pragma unroll
        for (int i = 0; i < G; ++i) tc::mbar_arrive(empty + (g0 + i) % STAGES);
}

// Epilogue of one 64-channel block of an item: this thread holds D[co][px] for the channels c0 + cw, c0 + cw + 8 and the
// pixels 8 j + 2 (lane % 4) + {0, 1}.  MASKED: the value is multiplied by the slope where its bit in `neg` (mask_bits) is set.
template <bool MASKED>
__device__ __forceinline__ void epilogue_block(const float (&acc)[BM / 2], const uint32_t (&neg)[2], const ConvParams& p, const TileAt& t,
                                               const float* bias, float* out, int c0, int cw, int lane) {
    bool cok[2];
    float bv[2], sum[2] = {0.f, 0.f}, sq[2] = {0.f, 0.f};
#pragma unroll
    for (int e = 0; e < 2; ++e) {
        cok[e] = c0 + cw + 8 * e < p.Cout;
        bv[e] = bias && cok[e] ? __ldg(bias + c0 + cw + 8 * e) : 0.f;
    }
    float* out0 = out + t.base + c0 + cw;
    // A zero the compiler cannot see through: the pixels' box coordinates and relative offsets do not depend on the item, and
    // hoisted out of the item loop they cost more registers than the kernel has.
    int q;
    asm volatile("mov.u32 %0, 0;" : "=r"(q));
    q += 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BM / 8; ++j) {
#pragma unroll
        for (int e1 = 0; e1 < 2; ++e1) {
            uint32_t rel;
            const bool valid = tile_pixel(p, t, 8 * j + q + e1, rel);
#pragma unroll
            for (int e2 = 0; e2 < 2; ++e2) {
                float v = acc[4 * j + 2 * e2 + e1];
                if constexpr (MASKED) v *= (neg[j / 8] >> (4 * (j % 8) + 2 * e2 + e1)) & 1u ? p.mslope : 1.f;
                v = valid ? v : 0.f;
                sum[e2] += v;
                sq[e2] += v * v;
                if (valid && cok[e2]) {
                    const float o = v + bv[e2];
                    out0[rel + 8 * e2] = o >= 0.f ? o : o * p.leaky;
                }
            }
        }
    }
    if (p.stats) {
        // the four lanes of a quad hold the channel's 128 pixels; warp w alone holds channels c0 + 16 w .. c0 + 16 w + 15
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            sum[e] += __shfl_xor_sync(0xffffffffu, sum[e], 1);
            sum[e] += __shfl_xor_sync(0xffffffffu, sum[e], 2);
            sq[e] += __shfl_xor_sync(0xffffffffu, sq[e], 1);
            sq[e] += __shfl_xor_sync(0xffffffffu, sq[e], 2);
            if ((lane & 3) == 0 && cok[e]) {
                atomicAdd(p.stats + c0 + cw + 8 * e, (double)sum[e]);
                if (!p.stats_sum) atomicAdd(p.stats + p.Cout + c0 + cw + 8 * e, (double)sq[e]);
            }
        }
    }
}

// registers move from the producer warpgroup (one thread issues TMA) to the consumers: the 128- and 256-wide consumers hold
// 128 accumulators, and gather a block's mask bits from 32 loaded values at a time next to them (at 232 that spills);
// 128 * (168 - 24) == 256 * (240 - 168)
constexpr int PRODUCER_REGS = 24, CONSUMER_REGS = 240;

// tmap_m: the mask (masked launches only), dims {OC, OW, OH, N}, box {32, osx (BW - 1) + 1, osy (BH - 1) + 1, BI} with
// element strides {1, osx, osy, 1}: pixel px of the box lands as row px of the tile, zero-filled outside the tensor
template <int BN, int STAGES, int KW>
__global__ void __launch_bounds__(NTHREADS, 1)
conv_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
                  const __grid_constant__ CUtensorMap tmap_m, const ConvParams p, const float* __restrict__ bias,
                  float* __restrict__ out, int tiles, int work_items) {
    using S = CSmem<BN, STAGES, KW>;
    constexpr bool COOP = kCoop<BN>;
    constexpr int OWNERS = COOP ? 1 : 2;               // rows of full barriers: one per warpgroup that owns items
    constexpr int G = kMaskGroup<BN>;
    static_assert(G <= STAGES, "the mask stages of one block do not fit the ring");
    extern __shared__ unsigned char smem_raw[];
    unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full = reinterpret_cast<uint64_t*>(base + STAGES * S::STAGE_BYTES);     // [OWNERS][STAGES]
    uint64_t* empty = full + OWNERS * STAGES;
    static_assert((OWNERS + 1) * STAGES * 8 <= 256, "barriers do not fit their area");
    if (threadIdx.x == 0) {
        tc::tma_prefetch_desc(&tmap_x);
        tc::tma_prefetch_desc(&tmap_w);
        if (p.mask) tc::tma_prefetch_desc(&tmap_m);
        for (int s = 0; s < STAGES; ++s) {
            for (int o = 0; o < OWNERS; ++o) tc::mbar_init(full + o * STAGES + s, 1);
            tc::mbar_init(empty + s, kEmptyArrivals<BN>);
        }
        tc::fence_barrier_init();
    }
    __syncthreads();
    const int KI = p.ntaps / KW * p.kslices;           // K steps: (taps or filter rows) x channel slices
    const int MS = p.mask ? BN / 32 : 0;               // mask stages per item
    const int wg = threadIdx.x >> 7;

    if (wg == 0) {
        tc::setmaxnreg_dec<PRODUCER_REGS>();
        if (threadIdx.x == 0) {
            uint32_t git = 0;
            for (int w = blockIdx.x, k = 0; w < work_items; w += gridDim.x, ++k) {
                uint64_t* fb = full + (COOP ? 0 : (k & 1) * STAGES);     // the owner's full barriers
                // classes are the fastest index: the CTAs that work on the same pixel tiles at the same time share them in L2
                const int cls = w % p.ncls, wq = w / p.ncls, tb = cls * p.ntaps;
                int t = wq % tiles;
                const int c0 = (wq / tiles) * BN;
                const int x0 = p.xbase + (t % p.tiles_x) * p.BW;
                t /= p.tiles_x;
                const int y0 = (t % p.tiles_y) * p.BH, n0 = (t / p.tiles_y) * p.BI;
                for (int it = 0; it < KI; ++it, ++git) {
                    const int s = git % STAGES;
                    tc::mbar_wait(empty + s, ((git / STAGES) & 1) ^ 1);
                    const int tap = it / p.kslices * KW, ks = it % p.kslices;        // KW > 1: first tap of the filter row
                    unsigned char* a = base + s * S::STAGE_BYTES;
                    tc::mbar_arrive_expect_tx(fb + s, S::TX_BYTES);
                    if (KW > 1)     // window of 128 + KW - 1 pixels of the row; one box with the row's KW weight tiles
                        tc::tma_load_4d(a, &tmap_x, fb + s, ks * BK, x0 + p.dx0, y0 + p.dy[tb + tap], n0);
                    else if (p.fold)     // box {8 ch, BW px, 4 rows}: lands as [row][pixel][8 floats] = four 32-byte-swizzled K-step tiles
                        tc::tma_load_4d(a, &tmap_x, fb + s, 0, x0 + p.dx[tb + tap], y0 + p.fold_y0 + 4 * ks, n0);
                    else
                        tc::tma_load_4d(a, &tmap_x, fb + s, ks * BK, p.sx * x0 + p.dx[tb + tap], p.sy * y0 + p.dy[tb + tap], n0);
                    tc::tma_load_3d(a + S::A_BYTES, &tmap_w, fb + s, ks * BK, c0, p.wtap[tb + tap]);
                }
                const int mx = p.osx * x0 + p.coox[cls], my = p.osy * y0 + p.cooy[cls];
                for (int m = 0; m < MS; ++m, ++git) {
                    const int s = git % STAGES;
                    tc::mbar_wait(empty + s, ((git / STAGES) & 1) ^ 1);
                    tc::mbar_arrive_expect_tx(fb + s, MASK_BYTES);
                    tc::tma_load_4d(base + s * S::STAGE_BYTES, &tmap_m, fb + s, c0 + mask_chunk_channel(m, G), mx, my, n0);
                }
            }
        }
        return;
    }
    tc::setmaxnreg_inc<CONSUMER_REGS>();

    const int h = wg - 1, tid = threadIdx.x & 127, lane = tid & 31;
    float acc[kBlocks<BN>][BM / 2];
#pragma unroll
    for (int m = 0; m < kBlocks<BN>; ++m)
#pragma unroll
        for (int i = 0; i < BM / 2; ++i) acc[m][i] = 0.f;
    uint32_t git = 0, phase = 0;
    const uint32_t ring = tc::smem_u32(base);
    TileAt at;
    at.lbw = __ffs(p.BW) - 1;
    at.lbwh = at.lbw + __ffs(p.BH) - 1;
    uint64_t* fb = full + (COOP ? 0 : h * STAGES);
    const int cb = COOP ? 128 * h : 0;                 // the warpgroup's first channel in the item's tile
    const int cw = (tid >> 5) * 16 + (lane >> 2);
    const int mine = (COOP ? 2 * h : 0) + (tid >> 6);  // which of a block's G mask stages holds this warp's 16 channels
    for (int k = COOP ? 0 : h;; k += COOP ? 1 : 2) {
        const int w = blockIdx.x + k * gridDim.x;
        if (w >= work_items) break;
        git = (uint32_t)k * (KI + MS);                                         // skip the other warpgroup's items
        const int wq = w / p.ncls, tile = wq % tiles, c0 = (wq / tiles) * BN + cb;
        tile_origin(p, at, tile, w % p.ncls);
        if (KW == 1 && p.fold) mainloop<BN, STAGES, KW, true>(acc, base, fb, empty, KI, git, phase, cb, tid == 0, p.shift);
        else mainloop<BN, STAGES, KW, false>(acc, base, fb, empty, KI, git, phase, cb, tid == 0, p.shift);
        uint32_t neg[kBlocks<BN>][2] = {};
        if (p.mask) {
            // every warp waits for all G stages of a block, so that its phase bits stay those of the barriers, and reads the
            // one that holds its channels; all of the item's mask stages are handed back before the first block's epilogue
#pragma unroll
            for (int m = 0; m < kBlocks<BN>; ++m, git += G) {
                uint32_t mstage = 0;
#pragma unroll
                for (int i = 0; i < G; ++i) {
                    const int s = (git + i) % STAGES;
                    tc::mbar_wait(fb + s, (phase >> s) & 1);
                    phase ^= 1u << s;
                    if (i == mine) mstage = ring + s * S::STAGE_BYTES;
                }
                mask_bits<G, STAGES>(neg[m], mstage, cw, lane, empty, git);
            }
        }
#pragma unroll
        for (int m = 0; m < kBlocks<BN>; ++m) {
            if (p.mask) epilogue_block<true>(acc[m], neg[m], p, at, bias, out, c0 + 64 * m, cw, lane);
            else epilogue_block<false>(acc[m], neg[m], p, at, bias, out, c0 + 64 * m, cw, lane);
        }
    }
}

// ----------------------------------------------------------------------------------------------
// wgrad:  dW[co, ci, r, s] += sum_{n,y,x} dY[n, y, x, co] * X[n, st*y + r - pad_y, st*x + s, ci]      (NHWC operands)
// GEMM with M = Cout (128), N = Cin (BN), K = output pixels.  In NHWC the reduction index (pixel) is the SLOW index
// of both operands, i.e. they are M/N-major: a K slice is a BWk x BHk box of 32 output pixels, loaded by TMA as
// [32 pixels][32 channels] boxes (four for dY, BN/32 for X, the X boxes shifted by the tap on the OUTER dims: zero fill =
// padding, element strides for stride 2) into an NRAW-deep staging ring.  wgmma reads tf32 operands from shared memory
// K-major only, so the producer warpgroup rewrites each X slice K-major into the swizzled stage the consumers read
// (wgrad_transpose: 16-byte shared-memory loads and stores around a 4 x 4 register transpose).  dY is the A operand, which wgmma also takes from registers: the consumers load their
// fragments straight from the staged dY tile (128-byte swizzled by TMA, conflict-free: dy_tile_offset) and hand the raw
// slot back as soon as the loads are done.  No NCHW copy is ever made.  T > 1 (row of taps): a K slice is a 32-pixel row
// segment, the X box is a window of 32 + T - 1 (rounded to 36) pixels, and the producer reads it once and writes T K-major
// B tiles from it — tap t is the window shifted by t pixels — which share the dY fragments: T accumulators per consumer warpgroup, T taps
// per byte of dY.  One CTA per (co tile, ci tile, tap group, K split); partial sums are reduced into dW with global atomics.
// ----------------------------------------------------------------------------------------------
struct WgradParams {
    int N, Hout, Wout, Cout, Cin;
    int BWk, BHk;                  // pixel box of one K slice, BWk * BHk == 32
    int kx, ky;                    // K slices along x and y per image
    int kh, kw, pad_y, st;
    int xoff;                      // the convolution reads x from column xoff on (a caller-side crop of the padded input)
    int splits;                    // K splits (gridDim.z / tap groups)
    int tapmajor;                  // dW layout: 0 = [Cout][Cin][kh][kw], 1 = tap-major [kh*kw][Cout][Cin] (the F layout)
    int tstep;                     // taps of one CTA are s0, s0 + tstep, ... (1: adjacent taps of a stride-1 conv,
                                   // 2: taps of equal parity of a stride-2 conv = adjacent pixels of the strided window)
};

// Stage: the T K-major X tiles.  Raw slot: the dY tile (offset 0, 1024-byte aligned: its 128-byte swizzle is the one
// dy_tile_offset describes) and the X boxes behind it.
template <int BN, int STAGES, int NRAW, int T>
struct WSmem {
    static constexpr int DY_BYTES = BM * BK * 4;
    static constexpr int STAGE_BYTES = T * BN * BK * 4;
    static constexpr int WROWS = T == 1 ? 32 : 36;                      // X pixels per 32-channel block of a raw slice
    static constexpr int RAW_X = (BN / 32) * WROWS * 128;
    static constexpr int RAW_BYTES = (DY_BYTES + RAW_X + 1023) / 1024 * 1024;
    static constexpr int TOTAL = STAGES * STAGE_BYTES + NRAW * RAW_BYTES + 1024 + 256;
};

// Row m (0..63) of a consumer warpgroup's m64 tile is output channel wgrad_row_co(m) of the warpgroup's 64: bits 2, 3, 4
// of m rotated to 3, 4, 2.  Within a warp's fragment load the eight lanes that share l % 4 then see channels c, c + 1,
// c + 2, c + 3, c + 16 ... c + 19, i.e. two 16-byte chunks of a 128-byte row that differ in chunk bit 2, while the four
// values of l % 4 (consecutive pixels) XOR the chunk index with four different values in bits 0-1.
__host__ __device__ constexpr int wgrad_row_co(int m) { return (m & 35) | ((m & 8) >> 1) | ((m & 16) >> 1) | ((m & 4) << 2); }

// Byte offset of dY[co][px] (co < 128 of the CTA's tile, px < 32 of the K slice) in the staged dY tile: TMA lands four
// [32 px][32 ch] boxes of 4 KB with the 128-byte swizzle (16-byte chunk index XOR row % 8).  With the rows of
// wgrad_row_co, each of a thread's fragment loads (A[m][k] of the layout in tc_common.cuh, k = px % 8 of K step px / 8)
// touches 32 different banks across the warp; K step k is 1024 bytes further.
__host__ __device__ constexpr int dy_tile_offset(int co, int px) {
    return (co >> 5) * 4096 + px * 128 + ((((co >> 2) & 7) ^ (px & 7)) << 4) + (co & 3) * 4;
}

// The producer's transpose of a raw X slice (per 32-channel block: wrows pixels of 128 bytes, unswizzled) into the K-major,
// 128-byte swizzled B tiles (row = channel, 16-byte chunk c = pixels 4c .. 4c + 3, stored at chunk c ^ (row % 8)).  Task i
// (0 .. 2 BN) covers block i / 64, channels 4 (i % 8) .. + 3 and chunk xt_chunk(i) of every tap's tile: T + 3 16-byte loads
// of consecutive window pixels (xt_src_offset), a 4 x 4 register transpose per tap, and 4 T 16-byte stores (xt_dst_offset).
// The eight tasks of a quarter warp have i % 8 = 0 .. 7, so their loads hit eight different chunk positions of a 128-byte row,
// and for each store their chunks xt_chunk(i) ^ (row % 8) are eight different values: both are conflict-free.
__host__ __device__ constexpr int xt_chunk(int i) { return (((i & 7) >> 1) ^ ((i >> 4) & 3)) | (((i >> 3) & 1) << 2); }
__host__ __device__ constexpr int xt_src_offset(int i, int px, int wrows) { return ((i >> 6) * wrows + px) * 128 + (i & 7) * 16; }
__host__ __device__ constexpr int xt_dst_offset(int i, int j) {     // channel j (0..3) of task i
    return ((i >> 6) * 32 + 4 * (i & 7) + j) * 128 + ((xt_chunk(i) ^ ((4 * (i & 7) + j) & 7)) << 4);
}
template <int BN, int T, int WROWS>
__device__ __forceinline__ void wgrad_transpose(uint32_t src, uint32_t dst, int tid) {
    // A producer warp is alone on its SM sub-partition, so nothing hides its load latency: every load of the thread's
    // tasks (tid, tid + 128) is issued before the first store, one wait per slice instead of one per task and tap.
    constexpr int NT = 2 * BN / 128;
    float4 v[NT][T + 3];                                      // task n: pixels 4q .. 4q + T + 2 of the window, channels 4 (i % 8) ..
#pragma unroll
    for (int n = 0; n < NT; ++n)
#pragma unroll
        for (int u = 0; u < T + 3; ++u) v[n][u] = tc::lds_f32x4(src + xt_src_offset(tid + 128 * n, 4 * xt_chunk(tid + 128 * n) + u, WROWS));
#pragma unroll
    for (int n = 0; n < NT; ++n) {
        const int i = tid + 128 * n;
#pragma unroll
        for (int t = 0; t < T; ++t) {
            const uint32_t d = dst + t * (BN * 128);
            const float4* w = v[n] + t;
            tc::sts_f32x4(d + xt_dst_offset(i, 0), w[0].x, w[1].x, w[2].x, w[3].x);
            tc::sts_f32x4(d + xt_dst_offset(i, 1), w[0].y, w[1].y, w[2].y, w[3].y);
            tc::sts_f32x4(d + xt_dst_offset(i, 2), w[0].z, w[1].z, w[2].z, w[3].z);
            tc::sts_f32x4(d + xt_dst_offset(i, 3), w[0].w, w[1].w, w[2].w, w[3].w);
        }
    }
}

// The consumer loop of both weight-gradient kernels, for one warpgroup: K slices first, first + step, ... < KI, each the
// dY fragments of its raw slot (aoff: dy_tile_offset of K step 0) against the T K-major B tiles (N channels each) of its
// stage.  One wgmma group stays in flight: the next slice's fragments load into the other register set while a slice's
// group runs, and the previous slice's stage is handed back once wgmma_wait<1> has retired its group.  The operand fences
// keep the retiring set's registers from being reused before then.
template <int N, int T, int STAGES, int NRAW, int RAW_BYTES, int STAGE_BYTES>
__device__ __forceinline__ void wgrad_consume(float (&acc)[T][N / 2], uint32_t raw_s, uint32_t stage_s, uint64_t* full,
                                              uint64_t* empty, uint64_t* rawfull, uint64_t* rawempty, const int (&aoff)[4],
                                              int first, int step, int KI, int tid, bool zero_first) {
    using Frag = uint32_t[BK / MMA_K][4];
    auto load = [&](Frag& f, int j) {
        const int rb = j % NRAW;
        tc::mbar_wait(rawfull + rb, (j / NRAW) & 1);
#pragma unroll
        for (int k = 0; k < BK / MMA_K; ++k)
#pragma unroll
            for (int e = 0; e < 4; ++e) f[k][e] = tc::lds_u32(raw_s + rb * RAW_BYTES + aoff[e] + k * 1024);
        __syncwarp();
        if ((tid & 31) == 0) tc::mbar_arrive(rawempty + rb);      // the loads are complete: TMA may refill the slot
    };
    auto slice = [&](int j, Frag& f, Frag& g) {              // f: slice j's fragments, g: the previous slice's
        const int st = j % STAGES;
        tc::mbar_wait(full + st, (j / STAGES) & 1);
        const uint32_t b = stage_s + st * STAGE_BYTES;
        tc::wgmma_fence();
#pragma unroll
        for (int t = 0; t < T; ++t)
#pragma unroll
            for (int k = 0; k < BK / MMA_K; ++k)
                tc::Wgmma<N>::mma_rs(acc[t], f[k], tc::desc_k128(b + t * (N * 128) + k * MMA_K * 4), (zero_first && j == first && k == 0) ? 0u : 1u);
        tc::wgmma_commit();
        tc::wgmma_wait<1>();
#pragma unroll
        for (int k = 0; k < BK / MMA_K; ++k)
#pragma unroll
            for (int e = 0; e < 4; ++e) tc::fence_operand(g[k][e]);
        if (j != first && tid == 0) tc::mbar_arrive(empty + (j - step) % STAGES);
        if (j + step < KI) load(g, j + step);
    };
    Frag f0, f1;
    if (first < KI) load(f0, first);
    for (int j = first; j < KI; j += 2 * step) {
        slice(j, f0, f1);
        if (j + step < KI) slice(j + step, f1, f0);
    }
    tc::wgmma_wait<0>();
#pragma unroll
    for (int k = 0; k < BK / MMA_K; ++k)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            tc::fence_operand(f0[k][e]);
            tc::fence_operand(f1[k][e]);
        }
#pragma unroll
    for (int t = 0; t < T; ++t)
#pragma unroll
        for (int i = 0; i < N / 2; ++i) tc::fence_operand(acc[t][i]);
    if (first < KI && tid == 0) tc::mbar_arrive(empty + (first + (KI - 1 - first) / step * step) % STAGES);
}

template <int BN, int STAGES, int NRAW, int T>
__global__ void __launch_bounds__(NTHREADS, 1)
wgrad_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_dy, const __grid_constant__ CUtensorMap tmap_x,
                   const WgradParams p, float* __restrict__ dw) {
    using S = WSmem<BN, STAGES, NRAW, T>;
    extern __shared__ unsigned char smem_raw[];
    unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    unsigned char* raw = base + STAGES * S::STAGE_BYTES;
    uint64_t* full = reinterpret_cast<uint64_t*>(raw + NRAW * S::RAW_BYTES);
    uint64_t* empty = full + STAGES;
    uint64_t* rawfull = empty + STAGES;
    uint64_t* rawempty = rawfull + NRAW;                  // dY fragments loaded: one arrival per consumer warp

    const int co0 = blockIdx.x * BM, ci0 = blockIdx.y * BN;
    const int gpr = p.kw / T;                             // tap groups per filter row
    const int groups = p.kh * gpr;
    const int grp = blockIdx.z % groups, split = blockIdx.z / groups;
    const int r = grp / gpr, s = grp % gpr;               // filter row and first tap of the group
    const int per_img = p.kx * p.ky;
    const long long ktotal = (long long)p.N * per_img;
    const long long k_lo = ktotal * split / p.splits, k_hi = ktotal * (split + 1) / p.splits;
    const int KI = (int)(k_hi - k_lo);
    // consumer warpgroups with output channels below Cout: the second one's 64 are all past it when Cout <= co0 + 64 (the
    // 64-channel layers of the generator), and it leaves at once instead of multiplying the zero-filled half of the dY tile
    const int nact = co0 + 64 < p.Cout ? 2 : 1;

    if (threadIdx.x == 0) {
        tc::tma_prefetch_desc(&tmap_dy);
        tc::tma_prefetch_desc(&tmap_x);
        for (int i = 0; i < STAGES; ++i) {
            tc::mbar_init(full + i, 128);
            tc::mbar_init(empty + i, nact);
        }
        for (int i = 0; i < NRAW; ++i) {
            tc::mbar_init(rawfull + i, 1);
            tc::mbar_init(rawempty + i, 4 * nact);
        }
        tc::fence_barrier_init();
    }
    __syncthreads();
    const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;

    // registers move from the producer (the window transpose holds up to 2 (T + 3) float4) to the consumers (T accumulators
    // and two sets of dY fragments); 128 * (168 - 80) >= 256 * (208 - 168)
    if (wg == 0) {
        tc::setmaxnreg_dec<80>();
        auto issue = [&](int j) {
            if (tid != 0) return;
            const long long k = k_lo + j;
            const int n = (int)(k / per_img), rem = (int)(k % per_img);
            const int x0 = (rem % p.kx) * p.BWk, y0 = (rem / p.kx) * p.BHk;
            const int rb = j % NRAW;
            unsigned char* dst = raw + rb * S::RAW_BYTES;
            tc::mbar_wait(rawempty + rb, ((j / NRAW) & 1) ^ 1);   // the consumers have loaded the dY fragments of slice j - NRAW
            // channels are split as (32, C/32) in the tensor maps: ONE 5-D box lands all 32-channel blocks back to back
            tc::mbar_arrive_expect_tx(rawfull + rb, S::DY_BYTES + S::RAW_X);
            tc::tma_load_5d(dst, &tmap_dy, rawfull + rb, 0, x0, y0, n, co0 / 32);
            tc::tma_load_5d(dst + S::DY_BYTES, &tmap_x, rawfull + rb, 0, p.st * x0 + s + p.xoff, p.st * y0 + r - p.pad_y, n, ci0 / 32);
        };
        for (int j = 0; j < NRAW - 1 && j < KI; ++j) issue(j);
        const uint32_t raw_s = tc::smem_u32(raw), base_s = tc::smem_u32(base);
        for (int it = 0; it < KI; ++it) {
            if (it + NRAW - 1 < KI) issue(it + NRAW - 1);     // its buffer was last read in iteration it - 1
            const int rb = it % NRAW, st = it % STAGES;
            tc::mbar_wait(rawfull + rb, (it / NRAW) & 1);
            tc::mbar_wait(empty + st, ((it / STAGES) & 1) ^ 1);
            wgrad_transpose<BN, T, S::WROWS>(raw_s + rb * S::RAW_BYTES + S::DY_BYTES, base_s + st * S::STAGE_BYTES, tid);
            tc::fence_proxy_async();
            tc::mbar_arrive(full + st);
            tc::named_sync(2, 128);                               // the raw X boxes are consumed before they are loaded again
        }
        return;
    }
    tc::setmaxnreg_inc<208>();

    const int h = wg - 1, lane = tid & 31;
    if (h >= nact) return;
    // this thread's fragment registers a[0..3] of K step 0 in the staged dY tile (K step k: + 1024 k)
    int aoff[4];
#pragma unroll
    for (int e = 0; e < 4; ++e)
        aoff[e] = dy_tile_offset(h * 64 + wgrad_row_co((tid >> 5) * 16 + (lane >> 2) + 8 * (e & 1)), (lane & 3) + 4 * (e >> 1));
    float acc[T][BN / 2];
#pragma unroll
    for (int t = 0; t < T; ++t)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[t][i] = 0.f;
    wgrad_consume<BN, T, STAGES, NRAW, S::RAW_BYTES, S::STAGE_BYTES>(acc, tc::smem_u32(raw), tc::smem_u32(base), full, empty, rawfull,
                                                                     rawempty, aoff, 0, 1, KI, tid, true);
    if (KI == 0) return;
    const int m_a = (tid >> 5) * 16 + (lane >> 2);                // this thread's accumulator rows m_a, m_a + 8
    const int cq = ci0 + 2 * (lane & 3);
#pragma unroll
    for (int t = 0; t < T; ++t) {
        const int sc = s + t * p.tstep;                       // filter column of accumulator t
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int co = co0 + h * 64 + wgrad_row_co(m_a + 8 * e);
            if (co >= p.Cout) continue;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int ci = cq + 8 * j;
                if (ci >= p.Cin) continue;                        // Cin % 32 == 0: ci + 1 < Cin as well
                const float v0 = acc[t][4 * j + 2 * e], v1 = acc[t][4 * j + 2 * e + 1];
                if (p.tapmajor) {
                    atomicAdd(reinterpret_cast<float2*>(dw + ((size_t)(r * p.kw + sc) * p.Cout + co) * p.Cin + ci), make_float2(v0, v1));
                } else {
                    atomicAdd(dw + (((size_t)co * p.Cin + ci) * p.kh + r) * p.kw + sc, v0);
                    atomicAdd(dw + (((size_t)co * p.Cin + ci + 1) * p.kh + r) * p.kw + sc, v1);
                }
            }
        }
    }
}

template <int BN, int STAGES, int NRAW, int T>
int launch_wgrad(const CUtensorMap& mdy, const CUtensorMap& mx, const WgradParams& p, float* dw, dim3 grid, cudaStream_t st) {
    using S = WSmem<BN, STAGES, NRAW, T>;
    static_assert(S::TOTAL <= 227 * 1024, "wgrad pipeline does not fit shared memory");
    B3D_CUDA_OK(cudaFuncSetAttribute(wgrad_wgmma_kernel<BN, STAGES, NRAW, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL));
    wgrad_wgmma_kernel<BN, STAGES, NRAW, T><<<grid, NTHREADS, S::TOTAL, st>>>(mdy, mx, p, dw);
    B3D_LAUNCH_OK();
    b3d::add_variant("wgrad_wgmma<%d,%d,%d,%d>", BN, STAGES, NRAW, T);
    return B3D_OK;
}

// ----------------------------------------------------------------------------------------------
// Stem wgrad from the RAW 8-channel input (fold_kh > 0): dW'[s][co][r*8 + ci] += sum dY[n,y,x,co] * X[n, y + r - pad_y, x + s, ci]
// — the weight gradient of the kh-folded stem (kh = 1, kw = 5 taps, Cin' = 64 folded channels) without the folded tensor.
// GEMM per tap s: M = 64 output channels, N = 64 folded channels (8 fold_kh real, the rest zero), K = output pixels in
// 32-pixel row segments.  One TMA box {8 ch, 36 px, fold_kh rows} of the raw input per K slice (TMA's zero fill = the y
// padding; the x padding is in the tensor) is expanded by the producer warpgroup into the five K-major B tiles of the
// slice (tap s = the window shifted by s pixels), so dY and X are each read once for all taps.  dY is the register A
// operand as in wgrad_wgmma_kernel (two 32-channel boxes).  The two consumer warpgroups take alternate K slices, each
// with five 64 x 64 accumulators over the whole 64-channel tile; both are reduced into dW by fp32 atomics.
// ----------------------------------------------------------------------------------------------
constexpr int STEM_KW = 5, STEM_STAGES = 4, STEM_NRAW = 3;
constexpr int STEM_BATCH = 3;                                         // producer expansion tasks whose loads are in flight together
struct StemSmem {
    static constexpr int DY_BYTES = 64 * BK * 4;
    static constexpr int WPX = BK + STEM_KW - 1;                       // raw pixels per K slice: 32 + 4
    static constexpr int RAW_X_MAX = 8 * WPX * 32;                     // fold_kh <= 8 rows of [36 px][8 ch]
    static constexpr int RAW_BYTES = (DY_BYTES + RAW_X_MAX + 1023) / 1024 * 1024;
    static constexpr int TILE_BYTES = 64 * BK * 4;                     // one tap's K-major [64 folded ch][32 px] tile
    static constexpr int STAGE_BYTES = STEM_KW * TILE_BYTES;
    static constexpr int TOTAL = STEM_STAGES * STAGE_BYTES + STEM_NRAW * RAW_BYTES + 1024 + 256;
};

__global__ void __launch_bounds__(NTHREADS, 1)
wgrad_stem_kernel(const __grid_constant__ CUtensorMap tmap_dy, const __grid_constant__ CUtensorMap tmap_x,
                  const WgradParams p, int fold_kh, float* __restrict__ dw) {
    using S = StemSmem;
    extern __shared__ unsigned char smem_raw[];
    unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    unsigned char* raw = base + STEM_STAGES * S::STAGE_BYTES;
    uint64_t* full = reinterpret_cast<uint64_t*>(raw + STEM_NRAW * S::RAW_BYTES);
    uint64_t* empty = full + STEM_STAGES;
    uint64_t* rawfull = empty + STEM_STAGES;
    uint64_t* rawempty = rawfull + STEM_NRAW;             // dY fragments loaded: one arrival per warp of the consumer

    const int co0 = blockIdx.x * 64, split = blockIdx.y;
    const int per_img = p.kx * p.ky;
    const long long ktotal = (long long)p.N * per_img;
    const long long k_lo = ktotal * split / p.splits, k_hi = ktotal * (split + 1) / p.splits;
    const int KI = (int)(k_hi - k_lo);
    const int creal = 8 * fold_kh;                        // folded channels that hold data
    const int xbytes = fold_kh * S::WPX * 32;

    if (threadIdx.x == 0) {
        tc::tma_prefetch_desc(&tmap_dy);
        tc::tma_prefetch_desc(&tmap_x);
        for (int i = 0; i < STEM_STAGES; ++i) {
            tc::mbar_init(full + i, 128);
            tc::mbar_init(empty + i, 1);
        }
        for (int i = 0; i < STEM_NRAW; ++i) {
            tc::mbar_init(rawfull + i, 1);
            tc::mbar_init(rawempty + i, 4);
        }
        tc::fence_barrier_init();
    }
    __syncthreads();
    const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;

    if (wg == 0) {
        tc::setmaxnreg_dec<56>();
        auto issue = [&](int j) {
            if (tid != 0) return;
            const long long k = k_lo + j;
            const int n = (int)(k / per_img), rem = (int)(k % per_img);
            const int x0 = (rem % p.kx) * BK, y0 = rem / p.kx;
            const int rb = j % STEM_NRAW;
            unsigned char* dst = raw + rb * S::RAW_BYTES;
            tc::mbar_wait(rawempty + rb, ((j / STEM_NRAW) & 1) ^ 1);
            tc::mbar_arrive_expect_tx(rawfull + rb, S::DY_BYTES + xbytes);
            tc::tma_load_5d(dst, &tmap_dy, rawfull + rb, 0, x0, y0, n, co0 / 32);
            tc::tma_load_4d(dst + S::DY_BYTES, &tmap_x, rawfull + rb, 0, x0, y0 - p.pad_y, n);
        };
        // the folded channels past creal are zero in every B tile: written once, never touched again
        for (int i = tid; i < STEM_STAGES * STEM_KW * (64 - creal) * 8; i += 128) {
            const int c = creal + (i >> 3) % (64 - creal), tile = (i >> 3) / (64 - creal);
            *reinterpret_cast<float4*>(base + tile * S::TILE_BYTES + c * 128 + (i & 7) * 16) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        for (int j = 0; j < STEM_NRAW - 1 && j < KI; ++j) issue(j);
        const int ntask = fold_kh * 8 * STEM_KW * 8;
        const uint32_t raw_s = tc::smem_u32(raw), base_s = tc::smem_u32(base);
        for (int it = 0; it < KI; ++it) {
            if (it + STEM_NRAW - 1 < KI) issue(it + STEM_NRAW - 1);
            const int rb = it % STEM_NRAW, st = it % STEM_STAGES;
            tc::mbar_wait(rawfull + rb, (it / STEM_NRAW) & 1);
            tc::mbar_wait(empty + st, ((it / STEM_STAGES) & 1) ^ 1);
            const uint32_t src = raw_s + rb * S::RAW_BYTES + S::DY_BYTES;       // [row][36 px][8 ch]
            const uint32_t dst = base_s + st * S::STAGE_BYTES;
            // task (r, q, s, ci), ci fastest: 16-byte chunk q (pixels 4q .. 4q + 3) of row c = 8r + ci of tap s's tile.  Eight
            // lanes of a store phase write chunks q ^ ci of eight rows (conflict-free); the reads of a warp's four (s, q)
            // groups start on pixels 4q + s, mostly different banks mod 4 pixels.  Shared-memory loads of STEM_BATCH tasks are
            // issued before their stores (the producer warp alone on its sub-partition would otherwise wait out each load).
            for (int i0 = tid; i0 < ntask; i0 += STEM_BATCH * 128) {
                float v[STEM_BATCH][4];
                uint32_t d[STEM_BATCH];
#pragma unroll
                for (int g = 0; g < STEM_BATCH; ++g) {
                    const int i = i0 + 128 * g;
                    if (i >= ntask) break;
                    const int ci = i & 7, u = i >> 3;
                    const int s = u % STEM_KW, q = (u / STEM_KW) & 7, r = u / (STEM_KW * 8);
                    const uint32_t a = src + ((r * S::WPX + 4 * q + s) * 8 + ci) * 4;
#pragma unroll
                    for (int e = 0; e < 4; ++e) v[g][e] = tc::lds_f32(a + 32 * e);
                    d[g] = dst + s * S::TILE_BYTES + (8 * r + ci) * 128 + ((q ^ ci) << 4);
                }
#pragma unroll
                for (int g = 0; g < STEM_BATCH; ++g) {
                    if (i0 + 128 * g >= ntask) break;
                    tc::sts_f32x4(d[g], v[g][0], v[g][1], v[g][2], v[g][3]);
                }
            }
            tc::fence_proxy_async();
            tc::mbar_arrive(full + st);
            tc::named_sync(2, 128);                               // the raw X box is consumed before it is loaded again
        }
        return;
    }
    tc::setmaxnreg_inc<224>();

    const int h = wg - 1, lane = tid & 31;
    int aoff[4];
#pragma unroll
    for (int e = 0; e < 4; ++e)
        aoff[e] = dy_tile_offset(wgrad_row_co((tid >> 5) * 16 + (lane >> 2) + 8 * (e & 1)), (lane & 3) + 4 * (e >> 1));
    float acc[STEM_KW][32];
#pragma unroll
    for (int t = 0; t < STEM_KW; ++t)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[t][i] = 0.f;
    static_assert(S::TILE_BYTES == 64 * 128, "a tap's B tile is 64 channel rows of 128 bytes");
    wgrad_consume<64, STEM_KW, STEM_STAGES, STEM_NRAW, S::RAW_BYTES, S::STAGE_BYTES>(acc, tc::smem_u32(raw), tc::smem_u32(base), full, empty,
                                                                                     rawfull, rawempty, aoff, h, 2, KI, tid, false);
    if (h >= KI) return;
    const int m_a = (tid >> 5) * 16 + (lane >> 2);
#pragma unroll
    for (int t = 0; t < STEM_KW; ++t) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int co = co0 + wgrad_row_co(m_a + 8 * e);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int ci = 8 * j + 2 * (lane & 3);
                if (ci >= creal) continue;                        // creal is even: ci + 1 < creal as well
                const float v0 = acc[t][4 * j + 2 * e], v1 = acc[t][4 * j + 2 * e + 1];
                if (p.tapmajor) {
                    atomicAdd(reinterpret_cast<float2*>(dw + ((size_t)t * p.Cout + co) * p.Cin + ci), make_float2(v0, v1));
                } else {
                    atomicAdd(dw + ((size_t)co * p.Cin + ci) * STEM_KW + t, v0);
                    atomicAdd(dw + ((size_t)co * p.Cin + ci + 1) * STEM_KW + t, v1);
                }
            }
        }
    }
}

// K splits of a weight-gradient grid of base_ctas CTAs per split (one CTA per SM): the count that minimises the modelled
// time  waves(s) * (ceil(K / s) + FIXED)  — a CTA's time is its share of the K slices plus a fixed cost (pipeline
// fill, the atomic epilogue), taken as 16 K slices; a partial last wave costs as much as a full one.  At least 8 K
// slices per CTA; ties go to the smaller count (fewer atomics).
int wgrad_splits(int base_ctas, long long ktotal) {
    constexpr long long FIXED = 16;
    const long long sms = tc::num_sms();
    long long smax = ktotal / 8;
    if (smax > 8 * sms) smax = 8 * sms;
    int best = 1;
    long long best_cost = -1;
    for (long long s = 1; s <= smax; ++s) {
        const long long cost = (base_ctas * s + sms - 1) / sms * ((ktotal + s - 1) / s + FIXED);
        if (best_cost < 0 || cost < best_cost) { best = (int)s; best_cost = cost; }
    }
    return best;
}

template <int BN, int STAGES, int KW = 1>
int launch_conv(const CUtensorMap& mx, const CUtensorMap& mw, const CUtensorMap& mm, const ConvParams& p, const float* bias, float* out,
                int tiles, cudaStream_t st) {
    using S = CSmem<BN, STAGES, KW>;
    static_assert(S::TOTAL <= 227 * 1024, "conv pipeline does not fit shared memory");
    B3D_CUDA_OK(cudaFuncSetAttribute(conv_wgmma_kernel<BN, STAGES, KW>, cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL));
    const int work = tiles * b3d::ceil_div(p.Cout, BN) * p.ncls;
    const int sms = tc::num_sms();
    conv_wgmma_kernel<BN, STAGES, KW><<<work < sms ? work : sms, NTHREADS, S::TOTAL, st>>>(mx, mw, mm, p, bias, out, tiles, work);
    B3D_LAUNCH_OK();
    if (KW > 1) b3d::add_variant("conv_wgmma_rowwin<%d,%d,%d>", BN, KW, STAGES);
    else b3d::add_variant("conv_wgmma<%d,%d>", BN, STAGES);
    return B3D_OK;
}

// row-window launch of a filter grid of rows of kw horizontally consecutive taps (stages: as many as fit ~200 KB)
template <int BN>
int launch_rowwin(int kw, const CUtensorMap& mx, const CUtensorMap& mw, const CUtensorMap& mm, const ConvParams& p, const float* bias,
                  float* out, int tiles, cudaStream_t st) {
    if (kw == 2) return launch_conv<BN, BN == 64 ? 5 : 4, 2>(mx, mw, mm, p, bias, out, tiles, st);
    if (kw == 3) return launch_conv<BN, BN == 64 ? 4 : 3, 3>(mx, mw, mm, p, bias, out, tiles, st);
    return launch_conv<BN, BN == 64 ? 3 : 2, 5>(mx, mw, mm, p, bias, out, tiles, st);
}

int pow2_floor(int v) {
    int p = 1;
    while (p * 2 <= v) p *= 2;
    return p;
}

}  // namespace

extern "C" {

// x   [N, H, W, Cin]  NHWC fp32, Cin % 32 == 0
// wt  [ntaps, Cout, Cin] fp32 (tap-major, K-major rows)
// out [N, OH, OW, OC]; the tile grid covers (Hout, Wout) logical outputs, written to (osy*y+ooy, osx*x+oox)
int b3d_conv2d_tf32(const float* x, const float* wt, const float* bias, float* out, int N, int H, int W, int Cin,
                    int Hout, int Wout, int Cout, int ntaps, const int* dy, const int* dx, int sy, int sx, int OH,
                    int OW, int OC, int osy, int osx, int ooy, int oox, float leaky, const int* wtap,
                    int wtaps_total, double* stats, int fold_kh, int fold_pad, const b3d_conv_opts* opts, void* stream) {
    B3D_REQUIRE(N > 0 && H > 0 && W > 0 && Hout > 0 && Wout > 0 && Cout > 0, B3D_EINVAL, "b3d_conv2d_tf32: bad sizes");
    B3D_REQUIRE(Cin > 0 && Cin % BK == 0, B3D_EINVAL, "b3d_conv2d_tf32: Cin=%d must be a multiple of %d", Cin, BK);
    B3D_REQUIRE(ntaps >= 1 && ntaps <= MAX_TAPS && dy && dx, B3D_EINVAL, "b3d_conv2d_tf32: bad taps");
    B3D_REQUIRE(x && wt && out, B3D_EINVAL, "b3d_conv2d_tf32: null pointer");
    B3D_REQUIRE(sy >= 1 && sy <= 2 && sx >= 1 && sx <= 2, B3D_EINVAL, "b3d_conv2d_tf32: stride must be 1 or 2");
    if (!wtap) wtaps_total = ntaps;
    B3D_REQUIRE(wtaps_total >= ntaps || wtap, B3D_EINVAL, "b3d_conv2d_tf32: bad weight tap count");
    for (int t = 0; wtap && t < ntaps; ++t)
        B3D_REQUIRE(wtap[t] >= 0 && wtap[t] < wtaps_total, B3D_EINVAL, "b3d_conv2d_tf32: weight tap %d out of range", wtap[t]);
    B3D_CHECK_ALIGNED(x);
    B3D_CHECK_ALIGNED(wt);
    b3d::clear_variant();

    const float* mask = opts ? opts->mask : nullptr;
    const float mslope = opts ? opts->mask_slope : 1.f;
    // the mask is read through a tensor map of the output's geometry: a 16-byte aligned base and 16-byte pixel strides
    B3D_REQUIRE(!mask || (reinterpret_cast<uintptr_t>(mask) % 16 == 0 && OC % 4 == 0), B3D_EINVAL,
                "b3d_conv2d_tf32: the mask needs a 16-byte aligned base and OC %% 4 == 0 (OC=%d)", OC);
    const int stats_sum = (opts && opts->stats_sum_only) ? 1 : 0;
    const int xpitch = (opts && opts->x_row_pitch) ? opts->x_row_pitch : W;
    // nclass > 1: the tap lists hold nclass groups of ntaps / nclass taps; class c writes at (class_ooy[c], class_oox[c])
    const int ncls = (opts && opts->nclass > 1) ? opts->nclass : 1;
    B3D_REQUIRE(ncls <= 4 && ntaps % ncls == 0 && (ncls == 1 || (sy == 1 && sx == 1 && fold_kh == 0)), B3D_EINVAL,
                "b3d_conv2d_tf32: nclass=%d needs <= 4 equal tap groups of a stride-1 launch", ncls);
    const int tpc = ntaps / ncls;                              // taps per class
    int cooy[4] = {ooy, ooy, ooy, ooy}, coox[4] = {oox, oox, oox, oox};
    for (int c = 0; c < ncls && ncls > 1; ++c) { cooy[c] = opts->class_ooy[c]; coox[c] = opts->class_oox[c]; }
    B3D_REQUIRE(xpitch >= W && (fold_kh == 0 || xpitch == W), B3D_EINVAL, "b3d_conv2d_tf32: x_row_pitch=%d must be >= W=%d (and absent with the on-the-fly fold)", xpitch, W);
    if (fold_kh > 0) {
        // x is the RAW stem input [N, H, W, 8]; the convolution is kh x kw with the kh rows folded into the K dimension:
        // Cin = 32 * ceil(8 kh / 32) "channels", taps = the kw horizontal ones (dy ignored), zero rows = the y padding
        B3D_REQUIRE(fold_kh <= 8 && Cin == 32 * ((8 * fold_kh + 31) / 32) && sy == 1 && sx == 1 && !wtap && Wout % BM == 0,
                    B3D_EINVAL, "b3d_conv2d_tf32: on-the-fly fold needs 8 input channels, stride 1 and Wout %% 128 == 0 (Wout=%d)", Wout);
    }
    // statistics are taken over the pixels the launch writes: the whole output when it is dense, or when four parity classes
    // at output stride 2 tile it (the forward of a 3x3 convolution of a x2-upsampled input, b3d/conv.py:_up_fprop)
    bool tiles = ncls == 4 && osy == 2 && osx == 2 && OH == 2 * Hout && OW == 2 * Wout;
    for (int c = 0, seen = 0; tiles && c < 4; ++c) {
        const int bit = 1 << (2 * cooy[c] + coox[c]);
        tiles = cooy[c] >= 0 && cooy[c] <= 1 && coox[c] >= 0 && coox[c] <= 1 && !(seen & bit);
        seen |= bit;
    }
    B3D_REQUIRE(!stats || mask || (osy == 1 && osx == 1) || tiles, B3D_EINVAL,
                "b3d_conv2d_tf32: statistics need a dense output, or four parity classes that tile it");
    // 256-wide output-channel tiles halve the input-tile bytes per FLOP through the L2 -> SM path when there are >= 256
    // output channels and enough work items to give every SM one.  Every launch of cfg3, cfg4 and cfg5 this rule gives
    // 256-wide tiles, timed against the same kernels forced to 128 (tools/time_conv128.py, H100 SXM, 700 W): 256 wins on
    // all such forwards (d1.conv4 at batch 64 0.92 vs 1.14 ms, d1.conv3 0.97 vs 1.00 ms, the cfg4 encoder's conv3e /
    // conv4e 0.14 / 0.12 vs 0.14 / 0.14 ms, blk4_tex.conv1 at batch 50 0.37 vs 0.43 ms) and on the 1x1 input gradients
    // (G.blk4.short 0.06 vs 0.07 ms); 128 wins on most 3x3 and stride-2 input gradients (G.blk3a 0.10 vs 0.12 ms,
    // d1.conv4 masked at batch 64 0.91 vs 0.95 ms).  Summed over those launches and cfg3's others 256 is ahead (17.5 vs
    // 18.0 ms), so the rule stays as it is.
    const bool bn256 = Cout % 256 == 0 && (long long)N * Hout * Wout / BM * (Cout / 256) * ncls >= tc::num_sms();
    const int BN = bn256 ? 256 : Cout > 64 ? 128 : 64;
    cudaStream_t st = (cudaStream_t)stream;
    CUtensorMap mw;
    {
        const uint64_t dims[3] = {(uint64_t)Cin, (uint64_t)Cout, (uint64_t)wtaps_total};
        const uint64_t strides[2] = {(uint64_t)Cin * 4, (uint64_t)Cout * Cin * 4};
        const uint32_t box[3] = {(uint32_t)BK, (uint32_t)BN, 1};
        if (int rc = tc::make_tmap_f32(&mw, wt, 3, dims, strides, box)) return rc;
    }

    // Filter-grid detection for the row window (stride 1, no fold): every class has kh rows of kw in {2, 3, 5} horizontally
    // consecutive taps (dx step +-1) whose weight taps form an arithmetic progression (step 1, or 2 for the stride-2
    // input gradient's parity classes), the same column pattern in every class.
    int g_kw = 0, g_step = 1, g_wstep = 1;
    if (sy == 1 && sx == 1 && fold_kh == 0) {
        int kw_ = 1;
        while (kw_ < tpc && dy[kw_] == dy[0]) ++kw_;
        const int step = kw_ > 1 ? dx[1] - dx[0] : 1;
        const int wstep = (wtap && kw_ > 1) ? wtap[1] - wtap[0] : 1;
        bool grid_ok = tpc % kw_ == 0 && (kw_ == 2 || kw_ == 3 || kw_ == 5) && (step == 1 || step == -1) && wstep >= 1 && wstep <= 2 &&
                       (ncls == 1 || wtap != nullptr);
        for (int t = 0; grid_ok && t < ntaps; ++t) {
            const int tc_ = t % tpc, t0 = t - tc_;
            grid_ok = dy[t] == dy[t0 + (tc_ / kw_) * kw_] && dx[t] == dx[0] + (tc_ % kw_) * step;
            if (wtap) grid_ok = grid_ok && wtap[t] == wtap[t0 + (tc_ / kw_) * kw_] + (tc_ % kw_) * wstep;
        }
        if (grid_ok && BN <= 128) { g_kw = kw_; g_step = step; g_wstep = wstep; }
    }

    // One launch covers output columns [xlo, xhi).  A width of "power of two + a few columns" (dgrad of an x-padded
    // input: 130, 66, 34 ...; stride-2 parity classes: 129, 65 ...) would leave a second, almost empty 128-pixel tile in
    // every row, so the remainder columns get a narrow strip launch of their own.
    auto run = [&](int xlo, int xhi) -> int {
        const int wspan = xhi - xlo;
        ConvParams p{};
        p.N = N; p.Hout = Hout; p.Wout = xhi; p.Cout = Cout; p.xbase = xlo;
        p.BW = pow2_floor(wspan < BM ? wspan : BM);
        p.BH = pow2_floor(Hout < BM / p.BW ? Hout : BM / p.BW);
        p.BI = BM / (p.BW * p.BH);
        p.tiles_x = b3d::ceil_div(wspan, p.BW);
        p.tiles_y = b3d::ceil_div(Hout, p.BH);
        const int tiles = p.tiles_x * p.tiles_y * b3d::ceil_div(N, p.BI);
        p.ntaps = tpc; p.kslices = Cin / BK; p.sy = sy; p.sx = sx; p.ncls = ncls;
        for (int t = 0; t < ntaps; ++t) { p.dy[t] = dy[t]; p.dx[t] = dx[t]; p.wtap[t] = wtap ? wtap[t] : t; }
        for (int c = 0; c < 4; ++c) { p.cooy[c] = cooy[c]; p.coox[c] = coox[c]; }
        p.OH = OH; p.OW = OW; p.OC = OC; p.osy = osy; p.osx = osx;
        p.leaky = leaky;
        p.stats = stats;
        p.mask = mask != nullptr; p.mslope = mslope; p.stats_sum = stats_sum;
        p.fold = fold_kh; p.fold_y0 = -fold_pad;
        {   // the epilogue addresses a tile's pixels relative to its first one in 32 bits
            const unsigned long long esn = p.BI > 1 ? (unsigned long long)OH * OW * OC : 0, esy = p.BH > 1 ? (unsigned long long)osy * OW * OC : 0,
                                     esx = (unsigned long long)osx * OC;
            B3D_REQUIRE((p.BI - 1) * esn + (p.BH - 1) * esy + (p.BW - 1) * esx + OC < (1ull << 32), B3D_EINVAL,
                        "b3d_conv2d_tf32: a %d x %d x %d pixel tile spans more than 2^32 elements of the output", p.BI, p.BH, p.BW);
            p.esn = (uint32_t)esn; p.esy = (uint32_t)esy; p.esx = (uint32_t)esx;
        }
        CUtensorMap mm{};                                      // the mask, with the output's geometry: one 32-channel chunk of a tile per box
        if (mask) {
            const uint64_t dims[4] = {(uint64_t)OC, (uint64_t)OW, (uint64_t)OH, (uint64_t)N};
            const uint64_t strides[3] = {(uint64_t)OC * 4, (uint64_t)OW * OC * 4, (uint64_t)OH * OW * OC * 4};
            const uint32_t box[4] = {(uint32_t)BK, (uint32_t)(osx * (p.BW - 1) + 1), (uint32_t)(osy * (p.BH - 1) + 1), (uint32_t)p.BI};
            const uint32_t es[4] = {1, (uint32_t)osx, (uint32_t)osy, 1};
            if (int rc = tc::make_tmap_f32(&mm, mask, 4, dims, strides, box, es)) return rc;
        }
        CUtensorMap mx;
        if (g_kw && wspan >= BM) {
            // row window: tiles are 128-pixel row segments (BW = 128, BH = BI = 1); one A box = 128 + kw - 1 pixels of a row,
            // one weight box = the kw weight tiles of a filter row (element stride g_wstep along the tap dimension)
            p.dx0 = g_step > 0 ? dx[0] : dx[g_kw - 1];
            for (int t = 0; t < g_kw; ++t) p.shift[t] = dx[t] - p.dx0;
            const uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)N};
            const uint64_t strides[3] = {(uint64_t)Cin * 4, (uint64_t)xpitch * Cin * 4, (uint64_t)H * xpitch * Cin * 4};
            const uint32_t box[4] = {(uint32_t)BK, (uint32_t)(BM + g_kw - 1), 1, 1};
            if (int rc = tc::make_tmap_f32(&mx, x, 4, dims, strides, box)) return rc;
            CUtensorMap mwr;
            const uint64_t wdims[3] = {(uint64_t)Cin, (uint64_t)Cout, (uint64_t)wtaps_total};
            const uint64_t wstrides[2] = {(uint64_t)Cin * 4, (uint64_t)Cout * Cin * 4};
            const uint32_t wbox[3] = {(uint32_t)BK, (uint32_t)BN, (uint32_t)((g_kw - 1) * g_wstep + 1)};
            const uint32_t wes[3] = {1, 1, (uint32_t)g_wstep};
            if (int rc = tc::make_tmap_f32(&mwr, wt, 3, wdims, wstrides, wbox, wes)) return rc;
            return BN == 128 ? launch_rowwin<128>(g_kw, mx, mwr, mm, p, bias, out, tiles, st)
                             : launch_rowwin<64>(g_kw, mx, mwr, mm, p, bias, out, tiles, st);
        }
        if (fold_kh > 0) {
            B3D_REQUIRE(p.BH == 1 && p.BI == 1, B3D_EINVAL, "b3d_conv2d_tf32: on-the-fly fold needs one-row tiles");
            const uint64_t dims[4] = {8, (uint64_t)W, (uint64_t)H, (uint64_t)N};                    // the raw NHWC tensor
            const uint64_t strides[3] = {32, (uint64_t)W * 32, (uint64_t)H * W * 32};
            const uint32_t box[4] = {8, (uint32_t)p.BW, 4, 1};                                     // 4 image rows per K slice
            if (int rc = tc::make_tmap_f32(&mx, x, 4, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_32B)) return rc;
        } else {
            const uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)N};
            const uint64_t strides[3] = {(uint64_t)Cin * 4, (uint64_t)xpitch * Cin * 4, (uint64_t)H * xpitch * Cin * 4};
            const uint32_t box[4] = {(uint32_t)BK, (uint32_t)(sx * (p.BW - 1) + 1), (uint32_t)(sy * (p.BH - 1) + 1), (uint32_t)p.BI};
            const uint32_t es[4] = {1, (uint32_t)sx, (uint32_t)sy, 1};
            if (int rc = tc::make_tmap_f32(&mx, x, 4, dims, strides, box, es)) return rc;
        }
        // ring depth: as many stages as fit next to the barrier area (~192 KB of operands)
        if (BN == 256) return launch_conv<256, 4>(mx, mw, mm, p, bias, out, tiles, st);
        if (BN == 128) return launch_conv<128, 6>(mx, mw, mm, p, bias, out, tiles, st);
        return launch_conv<64, 8>(mx, mw, mm, p, bias, out, tiles, st);
    };
    const int bw_full = pow2_floor(Wout < BM ? Wout : BM);
    const int rem = Wout % bw_full;
    if (rem != 0 && rem * 8 <= bw_full && Wout > bw_full) {
        const int rc = run(0, Wout - rem);
        return rc ? rc : run(Wout - rem, Wout);
    }
    return run(0, Wout);
}

// dy [N,Hout,Wout,Cout], x [N,H,W,Cin] NHWC (x already padded along x; Cin, Cout multiples of 32),
// dw [Cout,Cin,kh,kw] or tap-major [kh*kw,Cout,Cin] (accumulated into)
int b3d_conv2d_wgrad_tf32(const float* dy, const float* x, float* dw, int N, int H, int W, int Cin, int Hout, int Wout,
                          int Cout, int kh, int kw, int pad_y, int stride, int x_off, int tap_major, int fold_kh, int dy_row_pitch,
                          void* stream) {
    B3D_REQUIRE(N > 0 && Cin > 0 && Cout > 0 && H > 0 && W > 0 && Hout > 0 && Wout > 0, B3D_EINVAL,
                "b3d_conv2d_wgrad_tf32: bad sizes");
    // x_off < 0: the first taps of a row read left of x; TMA fills those columns with zeros
    B3D_REQUIRE(kh * kw <= MAX_TAPS && (stride == 1 || stride == 2) && x_off > -kw, B3D_EINVAL, "b3d_conv2d_wgrad_tf32: bad kernel/stride");
    B3D_REQUIRE(dy && x && dw, B3D_EINVAL, "b3d_conv2d_wgrad_tf32: null pointer");
    B3D_REQUIRE(Cin % 32 == 0 && Cout % 32 == 0, B3D_EINVAL,
                "b3d_conv2d_wgrad_tf32: Cin=%d and Cout=%d must be multiples of 32 (pad the channels with zeros)", Cin, Cout);
    B3D_CHECK_ALIGNED(dy);
    B3D_CHECK_ALIGNED(x);
    b3d::clear_variant();
    if (tap_major) B3D_CHECK_ALIGNED(dw);
    WgradParams p{};
    p.N = N; p.Hout = Hout; p.Wout = Wout; p.Cout = Cout; p.Cin = Cin;
    const uint64_t dpitch = dy_row_pitch > 0 ? dy_row_pitch : Wout;            // pixels per row of dy in memory
    B3D_REQUIRE(dpitch >= (uint64_t)Wout, B3D_EINVAL, "b3d_conv2d_wgrad_tf32: dy_row_pitch=%d must be >= Wout=%d", dy_row_pitch, Wout);
    cudaStream_t st = (cudaStream_t)stream;
    if (fold_kh > 0) {
        // raw 8-channel stem input: 32-pixel row segments of the output are the K slices
        B3D_REQUIRE(fold_kh > 4 && fold_kh <= 8 && Cin == 64 && kh == 1 && kw == STEM_KW && stride == 1 && x_off == 0 &&
                        Cout % 64 == 0 && W == Wout + STEM_KW - 1 && Hout == H + 2 * pad_y - fold_kh + 1,
                    B3D_EINVAL, "b3d_conv2d_wgrad_tf32: the raw-input stem weight gradient needs 4 < fold_kh <= 8 rows folded into "
                    "64 channels, a 1x5 stride-1 filter, Cout %% 64 == 0 and the x padding in the input");
        p.BWk = BK; p.BHk = 1;
        p.kx = b3d::ceil_div(Wout, BK);
        p.ky = Hout;
        p.kh = 1; p.kw = kw; p.pad_y = pad_y; p.st = 1; p.tapmajor = tap_major ? 1 : 0;
        p.splits = wgrad_splits(Cout / 64, (long long)N * p.kx * p.ky);
        CUtensorMap mdy, mx;
        {
            const uint64_t dims[5] = {32, (uint64_t)Wout, (uint64_t)Hout, (uint64_t)N, (uint64_t)Cout / 32};
            const uint64_t strides[4] = {(uint64_t)Cout * 4, dpitch * Cout * 4, (uint64_t)Hout * dpitch * Cout * 4, 128};
            const uint32_t box[5] = {32, (uint32_t)BK, 1, 1, 2};
            if (int rc = tc::make_tmap_f32(&mdy, dy, 5, dims, strides, box)) return rc;    // 128-byte swizzle: dy_tile_offset
        }
        {
            const uint64_t dims[4] = {8, (uint64_t)W, (uint64_t)H, (uint64_t)N};          // the raw NHWC tensor
            const uint64_t strides[3] = {32, (uint64_t)W * 32, (uint64_t)H * W * 32};
            const uint32_t box[4] = {8, (uint32_t)StemSmem::WPX, (uint32_t)fold_kh, 1};
            if (int rc = tc::make_tmap_f32(&mx, x, 4, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_NONE)) return rc;
        }
        B3D_CUDA_OK(cudaFuncSetAttribute(wgrad_stem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, StemSmem::TOTAL));
        wgrad_stem_kernel<<<dim3(Cout / 64, p.splits), NTHREADS, StemSmem::TOTAL, st>>>(mdy, mx, p, fold_kh, dw);
        B3D_LAUNCH_OK();
        b3d::add_variant("wgrad_stem<%d,%d,%d>", STEM_KW, STEM_STAGES, STEM_NRAW);
        return B3D_OK;
    }
    p.BWk = pow2_floor(Wout < BK ? Wout : BK);
    p.BHk = BK / p.BWk;
    p.kx = b3d::ceil_div(Wout, p.BWk);
    p.ky = b3d::ceil_div(Hout, p.BHk);
    p.kh = kh; p.kw = kw; p.pad_y = pad_y; p.st = stride; p.xoff = x_off; p.tapmajor = tap_major ? 1 : 0;
    const int BN = Cin > 64 ? 128 : 64;
    // a row of taps per CTA when the K slice is a 32-pixel row segment (Wout >= 32): the three taps of a 3x3 row at 64
    // input channels, the taps {0,2} / {1,3} of a 4-wide stride-2 row (adjacent pixels of its strided window).  T
    // accumulators of BN / 2 registers per thread must fit next to the rest (T * BN <= 256).
    int T = 1;
    p.tstep = 1;
    if (Wout >= BK) {
        if (stride == 1 && kw == 3 && BN == 64) T = 3;
        if (stride == 2 && kw == 4) { T = 2; p.tstep = 2; }
    }
    const int base_ctas = b3d::ceil_div(Cout, BM) * b3d::ceil_div(Cin, BN) * kh * (kw / T);
    const long long ktotal = (long long)N * p.kx * p.ky;
    const int splits = wgrad_splits(base_ctas, ktotal);
    p.splits = splits;

    CUtensorMap mdy, mx;
    {   // dims: (32 channels, W, H, N, channel block) — the block dim is outermost so that a box of BM/32 blocks is contiguous
        const uint64_t dims[5] = {32, (uint64_t)Wout, (uint64_t)Hout, (uint64_t)N, (uint64_t)Cout / 32};
        const uint64_t strides[4] = {(uint64_t)Cout * 4, dpitch * Cout * 4, (uint64_t)Hout * dpitch * Cout * 4, 128};
        const uint32_t box[5] = {32, (uint32_t)p.BWk, (uint32_t)p.BHk, 1, (uint32_t)(BM / 32)};
        if (int rc = tc::make_tmap_f32(&mdy, dy, 5, dims, strides, box)) return rc;    // 128-byte swizzle: dy_tile_offset
    }
    {
        const uint64_t dims[5] = {32, (uint64_t)W, (uint64_t)H, (uint64_t)N, (uint64_t)Cin / 32};
        const uint64_t strides[4] = {(uint64_t)Cin * 4, (uint64_t)W * Cin * 4, (uint64_t)H * W * Cin * 4, 128};
        const int wpx = T == 1 ? p.BWk : 36;                       // X pixels per slice: the K slice, or the window of T taps
        const uint32_t box[5] = {32, (uint32_t)(stride * (wpx - 1) + 1), (uint32_t)(stride * (p.BHk - 1) + 1), 1, (uint32_t)(BN / 32)};
        const uint32_t es[5] = {1, (uint32_t)stride, (uint32_t)stride, 1, 1};
        if (int rc = tc::make_tmap_f32(&mx, x, 5, dims, strides, box, es, CU_TENSOR_MAP_SWIZZLE_NONE)) return rc;
    }
    dim3 grid(b3d::ceil_div(Cout, BM), b3d::ceil_div(Cin, BN), kh * (kw / T) * splits);
    if (T == 3) return launch_wgrad<64, 3, 3, 3>(mdy, mx, p, dw, grid, st);
    if (T == 2) return BN == 128 ? launch_wgrad<128, 2, 3, 2>(mdy, mx, p, dw, grid, st) : launch_wgrad<64, 3, 3, 2>(mdy, mx, p, dw, grid, st);
    if (BN == 128) return launch_wgrad<128, 3, 3, 1>(mdy, mx, p, dw, grid, st);
    return launch_wgrad<64, 4, 4, 1>(mdy, mx, p, dw, grid, st);
}

}  // extern "C"
