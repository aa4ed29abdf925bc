// K8-beam: decoder cross-attention for beam search - the NQ beams of one window share one K / V stream (kv_div = beam size).
//
// One CTA = one (window, head): K then V of that head (Tlen x 64, 16-bit) stream once through a TMA ring (128-key tiles, 128B swizzle,
// rows past Tlen zero-filled by TMA) and serve all NQ queries.  The single-query kernel does its dot products on the FMA pipe, which is
// free there (one query: 2 flops per byte); with NQ = 5 queries per byte stream the same layout is instruction-bound (the first version of
// this kernel did it that way: 130 us per layer at 32 windows x 5 beams where the stream itself needs ~37 us; this one: 71 us, beam-5
// pass 515 -> 660 audio-s/s), so here both products run on the tensor cores with the queries as the 16-row A operand (rows >= NQ are zero):
//   scores = Q K^T      mma.sync m16n8k16, A = Q (hi + lo 16-bit split of the f32 query: two MMAs, ~16 mantissa bits),
//                       B = K tile rows straight from the swizzled ring with ldmatrix
//   out    = P V        A = P (f32 probabilities from smem, hi + lo split on the fly), B = V tile with ldmatrix.trans
// Softmax is exact two-pass over the f32 scores in shared memory (one warp per beam row, no block barriers inside).
// FP8 cache (FP8 = true): the TMA brings 64-byte rows of E4M3 codes, each consumer warp widens its rows exactly to 16-bit (mq_widen_fp8) and
// the MMA path is unchanged; the K row scale multiplies the scores, p carries the V row scale relative to the block's largest one.
// Packed bf16 cache (PK): the TMA brings the 96-byte primary slots, the consumers first copy the block's row headers to shared memory, and
// each warp rebuilds its rows' exact bf16 values into the same 16-bit buffer (mq_widen_packed; a raw row's last 32 bytes come from global
// memory - at most a few rows per tile).
// 4 consumer warps (each owns a quarter of every tile's keys) + 1 TMA producer warp; the K tiles do not depend on the upstream kernel
// (the cross K/V cache is written before the decode loop), so the producer starts before griddepcontrol.wait.
// Reference counterpart: the cross-attention inside TextDecoder.mlmodelc (Sources/WhisperKit/Core/TextDecoder.swift:394-417); beam
// semantics are the self-oracle's (oracle/beam_ref.py), the reference's own beam sampler being a stub (TokenSampler.swift:254-290).
#include <stdio.h>
#include <stdlib.h>

#include <type_traits>

#include "common.cuh"
#include "kernels.h"

namespace wk {

static constexpr int kMqThreads = 160;            // 4 consumer warps + 1 producer warp
static constexpr int kMqRows = 128;               // keys per tile
static constexpr int kMqStageBytes = kMqRows * 128;
static constexpr float kMqPScale = 1024.f;         // probabilities are carried as p * 2^10 through the P V product

__device__ __forceinline__ void mq_ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mq_ldsm_x4_trans(uint32_t addr, uint32_t (&r)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
// c (16 x 8, f32) += A (16 x 16: only rows 0..7 are non-zero, so a1 = a3 = 0) * B (16 x 8)
template <typename T> __device__ __forceinline__ void mq_mma(float (&c)[4], uint32_t a0, uint32_t a2, uint32_t b0, uint32_t b1);
template <> __device__ __forceinline__ void mq_mma<__nv_bfloat16>(float (&c)[4], uint32_t a0, uint32_t a2, uint32_t b0, uint32_t b1) {
    const uint32_t z = 0;
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a0), "r"(z), "r"(a2), "r"(z), "r"(b0), "r"(b1));
}
template <> __device__ __forceinline__ void mq_mma<__half>(float (&c)[4], uint32_t a0, uint32_t a2, uint32_t b0, uint32_t b1) {
    const uint32_t z = 0;
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a0), "r"(z), "r"(a2), "r"(z), "r"(b0), "r"(b1));
}
// x, y (f32) -> 16-bit pair hi and the 16-bit pair of what the rounding dropped: hi + lo carries ~16 mantissa bits through two MMAs
template <typename T> __device__ __forceinline__ void mq_split2(float x, float y, uint32_t& hi, uint32_t& lo) {
    hi = T16<T>::pack2(x, y);
    const float2 h = T16<T>::unpack2(hi);
    lo = T16<T>::pack2(x - h.x, y - h.y);
}

// FP8 cache: a warp widens its 32 rows of the E4M3 tile (rows 32 w .. 32 w + 31, the only rows its ldmatrix reads) exactly to 16-bit into
// its own 4 KiB buffer, in the 128B-swizzled layout the TMA gives the 16-bit tiles, so the MMA code below is the same for both caches
template <typename T>
__device__ __forceinline__ void mq_widen_fp8(const uint8_t* tile, uint8_t* wbuf, int warp, int lane) {
#pragma unroll 1
    for (int it = 0; it < 8; ++it) {
        const int idx = it * 32 + lane, row = idx >> 3, chunk = idx & 7;   // 8 codes -> 16-byte chunk `chunk` of the 16-bit row
        const uint2 u = *reinterpret_cast<const uint2*>(tile + (warp * 32 + row) * 64 + chunk * 8);
        uint32_t h[4];
        fp8x4_to_half2(u.x, h[0], h[1]);
        fp8x4_to_half2(u.y, h[2], h[3]);
        if constexpr (!std::is_same<T, __half>::value) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float2 a = T16<__half>::unpack2(h[k]);
                h[k] = T16<T>::pack2(a.x, a.y);
            }
        }
        *reinterpret_cast<uint4*>(wbuf + row * 128 + ((chunk ^ (row & 7)) << 4)) = make_uint4(h[0], h[1], h[2], h[3]);
    }
}

// Packed cache: a warp rebuilds its 32 rows of the tile (headers hdr[row of the tile]) into its 4 KiB buffer, same layout as mq_widen_fp8
__device__ __forceinline__ void mq_widen_packed(const uint8_t* tile, const uint8_t* hdr, const uint8_t* __restrict__ blk, int Tlen, int t0,
                                                uint8_t* wbuf, int warp, int lane) {
#pragma unroll 1
    for (int it = 0; it < 8; ++it) {
        const int idx = it * 32 + lane, row = idx >> 3, chunk = idx & 7, tr = warp * 32 + row;
        const uint8_t h = hdr[tr];
        const uint8_t* pr = tile + tr * kPackedRowBytes;
        uint4 u;
        if (h == kPackedRaw)
            u = chunk < 6 ? *reinterpret_cast<const uint4*>(pr + 16 * chunk)
                          : __ldg(reinterpret_cast<const uint4*>(blk + (long long)Tlen * kPackedRowBytes + (long long)(t0 + tr) * 32 + 16 * (chunk - 6)));
        else
            u = unpack_bf16x8(*reinterpret_cast<const uint2*>(pr + 8 * chunk), *reinterpret_cast<const uint32_t*>(pr + 64 + 4 * chunk), h);
        *reinterpret_cast<uint4*>(wbuf + row * 128 + ((chunk ^ (row & 7)) << 4)) = u;
    }
}

// F: 0 the 16-bit cache, 1 FP8, 2 packed bf16
template <typename T, int NQ, int STAGES, int F>
__global__ void __launch_bounds__(kMqThreads)
decoder_cross_attention_mq_kernel(const __grid_constant__ CUtensorMap tm_k, const __grid_constant__ CUtensorMap tm_v,
                                  const float* __restrict__ partial, int splits, int Bp, const float* __restrict__ bq, T* __restrict__ out, int H,
                                  int Tlen, int chunks, const int32_t* __restrict__ done, const float* __restrict__ kscale,
                                  const float* __restrict__ vscale, const uint8_t* __restrict__ kcross, const uint8_t* __restrict__ vcross,
                                  const uint8_t* __restrict__ khdr, const uint8_t* __restrict__ vhdr) {
    constexpr bool FP8 = F == 1, PK = F == 2, WIDE = FP8 || PK;
    constexpr int kStage = FP8 ? kMqRows * 64 : PK ? kMqRows * kPackedRowBytes : kMqStageBytes;   // bytes of one TMA tile
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* ring = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));   // STAGES x kStage
    const int Tp = chunks * kMqRows;
    float* scores = reinterpret_cast<float*>(ring + STAGES * kStage);          // [NQ][Tp]: raw scores, then probabilities
    float* sq = scores + NQ * Tp;                                              // [NQ][64]
    float* red = sq + NQ * 64;                                                 // [4][NQ][64]
    float* stat = red + 4 * NQ * 64;                                           // [NQ] 1 / row sum  (padded to 8)
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(stat + 8);
    uint64_t* empty_bar = full_bar + STAGES;
    // FP8 only: K / V row scales [Tp] each, the V-scale maximum (+ per-warp scratch), the widened 16-bit tiles [4 warps][32 rows][128 B]
    float* ksc = reinterpret_cast<float*>(empty_bar + STAGES);
    float* vsc = ksc + Tp;
    float* vmax_s = vsc + Tp;
    // packed: the widened tiles right after the barriers, then the K and V row headers [2][Tp] (rows past Tlen: 0)
    uint8_t* wbuf = PK ? reinterpret_cast<uint8_t*>(empty_bar + STAGES) : reinterpret_cast<uint8_t*>(vmax_s + 8);
    uint8_t* hdr_s = wbuf + 4 * 32 * 128;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int win = blockIdx.x / H, h = blockIdx.x % H;
    const int r0 = win * NQ;                 // first decode row of the window
    const int dm = H * 64;
    pdl_launch_dependents();
    // the group is skipped once all its rows have ended (beams end together; best-of samples one by one, and the rows a rung leaves
    // unused start ended)
    int ended = done != nullptr;
    if (done != nullptr)
#pragma unroll
        for (int j = 0; j < NQ; ++j) ended &= done[r0 + j] != 0;
    if (tid == 0) {
        tma_prefetch_desc(&tm_k);
        tma_prefetch_desc(&tm_v);
        for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 4); }
        fence_barrier_init();
    }
    __syncthreads();
    if (ended) { pdl_wait(); return; }   // (the wait still runs: this grid must not complete before its upstream does)
    if (warp == 4) {
        if (lane == 0) {
            for (int c = 0; c < 2 * chunks; ++c) {
                const int stage = c % STAGES;
                const uint32_t ph = (c / STAGES) & 1;
                mbar_wait_bounded(&empty_bar[stage], ph ^ 1);
                mbar_expect_tx(&full_bar[stage], kStage);
                tma_load_3d(ring + stage * kStage, c < chunks ? &tm_k : &tm_v, &full_bar[stage], 0, (c < chunks ? c : c - chunks) * kMqRows,
                            (int)blockIdx.x);
            }
        }
        return;
    }
    pdl_wait();                      // the q partials come from the upstream GEMM
    for (int i = tid; i < NQ * 64; i += 128) {
        const int j = i >> 6, e = i & 63;
        float q = bq[h * 64 + e];
        for (int s = 0; s < splits; ++s) q += partial[((long long)s * Bp + r0 + j) * dm + h * 64 + e];
        sq[i] = q * 0.125f;
    }
    if constexpr (FP8) {   // row scales of this (window, head); keys past Tlen get 0.  V scales are used relative to their maximum
        float vm = 0.f;
        for (int t = tid; t < Tp; t += 128) {
            ksc[t] = t < Tlen ? kscale[(long long)blockIdx.x * Tlen + t] : 0.f;
            vsc[t] = t < Tlen ? vscale[(long long)blockIdx.x * Tlen + t] : 0.f;
            vm = fmaxf(vm, vsc[t]);
        }
        vm = warp_max(vm);
        if (lane == 0) vmax_s[warp] = vm;
    }
    if constexpr (PK) {
        const long long hb = (long long)blockIdx.x * packed_hdr_stride(Tlen);
        for (int t = tid; t < Tp; t += 128) {
            hdr_s[t] = t < Tlen ? khdr[hb + t] : 0;
            hdr_s[Tp + t] = t < Tlen ? vhdr[hb + t] : 0;
        }
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    // FP8: p carries vsc[t] / vmax (at most 1, so the hi + lo split of p keeps its range) and the output is scaled back by vmax
    const float vmax = FP8 ? fmaxf(fmaxf(vmax_s[0], vmax_s[1]), fmaxf(vmax_s[2], vmax_s[3])) : 1.f;
    const float inv_vmax = vmax > 0.f ? 1.f / vmax : 0.f;
    const int g = lane >> 2, tq = lane & 3;          // fragment row (query) and column pair
    const int lm = lane >> 3, lr = lane & 7;         // ldmatrix: which of the four 8x8 matrices this lane addresses, and its row
    uint32_t qh[4][2], ql[4][2];                     // A fragments of Q per 16-wide k-step: columns 2tq.. and 8+2tq.., hi and lo halves
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int col = ks * 16 + half * 8 + 2 * tq;
            const float x = g < NQ ? sq[g * 64 + col] : 0.f, y = g < NQ ? sq[g * 64 + col + 1] : 0.f;
            mq_split2<T>(x, y, qh[ks][half], ql[ks][half]);
        }
    // ---- K phase: scores[j][t] = q_j . K[t]; warp w takes key groups 4w .. 4w+3 (8 keys each) of every tile
    for (int c = 0; c < chunks; ++c) {
        const int stage = c % STAGES;
        mbar_wait_bounded(&full_bar[stage], (c / STAGES) & 1);
        uint32_t tile = smem_u32(ring + stage * kStage);
        if constexpr (WIDE) {   // widen this warp's rows, release the stage, read the 16-bit copy (same row addressing)
            if constexpr (FP8) mq_widen_fp8<T>(ring + stage * kStage, wbuf + warp * 4096, warp, lane);
            else mq_widen_packed(ring + stage * kStage, hdr_s + c * kMqRows, kcross + (long long)blockIdx.x * Tlen * 128, Tlen, c * kMqRows,
                                 wbuf + warp * 4096, warp, lane);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[stage]);
            tile = smem_u32(wbuf + warp * 4096) - warp * 4096;
        }
#pragma unroll
        for (int gi = 0; gi < 4; ++gi) {
            const int kg = warp * 4 + gi;
            uint32_t b[2][4];
#pragma unroll
            for (int half = 0; half < 2; ++half)   // 16-byte chunks 4*half .. 4*half+3 of rows kg*8 .. +7 (physical chunk = logical ^ (row & 7))
                mq_ldsm_x4(tile + (kg * 8 + lr) * 128 + (((half * 4 + lm) ^ lr) << 4), b[half]);
            float cacc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                const uint32_t b0 = b[ks >> 1][(ks & 1) * 2], b1 = b[ks >> 1][(ks & 1) * 2 + 1];
                mq_mma<T>(cacc, qh[ks][0], qh[ks][1], b0, b1);
                mq_mma<T>(cacc, ql[ks][0], ql[ks][1], b0, b1);
            }
            if constexpr (FP8) {
                const int t = c * kMqRows + kg * 8 + 2 * tq;
                cacc[0] *= ksc[t]; cacc[1] *= ksc[t + 1];
            }
            if (g < NQ) *reinterpret_cast<float2*>(scores + g * Tp + c * kMqRows + kg * 8 + 2 * tq) = make_float2(cacc[0], cacc[1]);
        }
        __syncwarp();
        if (!WIDE && lane == 0) mbar_arrive(&empty_bar[stage]);
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    // ---- exact two-pass softmax, one warp per beam row; keys past Tlen (zero-filled K rows) get probability 0
    for (int j = warp; j < NQ; j += 4) {
        float* sc = scores + j * Tp;
        float mx = -INFINITY;
        for (int t = lane; t < Tlen; t += 32) mx = fmaxf(mx, sc[t]);
        mx = warp_max(mx);
        float sm = 0.f;
        for (int t = lane; t < Tlen; t += 32) {
            const float pr = __expf(sc[t] - mx);
            sc[t] = pr * kMqPScale;   // stored scaled: keeps the lo half of the 16-bit split out of the f16 subnormals (p ~ 1 / Tlen)
            sm += pr;
        }
        for (int t = Tlen + lane; t < Tp; t += 32) sc[t] = 0.f;
        sm = warp_sum(sm);
        if (lane == 0) stat[j] = (FP8 ? vmax : 1.f) / (sm * kMqPScale);
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    // ---- V phase: out_j[d] = sum_t p_j[t] V[t][d]; warp w takes k-steps 2w, 2w+1 (16 keys each) of every tile, all 64 output columns
    float acc[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[nt][e] = 0.f;
    for (int c = chunks; c < 2 * chunks; ++c) {
        const int stage = c % STAGES;
        mbar_wait_bounded(&full_bar[stage], (c / STAGES) & 1);
        uint32_t tile = smem_u32(ring + stage * kStage);
        if constexpr (WIDE) {   // widen this warp's rows, release the stage, read the 16-bit copy (same row addressing)
            if constexpr (FP8) mq_widen_fp8<T>(ring + stage * kStage, wbuf + warp * 4096, warp, lane);
            else mq_widen_packed(ring + stage * kStage, hdr_s + Tp + (c - chunks) * kMqRows, vcross + (long long)blockIdx.x * Tlen * 128, Tlen,
                                 (c - chunks) * kMqRows, wbuf + warp * 4096, warp, lane);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[stage]);
            tile = smem_u32(wbuf + warp * 4096) - warp * 4096;
        }
#pragma unroll
        for (int ki = 0; ki < 2; ++ki) {
            const int ks = warp * 2 + ki;
            const float* pr = scores + g * Tp + (c - chunks) * kMqRows + ks * 16 + 2 * tq;
            float2 p0 = g < NQ ? *reinterpret_cast<const float2*>(pr) : make_float2(0.f, 0.f);
            float2 p1 = g < NQ ? *reinterpret_cast<const float2*>(pr + 8) : make_float2(0.f, 0.f);
            if constexpr (FP8) {
                const float* vs = vsc + (c - chunks) * kMqRows + ks * 16 + 2 * tq;
                p0.x *= vs[0] * inv_vmax; p0.y *= vs[1] * inv_vmax; p1.x *= vs[8] * inv_vmax; p1.y *= vs[9] * inv_vmax;
            }
            uint32_t ah0, al0, ah2, al2;
            mq_split2<T>(p0.x, p0.y, ah0, al0);
            mq_split2<T>(p1.x, p1.y, ah2, al2);
#pragma unroll
            for (int np = 0; np < 4; ++np) {   // output column tiles 2np, 2np+1
                uint32_t bv[4];
                const int row = ks * 16 + (lm & 1) * 8 + lr;   // row & 7 == lr
                mq_ldsm_x4_trans(tile + row * 128 + (((np * 2 + (lm >> 1)) ^ lr) << 4), bv);
                mq_mma<T>(acc[2 * np], ah0, ah2, bv[0], bv[1]);
                mq_mma<T>(acc[2 * np], al0, al2, bv[0], bv[1]);
                mq_mma<T>(acc[2 * np + 1], ah0, ah2, bv[2], bv[3]);
                mq_mma<T>(acc[2 * np + 1], al0, al2, bv[2], bv[3]);
            }
        }
        __syncwarp();
        if (!WIDE && lane == 0) mbar_arrive(&empty_bar[stage]);
    }
    if (g < NQ) {
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) *reinterpret_cast<float2*>(red + (warp * NQ + g) * 64 + nt * 8 + 2 * tq) = make_float2(acc[nt][0], acc[nt][1]);
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    for (int i = tid; i < NQ * 64; i += 128) {
        const int j = i >> 6, e = i & 63;
        const float o = (red[(0 * NQ + j) * 64 + e] + red[(1 * NQ + j) * 64 + e] + red[(2 * NQ + j) * 64 + e] + red[(3 * NQ + j) * 64 + e]) * stat[j];
        out[(long long)(r0 + j) * dm + h * 64 + e] = T16<T>::from_f(o);
    }
}

// ------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiledMq)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                      const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                      CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

template <int NQ> static constexpr int mq_stages() { return NQ <= 5 ? 4 : 3; }
template <int NQ, int F> static size_t mq_smem_bytes(int chunks) {
    const size_t fp8_extra = F == 1 ? (size_t)2 * chunks * kMqRows * 4 + 8 * 4 + 4 * 32 * 128 : 0;   // row scales, V-scale maximum, widened tiles
    const size_t pk_extra = F == 2 ? (size_t)4 * 32 * 128 + 2 * chunks * kMqRows : 0;                // widened tiles, row headers
    const int stage = F == 1 ? kMqRows * 64 : F == 2 ? kMqRows * kPackedRowBytes : kMqStageBytes;
    return 1024 + (size_t)mq_stages<NQ>() * stage + (size_t)NQ * chunks * kMqRows * 4 + (size_t)NQ * 64 * 4 +
           (size_t)4 * NQ * 64 * 4 + 8 * 4 + 2 * mq_stages<NQ>() * 8 + fp8_extra + pk_extra + 64;
}

template <typename T, int NQ, int F>
static wk_status launch_mq(const CUtensorMap& tmk, const CUtensorMap& tmv, const float* partial, int splits, int Bp, const float* bq, void* out, int B, int H,
                           int Tlen, int chunks, const int32_t* done, const float* kscale, const float* vscale, const void* kcross, const void* vcross,
                           const uint8_t* khdr, const uint8_t* vhdr, cudaStream_t stream) {
    constexpr int ST = mq_stages<NQ>();
    const size_t smem = mq_smem_bytes<NQ, F>(chunks);
    if (smem > 227 * 1024) { set_error("decoder_cross_attention (beam): %d encoder positions do not fit shared memory", Tlen); return WK_ERR_INVALID_ARGUMENT; }
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(decoder_cross_attention_mq_kernel<T, NQ, ST, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
        if (e != cudaSuccess) { set_error("cudaFuncSetAttribute(cross mq): %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
        attr_set = true;
    }
    launch_k(decoder_cross_attention_mq_kernel<T, NQ, ST, F>, dim3((B / NQ) * H), dim3(kMqThreads), smem, stream, 4, tmk, tmv, partial, splits, Bp, bq, (T*)out, H,
             Tlen, chunks, done, kscale, vscale, (const uint8_t*)kcross, (const uint8_t*)vcross, khdr, vhdr);
    return WK_OK;
}

wk_status decoder_cross_attention_mq(const float* partial, int splits, int Bp, const float* bq, const void* kcross, const void* vcross, void* out, int B, int H,
                                     int Tlen, int dtype, cudaStream_t stream, const int32_t* done, int nq, const float* kscale,
                                     const float* vscale, const uint8_t* khdr, const uint8_t* vhdr) {
    if (nq < 2 || nq > 8 || B % nq != 0) { set_error("decoder_cross_attention (beam): %d rows, groups of %d", B, nq); return WK_ERR_INVALID_ARGUMENT; }
    static PFN_encodeTiledMq enc = nullptr;
    if (!enc) {
        void* fp = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
            set_error("cuTensorMapEncodeTiled entry point unavailable");
            return WK_ERR_CUDA;
        }
        enc = reinterpret_cast<PFN_encodeTiledMq>(fp);
    }
    const int chunks = (Tlen + kMqRows - 1) / kMqRows;
    const bool fp8 = kscale != nullptr, pk = khdr != nullptr;
    if (pk && (fp8 || dtype != WK_DTYPE_BF16 || !vhdr)) { set_error("decoder_cross_attention (beam): the packed cache is bf16 and needs both header vectors"); return WK_ERR_INVALID_ARGUMENT; }
    CUtensorMap tmk, tmv;
    // FP8: unswizzled 64-byte rows of codes; packed: unswizzled 96-byte primary slots in blocks of T x 128 bytes; both widened by the consumers
    const cuuint64_t row_bytes = fp8 ? 64 : pk ? kPackedRowBytes : 128;
    cuuint64_t gdim[3] = {pk ? (cuuint64_t)kPackedRowBytes : 64, (cuuint64_t)Tlen, (cuuint64_t)(B / nq) * H};
    cuuint64_t gstr[2] = {row_bytes, (cuuint64_t)Tlen * (pk ? 128 : row_bytes)};
    cuuint32_t box[3] = {pk ? (cuuint32_t)kPackedRowBytes : 64, (cuuint32_t)kMqRows, 1};
    cuuint32_t es[3] = {1, 1, 1};
    const CUtensorMapDataType dt = fp8 || pk ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : dtype == WK_DTYPE_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    const CUtensorMapSwizzle sw = fp8 || pk ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B;
    CUresult r = enc(&tmk, dt, 3, const_cast<void*>(kcross), gdim, gstr, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r == CUDA_SUCCESS)
        r = enc(&tmv, dt, 3, const_cast<void*>(vcross), gdim, gstr, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cross-attention tensor map encode failed: %d", (int)r); return WK_ERR_CUDA; }
    wk_status st = WK_OK;
#define WK_MQ_A(TT, N, F) launch_mq<TT, N, F>(tmk, tmv, partial, splits, Bp, bq, out, B, H, Tlen, chunks, done, kscale, vscale, kcross, vcross, khdr, vhdr, stream)
#define WK_MQ_T(N, F) (dtype == WK_DTYPE_F16 ? WK_MQ_A(__half, N, F) : WK_MQ_A(__nv_bfloat16, N, F))
#define WK_MQ(N) case N: st = pk ? WK_MQ_A(__nv_bfloat16, N, 2) : fp8 ? WK_MQ_T(N, 1) : WK_MQ_T(N, 0); break;
    switch (nq) { WK_MQ(2) WK_MQ(3) WK_MQ(4) WK_MQ(5) WK_MQ(6) WK_MQ(7) WK_MQ(8) default: break; }
#undef WK_MQ
#undef WK_MQ_T
#undef WK_MQ_A
    if (st != WK_OK) return st;
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("decoder_cross_attention (beam) launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

}  // namespace wk
