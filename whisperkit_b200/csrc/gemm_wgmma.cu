// Persistent warp-specialised wgmma GEMM for sm_90a.
//
//   D[rows, cols] = A[rows, K] * B[cols, K]^T      (both operands K-major, 16-bit, f32 accumulate in registers)
//
// One kernel serves every dense contraction of the Whisper hot path:
//   * encoder / cross-KV projections: A = activations (M = B*1500 rows), B = weights [N, K]; the cross-KV projection scatters head-major
//     16-bit rows, or (FP8 cache) E4M3 rows with one f32 scale each, quantized in the epilogue (gemm_epilogue_fp8_heads)
//   * conv stem as implicit GEMM: A is a 3-D tensor map, the 3 taps are extra K-blocks with a row shift
//   * decoder (M = batch <= 256): swap-AB, A = weights (128 output features per tile), B = activations,
//     split-K partials written transposed so the next fused reduce(+LN) kernel reads them coalesced.
//
// Structure (384 threads = 3 warpgroups, 1 CTA / SM, persistent over work items):
//   warpgroup 0   warp 0: TMA producer, cp.async.bulk.tensor (128B swizzle) into a ring of smem stages, mbarrier tx; warps 1-3 idle
//                 (the warpgroup gives its registers to the consumers with setmaxnreg)
//   warpgroups 1, 2  consumers: rows [64 * (wg - 1), +64) of the 128-row tile, wgmma m64nBNk16 from shared memory, the accumulator
//                 in registers, then the fused epilogue (see GemmEpi: TMA stores through a staging box, or stores from registers).
//                 A stage is released as soon as the wgmma group that read it has retired (wait_group 1 keeps one k-block of MMAs in
//                 flight).
// The WhisperKit reference has no counterpart source for this file: the contraction lives inside
// AudioEncoder.mlmodelc / TextDecoder.mlmodelc (Sources/WhisperKit/Core/AudioEncoder.swift:59-62,
// Sources/WhisperKit/Core/TextDecoder.swift:394-417).
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>
#include <type_traits>

#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace wk {

static constexpr int kBlockM = 128;
static constexpr int kBlockK = 64;   // 64 x 2 B = one 128-byte swizzle row
static constexpr int kStageA = kBlockM * kBlockK * 2;  // 16 KiB
static constexpr int kGemmThreads = 384;   // producer warpgroup + two consumer warpgroups
static constexpr int kMaxStages = 10;
static constexpr int kSmemMax = 227 * 1024;

struct GemmKParams {
    int tiles_per_batch, n_batches, tiles_n, splits, work;
    int kb_per_tap, kb_per_split, taps;
    int tap_row_shift[3];
    int tap_col_off[3];
    int a_is_3d;
    int m_rows_per_batch, n, bn;
    int stage_b_bytes, stages, store_bytes;
    int mode, gelu;
    void* out;
    long long ld_out, out_rows_per_batch, partial_cols;
    const float* bias;
    const float* pos;
    long long ld_pos;
    int heads_T, heads_B, heads_H, heads_dmodel;
    float* out_scale;
    uint8_t* out_hdr;
    int a_static;     // see GemmDesc::a_static
};

// How a GEMM leaves the accumulator (one kernel instantiation each):
//   kEpiPartialT  GEMM_OUT_PARTIAL_T, per-pair stores from the registers
//   kEpiFp8Heads  GEMM_OUT_FP8_HEADS, per-row quantization in registers (gemm_epilogue_fp8_heads)
//   kEpiStore16   GEMM_OUT_T16 / GEMM_OUT_T16_HEADS and kEpiStore32  GEMM_OUT_F32 / _F32_ADD / _F32_GELU_POS: the per-element math in
//                 registers, the tile through a shared-memory staging box and TMA bulk tensor stores (gemm_epilogue_store16 / _store32)
//   kEpiFp8Blocks GEMM_OUT_FP8_BLOCKS (FP8 kernel only), per-row block quantization in registers (gemm_epilogue_fp8_blocks)
//   kEpiPackedHeads GEMM_OUT_PACKED_HEADS, the packed bf16 rows from the registers (gemm_epilogue_packed_heads)
enum GemmEpi { kEpiPartialT = 0, kEpiFp8Heads = 1, kEpiStore16 = 2, kEpiStore32 = 3, kEpiFp8Blocks = 4, kEpiPackedHeads = 5 };
static int gemm_epi(int mode) {
    switch (mode) {
        case GEMM_OUT_PARTIAL_T: return kEpiPartialT;
        case GEMM_OUT_FP8_HEADS: return kEpiFp8Heads;
        case GEMM_OUT_PACKED_HEADS: return kEpiPackedHeads;
        case GEMM_OUT_T16: case GEMM_OUT_T16_HEADS: return kEpiStore16;
        default: return kEpiStore32;
    }
}

// Output staging of the TMA-store epilogues: per consumer warpgroup two boxes of 64 rows x 128 bytes (64 16-bit or 32 f32 columns),
// 128-byte swizzled like the output tensor map.  While one box drains to global memory the warpgroup fills the other; the consumers
// go on to the next work item's mainloop as soon as the last box of a tile is handed to TMA.
static constexpr int kStoreBox = 64 * 128;
static constexpr int kStoreBytes = 2 /*warpgroups*/ * 2 /*boxes*/ * kStoreBox;

// byte offset of 16-byte chunk `chunk` of row `row` in a 128-byte-swizzled box (16-byte chunk index XOR row % 8)
__device__ __forceinline__ uint32_t swz128(int row, int chunk) { return (uint32_t)(row * 128 + ((chunk ^ (row & 7)) << 4)); }

// hand staging box `box` to TMA after the warpgroup has written it.  Thread 0 of the warpgroup first waits until the previous box's
// store has read shared memory, so that the next chunk may overwrite that box once every thread has passed the barrier.
__device__ __forceinline__ void store_box_begin(int wg_tid, int cw) {
    fence_proxy_async();
    if (wg_tid == 0) bulk_wait_read_all();
    warpgroup_bar(1 + cw);
}

// GEMM_OUT_T16 / GEMM_OUT_T16_HEADS epilogue of one consumer warpgroup: rows [row0, row0 + 64) of batch `batch`, columns
// [col_base, col_base + BN).  Per 64-column chunk: bias, GELU and T16::pack2 in registers, stmatrix into the staging box, one TMA store.
// T16_HEADS: the chunk is one head; the output map is {64, T, blocks} over the [which][b][h][t][64] cache, so the chunk's 64 rows are one
// box at (0, t0, block), clipped at T.  When they run past the end of window b, the warpgroup copies rows [T - t0, 64) of the box to the
// start of block + H (window b + 1) with 16-byte stores: a TMA store box that starts at a negative row is an illegal instruction.
template <typename T, int BN>
__device__ __forceinline__ void gemm_epilogue_store16(const GemmKParams& p, const CUtensorMap* tmO, const float (&acc)[BN / 2],
                                                      uint8_t* stage, int& sbuf, int wg_tid, int cw, int batch, int row0, int col_base) {
    const int lane = wg_tid & 31;
    const int q = lane & 3;
    // stmatrix: lane l addresses row l % 8 of matrix l / 8; matrices (j, rows +0), (j, rows +8), (j + 1, +0), (j + 1, +8)
    const int mrow = 16 * (wg_tid >> 5) + 8 * ((lane >> 3) & 1) + (lane & 7);
    const int mj = lane >> 4;
    const bool heads = p.mode == GEMM_OUT_T16_HEADS;
    int hb = 0, ht0 = 0;
    bool straddle = false;
    if (heads) {
        hb = row0 / p.heads_T;
        ht0 = row0 - hb * p.heads_T;
        straddle = ht0 + 64 > p.heads_T && (hb + 1) * p.heads_T < p.m_rows_per_batch;
    }
#pragma unroll
    for (int c = 0; c < BN / 64; ++c) {
        const int col0 = col_base + 64 * c;
        if (col0 >= p.n) break;
        uint8_t* buf = stage + sbuf * kStoreBox;
        const uint32_t sb = smem_u32(buf);
#pragma unroll
        for (int jp = 0; jp < 4; ++jp) {
            uint32_t r[4];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int j = 8 * c + 2 * jp + h;
                const int col = col_base + 8 * j + 2 * q;
                float v0 = acc[4 * j], v1 = acc[4 * j + 1], v2 = acc[4 * j + 2], v3 = acc[4 * j + 3];
                if (p.bias && col < p.n) {
                    const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias + col));
                    v0 += bb.x; v1 += bb.y; v2 += bb.x; v3 += bb.y;
                }
                if (p.gelu) {
                    const float2 g0 = gelu_erf2(make_float2(v0, v1)), g1 = gelu_erf2(make_float2(v2, v3));
                    v0 = g0.x; v1 = g0.y; v2 = g1.x; v3 = g1.y;
                }
                r[2 * h] = T16<T>::pack2(v0, v1);
                r[2 * h + 1] = T16<T>::pack2(v2, v3);
            }
            stmatrix_x4(sb + swz128(mrow, 2 * jp + mj), r[0], r[1], r[2], r[3]);
        }
        store_box_begin(wg_tid, cw);
        int blk = 0;
        if (heads) {
            const int which = col0 / p.heads_dmodel;
            blk = (which * p.heads_B + hb) * p.heads_H + ((col0 - which * p.heads_dmodel) >> 6);
        }
        if (wg_tid == 0) {
            if (heads) tma_store_3d(tmO, buf, 0, ht0, blk);
            else tma_store_3d(tmO, buf, col0, row0, batch);
            bulk_commit();
        }
        if (straddle) {
            const int s = p.heads_T - ht0;
            uint8_t* dst = reinterpret_cast<uint8_t*>(p.out) + (long long)(blk + p.heads_H) * p.heads_T * 128;
            for (int i = wg_tid; i < (64 - s) * 8; i += 128) {
                const int r = s + (i >> 3), ch = i & 7;
                *reinterpret_cast<uint4*>(dst + (long long)(r - s) * 128 + ch * 16) = *reinterpret_cast<const uint4*>(buf + swz128(r, ch));
            }
        }
        sbuf ^= 1;
    }
}

// GEMM_OUT_F32 / GEMM_OUT_F32_ADD / GEMM_OUT_F32_GELU_POS epilogue of one consumer warpgroup, per 32-column chunk.  F32_ADD: the chunk of
// the residual x was TMA-loaded into the staging box (chunks 0 and 1 during the tile's mainloop, chunk c + 1 while chunk c is being
// computed); each thread reads its x from the box and writes x + (acc + bias) back in place before the box is stored.
template <int BN>
__device__ __forceinline__ void gemm_epilogue_store32(const GemmKParams& p, const CUtensorMap* tmO, const float (&acc)[BN / 2],
                                                      uint8_t* stage, uint64_t* rbar, int& sbuf, uint32_t& rphase, int wg_tid, int cw,
                                                      int batch, int row0, int col_base) {
    const int lane = wg_tid & 31;
    const int q = lane & 3;
    const int r_top = 16 * (wg_tid >> 5) + (lane >> 2);   // and r_top + 8 (same row % 8, so the same swizzle)
    const bool add = p.mode == GEMM_OUT_F32_ADD, pos = p.mode == GEMM_OUT_F32_GELU_POS;
#pragma unroll
    for (int c = 0; c < BN / 32; ++c) {
        const int col0 = col_base + 32 * c;
        if (col0 >= p.n) break;
        uint8_t* buf = stage + sbuf * kStoreBox;
        if (add) {
            if (wg_tid == 0 && c >= 1 && c + 1 < BN / 32 && col0 + 32 < p.n) {
                bulk_wait_read_all();   // the other box's store (chunk c - 1) has left shared memory
                mbar_expect_tx(&rbar[sbuf ^ 1], kStoreBox);
                tma_load_3d(stage + (sbuf ^ 1) * kStoreBox, tmO, &rbar[sbuf ^ 1], col0 + 32, row0, batch);
            }
            mbar_wait(&rbar[sbuf], (rphase >> sbuf) & 1u);
            rphase ^= 1u << sbuf;
        }
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
            const int j = 4 * c + jj;
            const int col = col_base + 8 * j + 2 * q;
            float v[4] = {acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]};
            if (p.bias && col < p.n) {
                const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias + col));
                v[0] += bb.x; v[1] += bb.y; v[2] += bb.x; v[3] += bb.y;
            }
            if (p.gelu) {
                const float2 g0 = gelu_erf2(make_float2(v[0], v[1])), g1 = gelu_erf2(make_float2(v[2], v[3]));
                v[0] = g0.x; v[1] = g0.y; v[2] = g1.x; v[3] = g1.y;
            }
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const int r = r_top + 8 * half;
                float2* s = reinterpret_cast<float2*>(buf + swz128(r, 2 * jj + (q >> 1)) + (q & 1) * 8);
                float2 o = make_float2(v[2 * half], v[2 * half + 1]);
                if (add) {
                    const float2 x = *s;
                    o = make_float2(x.x + o.x, x.y + o.y);
                } else if (pos) {
                    const int row_in_batch = row0 + r;
                    if (row_in_batch < p.m_rows_per_batch && col < p.n) {
                        const float2 pp = __ldg(reinterpret_cast<const float2*>(p.pos + (long long)row_in_batch * p.ld_pos + col));
                        o = make_float2(o.x + pp.x, o.y + pp.y);
                    }
                }
                *s = o;
            }
        }
        store_box_begin(wg_tid, cw);
        if (wg_tid == 0) {
            tma_store_3d(tmO, buf, col0, row0, batch);
            bulk_commit();
        }
        sbuf ^= 1;
    }
}

// GEMM_OUT_FP8_HEADS epilogue of one thread: rows r_lo and r_lo + 8, columns 8 j + c_lo, + 1.  The 64 columns of a head are j = 8 hh ..
// 8 hh + 7 of the 4 lanes of a quad (16 values each), so the row's amax is two quad shuffles; every lane then encodes its 16 values and
// the lane with c_lo == 0 stores the row's scale.  Rows past the tile's valid rows take part in the shuffles but store nothing.
template <int BN>
__device__ __forceinline__ void gemm_epilogue_fp8_heads(const GemmKParams& p, int batch, int tile_row0, int r_lo, int c_lo, int col_base,
                                                        const float (&acc)[BN / 2]) {
    static_assert(BN % 64 == 0, "FP8 heads epilogue needs head-aligned N tiles");
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const int row_in_batch = tile_row0 + r_lo + 8 * half;
        const long long grow = (long long)batch * p.out_rows_per_batch + row_in_batch;
        const int b = (int)(grow / p.heads_T);
        const int tt = (int)(grow - (long long)b * p.heads_T);
#pragma unroll
        for (int hh = 0; hh < BN / 64; ++hh) {
            const int col0 = col_base + hh * 64;   // n is a multiple of 64: a head is wholly inside or wholly past n
            const bool col_ok = col0 < p.n;
            float v[16];
            float amax = 0.f;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                const int j = hh * 8 + jj;
                float v0 = acc[4 * j + 2 * half], v1 = acc[4 * j + 2 * half + 1];
                if (p.bias && col_ok) {
                    const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias + col0 + 8 * jj + c_lo));
                    v0 += bb.x; v1 += bb.y;
                }
                v[2 * jj] = v0; v[2 * jj + 1] = v1;
                amax = fmaxf(amax, fmaxf(fabsf(v0), fabsf(v1)));
            }
            amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
            amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
            if (!col_ok || row_in_batch >= p.m_rows_per_batch) continue;
            const int which = col0 / p.heads_dmodel;
            const int h = (col0 - which * p.heads_dmodel) >> 6;
            const long long row = (((long long)which * p.heads_B + b) * p.heads_H + h) * p.heads_T + tt;
            const float s = fp8_row_scale(amax);
            uint8_t* o = reinterpret_cast<uint8_t*>(p.out) + row * 64 + c_lo;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
                *reinterpret_cast<uint16_t*>(o + 8 * jj) = (uint16_t)(fp8_encode(v[2 * jj], s) | (fp8_encode(v[2 * jj + 1], s) << 8));
            if (c_lo == 0) p.out_scale[row] = s;
        }
    }
}

// GEMM_OUT_PACKED_HEADS epilogue of one thread, same fragments as gemm_epilogue_fp8_heads: acc + bias rounded to bf16 as the T16 heads
// path rounds it, the row's exponent range from quad shuffles, then the packed row (common.cuh): lane q holds values 8 jj + 2q, + 1 of every
// group jj, so it writes their two sign|mantissa bytes and, once the quad has OR-ed its nibbles together, the nibble words of groups 2q, 2q + 1
template <int BN>
__device__ __forceinline__ void gemm_epilogue_packed_heads(const GemmKParams& p, int batch, int tile_row0, int r_lo, int c_lo, int col_base,
                                                           const float (&acc)[BN / 2]) {
    static_assert(BN % 64 == 0, "packed heads epilogue needs head-aligned N tiles");
    const int q = c_lo >> 1;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const int row_in_batch = tile_row0 + r_lo + 8 * half;
        const long long grow = (long long)batch * p.out_rows_per_batch + row_in_batch;
        const int b = (int)(grow / p.heads_T);
        const int tt = (int)(grow - (long long)b * p.heads_T);
#pragma unroll
        for (int hh = 0; hh < BN / 64; ++hh) {
            const int col0 = col_base + hh * 64;
            const bool col_ok = col0 < p.n;
            uint32_t w[8];
            uint32_t emax = 0, emin = 255;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                const int j = hh * 8 + jj;
                float v0 = acc[4 * j + 2 * half], v1 = acc[4 * j + 2 * half + 1];
                if (p.bias && col_ok) {
                    const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias + col0 + 8 * jj + c_lo));
                    v0 += bb.x; v1 += bb.y;
                }
                w[jj] = T16<__nv_bfloat16>::pack2(v0, v1);
                const uint32_t e0 = (w[jj] >> 7) & 0xffu, e1 = (w[jj] >> 23) & 0xffu;
                emax = max(emax, max(e0, e1));
                emin = min(emin, min(e0, e1));
            }
            emax = max(emax, __shfl_xor_sync(0xffffffffu, emax, 1));
            emax = max(emax, __shfl_xor_sync(0xffffffffu, emax, 2));
            emin = min(emin, __shfl_xor_sync(0xffffffffu, emin, 1));
            emin = min(emin, __shfl_xor_sync(0xffffffffu, emin, 2));
            const bool raw = emax == 255u || emax - emin > 15u;   // uniform over the quad
            uint32_t nib[8];
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                nib[jj] = raw ? 0u : ((emax - ((w[jj] >> 7) & 0xffu)) << (4 * q)) | ((emax - ((w[jj] >> 23) & 0xffu)) << (16 + 4 * q));
                nib[jj] |= __shfl_xor_sync(0xffffffffu, nib[jj], 1);
                nib[jj] |= __shfl_xor_sync(0xffffffffu, nib[jj], 2);
            }
            if (!col_ok || row_in_batch >= p.m_rows_per_batch) continue;
            const int which = col0 / p.heads_dmodel;
            const int h = (col0 - which * p.heads_dmodel) >> 6;
            const long long blk = ((long long)which * p.heads_B + b) * p.heads_H + h;
            uint8_t* base = reinterpret_cast<uint8_t*>(p.out) + blk * p.heads_T * 128;
            uint8_t* row = base + (long long)tt * kPackedRowBytes;
            if (raw) {
#pragma unroll
                for (int jj = 0; jj < 8; ++jj) {
                    uint8_t* dst = jj < 6 ? row + 16 * jj + 2 * c_lo : base + (long long)p.heads_T * kPackedRowBytes + (long long)tt * 32 + 16 * (jj - 6) + 2 * c_lo;
                    *reinterpret_cast<uint32_t*>(dst) = w[jj];
                }
            } else {
#pragma unroll
                for (int jj = 0; jj < 8; ++jj) {   // sign|mantissa bytes of values 8 jj + c_lo, + 1
                    const uint32_t lo = ((w[jj] >> 8) & 0x80u) | (w[jj] & 0x7fu), hi = ((w[jj] >> 24) & 0x80u) | ((w[jj] >> 16) & 0x7fu);
                    *reinterpret_cast<uint16_t*>(row + 8 * jj + c_lo) = (uint16_t)(lo | (hi << 8));
                }
#pragma unroll
                for (int jj = 0; jj < 8; jj += 2)
                    if ((jj >> 1) == q) *reinterpret_cast<uint2*>(row + 64 + 4 * jj) = make_uint2(nib[jj], nib[jj + 1]);
            }
            if (c_lo == 0) p.out_hdr[blk * packed_hdr_stride(p.heads_T) + tt] = raw ? kPackedRaw : (uint8_t)emax;
        }
    }
}

template <typename T, int BN, int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmO,
                  const GemmKParams p) {
    constexpr bool kStore = EPI == kEpiStore16 || EPI == kEpiStore32;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // manual 1024-byte alignment (SWIZZLE_128B atoms are 1024 B)
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int stage_bytes = kStageA + p.stage_b_bytes;
    uint8_t* store_stage = smem + (size_t)p.stages * stage_bytes;   // kStoreBytes for the TMA-store epilogues, else nothing
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(store_stage + p.store_bytes);
    uint64_t* empty_bar = full_bar + kMaxStages;
    uint64_t* res_bar = empty_bar + kMaxStages;   // [warpgroup][box]: F32_ADD residual loads

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    pdl_launch_dependents();   // the next kernel may start its prologue; it still waits for our completion

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        if (kStore) tma_prefetch_desc(&tmO);
        for (int i = 0; i < p.stages; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 8);   // one arrive per consumer warp
        }
        for (int i = 0; i < 4; ++i) mbar_init(&res_bar[i], 1);
        fence_barrier_init();
    }
    __syncthreads();
    // upstream results visible from here on.  With a static A operand the producer warp waits later, after it has put the first weight
    // tiles in flight; every other warp only sees data that arrived after that wait.
    const bool early_a = p.a_static != 0;
    if (!(early_a && warp == 0)) pdl_wait();

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp != 0) return;
        // ===================== TMA producer =====================
        // the whole warp runs this converged; the TMA / mbarrier instructions are predicated on the elect.sync lane (common.cuh)
        int stage = 0;
        uint32_t phase = 0;
        bool need_wait = early_a;
        auto issue = [&](int kb, int st, int row0, int batch, int n_tile, bool do_a, bool do_b) {
            const int tap = kb / p.kb_per_tap;
            const int kk = kb - tap * p.kb_per_tap;
            uint8_t* sa = smem + (size_t)st * stage_bytes;
            uint8_t* sb = sa + kStageA;
            if (do_a) {
                mbar_expect_tx_elect(&full_bar[st], (uint32_t)stage_bytes);
                const int ac0 = p.tap_col_off[tap] + kk * kBlockK;
                const int ar = row0 + p.tap_row_shift[tap];
                if (p.a_is_3d) tma_load_3d_elect(sa, &tmA, &full_bar[st], ac0, ar, batch);
                else tma_load_2d_elect(sa, &tmA, &full_bar[st], ac0, ar);
            }
            if (do_b) tma_load_2d_elect(sb, &tmB, &full_bar[st], kb * kBlockK, n_tile * BN);
        };
        for (int w = blockIdx.x; w < p.work; w += gridDim.x) {
            const int split = w % p.splits;
            const int t = w / p.splits;
            const int n_tile = t % p.tiles_n;
            const int m_tile = t / p.tiles_n;
            const int batch = m_tile / p.tiles_per_batch;
            const int row0 = (m_tile % p.tiles_per_batch) * kBlockM;
            const int kb0 = split * p.kb_per_split;
            int kb = kb0;
            if (need_wait) {
                // first work item, fresh ring: weight tiles go out before griddepcontrol.wait, activation tiles after it
                const int n_pre = p.kb_per_split < p.stages ? p.kb_per_split : p.stages;
                for (int i = 0; i < n_pre; ++i) issue(kb0 + i, i, row0, batch, n_tile, true, false);
                pdl_wait();
                for (int i = 0; i < n_pre; ++i) issue(kb0 + i, i, row0, batch, n_tile, false, true);
                kb = kb0 + n_pre;
                if (n_pre == p.stages) { stage = 0; phase ^= 1; } else stage = n_pre;
                need_wait = false;
            }
            for (; kb < kb0 + p.kb_per_split; ++kb) {
                mbar_wait(&empty_bar[stage], phase ^ 1);
                __syncwarp();
                issue(kb, stage, row0, batch, n_tile, true, true);
                if (++stage == p.stages) { stage = 0; phase ^= 1; }
            }
        }
        if (need_wait) pdl_wait();
        return;
    }

    // ===================== consumer warpgroups =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int cw = (warp >> 2) - 1;                       // 0 / 1: rows [64 cw, 64 cw + 64) of the tile
    const int wg_tid = threadIdx.x & 127;
    const int r_lo = cw * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's rows: r_lo and r_lo + 8
    const int c_lo = 2 * (lane & 3);                      // and columns 8 j + c_lo, + 1
    uint8_t* my_stage = store_stage + cw * 2 * kStoreBox;
    uint64_t* my_res_bar = res_bar + 2 * cw;
    int sbuf = 0;            // staging box the next chunk goes to
    uint32_t rphase = 0;     // parity of my_res_bar[0 / 1]
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
    for (int w = blockIdx.x; w < p.work; w += gridDim.x) {
        const int split = w % p.splits;
        const int t = w / p.splits;
        const int n_tile = t % p.tiles_n;
        const int m_tile = t / p.tiles_n;
        const int batch = m_tile / p.tiles_per_batch;
        const int tile_row0 = (m_tile % p.tiles_per_batch) * kBlockM;
        const int col_base = n_tile * BN;
        const int wg_row0 = tile_row0 + 64 * cw;         // this warpgroup's first row (in its batch)
        const bool wg_rows = wg_row0 < p.m_rows_per_batch;

        int prev = -1;
        for (int kb = 0; kb < p.kb_per_split; ++kb) {
            mbar_wait(&full_bar[stage], phase);
            const uint32_t sa = smem_u32(smem + (size_t)stage * stage_bytes);
            const uint64_t adesc = wgmma_desc_sw128(sa + cw * 64 * 128);
            const uint64_t bdesc = wgmma_desc_sw128(sa + kStageA);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < kBlockK / 16; ++k)   // +32 bytes per 16 K elements inside the swizzle row (>> 4 -> +2k)
                Wgmma<T, BN>::ss(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (kb > 0 || k > 0) ? 1u : 0u);
            wgmma_commit();
            if (EPI == kEpiStore32 && kb == 0 && p.mode == GEMM_OUT_F32_ADD && wg_tid == 0 && wg_rows) {
                // residual chunks 0 and 1 of this tile, fetched while the MMAs run; the boxes are free once the previous tile's stores
                // have read them
                bulk_wait_read_all();
                for (int c = 0; c < 2 && c < BN / 32 && col_base + 32 * c < p.n; ++c) {
                    const int b = sbuf ^ c;
                    mbar_expect_tx(&my_res_bar[b], kStoreBox);
                    tma_load_3d(my_stage + b * kStoreBox, &tmO, &my_res_bar[b], col_base + 32 * c, wg_row0, batch);
                }
            }
            wgmma_wait<1>();   // the MMAs of the previous k-block have retired: its stage may be refilled
            if (prev >= 0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty_bar[prev]);
            }
            prev = stage;
            if (++stage == p.stages) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);

        if constexpr (EPI == kEpiFp8Heads) {
            gemm_epilogue_fp8_heads<BN>(p, batch, tile_row0, r_lo, c_lo, col_base, acc);
        } else if constexpr (EPI == kEpiPackedHeads) {
            gemm_epilogue_packed_heads<BN>(p, batch, tile_row0, r_lo, c_lo, col_base, acc);
        } else if constexpr (EPI == kEpiStore16) {
            if (wg_rows) gemm_epilogue_store16<T, BN>(p, &tmO, acc, my_stage, sbuf, wg_tid, cw, batch, wg_row0, col_base);
        } else if constexpr (EPI == kEpiStore32) {
            if (wg_rows) gemm_epilogue_store32<BN>(p, &tmO, acc, my_stage, my_res_bar, sbuf, rphase, wg_tid, cw, batch, wg_row0, col_base);
        } else {
            // GEMM_OUT_PARTIAL_T: out32[split][col][row] = acc, columns past partial_cols dropped
            float* o = reinterpret_cast<float*>(p.out);
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const int row_in_batch = tile_row0 + r_lo + 8 * half;
                if (row_in_batch >= p.m_rows_per_batch) continue;
                const long long grow = (long long)batch * p.out_rows_per_batch + row_in_batch;
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
                    const int col = col_base + 8 * j + c_lo;
                    if (col < p.partial_cols) o[((long long)split * p.partial_cols + col) * p.ld_out + grow] = acc[4 * j + 2 * half];
                    if (col + 1 < p.partial_cols) o[((long long)split * p.partial_cols + col + 1) * p.ld_out + grow] = acc[4 * j + 2 * half + 1];
                }
            }
        }
    }
    // the grid counts as complete (PDL dependents, stream order) only once its bulk stores are done
    if (kStore && wg_tid == 0) bulk_wait_all();
}

// ------------------------------------------------------------------------------------------------ FP8 (E4M3) encoder GEMMs
// The same producer / two-consumer structure with E4M3 operands: a k-block is 128 codes (one 128-byte swizzle row), so it is also one
// activation scale block.  A stage holds the A tile, the B tile and the tile's 128 row scales of that k-block (a 512-byte bulk copy
// from a_scale [K / 128][a_scale_ld]).  Each k-block's four m64n128k32 MMAs go into a temporary accumulator, which is then promoted:
// acc += tmp * a_scale[kb][row].  The weight scale (one per output channel) multiplies acc once before the epilogue.
static constexpr int kFp8BN = 128;
static constexpr int kStageB8 = kFp8BN * kFp8Block;          // 16 KiB
static constexpr int kStage8 = kStageA + kStageB8 + 1024;    // + the 512-byte scale row, padded to keep stages 1024-aligned

struct GemmFp8Params {
    GemmKParams g;
    const float* a_scale;
    long long a_scale_ld;
    const float* w_scale;
};

// GEMM_OUT_FP8_BLOCKS epilogue of one consumer warpgroup (FC1 under the FP8 encoder policy): v = act(acc + bias) in f32, then per row
// one scale over the tile's 128 columns - the 4 lanes of a quad hold a row, so its amax is two shuffles - and the codes into one
// 64-row x 128-byte staging box, one TMA store.  The lane with c_lo == 0 stores the row's scale to out_scale[col_base / 128][row].
__device__ __forceinline__ void gemm_epilogue_fp8_blocks(const GemmFp8Params& q, const CUtensorMap* tmO, float (&acc)[kFp8BN / 2],
                                                         uint8_t* stage, int& sbuf, int wg_tid, int cw, int row0, int col_base) {
    const GemmKParams& p = q.g;
    const int lane = wg_tid & 31;
    const int c_lo = 2 * (lane & 3);
    const int r_top = 16 * (wg_tid >> 5) + (lane >> 2);   // and r_top + 8
    float amax[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < kFp8BN / 8; ++j) {
        const int col = col_base + 8 * j + c_lo;
        float v0 = acc[4 * j], v1 = acc[4 * j + 1], v2 = acc[4 * j + 2], v3 = acc[4 * j + 3];
        if (p.bias) {
            const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias + col));
            v0 += bb.x; v1 += bb.y; v2 += bb.x; v3 += bb.y;
        }
        if (p.gelu) {
            const float2 g0 = gelu_erf2(make_float2(v0, v1)), g1 = gelu_erf2(make_float2(v2, v3));
            v0 = g0.x; v1 = g0.y; v2 = g1.x; v3 = g1.y;
        }
        acc[4 * j] = v0; acc[4 * j + 1] = v1; acc[4 * j + 2] = v2; acc[4 * j + 3] = v3;
        amax[0] = fmaxf(amax[0], fmaxf(fabsf(v0), fabsf(v1)));
        amax[1] = fmaxf(amax[1], fmaxf(fabsf(v2), fabsf(v3)));
    }
    uint8_t* buf = stage + sbuf * kStoreBox;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float a = fmaxf(amax[h], __shfl_xor_sync(0xffffffffu, amax[h], 1));
        a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, 2));
        const float s = fp8_row_scale(a);
        const int r = r_top + 8 * h;
        // column 8 j + c_lo is byte 8 (j & 1) + c_lo of the row's 16-byte chunk j / 2
#pragma unroll
        for (int j = 0; j < kFp8BN / 8; ++j)
            *reinterpret_cast<uint16_t*>(buf + swz128(r, j >> 1) + 8 * (j & 1) + c_lo) =
                (uint16_t)(fp8_encode(acc[4 * j + 2 * h], s) | (fp8_encode(acc[4 * j + 2 * h + 1], s) << 8));
        if (c_lo == 0 && row0 + r < p.m_rows_per_batch) p.out_scale[(long long)(col_base / kFp8Block) * q.a_scale_ld + row0 + r] = s;
    }
    store_box_begin(wg_tid, cw);
    if (wg_tid == 0) {
        tma_store_3d(tmO, buf, col_base, row0, 0);
        bulk_commit();
    }
    sbuf ^= 1;
}

template <typename T, int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmO,
                const GemmFp8Params q) {
    constexpr int BN = kFp8BN;
    const GemmKParams& p = q.g;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* store_stage = smem + (size_t)p.stages * kStage8;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(store_stage + kStoreBytes);
    uint64_t* empty_bar = full_bar + kMaxStages;
    uint64_t* res_bar = empty_bar + kMaxStages;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    pdl_launch_dependents();

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        tma_prefetch_desc(&tmO);
        for (int i = 0; i < p.stages; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 8);
        }
        for (int i = 0; i < 4; ++i) mbar_init(&res_bar[i], 1);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp != 0) return;
        // ===================== TMA producer =====================
        int stage = 0;
        uint32_t phase = 0;
        for (int w = blockIdx.x; w < p.work; w += gridDim.x) {
            const int n_tile = w % p.tiles_n;
            const int row0 = (w / p.tiles_n) * kBlockM;
            for (int kb = 0; kb < p.kb_per_split; ++kb) {
                mbar_wait(&empty_bar[stage], phase ^ 1);
                __syncwarp();
                uint8_t* sa = smem + (size_t)stage * kStage8;
                mbar_expect_tx_elect(&full_bar[stage], (uint32_t)(kStageA + kStageB8 + kBlockM * 4));
                tma_load_2d_elect(sa, &tmA, &full_bar[stage], kb * kFp8Block, row0);
                tma_load_2d_elect(sa + kStageA, &tmB, &full_bar[stage], kb * kFp8Block, n_tile * BN);
                bulk_load_1d_elect(sa + kStageA + kStageB8, q.a_scale + (long long)kb * q.a_scale_ld + row0, kBlockM * 4, &full_bar[stage]);
                if (++stage == p.stages) { stage = 0; phase ^= 1; }
            }
        }
        return;
    }

    // ===================== consumer warpgroups =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int cw = (warp >> 2) - 1;
    const int wg_tid = threadIdx.x & 127;
    const int r_lo = cw * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's rows in the tile: r_lo and r_lo + 8
    const int c_lo = 2 * (lane & 3);
    uint8_t* my_stage = store_stage + cw * 2 * kStoreBox;
    uint64_t* my_res_bar = res_bar + 2 * cw;
    int sbuf = 0;
    uint32_t rphase = 0;
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2], tmp[BN / 2];
    for (int w = blockIdx.x; w < p.work; w += gridDim.x) {
        const int n_tile = w % p.tiles_n;
        const int tile_row0 = (w / p.tiles_n) * kBlockM;
        const int col_base = n_tile * BN;
        const int wg_row0 = tile_row0 + 64 * cw;
        const bool wg_rows = wg_row0 < p.m_rows_per_batch;

        for (int kb = 0; kb < p.kb_per_split; ++kb) {
            mbar_wait(&full_bar[stage], phase);
            uint8_t* sa = smem + (size_t)stage * kStage8;
            const uint64_t adesc = wgmma_desc_sw128(smem_u32(sa) + cw * 64 * 128);
            const uint64_t bdesc = wgmma_desc_sw128(smem_u32(sa + kStageA));
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < kFp8Block / 32; ++k)   // +32 bytes per 32 K codes inside the swizzle row
                WgmmaE4M3x128::ss(tmp, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), k > 0 ? 1u : 0u);
            wgmma_commit();
            if (EPI == kEpiStore32 && kb == 0 && wg_tid == 0 && wg_rows) {
                // residual chunks 0 and 1 of this tile (GEMM_OUT_F32_ADD), fetched while the MMAs run
                bulk_wait_read_all();
                for (int c = 0; c < 2 && col_base + 32 * c < p.n; ++c) {
                    const int b = sbuf ^ c;
                    mbar_expect_tx(&my_res_bar[b], kStoreBox);
                    tma_load_3d(my_stage + b * kStoreBox, &tmO, &my_res_bar[b], col_base + 32 * c, wg_row0, 0);
                }
            }
            const float* sc = reinterpret_cast<const float*>(sa + kStageA + kStageB8);
            const float s0 = sc[r_lo], s1 = sc[r_lo + 8];
            wgmma_wait<0>();
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[stage]);
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                if (kb == 0) {
                    acc[4 * j] = tmp[4 * j] * s0; acc[4 * j + 1] = tmp[4 * j + 1] * s0;
                    acc[4 * j + 2] = tmp[4 * j + 2] * s1; acc[4 * j + 3] = tmp[4 * j + 3] * s1;
                } else {
                    acc[4 * j] = fmaf(tmp[4 * j], s0, acc[4 * j]); acc[4 * j + 1] = fmaf(tmp[4 * j + 1], s0, acc[4 * j + 1]);
                    acc[4 * j + 2] = fmaf(tmp[4 * j + 2], s1, acc[4 * j + 2]); acc[4 * j + 3] = fmaf(tmp[4 * j + 3], s1, acc[4 * j + 3]);
                }
            }
            if (++stage == p.stages) { stage = 0; phase ^= 1; }
        }
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {   // dequantize: the weight scale of each output channel (n is a multiple of 128)
            const float2 ws = __ldg(reinterpret_cast<const float2*>(q.w_scale + col_base + 8 * j + c_lo));
            acc[4 * j] *= ws.x; acc[4 * j + 1] *= ws.y; acc[4 * j + 2] *= ws.x; acc[4 * j + 3] *= ws.y;
        }
        if (!wg_rows) continue;
        if constexpr (EPI == kEpiStore16) gemm_epilogue_store16<T, BN>(p, &tmO, acc, my_stage, sbuf, wg_tid, cw, 0, wg_row0, col_base);
        else if constexpr (EPI == kEpiStore32) gemm_epilogue_store32<BN>(p, &tmO, acc, my_stage, my_res_bar, sbuf, rphase, wg_tid, cw, 0, wg_row0, col_base);
        else gemm_epilogue_fp8_blocks(q, &tmO, acc, my_stage, sbuf, wg_tid, cw, wg_row0, col_base);
    }
    if (wg_tid == 0) bulk_wait_all();
}

// ------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_encodeTiled>(p);
    }
    return fn;
}

static wk_status make_tmap(CUtensorMap* tm, const void* base, int dtype, int ndim, const uint64_t* dims,
                           const uint64_t* strides_bytes, const uint32_t* box) {
    PFN_encodeTiled enc = get_encode_fn();
    if (!enc) {
        set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
        return WK_ERR_CUDA;
    }
    cuuint64_t gdim[3];
    cuuint64_t gstr[2];
    cuuint32_t bx[3];
    cuuint32_t es[3] = {1, 1, 1};
    for (int i = 0; i < ndim; ++i) { gdim[i] = dims[i]; bx[i] = box[i]; }
    for (int i = 0; i < ndim - 1; ++i) gstr[i] = strides_bytes[i];
    const CUtensorMapDataType ty = dtype == WK_DTYPE_F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                   : dtype == WK_DTYPE_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                                   : dtype == WK_DTYPE_FP8_E4M3 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    CUresult r = enc(tm, ty,
                     (cuuint32_t)ndim, const_cast<void*>(base), gdim, gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed: %d (ndim %d dims %llu %llu stride %llu box %u %u)", (int)r, ndim,
                  (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)strides_bytes[0], box[0],
                  box[1]);
        return WK_ERR_CUDA;
    }
    return WK_OK;
}

int wgmma_tile_n(int bn) {
    int t = 16;
    while (t < bn) t <<= 1;
    return t;
}

template <typename T, int BN, int EPI>
static cudaError_t launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmO, const GemmKParams& p, int grid,
                               size_t smem, int pdl, cudaStream_t stream) {
    static bool attr_set = false;
    if (!attr_set) {
        const cudaError_t e = cudaFuncSetAttribute(gemm_wgmma_kernel<T, BN, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax);
        if (e != cudaSuccess) return e;
        attr_set = true;
    }
    return launch_k(gemm_wgmma_kernel<T, BN, EPI>, dim3(grid), dim3(kGemmThreads), smem, stream, pdl, tmA, tmB, tmO, p);
}

// the TMA-store epilogues run 64-, 128- or 256-column tiles (gemm_wgmma rounds bn up to 64 for them)
template <typename T, int EPI>
static cudaError_t launch_gemm_store(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmO, const GemmKParams& p, int grid,
                                     size_t smem, int pdl, cudaStream_t stream) {
    switch (p.bn) {
        case 64: return launch_gemm<T, 64, EPI>(tmA, tmB, tmO, p, grid, smem, pdl, stream);
        case 128: return launch_gemm<T, 128, EPI>(tmA, tmB, tmO, p, grid, smem, pdl, stream);
        default: return launch_gemm<T, 256, EPI>(tmA, tmB, tmO, p, grid, smem, pdl, stream);
    }
}

template <typename T>
static cudaError_t launch_gemm_n(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmO, const GemmKParams& p, int grid,
                                 size_t smem, int pdl, cudaStream_t stream) {
    switch (gemm_epi(p.mode)) {
        case kEpiFp8Heads: return launch_gemm<T, 256, kEpiFp8Heads>(tmA, tmB, tmO, p, grid, smem, pdl, stream);   // bn checked by gemm_wgmma
        case kEpiPackedHeads:
            if constexpr (std::is_same<T, __nv_bfloat16>::value) return launch_gemm<T, 256, kEpiPackedHeads>(tmA, tmB, tmO, p, grid, smem, pdl, stream);
            return cudaErrorInvalidValue;   // bf16 only (checked by gemm_wgmma)
        case kEpiStore16: return launch_gemm_store<T, kEpiStore16>(tmA, tmB, tmO, p, grid, smem, pdl, stream);
        case kEpiStore32: return launch_gemm_store<T, kEpiStore32>(tmA, tmB, tmO, p, grid, smem, pdl, stream);
        default: break;
    }
    switch (p.bn) {
        case 16: return launch_gemm<T, 16, kEpiPartialT>(tmA, tmB, tmO, p, grid, smem, pdl, stream);
        case 32: return launch_gemm<T, 32, kEpiPartialT>(tmA, tmB, tmO, p, grid, smem, pdl, stream);
        case 64: return launch_gemm<T, 64, kEpiPartialT>(tmA, tmB, tmO, p, grid, smem, pdl, stream);
        case 128: return launch_gemm<T, 128, kEpiPartialT>(tmA, tmB, tmO, p, grid, smem, pdl, stream);
        default: return launch_gemm<T, 256, kEpiPartialT>(tmA, tmB, tmO, p, grid, smem, pdl, stream);
    }
}

wk_status gemm_wgmma(const GemmDesc& d, int num_sms, cudaStream_t stream) {
    if (d.k % kBlockK != 0 || d.bn % 16 != 0 || d.bn < 16 || d.bn > 256 || d.taps < 1 || d.taps > 3) {
        set_error("gemm_wgmma: unsupported shape k=%d bn=%d taps=%d", d.k, d.bn, d.taps);
        return WK_ERR_INVALID_ARGUMENT;
    }
    if (d.mode != GEMM_OUT_PARTIAL_T && (d.n % 32 != 0 || d.splits != 1)) {
        set_error("gemm_wgmma: n=%d must be a multiple of 32 and splits 1 for mode %d", d.n, d.mode);
        return WK_ERR_INVALID_ARGUMENT;
    }
    GemmKParams p;
    memset(&p, 0, sizeof(p));
    p.kb_per_tap = d.k / kBlockK;
    const int total_kb = p.kb_per_tap * d.taps;
    p.splits = d.splits < 1 ? 1 : d.splits;
    if (total_kb % p.splits != 0) {
        set_error("gemm_wgmma: splits %d does not divide %d k-blocks", p.splits, total_kb);
        return WK_ERR_INVALID_ARGUMENT;
    }
    p.kb_per_split = total_kb / p.splits;
    p.taps = d.taps;
    for (int i = 0; i < 3; ++i) { p.tap_row_shift[i] = d.tap_row_shift[i]; p.tap_col_off[i] = d.tap_col_off[i]; }
    p.a_is_3d = d.a_3d ? 1 : 0;
    p.n_batches = d.a_3d ? d.a_batches : 1;
    p.m_rows_per_batch = d.m_rows_per_batch;
    p.tiles_per_batch = (d.m_rows_per_batch + kBlockM - 1) / kBlockM;
    p.n = d.n;
    // wgmma tile width: the requested bn rounded up to a power of two (columns past n / partial_cols are zero-filled by TMA and never stored)
    p.bn = wgmma_tile_n(d.bn);
    const int epi = gemm_epi(d.mode);
    const bool tma_store = epi == kEpiStore16 || epi == kEpiStore32;
    if (tma_store && p.bn < 64) p.bn = 64;   // whole 64-row x 128-byte staging boxes
    p.tiles_n = (d.n + p.bn - 1) / p.bn;
    p.work = p.tiles_per_batch * p.n_batches * p.tiles_n * p.splits;
    p.stage_b_bytes = p.bn * kBlockK * 2;
    // B stage must keep 1024-byte alignment of the following A stage
    if (p.stage_b_bytes % 1024 != 0) p.stage_b_bytes = (p.stage_b_bytes + 1023) / 1024 * 1024;
    const int stage_bytes = kStageA + p.stage_b_bytes;
    p.store_bytes = tma_store ? kStoreBytes : 0;
    const int smem_budget = kSmemMax - 1024 /*align slack*/ - 256 /*barriers*/ - p.store_bytes;
    int stages = smem_budget / stage_bytes;
    if (stages > kMaxStages) stages = kMaxStages;
    if (stages > total_kb / p.splits + 2) stages = total_kb / p.splits + 2;
    if (stages < 2) stages = 2;
    if (d.max_stages > 0 && stages > d.max_stages) stages = d.max_stages;
    p.stages = stages;
    p.a_static = d.a_static;
    p.mode = d.mode;
    p.gelu = d.gelu;
    p.out = d.out;
    p.ld_out = d.ld_out;
    p.out_rows_per_batch = d.out_rows_per_batch;
    p.partial_cols = d.partial_cols;
    p.bias = d.bias;
    p.pos = d.pos;
    p.ld_pos = d.ld_pos;
    p.heads_T = d.heads_T; p.heads_B = d.heads_B; p.heads_H = d.heads_H; p.heads_dmodel = d.heads_dmodel;
    p.out_scale = d.out_scale;
    p.out_hdr = d.out_hdr;
    if (d.mode == GEMM_OUT_PACKED_HEADS && (p.bn != 256 || d.n % 64 != 0 || d.heads_dmodel % 64 != 0 || !d.out_hdr || d.in_dtype != WK_DTYPE_BF16)) {
        set_error("gemm_wgmma: the packed heads epilogue needs bf16, 256-column tiles and head-aligned columns (bn %d n %d d %d)", p.bn, d.n, d.heads_dmodel);
        return WK_ERR_INVALID_ARGUMENT;
    }
    if (d.mode == GEMM_OUT_FP8_HEADS && (p.bn != 256 || d.n % 64 != 0 || d.heads_dmodel % 64 != 0 || !d.out_scale)) {
        // the row amax is taken over whole heads inside one N tile
        set_error("gemm_wgmma: the FP8 heads epilogue needs 256-column tiles and head-aligned columns (bn %d n %d d %d)", p.bn, d.n, d.heads_dmodel);
        return WK_ERR_INVALID_ARGUMENT;
    }
    if (d.mode == GEMM_OUT_T16_HEADS &&
        (p.n_batches != 1 || d.n % 64 != 0 || d.heads_dmodel % 64 != 0 || d.n % d.heads_dmodel != 0 || d.m_rows_per_batch % d.heads_T != 0)) {
        // a 64-column chunk is one head; rows are whole windows of heads_T
        set_error("gemm_wgmma: the 16-bit heads epilogue needs head-aligned columns and whole windows (n %d d %d rows %d T %d)", d.n,
                  d.heads_dmodel, d.m_rows_per_batch, d.heads_T);
        return WK_ERR_INVALID_ARGUMENT;
    }

    CUtensorMap tmA, tmB, tmO;
    memset(&tmO, 0, sizeof(tmO));
    wk_status st;
    if (p.a_is_3d) {
        uint64_t dims[3] = {(uint64_t)d.a_cols, (uint64_t)d.a_rows, (uint64_t)d.a_batches};
        uint64_t str[2] = {(uint64_t)d.a_ld * 2, (uint64_t)d.a_batch_stride * 2};
        uint32_t box[3] = {kBlockK, kBlockM, 1};
        st = make_tmap(&tmA, d.a, d.in_dtype, 3, dims, str, box);
    } else {
        uint64_t dims[2] = {(uint64_t)d.a_cols, (uint64_t)d.a_rows};
        uint64_t str[1] = {(uint64_t)d.a_ld * 2};
        uint32_t box[2] = {kBlockK, kBlockM};
        st = make_tmap(&tmA, d.a, d.in_dtype, 2, dims, str, box);
    }
    if (st != WK_OK) return st;
    {
        uint64_t dims[2] = {(uint64_t)d.k * d.taps, (uint64_t)d.b_rows};
        uint64_t str[1] = {(uint64_t)d.b_ld * 2};
        uint32_t box[2] = {kBlockK, (uint32_t)p.bn};
        st = make_tmap(&tmB, d.b, d.in_dtype, 2, dims, str, box);
        if (st != WK_OK) return st;
    }
    if (d.mode == GEMM_OUT_T16_HEADS) {
        // the [which][b][h][t][64] cache as {64, T, which * b * h}: the 64 rows of one head of a warpgroup are one box
        uint64_t dims[3] = {64, (uint64_t)d.heads_T, (uint64_t)(d.n / d.heads_dmodel) * d.heads_B * d.heads_H};
        uint64_t str[2] = {128, (uint64_t)d.heads_T * 128};
        uint32_t box[3] = {64, 64, 1};
        st = make_tmap(&tmO, d.out, d.in_dtype, 3, dims, str, box);
    } else if (tma_store) {
        // [batch][rows][ld_out] with m_rows_per_batch valid rows and n valid columns per batch: TMA clips ragged tiles
        const int out_dtype = epi == kEpiStore16 ? d.in_dtype : WK_DTYPE_F32;
        const uint64_t es = epi == kEpiStore16 ? 2 : 4;
        uint64_t dims[3] = {(uint64_t)d.n, (uint64_t)d.m_rows_per_batch, (uint64_t)p.n_batches};
        uint64_t str[2] = {(uint64_t)d.ld_out * es, (uint64_t)d.out_rows_per_batch * d.ld_out * es};
        uint32_t box[3] = {(uint32_t)(128 / es), 64, 1};
        st = make_tmap(&tmO, d.out, out_dtype, 3, dims, str, box);
    }
    if (st != WK_OK) return st;
    const size_t smem_bytes = (size_t)stages * stage_bytes + p.store_bytes + 1024 + 256;
    int grid = p.work < num_sms ? p.work : num_sms;
    if (grid < 1) return WK_OK;
    const int pdl = d.pdl != 0 ? 16 : 0;
    cudaError_t e = d.in_dtype == WK_DTYPE_F16 ? launch_gemm_n<__half>(tmA, tmB, tmO, p, grid, smem_bytes, pdl, stream)
                                               : launch_gemm_n<__nv_bfloat16>(tmA, tmB, tmO, p, grid, smem_bytes, pdl, stream);
    count_launch();
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("gemm_wgmma launch: %s", cudaGetErrorString(e));
        return WK_ERR_CUDA;
    }
    return WK_OK;
}

template <typename T, int EPI>
static cudaError_t launch_gemm_fp8(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmO, const GemmFp8Params& q, int grid,
                                   size_t smem, cudaStream_t stream) {
    static bool attr_set = false;
    if (!attr_set) {
        const cudaError_t e = cudaFuncSetAttribute(gemm_fp8_kernel<T, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax);
        if (e != cudaSuccess) return e;
        attr_set = true;
    }
    return launch_k(gemm_fp8_kernel<T, EPI>, dim3(grid), dim3(kGemmThreads), smem, stream, 0, tmA, tmB, tmO, q);
}

template <typename T>
static cudaError_t launch_gemm_fp8_mode(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmO, const GemmFp8Params& q,
                                        int grid, size_t smem, cudaStream_t stream) {
    switch (q.g.mode) {
        case GEMM_OUT_T16: return launch_gemm_fp8<T, kEpiStore16>(tmA, tmB, tmO, q, grid, smem, stream);
        case GEMM_OUT_F32_ADD: return launch_gemm_fp8<T, kEpiStore32>(tmA, tmB, tmO, q, grid, smem, stream);
        default: return launch_gemm_fp8<T, kEpiFp8Blocks>(tmA, tmB, tmO, q, grid, smem, stream);
    }
}

wk_status gemm_wgmma_fp8(const GemmDesc& d, int num_sms, cudaStream_t stream) {
    if (d.k % kFp8Block != 0 || d.n % kFp8BN != 0 || d.k < kFp8Block || d.n < kFp8BN || d.m_rows_per_batch < 1 || d.a_3d || d.taps != 1 ||
        (d.mode != GEMM_OUT_T16 && d.mode != GEMM_OUT_F32_ADD && d.mode != GEMM_OUT_FP8_BLOCKS) || !d.a_scale || !d.w_scale ||
        d.a_scale_ld % kBlockM != 0 || d.a_scale_ld < d.m_rows_per_batch || (d.mode == GEMM_OUT_FP8_BLOCKS && !d.out_scale) ||
        (d.in_dtype != WK_DTYPE_BF16 && d.in_dtype != WK_DTYPE_F16)) {
        set_error("gemm_wgmma_fp8: unsupported problem (m %d n %d k %d mode %d scale ld %lld)", d.m_rows_per_batch, d.n, d.k, d.mode,
                  (long long)d.a_scale_ld);
        return WK_ERR_INVALID_ARGUMENT;
    }
    GemmFp8Params q;
    memset(&q, 0, sizeof(q));
    GemmKParams& p = q.g;
    p.kb_per_tap = p.kb_per_split = d.k / kFp8Block;
    p.splits = 1; p.taps = 1; p.n_batches = 1;
    p.m_rows_per_batch = d.m_rows_per_batch;
    p.tiles_per_batch = (d.m_rows_per_batch + kBlockM - 1) / kBlockM;
    p.n = d.n; p.bn = kFp8BN;
    p.tiles_n = d.n / kFp8BN;
    p.work = p.tiles_per_batch * p.tiles_n;
    p.stage_b_bytes = kStageB8;
    p.store_bytes = kStoreBytes;
    int stages = (kSmemMax - 1024 - 256 - kStoreBytes) / kStage8;
    if (stages > kMaxStages) stages = kMaxStages;
    p.stages = stages;
    p.mode = d.mode; p.gelu = d.gelu; p.out = d.out; p.ld_out = d.ld_out; p.out_rows_per_batch = d.m_rows_per_batch;
    p.bias = d.bias; p.out_scale = d.out_scale;
    q.a_scale = d.a_scale; q.a_scale_ld = d.a_scale_ld; q.w_scale = d.w_scale;

    CUtensorMap tmA, tmB, tmO;
    {
        uint64_t dims[2] = {(uint64_t)d.k, (uint64_t)d.a_rows};
        uint64_t str[1] = {(uint64_t)d.a_ld};
        uint32_t box[2] = {kFp8Block, kBlockM};
        WK_CHECK(make_tmap(&tmA, d.a, WK_DTYPE_FP8_E4M3, 2, dims, str, box));
    }
    {
        uint64_t dims[2] = {(uint64_t)d.k, (uint64_t)d.b_rows};
        uint64_t str[1] = {(uint64_t)d.b_ld};
        uint32_t box[2] = {kFp8Block, kFp8BN};
        WK_CHECK(make_tmap(&tmB, d.b, WK_DTYPE_FP8_E4M3, 2, dims, str, box));
    }
    {
        // [rows][ld_out] with n valid columns: 64 rows x 128 bytes per staging box (64 16-bit, 32 f32 or 128 E4M3 columns)
        const int out_dtype = d.mode == GEMM_OUT_T16 ? d.in_dtype : d.mode == GEMM_OUT_F32_ADD ? WK_DTYPE_F32 : WK_DTYPE_FP8_E4M3;
        const uint64_t es = d.mode == GEMM_OUT_T16 ? 2 : d.mode == GEMM_OUT_F32_ADD ? 4 : 1;
        uint64_t dims[3] = {(uint64_t)d.n, (uint64_t)d.m_rows_per_batch, 1};
        uint64_t str[2] = {(uint64_t)d.ld_out * es, (uint64_t)d.m_rows_per_batch * d.ld_out * es};
        uint32_t box[3] = {(uint32_t)(128 / es), 64, 1};
        WK_CHECK(make_tmap(&tmO, d.out, out_dtype, 3, dims, str, box));
    }
    const size_t smem_bytes = (size_t)stages * kStage8 + kStoreBytes + 1024 + 256;
    const int grid = p.work < num_sms ? p.work : num_sms;
    cudaError_t e = d.in_dtype == WK_DTYPE_F16 ? launch_gemm_fp8_mode<__half>(tmA, tmB, tmO, q, grid, smem_bytes, stream)
                                               : launch_gemm_fp8_mode<__nv_bfloat16>(tmA, tmB, tmO, q, grid, smem_bytes, stream);
    count_launch();
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("gemm_wgmma_fp8 launch: %s", cudaGetErrorString(e));
        return WK_ERR_CUDA;
    }
    return WK_OK;
}

}  // namespace wk
