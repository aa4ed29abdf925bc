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
//                 in registers, then the fused epilogue straight from those registers to HBM.  A stage is released as soon as the
//                 wgmma group that read it has retired (wait_group 1 keeps one k-block of MMAs in flight).
// The WhisperKit reference has no counterpart source for this file: the contraction lives inside
// AudioEncoder.mlmodelc / TextDecoder.mlmodelc (Sources/WhisperKit/Core/AudioEncoder.swift:59-62,
// Sources/WhisperKit/Core/TextDecoder.swift:394-417).
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>

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
    int stage_b_bytes, stages;
    int mode, gelu;
    void* out;
    long long ld_out, out_rows_per_batch, partial_cols;
    const float* bias;
    const float* pos;
    long long ld_pos;
    int heads_T, heads_B, heads_H, heads_dmodel;
    float* out_scale;
    int a_static;     // see GemmDesc::a_static
};

// fused epilogue of two adjacent accumulator columns (col, col + 1) of one output row
template <typename T>
__device__ __forceinline__ void gemm_epilogue_pair(const GemmKParams& p, int split, long long grow, int row_in_batch, int col, float v0,
                                                   float v1) {
    if (p.mode == GEMM_OUT_PARTIAL_T) {
        float* o = reinterpret_cast<float*>(p.out);
        if (col < p.partial_cols) o[((long long)split * p.partial_cols + col) * p.ld_out + grow] = v0;
        if (col + 1 < p.partial_cols) o[((long long)split * p.partial_cols + col + 1) * p.ld_out + grow] = v1;
        return;
    }
    if (col >= p.n) return;   // n is a multiple of 32: col + 1 < n as well
    if (p.bias) {
        const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias + col));
        v0 += bb.x; v1 += bb.y;
    }
    if (p.gelu) {
        const float2 g = gelu_erf2(make_float2(v0, v1));
        v0 = g.x; v1 = g.y;
    }
    if (p.mode == GEMM_OUT_T16) {
        *reinterpret_cast<uint32_t*>(reinterpret_cast<T*>(p.out) + grow * p.ld_out + col) = T16<T>::pack2(v0, v1);
    } else if (p.mode == GEMM_OUT_T16_HEADS) {
        const int b = (int)(grow / p.heads_T);
        const int tt = (int)(grow - (long long)b * p.heads_T);
        const int which = col / p.heads_dmodel;
        const int rem = col - which * p.heads_dmodel;
        const int h = rem >> 6;
        const int dd = rem & 63;
        T* o = reinterpret_cast<T*>(p.out) + ((((long long)which * p.heads_B + b) * p.heads_H + h) * p.heads_T + tt) * 64 + dd;
        *reinterpret_cast<uint32_t*>(o) = T16<T>::pack2(v0, v1);
    } else {
        float2* o = reinterpret_cast<float2*>(reinterpret_cast<float*>(p.out) + grow * p.ld_out + col);
        if (p.mode == GEMM_OUT_F32_ADD) {
            float2 x = *o;
            x.x += v0; x.y += v1;
            *o = x;
        } else if (p.mode == GEMM_OUT_F32_GELU_POS) {
            const float2 pp = __ldg(reinterpret_cast<const float2*>(p.pos + (long long)row_in_batch * p.ld_pos + col));
            *o = make_float2(v0 + pp.x, v1 + pp.y);
        } else {
            *o = make_float2(v0, v1);
        }
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

template <typename T, int BN, bool FP8_HEADS = false>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmKParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // manual 1024-byte alignment (SWIZZLE_128B atoms are 1024 B)
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int stage_bytes = kStageA + p.stage_b_bytes;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + (size_t)p.stages * stage_bytes);
    uint64_t* empty_bar = full_bar + kMaxStages;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    pdl_launch_dependents();   // the next kernel may start its prologue; it still waits for our completion

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int i = 0; i < p.stages; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 8);   // one arrive per consumer warp
        }
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
    const int r_lo = cw * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's rows: r_lo and r_lo + 8
    const int c_lo = 2 * (lane & 3);                      // and columns 8 j + c_lo, + 1
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

        const int col_base = n_tile * BN;
        if constexpr (FP8_HEADS) {
            gemm_epilogue_fp8_heads<BN>(p, batch, tile_row0, r_lo, c_lo, col_base, acc);
        } else {
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const int row_in_batch = tile_row0 + r_lo + 8 * half;
                if (row_in_batch >= p.m_rows_per_batch) continue;
                const long long grow = (long long)batch * p.out_rows_per_batch + row_in_batch;
#pragma unroll
                for (int j = 0; j < BN / 8; ++j)
                    gemm_epilogue_pair<T>(p, split, grow, row_in_batch, col_base + 8 * j + c_lo, acc[4 * j + 2 * half], acc[4 * j + 2 * half + 1]);
            }
        }
    }
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
    CUresult r = enc(tm, dtype == WK_DTYPE_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16,
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

// 2-D, 128-byte-swizzled, 16-bit tensor map over a row-major [rows][ld] matrix with a [box_rows][box_cols] box (used by fused_chain.cu)
wk_status make_tmap_2d(void* tm, const void* base, int dtype, uint64_t cols, uint64_t rows, uint64_t ld_elems, uint32_t box_cols, uint32_t box_rows) {
    uint64_t dims[2] = {cols, rows};
    uint64_t str[1] = {ld_elems * 2};
    uint32_t box[2] = {box_cols, box_rows};
    return make_tmap(reinterpret_cast<CUtensorMap*>(tm), base, dtype, 2, dims, str, box);
}

int wgmma_tile_n(int bn) {
    int t = 16;
    while (t < bn) t <<= 1;
    return t;
}

template <typename T, int BN, bool FP8_HEADS = false>
static cudaError_t launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmKParams& p, int grid, size_t smem, int pdl,
                               cudaStream_t stream) {
    static bool attr_set = false;
    if (!attr_set) {
        const cudaError_t e = cudaFuncSetAttribute(gemm_wgmma_kernel<T, BN, FP8_HEADS>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax);
        if (e != cudaSuccess) return e;
        attr_set = true;
    }
    return launch_k(gemm_wgmma_kernel<T, BN, FP8_HEADS>, dim3(grid), dim3(kGemmThreads), smem, stream, pdl, tmA, tmB, p);
}

template <typename T>
static cudaError_t launch_gemm_n(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmKParams& p, int grid, size_t smem, int pdl,
                                 cudaStream_t stream) {
    if (p.mode == GEMM_OUT_FP8_HEADS) return launch_gemm<T, 256, true>(tmA, tmB, p, grid, smem, pdl, stream);   // bn checked by gemm_wgmma
    switch (p.bn) {
        case 16: return launch_gemm<T, 16>(tmA, tmB, p, grid, smem, pdl, stream);
        case 32: return launch_gemm<T, 32>(tmA, tmB, p, grid, smem, pdl, stream);
        case 64: return launch_gemm<T, 64>(tmA, tmB, p, grid, smem, pdl, stream);
        case 128: return launch_gemm<T, 128>(tmA, tmB, p, grid, smem, pdl, stream);
        default: return launch_gemm<T, 256>(tmA, tmB, p, grid, smem, pdl, stream);
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
    p.tiles_n = (d.n + p.bn - 1) / p.bn;
    p.work = p.tiles_per_batch * p.n_batches * p.tiles_n * p.splits;
    p.stage_b_bytes = p.bn * kBlockK * 2;
    // B stage must keep 1024-byte alignment of the following A stage
    if (p.stage_b_bytes % 1024 != 0) p.stage_b_bytes = (p.stage_b_bytes + 1023) / 1024 * 1024;
    const int stage_bytes = kStageA + p.stage_b_bytes;
    const int smem_budget = kSmemMax - 1024 /*align slack*/ - 256 /*barriers*/;
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
    if (d.mode == GEMM_OUT_FP8_HEADS && (p.bn != 256 || d.n % 64 != 0 || d.heads_dmodel % 64 != 0 || !d.out_scale)) {
        // the row amax is taken over whole heads inside one N tile
        set_error("gemm_wgmma: the FP8 heads epilogue needs 256-column tiles and head-aligned columns (bn %d n %d d %d)", p.bn, d.n, d.heads_dmodel);
        return WK_ERR_INVALID_ARGUMENT;
    }

    CUtensorMap tmA, tmB;
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
    const size_t smem_bytes = (size_t)stages * stage_bytes + 1024 + 256;
    int grid = p.work < num_sms ? p.work : num_sms;
    if (grid < 1) return WK_OK;
    const int pdl = d.pdl != 0 ? 16 : 0;
    cudaError_t e = d.in_dtype == WK_DTYPE_F16 ? launch_gemm_n<__half>(tmA, tmB, p, grid, smem_bytes, pdl, stream)
                                               : launch_gemm_n<__nv_bfloat16>(tmA, tmB, p, grid, smem_bytes, pdl, stream);
    count_launch();
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("gemm_wgmma launch: %s", cudaGetErrorString(e));
        return WK_ERR_CUDA;
    }
    return WK_OK;
}

}  // namespace wk
