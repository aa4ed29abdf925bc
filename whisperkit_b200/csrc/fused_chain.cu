// fused_chain.cu - decoder phase chains: one persistent kernel runs a CHAIN of decoder phases that today are separate launches:
//     swap-AB split-K GEMM -> split-K reduce (+bias +residual +LayerNorm | +bias +GELU) -> GEMM -> ...
// with a grid-wide barrier between phases instead of a kernel boundary.  Motivation: a decoder GEMM launch is a few
// microseconds of fixed cost around about one microsecond of weight streaming, 11 such launches per layer; inside one kernel the mbarriers
// and tensor maps are set up once, the WEIGHT tiles of the next GEMM phase are put in flight before the barrier (weights are static), and
// a phase boundary costs one barrier.  Chains per decoder layer (engine.cu, decoder_forward):
//     B: out-proj GEMM -> reduce+LN -> cross-Q GEMM                                                  (between self- and cross-attention)
//     C: cross-out GEMM -> reduce+LN -> FC1 -> reduce+GELU -> FC2 -> reduce+LN -> next layer's QKV GEMM  (between cross- and self-attention)
//
// Structure: grid = one CTA per SM (all co-resident), 384 threads = 3 warpgroups.  GEMM phase: warp 0 = TMA producer, warpgroups 1 and 2
// = wgmma consumers (64 weight rows each, accumulator in registers) whose epilogue stores the transposed f32 partials, work item =
// (128-row weight tile, K split), one per CTA (single wave by the split rule).  Reduce phase: all 384 threads, CTA b reduces batch rows
// b, b + grid, ... in the fixed split order (deterministic).  Pipeline state (ring stage / parity) lives in registers across phases.  Memory ordering at a phase boundary: every thread
// fences its generic-proxy global writes towards the async proxy (the next GEMM phase reads activations with TMA), then
// bar.sync + __threadfence + atomic arrive / acquire spin (the cooperative-groups grid.sync recipe).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <string.h>

#include <algorithm>

#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

#define WK_CHECK_STATUS(expr)             \
    do {                                  \
        wk_status _s = (expr);            \
        if (_s != WK_OK) return _s;       \
    } while (0)

namespace wk {

namespace {

constexpr int kM = 128, kK = 64;
constexpr int kStageABytes = kM * kK * 2;
constexpr int kThreads = 384;
constexpr int kRingMax = 8;
constexpr int kMaxSplitsR = 20;

struct PhaseK {
    int kind;
    int map;                    // GEMM: index into the tensor-map arrays
    int n, kb_per_split, splits, tiles;
    int red_n, red_splits;      // reduce: row length and partial count
    const float* bias; const float* gamma; const float* beta;
    void* out16;
};
struct ChainK {
    int n_phases;
    PhaseK ph[kChainMaxPhases];
    float* partial; float* x;
    int B, Bp, d;
    int stages, stage_b_bytes;
    unsigned int* counters;
    unsigned int* reset;
};
struct ChainMaps {
    CUtensorMap a[kChainMaxGemms];
    CUtensorMap b[kChainMaxGemms];
};

__device__ __forceinline__ void fence_generic_to_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

__device__ __forceinline__ unsigned int ld_acquire_gpu(const unsigned int* p) {
    unsigned int v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// grid-wide barrier: every CTA of the (fully co-resident) grid arrives once on `ctr` (zero before the launch).  Release / acquire at gpu
// scope through one elected thread per CTA, made cumulative over the CTA by the bar.sync on either side.  `tma_reads_next`: this CTA's
// generic-proxy stores of the phase are read by TMA (async proxy) in the next phase - the writers fence towards that proxy first.
__device__ __forceinline__ void grid_barrier(unsigned int* ctr, unsigned int n_ctas, bool tma_reads_next) {
    if (tma_reads_next) fence_generic_to_async_global();
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory");
        if (ld_acquire_gpu(ctr) < n_ctas) {
            const unsigned long long t0 = globaltimer_ns();
            unsigned int spins = 0;
            while (ld_acquire_gpu(ctr) < n_ctas) {
                if ((++spins & 0xfffu) == 0 && globaltimer_ns() - t0 > kSpinLimitNs) {
                    printf("wkb200: grid barrier timed out (block %d: %u of %u CTAs arrived)\n", (int)blockIdx.x, ld_acquire_gpu(ctr), n_ctas);
                    __trap();
                }
            }
        }
    }
    __syncthreads();
}

template <typename T>
__device__ __forceinline__ void reduce_ln_row(const ChainK& p, const PhaseK& P, int b, float* scratch) {
    // the body of decoder_reduce_resid_ln_kernel (decoder_ops.cu): x[b] += bias + sum_s partial[s][b]; out16[b] = LN(x[b])
    const int tid = threadIdx.x, d = P.red_n, d4 = d >> 2, splits = P.red_splits;
    T* xn = reinterpret_cast<T*>(P.out16);
    float4 v[2];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const int i4 = tid + k * kThreads;
        v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i4 < d4) {
            float4 pr[kMaxSplitsR];
#pragma unroll
            for (int sp = 0; sp < kMaxSplitsR; ++sp)
                if (sp < splits) pr[sp] = __ldcg(reinterpret_cast<const float4*>(p.partial + ((long long)sp * p.Bp + b) * d) + i4);
            float4 a = reinterpret_cast<const float4*>(p.x + (long long)b * d)[i4];
            if (P.bias) {
                const float4 bb = __ldg(reinterpret_cast<const float4*>(P.bias) + i4);
                a.x += bb.x; a.y += bb.y; a.z += bb.z; a.w += bb.w;
            }
#pragma unroll
            for (int sp = 0; sp < kMaxSplitsR; ++sp)
                if (sp < splits) { a.x += pr[sp].x; a.y += pr[sp].y; a.z += pr[sp].z; a.w += pr[sp].w; }
            v[k] = a;
            reinterpret_cast<float4*>(p.x + (long long)b * d)[i4] = a;
            s += a.x + a.y + a.z + a.w;
        }
    }
    // block_sum over kThreads threads
    auto bsum = [&](float val) -> float {
        val = warp_sum(val);
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        __syncthreads();
        if (lane == 0) scratch[warp] = val;
        __syncthreads();
        float r = (lane < kThreads / 32) ? scratch[lane] : 0.f;
        return warp_sum(r);
    };
    const float mean = bsum(s) / d;
    float q = 0.f;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const int i4 = tid + k * kThreads;
        if (i4 < d4) {
            const float a0 = v[k].x - mean, a1 = v[k].y - mean, a2 = v[k].z - mean, a3 = v[k].w - mean;
            q += a0 * a0 + a1 * a1 + a2 * a2 + a3 * a3;
        }
    }
    const float rstd = rsqrtf(bsum(q) / d + 1e-5f);
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const int i4 = tid + k * kThreads;
        if (i4 < d4) {
            const float4 g = __ldg(reinterpret_cast<const float4*>(P.gamma) + i4), bb = __ldg(reinterpret_cast<const float4*>(P.beta) + i4);
            uint2 pk;
            pk.x = T16<T>::pack2((v[k].x - mean) * rstd * g.x + bb.x, (v[k].y - mean) * rstd * g.y + bb.y);
            pk.y = T16<T>::pack2((v[k].z - mean) * rstd * g.z + bb.z, (v[k].w - mean) * rstd * g.w + bb.w);
            reinterpret_cast<uint2*>(xn + (long long)b * d)[i4] = pk;
        }
    }
}

template <typename T>
__device__ __forceinline__ void reduce_gelu_all(const ChainK& p, const PhaseK& P) {
    // the body of decoder_reduce_bias_gelu_kernel spread over the whole grid: out16[b][i] = gelu(bias[i] + sum_s partial[s][b][i])
    const int n = P.red_n, splits = P.red_splits;
    T* out = reinterpret_cast<T*>(P.out16);
    const long long total4 = (long long)p.B * n / 4;
    for (long long q = (long long)blockIdx.x * kThreads + threadIdx.x; q < total4; q += (long long)gridDim.x * kThreads) {
        const long long idx = q * 4;
        const int b = (int)(idx / n), i = (int)(idx - (long long)b * n);
        float4 a = *reinterpret_cast<const float4*>(P.bias + i);
        for (int sp = 0; sp < splits; ++sp) {
            const float4 pp = __ldcg(reinterpret_cast<const float4*>(p.partial + ((long long)sp * p.Bp + b) * n + i));
            a.x += pp.x; a.y += pp.y; a.z += pp.z; a.w += pp.w;
        }
        uint2 pk;
        pk.x = T16<T>::pack2(gelu_erf(a.x), gelu_erf(a.y));
        pk.y = T16<T>::pack2(gelu_erf(a.z), gelu_erf(a.w));
        *reinterpret_cast<uint2*>(out + (long long)b * n + i) = pk;
    }
}

template <typename T, int BN>
__global__ void __launch_bounds__(kThreads, 1)
decoder_chain_kernel(const __grid_constant__ ChainMaps maps, const ChainK p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int stage_bytes = kStageABytes + p.stage_b_bytes;
    uint8_t* tail = smem + (size_t)p.stages * stage_bytes;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(tail);
    uint64_t* empty_bar = full_bar + kRingMax;
    float* scratch = reinterpret_cast<float*>(empty_bar + kRingMax);   // 32 floats

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    pdl_launch_dependents();
    if (warp == 0 && lane == 0) {
        for (int g = 0; g < kChainMaxGemms; ++g) { tma_prefetch_desc(&maps.a[g]); tma_prefetch_desc(&maps.b[g]); }
        for (int i = 0; i < p.stages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 8); }   // empty: one arrive per consumer warp
        fence_barrier_init();
    }
    __syncthreads();

    // ---- pipeline state that survives the phases
    int p_stage = 0; uint32_t p_phase = 0;      // producer (warp 0, lane 0)
    int pre_stage0 = 0, pre_n = 0, pre_for = -1; // weight tiles already in flight for GEMM phase `pre_for`
    int m_stage = 0; uint32_t m_phase = 0;      // consumer warpgroups (both walk the ring in step)

    auto work_of = [&](const PhaseK& P, int* tile, int* split) -> bool {
        const int w = blockIdx.x;
        if (w >= P.tiles * P.splits) return false;
        *split = w % P.splits;
        *tile = w / P.splits;
        return true;
    };
    // producer thread only: put the weight (A) tiles of GEMM phase `g` in flight; legal before the data dependency on the previous
    // phase is resolved because weights never change
    auto prefetch_weights = [&](int g) {
        const PhaseK& P = p.ph[g];
        int tile, split;
        pre_for = g; pre_n = 0; pre_stage0 = p_stage;
        if (!work_of(P, &tile, &split)) return;
        const int n_pre = P.kb_per_split < p.stages ? P.kb_per_split : p.stages;
        for (int i = 0; i < n_pre; ++i) {
            mbar_wait_bounded(&empty_bar[p_stage], p_phase ^ 1);
            uint8_t* sa = smem + (size_t)p_stage * stage_bytes;
            mbar_expect_tx(&full_bar[p_stage], (uint32_t)stage_bytes);
            tma_load_2d(sa, &maps.a[P.map], &full_bar[p_stage], (split * P.kb_per_split + i) * kK, tile * kM);
            if (++p_stage == p.stages) { p_stage = 0; p_phase ^= 1; }
        }
        pre_n = n_pre;
    };

    // the first phase is always a GEMM: its weights go out before griddepcontrol.wait, everything else after
    if (warp == 0 && lane == 0 && p.ph[0].kind == 0) prefetch_weights(0);
    pdl_wait();
    // every kernel upstream of this one has completed: the barrier words of the sibling chain (last used before this launch) can be
    // re-armed here, which keeps memset nodes out of the step graph
    if (blockIdx.x == 0 && threadIdx.x < 8 && p.reset != nullptr) p.reset[threadIdx.x] = 0u;

    for (int ph = 0; ph < p.n_phases; ++ph) {
        const PhaseK& P = p.ph[ph];
        if (P.kind == 0) {
            int tile = 0, split = 0;
            const bool has = work_of(P, &tile, &split);
            if (has && warp == 0) {
                if (lane == 0) {
                    // ===================== TMA producer =====================
                    if (pre_for != ph) prefetch_weights(ph);   // (only if the previous phase could not prefetch)
                    const int kb0 = split * P.kb_per_split;
                    fence_generic_to_async_global();           // the activations were written with generic stores by other CTAs (acquired at the barrier)
                    for (int i = 0; i < pre_n; ++i) {          // activations for the weight tiles already in flight
                        const int st = (pre_stage0 + i) % p.stages;
                        tma_load_2d(smem + (size_t)st * stage_bytes + kStageABytes, &maps.b[P.map], &full_bar[st], (kb0 + i) * kK, 0);
                    }
                    for (int kb = kb0 + pre_n; kb < kb0 + P.kb_per_split; ++kb) {
                        mbar_wait_bounded(&empty_bar[p_stage], p_phase ^ 1);
                        uint8_t* sa = smem + (size_t)p_stage * stage_bytes;
                        mbar_expect_tx(&full_bar[p_stage], (uint32_t)stage_bytes);
                        tma_load_2d(sa, &maps.a[P.map], &full_bar[p_stage], kb * kK, tile * kM);
                        tma_load_2d(sa + kStageABytes, &maps.b[P.map], &full_bar[p_stage], kb * kK, 0);
                        if (++p_stage == p.stages) { p_stage = 0; p_phase ^= 1; }
                    }
                    pre_for = -1;
                }
            } else if (has && warp >= 4) {
                // ===================== wgmma consumers: weight rows [64 cw, 64 cw + 64) of the tile =====================
                const int cw = (warp >> 2) - 1;
                float acc[BN / 2];
                int prev = -1;
                for (int kb = 0; kb < P.kb_per_split; ++kb) {
                    mbar_wait_bounded(&full_bar[m_stage], m_phase);
                    const uint32_t sa = smem_u32(smem + (size_t)m_stage * stage_bytes);
                    const uint64_t adesc = wgmma_desc_sw128(sa + cw * 64 * 128);
                    const uint64_t bdesc = wgmma_desc_sw128(sa + kStageABytes);
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < kK / 16; ++k)
                        Wgmma<T, BN>::ss(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (kb > 0 || k > 0) ? 1u : 0u);
                    wgmma_commit();
                    wgmma_wait<1>();
                    if (prev >= 0) {
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&empty_bar[prev]);
                    }
                    prev = m_stage;
                    if (++m_stage == p.stages) { m_stage = 0; m_phase ^= 1; }
                }
                wgmma_wait<0>();
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty_bar[prev]);
                // ===================== epilogue: transposed f32 partial store [split][b][n] =====================
                const int c_lo = 2 * (lane & 3);
#pragma unroll
                for (int hf = 0; hf < 2; ++hf) {
                    const int row = tile * kM + cw * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * hf;
                    if (row >= P.n) continue;
#pragma unroll
                    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int col = 8 * j + c_lo + e;
                            if (col < p.Bp) p.partial[((long long)split * p.Bp + col) * P.n + row] = acc[4 * j + 2 * hf + e];
                        }
                }
            }
        } else {
            // the producer thread first puts the NEXT GEMM phase's weight tiles in flight (all ring stages are free: the grid barrier
            // after the previous GEMM phase implies its MMAs have retired), then joins the reduction
            if (warp == 0 && lane == 0 && ph + 1 < p.n_phases && p.ph[ph + 1].kind == 0) prefetch_weights(ph + 1);
            __syncwarp();
            if (P.kind == 1) {
                for (int b = blockIdx.x; b < p.B; b += gridDim.x) reduce_ln_row<T>(p, P, b, scratch);   // rows beyond one per CTA (beam search: up to 256 rows)
            } else {
                reduce_gelu_all<T>(p, P);
            }
        }
        if (ph + 1 < p.n_phases) grid_barrier(p.counters + ph, gridDim.x, P.kind != 0);
    }
}

template <typename T, int BN>
cudaError_t launch_chain(const ChainMaps& maps, const ChainK& p, int grid, size_t smem, int pdl, cudaStream_t stream) {
    static bool attr = false;
    if (!attr) {
        const cudaError_t e = cudaFuncSetAttribute(decoder_chain_kernel<T, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 210 * 1024);
        if (e != cudaSuccess) return e;
        attr = true;
    }
    return launch_k(decoder_chain_kernel<T, BN>, dim3(grid), dim3(kThreads), smem, stream, pdl, maps, p);
}

template <typename T>
cudaError_t launch_chain_n(int bn, const ChainMaps& maps, const ChainK& p, int grid, size_t smem, int pdl, cudaStream_t stream) {
    switch (bn) {
        case 16: return launch_chain<T, 16>(maps, p, grid, smem, pdl, stream);
        case 32: return launch_chain<T, 32>(maps, p, grid, smem, pdl, stream);
        case 64: return launch_chain<T, 64>(maps, p, grid, smem, pdl, stream);
        case 128: return launch_chain<T, 128>(maps, p, grid, smem, pdl, stream);
        default: return launch_chain<T, 256>(maps, p, grid, smem, pdl, stream);
    }
}

}  // namespace

wk_status decoder_chain(const ChainDesc& c, int num_sms, cudaStream_t stream) {
    if (c.n_phases < 1 || c.n_phases > kChainMaxPhases || c.Bp % 16 != 0 || c.Bp < 16 || c.Bp > 256 || c.ph[0].kind != 0) {
        set_error("decoder_chain: unsupported chain (phases %d, Bp %d)", c.n_phases, c.Bp);
        return WK_ERR_INVALID_ARGUMENT;
    }
    ChainMaps maps;
    ChainK p;
    memset(&maps, 0, sizeof(maps));
    memset(&p, 0, sizeof(p));
    p.n_phases = c.n_phases; p.partial = c.partial; p.x = c.x; p.B = c.B; p.Bp = c.Bp; p.d = c.d; p.counters = c.counters; p.reset = c.reset_counters;
    const int bn = wgmma_tile_n(c.Bp);   // wgmma N: Bp rounded up to a power of two (rows past Bp are zero-filled by TMA)
    p.stage_b_bytes = bn * kK * 2;
    if (p.stage_b_bytes % 1024) p.stage_b_bytes = (p.stage_b_bytes + 1023) / 1024 * 1024;
    int n_gemm = 0, max_kb = 1, last_gemm = -1;
    for (int i = 0; i < c.n_phases; ++i) {
        const ChainPhaseDesc& s = c.ph[i];
        PhaseK& k = p.ph[i];
        k.kind = s.kind;
        if (s.kind == 0) {
            if (n_gemm >= kChainMaxGemms || s.k % kK || s.splits < 1 || (s.k / kK) % s.splits) { set_error("decoder_chain: bad GEMM phase %d", i); return WK_ERR_INVALID_ARGUMENT; }
            k.map = n_gemm; k.n = s.n; k.splits = s.splits; k.kb_per_split = s.k / kK / s.splits; k.tiles = (s.n + kM - 1) / kM;
            if (k.tiles * k.splits > num_sms) { set_error("decoder_chain: GEMM phase %d needs %d CTAs (> %d SMs)", i, k.tiles * k.splits, num_sms); return WK_ERR_INVALID_ARGUMENT; }
            WK_CHECK_STATUS(make_tmap_2d(&maps.a[n_gemm], s.w, c.dtype, (uint64_t)s.k, (uint64_t)s.n, (uint64_t)s.k, kK, kM));
            WK_CHECK_STATUS(make_tmap_2d(&maps.b[n_gemm], s.act, c.dtype, (uint64_t)s.k, (uint64_t)c.Bp, (uint64_t)s.k, kK, (uint32_t)bn));
            max_kb = std::max(max_kb, k.kb_per_split);
            last_gemm = i;
            ++n_gemm;
        } else {
            if (last_gemm != i - 1) { set_error("decoder_chain: reduce phase %d must follow a GEMM phase", i); return WK_ERR_INVALID_ARGUMENT; }
            k.red_n = p.ph[i - 1].n; k.red_splits = p.ph[i - 1].splits;
            k.bias = s.bias; k.gamma = s.gamma; k.beta = s.beta; k.out16 = s.out16;
            if (k.red_splits > kMaxSplitsR || (k.red_n & 3) || (s.kind == 1 && (k.red_n != c.d || c.d > 8 * kThreads))) {
                set_error("decoder_chain: unsupported reduce phase %d", i); return WK_ERR_INVALID_ARGUMENT;
            }
        }
    }
    // unused tensor-map slots must still be valid descriptors (they are prefetched): repeat the first pair
    for (int g = n_gemm; g < kChainMaxGemms; ++g) { maps.a[g] = maps.a[0]; maps.b[g] = maps.b[0]; }
    const int stage_bytes = kStageABytes + p.stage_b_bytes;
    p.stages = std::min(kRingMax, std::max(2, max_kb));
    while ((size_t)p.stages * stage_bytes + 2048 > 200 * 1024 && p.stages > 2) --p.stages;
    const size_t smem = (size_t)p.stages * stage_bytes + 1024 + 1024;
    cudaError_t e = c.dtype == WK_DTYPE_F16 ? launch_chain_n<__half>(bn, maps, p, num_sms, smem, c.pdl ? 16 : 0, stream)
                                            : launch_chain_n<__nv_bfloat16>(bn, maps, p, num_sms, smem, c.pdl ? 16 : 0, stream);
    count_launch();
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("decoder_chain launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

}  // namespace wk
