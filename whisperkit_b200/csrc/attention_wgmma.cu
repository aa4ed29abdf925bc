// K4: encoder self-attention (non-causal, head dim 64, S = 1500) on Hopper warpgroup MMAs (wgmma) with the probabilities kept in registers.
//
// One CTA = one (window, head, 128-query block).  384 threads = 3 warpgroups:
//   warpgroup 0     warp 0: TMA producer - Q once, then K / V tiles of 128 keys through 4-deep smem rings (128B swizzle); the rest of the
//                   warpgroup idles and hands its registers to the consumers (setmaxnreg)
//   warpgroups 1, 2 64 query rows each, per key tile j:
//                       S  = Q K_j^T        wgmma m64n128k16 x4, Q and K from shared memory, S in registers
//                       online softmax of S in registers (exact running maximum, 4 threads per row)
//                       O += P V_j          wgmma m64n64k16 x8, A = P from REGISTERS (the S accumulator layout is the A fragment
//                                           layout, so P never touches shared memory), B = V_j MN-major from shared memory
//                   Two consumer warpgroups share every K / V tile; while one runs its softmax the other's MMAs use the tensor cores.
// Q/K/V are read in place from the packed qkv activation [B*T, 3*d_model] through one 3-D tensor map (per-window out-of-bounds rows are
// zero-filled by TMA; keys >= T are masked to -inf before the softmax).
// Reference counterpart: inside AudioEncoder.mlmodelc (Sources/WhisperKit/Core/AudioEncoder.swift:59-62).
#include <stdio.h>
#include <stdlib.h>

#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace wk {

static constexpr int kFaThreads = 384;     // producer warpgroup + two consumer warpgroups
static constexpr int kFaBM = 128;          // queries per CTA (64 per consumer warpgroup)
static constexpr int kFaBN = 128;          // keys per tile
static constexpr int kFaD = 64;
static constexpr int kFaTile = kFaBN * kFaD * 2;   // 16 KiB: one K or V or Q tile, 128-byte rows
static constexpr int kFaStages = 4;
static constexpr int kFaSmem = kFaTile /*Q*/ + 2 * kFaStages * kFaTile /*K, V rings*/ + 1024 /*align*/ + 256 /*barriers*/;

struct FaParams {
    int T, H, dm, n_kv_tiles;
    float scale_log2e;
};

__device__ __forceinline__ float fa_ex2(float x) {   // MUFU.EX2: 2^x, ex2(-inf) = +0
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

template <typename T>
__global__ void __launch_bounds__(kFaThreads, 1)
encoder_attention_wgmma_kernel(const __grid_constant__ CUtensorMap tm_qkv, T* __restrict__ out, const FaParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sQ = smem;
    uint8_t* sK = sQ + kFaTile;
    uint8_t* sV = sK + kFaStages * kFaTile;
    uint64_t* bars = reinterpret_cast<uint64_t*>(sV + kFaStages * kFaTile);
    uint64_t* q_full = bars;                      // 1
    uint64_t* k_full = bars + 1;                  // kFaStages
    uint64_t* k_empty = k_full + kFaStages;
    uint64_t* v_full = k_empty + kFaStages;
    uint64_t* v_empty = v_full + kFaStages;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int bh = blockIdx.y;
    const int b = bh / p.H, h = bh % p.H;
    const int q0 = blockIdx.x * kFaBM;
    const int n = p.n_kv_tiles;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tm_qkv);
        mbar_init(q_full, 1);
        for (int i = 0; i < kFaStages; ++i) {
            mbar_init(&k_full[i], 1); mbar_init(&k_empty[i], 8);   // empty: one arrive per consumer warp
            mbar_init(&v_full[i], 1); mbar_init(&v_empty[i], 8);
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        // ============================ TMA producer ============================
        if (warp == 0 && lane == 0) {
            mbar_expect_tx(q_full, kFaTile);
            tma_load_3d(sQ, &tm_qkv, q_full, h * kFaD, q0, b);
            for (int j = 0; j < n; ++j) {
                const int st = j % kFaStages;
                const uint32_t ph = (j / kFaStages) & 1;
                mbar_wait_bounded(&k_empty[st], ph ^ 1);
                mbar_expect_tx(&k_full[st], kFaTile);
                tma_load_3d(sK + st * kFaTile, &tm_qkv, &k_full[st], p.dm + h * kFaD, j * kFaBN, b);
                mbar_wait_bounded(&v_empty[st], ph ^ 1);
                mbar_expect_tx(&v_full[st], kFaTile);
                tma_load_3d(sV + st * kFaTile, &tm_qkv, &v_full[st], 2 * p.dm + h * kFaD, j * kFaBN, b);
            }
        }
        return;
    }

    // ============================ consumers: 64 query rows per warpgroup ============================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int cw = (warp >> 2) - 1;
    const int c_lo = 2 * (lane & 3);           // this thread's columns inside every 8-column group
    const float c = p.scale_log2e;
    // K-major Q / K descriptors (SBO 1024); V is MN-major (d contiguous): 8-key groups 1024 B apart, 16 keys = 2 KiB per k-step
    const uint64_t qd = wgmma_desc_sw128(smem_u32(sQ + cw * 64 * 128));
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // rows r and r + 8 of this thread

    mbar_wait_bounded(q_full, 0);
    for (int j = 0; j < n; ++j) {
        const int st = j % kFaStages;
        const uint32_t ph = (j / kFaStages) & 1;
        float s[64];
        mbar_wait_bounded(&k_full[st], ph);
        const uint64_t kd = wgmma_desc_sw128(smem_u32(sK + st * kFaTile));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kFaD / 16; ++k) Wgmma<T, 128>::ss(s, qd + (uint64_t)(2 * k), kd + (uint64_t)(2 * k), k > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&k_empty[st]);

        const int valid = p.T - j * kFaBN;   // keys of this tile that exist (>= 128 except at the end)
        if (valid < kFaBN) {
#pragma unroll
            for (int jj = 0; jj < 16; ++jj)
#pragma unroll
                for (int e = 0; e < 4; ++e)
                    if (8 * jj + c_lo + (e & 1) >= valid) s[4 * jj + e] = -INFINITY;
        }
        uint32_t pa[8][4];
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            float mx = m_run[hf];
#pragma unroll
            for (int jj = 0; jj < 16; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * hf], s[4 * jj + 2 * hf + 1]));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            const float corr = fa_ex2((m_run[hf] - mx) * c);   // 0 on the first tile (m_run = -inf)
            m_run[hf] = mx;
            const float nmc = -mx * c;
            float sum = 0.f;
#pragma unroll
            for (int jj = 0; jj < 16; ++jj) {
                const float e0 = fa_ex2(fmaf(s[4 * jj + 2 * hf], c, nmc));
                const float e1 = fa_ex2(fmaf(s[4 * jj + 2 * hf + 1], c, nmc));
                sum += e0 + e1;
                // A fragment of k-step jj / 2: registers {row, keys 0-7}, {row + 8, keys 0-7}, {row, keys 8-15}, {row + 8, keys 8-15}
                pa[jj >> 1][(jj & 1) * 2 + hf] = T16<T>::pack2(e0, e1);
            }
            l_run[hf] = l_run[hf] * corr + sum;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) { o[4 * jj + 2 * hf] *= corr; o[4 * jj + 2 * hf + 1] *= corr; }
        }

        mbar_wait_bounded(&v_full[st], ph);
        const uint32_t vs = smem_u32(sV + st * kFaTile);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kFaBN / 16; ++kk) Wgmma<T, 64>::rs_bt(o, pa[kk], wgmma_desc_sw128(vs + kk * 2048), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&v_empty[st]);
    }

    // ---- epilogue: O / l, 16-bit, rows r and r + 8
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
        float l = l_run[hf];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        const float inv = 1.f / l;
        const int q = q0 + cw * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * hf;
        if (q >= p.T) continue;
        T* dst = out + ((long long)b * p.T + q) * p.dm + h * kFaD + c_lo;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
            *reinterpret_cast<uint32_t*>(dst + 8 * jj) = T16<T>::pack2(o[4 * jj + 2 * hf] * inv, o[4 * jj + 2 * hf + 1] * inv);
    }
}

// ------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                      const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                      CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

wk_status encoder_attention_wgmma(const void* qkv, void* out, int B, int T, int n_heads, int dtype, cudaStream_t stream) {
    static PFN_encodeTiled enc = nullptr;
    if (!enc) {
        void* fp = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
            set_error("cuTensorMapEncodeTiled entry point unavailable");
            return WK_ERR_CUDA;
        }
        enc = reinterpret_cast<PFN_encodeTiled>(fp);
    }
    const int dm = n_heads * 64;
    CUtensorMap tm;
    cuuint64_t gdim[3] = {(cuuint64_t)3 * dm, (cuuint64_t)T, (cuuint64_t)B};
    cuuint64_t gstr[2] = {(cuuint64_t)3 * dm * 2, (cuuint64_t)T * 3 * dm * 2};
    cuuint32_t box[3] = {64, 128, 1};
    cuuint32_t es[3] = {1, 1, 1};
    CUresult r = enc(&tm, dtype == WK_DTYPE_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3,
                     const_cast<void*>(qkv), gdim, gstr, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("attention tensor map encode failed: %d", (int)r); return WK_ERR_CUDA; }
    FaParams p;
    p.T = T; p.H = n_heads; p.dm = dm;
    p.n_kv_tiles = (T + kFaBN - 1) / kFaBN;
    p.scale_log2e = 0.125f * 1.4426950408889634f;
    dim3 grid((T + kFaBM - 1) / kFaBM, B * n_heads);
    cudaError_t e = cudaSuccess;
    if (dtype == WK_DTYPE_F16) {
        static bool set = false;
        if (!set) { e = cudaFuncSetAttribute(encoder_attention_wgmma_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFaSmem); set = e == cudaSuccess; }
        if (e == cudaSuccess) encoder_attention_wgmma_kernel<__half><<<grid, kFaThreads, kFaSmem, stream>>>(tm, (__half*)out, p);
    } else {
        static bool set = false;
        if (!set) { e = cudaFuncSetAttribute(encoder_attention_wgmma_kernel<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFaSmem); set = e == cudaSuccess; }
        if (e == cudaSuccess) encoder_attention_wgmma_kernel<__nv_bfloat16><<<grid, kFaThreads, kFaSmem, stream>>>(tm, (__nv_bfloat16*)out, p);
    }
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute(fa): %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    count_launch();
    e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("encoder_attention_wgmma launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

}  // namespace wk
