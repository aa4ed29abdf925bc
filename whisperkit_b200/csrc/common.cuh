// Common device helpers for the wkb200 kernels (sm_90a).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

namespace wk {

// ------------------------------------------------------------------ 16-bit type traits
template <typename T> struct T16;
template <> struct T16<__nv_bfloat16> {
    __device__ __forceinline__ static float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
    __device__ __forceinline__ static __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
    __device__ __forceinline__ static uint32_t pack2(float a, float b) {
        __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
        return *reinterpret_cast<uint32_t*>(&t);
    }
    __device__ __forceinline__ static float2 unpack2(uint32_t u) {
        __nv_bfloat162 t = *reinterpret_cast<__nv_bfloat162*>(&u);
        return __bfloat1622float2(t);
    }
};
template <> struct T16<__half> {
    __device__ __forceinline__ static float to_f(__half v) { return __half2float(v); }
    __device__ __forceinline__ static __half from_f(float v) { return __float2half_rn(v); }
    __device__ __forceinline__ static uint32_t pack2(float a, float b) {
        __half2 t = __floats2half2_rn(a, b);
        return *reinterpret_cast<uint32_t*>(&t);
    }
    __device__ __forceinline__ static float2 unpack2(uint32_t u) {
        __half2 t = *reinterpret_cast<__half2*>(&u);
        return __half22float2(t);
    }
};

// ------------------------------------------------------------------ FP8 (E4M3) quantization
// A group of values (a 64-value cross-attention K/V row; under the FP8 encoder policy a 128-column block of an activation row, or a
// whole weight row) is stored as E4M3 codes plus one f32 scale s = amax(|group|) / 448; code = cvt.rn.satfinite.e4m3(x / s) and the
// stored value is code * s.  A group whose amax is 0 gets s = 0 and all-zero codes.  The GEMM epilogues (gemm_wgmma.cu), the FP8
// LayerNorm and weight quantizer (encoder_ops.cu) and the host test entries (wk_cross_kv_quantize_rows, wk_fp8_quantize_blocks) all go
// through these two functions, so the CPU tests pin the rounding the GPU does.
constexpr float kFp8E4M3Max = 448.f;
constexpr int kFp8Block = 128;   // columns per activation scale of the FP8 encoder GEMMs (one 128-byte swizzle row, one k-block)
__host__ __device__ __forceinline__ float fp8_row_scale(float amax) { return amax / kFp8E4M3Max; }
__host__ __device__ __forceinline__ uint8_t fp8_encode(float x, float s) {
    return s > 0.f ? (uint8_t)__nv_cvt_float_to_fp8(x / s, __NV_SATFINITE, __NV_E4M3) : (uint8_t)0;
}
__host__ __device__ inline void fp8_quantize_row(const float* x, int n, uint8_t* codes, float* scale) {
    float amax = 0.f;
    for (int i = 0; i < n; ++i) amax = fmaxf(amax, fabsf(x[i]));
    const float s = fp8_row_scale(amax);
    for (int i = 0; i < n; ++i) codes[i] = fp8_encode(x[i], s);
    *scale = s;
}
// code -> value (exact: every E4M3 value is a f16 value)
__host__ __device__ inline float fp8_decode(uint8_t code) {
    const __half_raw h = __nv_cvt_fp8_to_halfraw((__nv_fp8_storage_t)code, __NV_E4M3);
    return __half2float(__half(h));
}
// four codes (little-endian in a word) -> two exact f16 pairs (cvt.rn.f16x2.e4m3x2)
__device__ __forceinline__ void fp8x4_to_half2(uint32_t w, uint32_t& lo, uint32_t& hi) {
    const __half2_raw a = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(w & 0xffffu), __NV_E4M3);
    const __half2_raw b = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(w >> 16), __NV_E4M3);
    lo = (uint32_t)a.x | ((uint32_t)a.y << 16);
    hi = (uint32_t)b.x | ((uint32_t)b.y << 16);
}

// Packed bf16 cross K/V cache (12 bits per value, lossless).  Block (layer, K|V, slot, head) keeps its T x 128-byte region:
//   primary slot of row t at t * 96: 64 sign|mantissa bytes (value i -> byte i: sign in bit 7, mantissa in bits 0..6), then 32 bytes of
//     exponent offsets, 4 bytes per group of 8 values (group g at 64 + 4 g); value 8 g + j sits at bit 16 (j & 1) + 4 (j >> 1) of its word
//   secondary slot of row t at T * 96 + t * 32: bytes 96..127 of a raw row
//   header byte of row t (a separate [block][round_up(T, 16)] vector): the row's largest exponent field `base`, offset = base - field
//   (0..15), or kPackedRaw: the row spans more than 16 binades or holds Inf/NaN and keeps its 128 raw bytes (0..95 primary, 96..127
//   secondary).  Exponent fields are coded as bits, so zeros and subnormals (field 0) need no special case.
static constexpr int kPackedRowBytes = 96;
static constexpr uint8_t kPackedRaw = 255;
__host__ __device__ inline int packed_hdr_stride(int T) { return (T + 15) & ~15; }
// the bf16 bits of one group of 8 values of a packed row, as the uint4 the raw row holds there
__device__ __forceinline__ uint4 unpack_bf16x8(uint2 sm, uint32_t nib, uint32_t base) {
    const uint32_t b7 = (base << 7) | (base << 23);
    const uint32_t nh = nib >> 8;
    // prmt: sign|mantissa byte k into bits 0..7 of its 16-bit half and its sign replicated into bits 8..15; & 0x807f keeps sign and mantissa
    uint4 u;
    u.x = (__byte_perm(sm.x, 0, 0x9180) & 0x807f807fu) | (b7 - (nib & 0x000f000fu) * 128u);
    u.y = (__byte_perm(sm.x, 0, 0xb3a2) & 0x807f807fu) | (b7 - (nib & 0x00f000f0u) * 8u);
    u.z = (__byte_perm(sm.y, 0, 0x9180) & 0x807f807fu) | (b7 - (nh & 0x000f000fu) * 128u);
    u.w = (__byte_perm(sm.y, 0, 0xb3a2) & 0x807f807fu) | (b7 - (nh & 0x00f000f0u) * 8u);
    return u;
}
// 8 values (16 bytes) of row t of a packed block: group g of a coded row, or bytes 16 g .. 16 g + 15 of a raw row
__device__ __forceinline__ uint4 packed_group(const uint8_t* blk, int T, int t, int g, uint8_t hdr) {
    const uint8_t* row = blk + (long long)t * kPackedRowBytes;
    if (hdr == kPackedRaw)
        return *reinterpret_cast<const uint4*>(g < 6 ? row + 16 * g : blk + (long long)T * kPackedRowBytes + (long long)t * 32 + 16 * (g - 6));
    return unpack_bf16x8(*reinterpret_cast<const uint2*>(row + 8 * g), *reinterpret_cast<const uint32_t*>(row + 64 + 4 * g), hdr);
}

__device__ __forceinline__ float gelu_erf(float x) {
    // exact (erf) GELU with erf from Abramowitz-Stegun 7.1.26 (|error| <= 1.5e-7, far below the 16-bit storage step of the output):
    // ~13 instructions and 2 MUFU ops against libdevice erff's two divergent polynomial branches - the FC1 epilogue is bound by this
    const float z = fabsf(x) * 0.70710678118654752440f;
    const float t = __fdividef(1.0f, fmaf(0.3275911f, z, 1.0f));
    float poly = fmaf(1.061405429f, t, -1.453152027f);
    poly = fmaf(poly, t, 1.421413741f);
    poly = fmaf(poly, t, -0.284496736f);
    poly = fmaf(poly, t, 0.254829592f);
    const float erf_abs = fmaf(-poly * t, __expf(-z * z), 1.0f);
    return 0.5f * x * (1.0f + copysignf(erf_abs, x));
}

// f32 pair arithmetic: the pair helpers keep the epilogue code written two values at a time
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(a.x * b.x, a.y * b.y); }
// gelu_erf on two values at once (the FC1 epilogue is bound by its instruction issue: ex2.approx instead of __expf's range handling)
__device__ __forceinline__ float2 gelu_erf2(float2 x) {
    const float2 z = make_float2(fabsf(x.x) * 0.70710678118654752440f, fabsf(x.y) * 0.70710678118654752440f);
    const float2 den = fma2(make_float2(0.3275911f, 0.3275911f), z, make_float2(1.0f, 1.0f));
    const float2 t = make_float2(__fdividef(1.0f, den.x), __fdividef(1.0f, den.y));
    float2 poly = fma2(make_float2(1.061405429f, 1.061405429f), t, make_float2(-1.453152027f, -1.453152027f));
    poly = fma2(poly, t, make_float2(1.421413741f, 1.421413741f));
    poly = fma2(poly, t, make_float2(-0.284496736f, -0.284496736f));
    poly = fma2(poly, t, make_float2(0.254829592f, 0.254829592f));
    const float2 nz2 = mul2(mul2(z, z), make_float2(-1.4426950408889634f, -1.4426950408889634f));   // -z^2 * log2(e)
    float2 e;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e.x) : "f"(nz2.x));
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e.y) : "f"(nz2.y));
    const float2 pt = mul2(make_float2(-poly.x, -poly.y), t);
    const float2 erf_abs = fma2(pt, e, make_float2(1.0f, 1.0f));
    const float2 hx = mul2(make_float2(0.5f, 0.5f), x);
    return fma2(hx, make_float2(copysignf(erf_abs.x, x.x), copysignf(erf_abs.y, x.y)), hx);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
// raise the transaction count of the current phase without arriving
__device__ __forceinline__ void mbar_expect_tx_only(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// Bounded mbarrier wait: a protocol bug must end as a trapped launch that the host reports, never as a GPU that spins until something
// kills the process.  2 s is >1000x the longest legitimate wait.
constexpr unsigned long long kSpinLimitNs = 2000000000ull;
__device__ __forceinline__ void mbar_wait_bounded(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const unsigned long long t0 = globaltimer_ns();
    unsigned int spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if ((++spins & 0xfffu) == 0 && globaltimer_ns() - t0 > kSpinLimitNs) {
            printf("wkb200: mbarrier wait timed out (block %d thread %d)\n", (int)blockIdx.x, (int)threadIdx.x);
            __trap();
        }
    }
}

// ------------------------------------------------------------------ TMA
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1,
                                            int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], "
        "[%2];" ::"r"(smem_u32(smem_dst)),
        "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
// The same loads for a CONVERGED warp: every lane calls, the instruction is predicated on the lane elect.sync picks, so the issue
// path stays straight-line code (UTMALDG takes uniform-register operands; from an `if (lane == 0)` branch the compiler rebuilds them).
__device__ __forceinline__ void tma_load_2d_elect(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "{\n\t.reg .pred q;\n\t"
        "elect.sync _|q, 0xffffffff;\n\t"
        "@q cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];\n\t}"
        ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d_elect(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "{\n\t.reg .pred q;\n\t"
        "elect.sync _|q, 0xffffffff;\n\t"
        "@q cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];\n\t}"
        ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void bulk_load_1d_elect(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "{\n\t.reg .pred q;\n\t"
        "elect.sync _|q, 0xffffffff;\n\t"
        "@q cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n\t}"
        ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void mbar_expect_tx_elect(uint64_t* bar, uint32_t bytes) {
    asm volatile(
        "{\n\t.reg .pred q;\n\t"
        "elect.sync _|q, 0xffffffff;\n\t"
        "@q mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n\t}" ::"r"(smem_u32(bar)), "r"(bytes)
        : "memory");
}
// Shared -> global tensor store of one box (the tensor map clips what lies outside the tensor), tracked by bulk async-groups.  The
// smem writes it reads must be made visible to the async proxy first (fence_proxy_async + a barrier over the writing threads).
__device__ __forceinline__ void tma_store_3d(const void* tmap, const void* smem_src, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
                 ::"l"(tmap), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// every committed bulk store has finished reading shared memory (its source buffer may be rewritten)
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// every committed bulk store has completed (its writes are done)
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// barrier over the 128 threads of one warpgroup (named barrier `id`, 1..15; 0 is __syncthreads)
__device__ __forceinline__ void warpgroup_bar(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }
// four 8x8 16-bit matrices to shared memory: lane l gives the address of row l % 8 of matrix l / 8; register i of every lane holds
// matrix i's elements (row lane / 4, columns 2 (lane % 4), + 1) - the layout of a wgmma accumulator pair
__device__ __forceinline__ void stmatrix_x4(uint32_t smem_addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
    asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(smem_addr), "r"(r0), "r"(r1), "r"(r2), "r"(r3)
                 : "memory");
}
// 1-D bulk copy global -> shared, completion on an mbarrier (UBLKCP).
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(smem_dst)),
        "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}

// ------------------------------------------------------------------ programmatic dependent launch (PDL)
// launch_dependents: lets the next kernel in the stream start its prologue while this grid is still running;
// wait: blocks until the upstream grid has completed and its memory is visible.  Both are no-ops when the kernel
// was launched without the programmatic-serialization attribute.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ------------------------------------------------------------------ misc
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, bool pred) {
    uint32_t sz = pred ? 16u : 0u;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(sz)
                 : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// Host-side launcher: cudaLaunchKernelEx with the PDL attribute when enabled (WKB200_NO_PDL=1 disables it).
bool pdl_enabled();
// Bit mask of the kernel classes launched as programmatic dependents: 1 embed, 2 self-attention, 4 cross-attention, 8 sampler/advance,
// 16 GEMM, 32 split-K reduce.  Default 53; WKB200_PDL = 0 off, 1 all (63), 2 GEMM + reduce (48), 3 reduce only; WKB200_PDL_MASK overrides.
int pdl_mode();
void pdl_disable();
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, int pdl,
                            Args&&... args) {   // pdl: 0 never, else the class bit (see pdl_mode)
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = (pdl & pdl_mode()) ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace wk

#define WK_CUDA_CHECK(expr)                                                                   \
    do {                                                                                      \
        cudaError_t _e = (expr);                                                              \
        if (_e != cudaSuccess) {                                                              \
            wk::set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            return WK_ERR_CUDA;                                                               \
        }                                                                                     \
    } while (0)
