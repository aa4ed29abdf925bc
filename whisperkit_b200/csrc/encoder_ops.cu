// Encoder-side kernels besides the GEMM: LayerNorm, non-causal multi-head attention (S = 1500, d_head = 64),
// layout conversion for host readback, weight initialisation.
// Reference counterpart: the inside of AudioEncoder.mlmodelc (Sources/WhisperKit/Core/AudioEncoder.swift:50-63).
#include <curand_kernel.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "kernels.h"

namespace wk {

// =====================================================================================================
// LayerNorm: one warp per row, row kept in registers (two-pass mean / variance in fp32, eps 1e-5)
// =====================================================================================================
// the row's (mean, rstd) from its NV float4 per lane
template <int NV>
__device__ __forceinline__ float2 ln_stats(const float4 (&v)[NV], int d) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) s += v[i].x + v[i].y + v[i].z + v[i].w;
    const float mean = warp_sum(s) / d;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, e = v[i].w - mean;
        q += a * a + b * b + c * c + e * e;
    }
    return make_float2(mean, rsqrtf(warp_sum(q) / d + 1e-5f));
}

template <int NV, typename OutT>
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                 OutT* __restrict__ out, long long rows, int d) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long row = (long long)blockIdx.x * 8 + warp;
    if (row >= rows) return;
    const float4* xr = reinterpret_cast<const float4*>(x + row * d);
    float4 v[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) v[i] = xr[lane + 32 * i];
    const float2 st = ln_stats<NV>(v, d);
    const float mean = st.x, rstd = st.y;
    const float4* g4 = reinterpret_cast<const float4*>(gamma);
    const float4* b4 = reinterpret_cast<const float4*>(beta);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const float4 g = __ldg(g4 + lane + 32 * i), bb = __ldg(b4 + lane + 32 * i);
        const float o0 = (v[i].x - mean) * rstd * g.x + bb.x, o1 = (v[i].y - mean) * rstd * g.y + bb.y;
        const float o2 = (v[i].z - mean) * rstd * g.z + bb.z, o3 = (v[i].w - mean) * rstd * g.w + bb.w;
        if constexpr (sizeof(OutT) == 4) {
            reinterpret_cast<float4*>(out + row * d)[lane + 32 * i] = make_float4(o0, o1, o2, o3);
        } else {
            uint2 pk;
            pk.x = T16<OutT>::pack2(o0, o1);
            pk.y = T16<OutT>::pack2(o2, o3);
            reinterpret_cast<uint2*>(out + row * d)[lane + 32 * i] = pk;
        }
    }
}

// The FP8 encoder policy's LayerNorm: the same f32 output, quantized without a 16-bit rounding.  The warp's v[i] is the row's 128-column
// block i, so the block's amax is one warp reduction; every lane stores its 4 codes, lane 0 the block scale to scales[i][row].
template <int NV>
__global__ void __launch_bounds__(256)
layernorm_fp8_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                     uint8_t* __restrict__ codes, float* __restrict__ scales, long long scale_ld, long long rows, int d) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long row = (long long)blockIdx.x * 8 + warp;
    if (row >= rows) return;
    const float4* xr = reinterpret_cast<const float4*>(x + row * d);
    float4 v[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) v[i] = xr[lane + 32 * i];
    const float2 st = ln_stats<NV>(v, d);
    const float mean = st.x, rstd = st.y;
    const float4* g4 = reinterpret_cast<const float4*>(gamma);
    const float4* b4 = reinterpret_cast<const float4*>(beta);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const float4 g = __ldg(g4 + lane + 32 * i), bb = __ldg(b4 + lane + 32 * i);
        const float o0 = (v[i].x - mean) * rstd * g.x + bb.x, o1 = (v[i].y - mean) * rstd * g.y + bb.y;
        const float o2 = (v[i].z - mean) * rstd * g.z + bb.z, o3 = (v[i].w - mean) * rstd * g.w + bb.w;
        const float s = fp8_row_scale(warp_max(fmaxf(fmaxf(fabsf(o0), fabsf(o1)), fmaxf(fabsf(o2), fabsf(o3)))));
        reinterpret_cast<uint32_t*>(codes + row * d)[lane + 32 * i] =
            (uint32_t)fp8_encode(o0, s) | ((uint32_t)fp8_encode(o1, s) << 8) | ((uint32_t)fp8_encode(o2, s) << 16) |
            ((uint32_t)fp8_encode(o3, s) << 24);
        if (lane == 0) scales[(long long)i * scale_ld + row] = s;
    }
}

template <typename OutT>
static wk_status launch_ln(const float* x, const float* g, const float* b, OutT* out, int64_t rows, int d, cudaStream_t st) {
    const unsigned grid = (unsigned)((rows + 7) / 8);
    switch (d / 128) {
        case 1: layernorm_kernel<1, OutT><<<grid, 256, 0, st>>>(x, g, b, out, rows, d); break;
        case 2: layernorm_kernel<2, OutT><<<grid, 256, 0, st>>>(x, g, b, out, rows, d); break;
        case 3: layernorm_kernel<3, OutT><<<grid, 256, 0, st>>>(x, g, b, out, rows, d); break;
        case 4: layernorm_kernel<4, OutT><<<grid, 256, 0, st>>>(x, g, b, out, rows, d); break;
        case 6: layernorm_kernel<6, OutT><<<grid, 256, 0, st>>>(x, g, b, out, rows, d); break;
        case 8: layernorm_kernel<8, OutT><<<grid, 256, 0, st>>>(x, g, b, out, rows, d); break;
        case 10: layernorm_kernel<10, OutT><<<grid, 256, 0, st>>>(x, g, b, out, rows, d); break;
        default: set_error("layernorm: unsupported d_model %d", d); return WK_ERR_INVALID_ARGUMENT;
    }
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("layernorm launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

wk_status layernorm_f32_to_16(const float* x, const float* gamma, const float* beta, void* out, int64_t rows, int d, int dtype,
                              cudaStream_t stream) {
    if (d % 128 != 0) { set_error("layernorm: d_model %d not a multiple of 128", d); return WK_ERR_INVALID_ARGUMENT; }
    if (dtype == WK_DTYPE_F16) return launch_ln<__half>(x, gamma, beta, (__half*)out, rows, d, stream);
    return launch_ln<__nv_bfloat16>(x, gamma, beta, (__nv_bfloat16*)out, rows, d, stream);
}
wk_status layernorm_f32_to_f32(const float* x, const float* gamma, const float* beta, float* out, int64_t rows, int d,
                               cudaStream_t stream) {
    if (d % 128 != 0) { set_error("layernorm: d_model %d not a multiple of 128", d); return WK_ERR_INVALID_ARGUMENT; }
    return launch_ln<float>(x, gamma, beta, out, rows, d, stream);
}

wk_status layernorm_f32_to_fp8(const float* x, const float* gamma, const float* beta, uint8_t* codes, float* scales, int64_t scale_ld,
                               int64_t rows, int d, cudaStream_t st) {
    const unsigned grid = (unsigned)((rows + 7) / 8);
    switch (d / 128) {
        case 1: layernorm_fp8_kernel<1><<<grid, 256, 0, st>>>(x, gamma, beta, codes, scales, scale_ld, rows, d); break;
        case 2: layernorm_fp8_kernel<2><<<grid, 256, 0, st>>>(x, gamma, beta, codes, scales, scale_ld, rows, d); break;
        case 3: layernorm_fp8_kernel<3><<<grid, 256, 0, st>>>(x, gamma, beta, codes, scales, scale_ld, rows, d); break;
        case 4: layernorm_fp8_kernel<4><<<grid, 256, 0, st>>>(x, gamma, beta, codes, scales, scale_ld, rows, d); break;
        case 6: layernorm_fp8_kernel<6><<<grid, 256, 0, st>>>(x, gamma, beta, codes, scales, scale_ld, rows, d); break;
        case 8: layernorm_fp8_kernel<8><<<grid, 256, 0, st>>>(x, gamma, beta, codes, scales, scale_ld, rows, d); break;
        case 10: layernorm_fp8_kernel<10><<<grid, 256, 0, st>>>(x, gamma, beta, codes, scales, scale_ld, rows, d); break;
        default: set_error("layernorm: unsupported d_model %d", d); return WK_ERR_INVALID_ARGUMENT;
    }
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("layernorm launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

// One output channel (weight row) per block: s = amax(|row|) / 448 over the whole row, then the row's codes
template <typename T>
__global__ void __launch_bounds__(256)
quantize_weight_rows_kernel(const T* __restrict__ w, uint8_t* __restrict__ codes, float* __restrict__ scales, int k) {
    __shared__ float red[8];
    const T* wr = w + (long long)blockIdx.x * k;
    float amax = 0.f;
    for (int i = threadIdx.x; i < k; i += 256) amax = fmaxf(amax, fabsf(T16<T>::to_f(wr[i])));
    amax = warp_max(amax);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = amax;
    __syncthreads();
    amax = red[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) amax = fmaxf(amax, red[i]);
    const float s = fp8_row_scale(amax);
    for (int i = threadIdx.x; i < k; i += 256) codes[(long long)blockIdx.x * k + i] = fp8_encode(T16<T>::to_f(wr[i]), s);
    if (threadIdx.x == 0) scales[blockIdx.x] = s;
}

wk_status quantize_weight_rows_fp8(const void* w, int dtype, uint8_t* codes, float* scales, int64_t rows, int k, cudaStream_t stream) {
    if (dtype == WK_DTYPE_F16) quantize_weight_rows_kernel<__half><<<(unsigned)rows, 256, 0, stream>>>((const __half*)w, codes, scales, k);
    else quantize_weight_rows_kernel<__nv_bfloat16><<<(unsigned)rows, 256, 0, stream>>>((const __nv_bfloat16*)w, codes, scales, k);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("quantize_weight_rows_fp8 launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

// Encoder attention lives in attention_wgmma.cu (TMA + wgmma); this is only its entry point.
wk_status encoder_attention(const void* qkv, void* out, int B, int T, int n_heads, int dtype, cudaStream_t stream) {
    return encoder_attention_wgmma(qkv, out, B, T, n_heads, dtype, stream);
}

// =====================================================================================================
// Helpers: host-layout readback, random init, dtype conversion
// =====================================================================================================
// dst[b][c][r] (f32) = src[b][row_off + r][c]   (time-major device layout -> channel-major reference layout)
template <typename T>
__global__ void transpose_to_host_kernel(const T* __restrict__ src, float* __restrict__ dst, long long rows, long long cols,
                                         long long src_rows_alloc, long long row_off, long long src_ld) {
    __shared__ float tile[32][33];
    const long long b = blockIdx.z;
    const long long r0 = (long long)blockIdx.x * 32, c0 = (long long)blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += 8) {
        const long long r = r0 + i, c = c0 + threadIdx.x;
        float v = 0.f;
        if (r < rows && c < cols) {
            const T* p = src + (b * src_rows_alloc + row_off + r) * src_ld + c;
            if constexpr (sizeof(T) == 4) v = *p; else v = T16<T>::to_f(*p);
        }
        tile[i][threadIdx.x] = v;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += 8) {
        const long long c = c0 + i, r = r0 + threadIdx.x;
        if (r < rows && c < cols) dst[(b * cols + c) * rows + r] = tile[threadIdx.x][i];
    }
}

wk_status transpose_to_host_layout(const void* src, float* dst, int64_t B, int64_t rows, int64_t cols, int64_t src_rows_alloc,
                                   int64_t src_row_off, int64_t src_ld, int dtype, cudaStream_t stream) {
    dim3 grid((unsigned)((rows + 31) / 32), (unsigned)((cols + 31) / 32), (unsigned)B), block(32, 8);
    if (dtype == WK_DTYPE_F32) transpose_to_host_kernel<float><<<grid, block, 0, stream>>>((const float*)src, dst, rows, cols, src_rows_alloc, src_row_off, src_ld);
    else if (dtype == WK_DTYPE_F16) transpose_to_host_kernel<__half><<<grid, block, 0, stream>>>((const __half*)src, dst, rows, cols, src_rows_alloc, src_row_off, src_ld);
    else transpose_to_host_kernel<__nv_bfloat16><<<grid, block, 0, stream>>>((const __nv_bfloat16*)src, dst, rows, cols, src_rows_alloc, src_row_off, src_ld);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("transpose launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

template <typename T>
__global__ void fill_random_kernel(T* dst, long long n, unsigned long long seed, float std, float mean) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long base = i * 4;
    if (base >= n) return;
    curandStatePhilox4_32_10_t st;
    curand_init(seed, (unsigned long long)i, 0, &st);
    const float4 r = curand_normal4(&st);
    const float v[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int k = 0; k < 4; ++k)
        if (base + k < n) {
            const float f = mean + std * v[k];
            if constexpr (sizeof(T) == 4) dst[base + k] = f; else dst[base + k] = T16<T>::from_f(f);
        }
}

wk_status fill_random_16(void* dst, int64_t n, uint64_t seed, float std, float mean, int dtype, cudaStream_t stream) {
    const unsigned grid = (unsigned)((n / 4 + 256) / 256);
    if (dtype == WK_DTYPE_F16) fill_random_kernel<__half><<<grid, 256, 0, stream>>>((__half*)dst, n, seed, std, mean);
    else fill_random_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>((__nv_bfloat16*)dst, n, seed, std, mean);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("fill_random launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}
wk_status fill_random_f32(float* dst, int64_t n, uint64_t seed, float std, float mean, cudaStream_t stream) {
    const unsigned grid = (unsigned)((n / 4 + 256) / 256);
    fill_random_kernel<float><<<grid, 256, 0, stream>>>(dst, n, seed, std, mean);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("fill_random launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

template <typename S, typename D>
__global__ void convert_kernel(const S* __restrict__ src, D* __restrict__ dst, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float v;
    if constexpr (sizeof(S) == 4) v = src[i]; else v = T16<S>::to_f(src[i]);
    if constexpr (sizeof(D) == 4) dst[i] = v; else dst[i] = T16<D>::from_f(v);
}

wk_status convert_to_16(const void* src, int src_dtype, void* dst, int dst_dtype, int64_t n, cudaStream_t stream) {
    const unsigned grid = (unsigned)((n + 255) / 256);
#define WK_CVT(S, D) convert_kernel<S, D><<<grid, 256, 0, stream>>>((const S*)src, (D*)dst, n)
    if (src_dtype == WK_DTYPE_F32 && dst_dtype == WK_DTYPE_BF16) WK_CVT(float, __nv_bfloat16);
    else if (src_dtype == WK_DTYPE_F32 && dst_dtype == WK_DTYPE_F16) WK_CVT(float, __half);
    else if (src_dtype == WK_DTYPE_F32 && dst_dtype == WK_DTYPE_F32) WK_CVT(float, float);
    else if (src_dtype == WK_DTYPE_BF16 && dst_dtype == WK_DTYPE_BF16) WK_CVT(__nv_bfloat16, __nv_bfloat16);
    else if (src_dtype == WK_DTYPE_BF16 && dst_dtype == WK_DTYPE_F16) WK_CVT(__nv_bfloat16, __half);
    else if (src_dtype == WK_DTYPE_BF16 && dst_dtype == WK_DTYPE_F32) WK_CVT(__nv_bfloat16, float);
    else if (src_dtype == WK_DTYPE_F16 && dst_dtype == WK_DTYPE_F16) WK_CVT(__half, __half);
    else if (src_dtype == WK_DTYPE_F16 && dst_dtype == WK_DTYPE_BF16) WK_CVT(__half, __nv_bfloat16);
    else if (src_dtype == WK_DTYPE_F16 && dst_dtype == WK_DTYPE_F32) WK_CVT(__half, float);
    else { set_error("convert: unsupported dtype pair %d -> %d", src_dtype, dst_dtype); return WK_ERR_INVALID_ARGUMENT; }
#undef WK_CVT
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("convert launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

}  // namespace wk
