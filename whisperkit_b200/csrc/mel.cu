// K1: fused log-mel front end (FeatureExtracting.logMelSpectrogram,
// Sources/WhisperKit/Core/FeatureExtractor.swift:40-56; padOrTrimAudio folded into the load,
// Sources/WhisperKit/Core/Audio/AudioProcessor.swift:151-174).
//
// HBM-bound by design: per 30 s window the kernel reads 480000 f32 once (float4, coalesced; reflect /
// zero padding resolved at load) and writes n_mels x 3000 16-bit values once.  Pass 1 stages 32 frames per
// CTA in shared memory, runs the 16x25 split real FFT + sparse mel + log10 entirely on chip and stores a
// u16 fixed-point code in the output buffer; pass 2 rewrites the (L2-resident) codes in place as f16 after the
// per-window max is known.  Output layout is time-major [window][3002][128] f16 with a zero row on both sides,
// i.e. exactly the K-major A operand of the conv-stem implicit GEMM (rows 1..3000 are frames 0..2999).
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <vector>

#include "common.cuh"
#include "kernels.h"
#include "mel_core.cuh"
#include "mel_tables.h"

namespace wk {

using namespace mel;

static constexpr int kPStride = kBins;  // floats per frame in the power buffer
static constexpr int kRegionA = (kF * kPStride > kSamplesPerCta ? kF * kPStride : kSamplesPerCta);  // samples | power

struct __align__(16) MelSmem {
    float a[kRegionA];               // phase 0/1: samples; phase 3/mel: power spectrum
    cf y[kF * kYPerFrame];           // twiddled 16-point outputs
    float win[kNfft];
    cf tw400[25 * kK1];
    cf tw25[25];
    float wts[kMaxTaps * kMelCols];
    int start[kMelCols];
};

__global__ void __launch_bounds__(kThreads, 2)
mel_pass1_kernel(const float* __restrict__ pcm, long long stride, const int* __restrict__ n_valid, MelTables t,
                 uint16_t* __restrict__ out, int* __restrict__ gmax, int ctas_per_window) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    MelSmem& s = *reinterpret_cast<MelSmem*>(smem_raw);
    const int tid = threadIdx.x;
    const int b = blockIdx.x / ctas_per_window;
    const int f0 = (blockIdx.x % ctas_per_window) * kF;
    const int nf = min(kF, kFramesPerWindow - f0);
    const float* x = pcm + (long long)b * stride;
    const int nv = n_valid ? n_valid[b] : kWindowSamples;

    // ---- tables -> smem
    for (int i = tid; i < kNfft; i += kThreads) s.win[i] = t.win[i];
    for (int i = tid; i < 25 * kK1; i += kThreads) s.tw400[i] = t.tw400[i];
    if (tid < 25) s.tw25[tid] = t.tw25[tid];
    for (int i = tid; i < kMaxTaps * kMelCols; i += kThreads) s.wts[i] = t.wts[i];
    if (tid < kMelCols) s.start[tid] = t.start[tid];

    // ---- phase 0: stage the samples of these frames (coalesced float4 on the interior)
    const int i0 = f0 * kHop - kNfft / 2;
    const int ns = (nf - 1) * kHop + kNfft;
    const bool interior = (i0 >= 0) && (i0 + ns <= nv) && ((stride & 3) == 0) &&
                          ((reinterpret_cast<uintptr_t>(pcm) & 15) == 0);
    if (interior) {
        const float4* x4 = reinterpret_cast<const float4*>(x + i0);  // i0 is a multiple of 8
        float4* a4 = reinterpret_cast<float4*>(s.a);
        for (int i = tid; i < ns / 4; i += kThreads) a4[i] = __ldg(x4 + i);
    } else {
        for (int i = tid; i < ns; i += kThreads) {
            const int j = reflect_index(i0 + i);
            s.a[i] = (j < nv) ? __ldg(x + j) : 0.f;
        }
    }
    __syncthreads();

    // ---- phase 1: 25 x 16-point real DFTs per frame
    for (int task = tid; task < nf * 25; task += kThreads) {
        const int f = task / 25, n2 = task - f * 25;
        phase1_task(s.a + f * kHop, s.win, s.tw400, n2, s.y + f * kYPerFrame);
    }
    __syncthreads();

    // ---- phase 3: 9 x 25-point DFTs per frame -> power spectrum (overwrites the sample region)
    for (int task = tid; task < nf * kK1; task += kThreads) {
        const int f = task / kK1, k1 = task - f * kK1;
        phase3_task(s.y + f * kYPerFrame, s.tw25, k1, s.a + f * kPStride);
    }
    __syncthreads();

    // ---- mel filterbank + log10 -> u16 code, coalesced 16-bit stores (128 mels = 256 B per frame row)
    int lmax = 0;
    const int n_mels = t.n_mels;
    for (int task = tid; task < nf * n_mels; task += kThreads) {
        const int f = task / n_mels, m = task - f * n_mels;
        const uint32_t q = mel_task(s.a + f * kPStride, s.wts, s.start, m, kMelCols);
        lmax = max(lmax, (int)q);
        out[((long long)b * kMelRows + 1 + f0 + f) * kMelCols + m] = (uint16_t)q;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) lmax = max(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
    if ((tid & 31) == 0) atomicMax(&gmax[b], lmax);
}

__global__ void __launch_bounds__(256)
mel_pass2_kernel(uint16_t* __restrict__ io, const int* __restrict__ gmax, int n_mels, long long n_rows_total) {
    // one thread per 8 mel columns (16 B); rows = windows * 3000 frames
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int cols8 = kMelCols / 8;
    const long long row = idx / cols8;
    const int c8 = (int)(idx - row * cols8);
    if (row >= n_rows_total) return;
    const long long b = row / kFramesPerWindow;
    const long long f = row - b * kFramesPerWindow;
    if (c8 * 8 >= n_mels) return;
    uint4* p = reinterpret_cast<uint4*>(io + (b * kMelRows + 1 + f) * kMelCols + c8 * 8);
    const uint32_t qmax = (uint32_t)gmax[b];
    uint4 v = *p;
    uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float lo = mel_normalise(w[i] & 0xffffu, qmax);
        const float hi = mel_normalise(w[i] >> 16, qmax);
        __half2 h = __floats2half2_rn(lo, hi);
        w[i] = *reinterpret_cast<uint32_t*>(&h);
    }
    *p = make_uint4(w[0], w[1], w[2], w[3]);
}

// ------------------------------------------------------------------------------------------------
wk_status mel_tables_create(int n_mels, Buffers& mem, MelTables* t) {
    if (n_mels != 80 && n_mels != 128) {
        set_error("mel: n_mels must be 80 or 128 (got %d)", n_mels);
        return WK_ERR_INVALID_ARGUMENT;
    }
    std::vector<float> win, wts;
    std::vector<cf> tw400, tw25;
    std::vector<int> start;
    mel_host_tables(n_mels, win, tw400, tw25, wts, start);
    t->n_mels = n_mels;
    WK_CHECK(mem.dmalloc(&t->win, win.size(), false));
    WK_CHECK(mem.dmalloc(&t->tw400, tw400.size(), false));
    WK_CHECK(mem.dmalloc(&t->tw25, tw25.size(), false));
    WK_CHECK(mem.dmalloc(&t->wts, wts.size(), false));
    WK_CHECK(mem.dmalloc(&t->start, start.size(), false));
    WK_CUDA_CHECK(cudaMemcpy(t->win, win.data(), win.size() * sizeof(float), cudaMemcpyHostToDevice));
    WK_CUDA_CHECK(cudaMemcpy(t->tw400, tw400.data(), tw400.size() * sizeof(cf), cudaMemcpyHostToDevice));
    WK_CUDA_CHECK(cudaMemcpy(t->tw25, tw25.data(), tw25.size() * sizeof(cf), cudaMemcpyHostToDevice));
    WK_CUDA_CHECK(cudaMemcpy(t->wts, wts.data(), wts.size() * sizeof(float), cudaMemcpyHostToDevice));
    WK_CUDA_CHECK(cudaMemcpy(t->start, start.data(), start.size() * sizeof(int), cudaMemcpyHostToDevice));
    WK_CUDA_CHECK(cudaFuncSetAttribute(mel_pass1_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(MelSmem)));
    return WK_OK;
}

wk_status mel_forward(const MelTables* t, const float* pcm, int64_t n_windows, int64_t stride, const int32_t* n_valid,
                      void* out_f16, int32_t* gmax_scratch, cudaStream_t stream) {
    if (n_windows <= 0) return WK_OK;
    WK_CUDA_CHECK(cudaMemsetAsync(gmax_scratch, 0, n_windows * sizeof(int32_t), stream));
    const int ctas_per_window = (kFramesPerWindow + kF - 1) / kF;
    mel_pass1_kernel<<<(unsigned)(n_windows * ctas_per_window), kThreads, sizeof(MelSmem), stream>>>(
        pcm, (long long)stride, n_valid, *t, reinterpret_cast<uint16_t*>(out_f16), gmax_scratch, ctas_per_window);
    const long long rows = (long long)n_windows * kFramesPerWindow;
    const long long threads = rows * (kMelCols / 8);
    mel_pass2_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(reinterpret_cast<uint16_t*>(out_f16), gmax_scratch,
                                                                           t->n_mels, rows);
    count_launch(2);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("mel launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

}  // namespace wk
