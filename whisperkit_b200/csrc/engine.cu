// libwkb200 engine: the model object (weights, mel tables, alignment heads), weight ingestion, the mel + encoder schedule, the
// piecewise protocol entry points wk_mel / wk_encode and the kernel-level hooks.  Decode sessions and the window scheduler are in
// session.cu.  Host-side control flow mirrors the reference's per-window body
// (Sources/WhisperKit/Core/TranscribeTask.swift:116-278); all arithmetic runs in the sm_90a kernels of this directory.
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <dirent.h>

#include <algorithm>
#include <atomic>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "common.cuh"
#include "engine.h"

namespace wk {

// ------------------------------------------------------------------------------------------------ errors / counters
static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
const char* last_error_cstr() { return g_err; }
static std::atomic<long long> g_launches{0};
static std::atomic<int64_t> g_live_bytes[2] = {{0}, {0}};   // held through Buffers: [0] device, [1] pinned host
static std::atomic<int> g_pdl{-1};
int pdl_mode() {
    // Programmatic dependent launch along the decode step.  Mask 53 = embed | cross-attention (its K chunks are static and prefetched
    // before griddepcontrol.wait) | GEMM | reduce: the kernels with a real prologue to hide under the upstream kernel's tail.
    // WKB200_PDL_MASK (read once per process) overrides it for A/B measurements.
    int v = g_pdl.load(std::memory_order_relaxed);
    if (v < 0) {
        v = 53;
        if (const char* e = getenv("WKB200_PDL_MASK")) v = (int)strtol(e, nullptr, 0) & 63;
        g_pdl.store(v, std::memory_order_relaxed);
    }
    return v;
}
bool pdl_enabled() { return pdl_mode() > 0; }
void pdl_disable() { g_pdl.store(0, std::memory_order_relaxed); }
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
long long launch_counter_load() { return g_launches.load(); }
void launch_counter_sub(long long n) { g_launches.fetch_sub(n); }

// ------------------------------------------------------------------------------------------------ buffer owner
wk_status Buffers::alloc(void** p, size_t bytes, bool pinned, bool zero) {
    cudaError_t e = pinned ? cudaHostAlloc(p, bytes, cudaHostAllocDefault) : cudaMalloc(p, bytes);
    if (e != cudaSuccess) {
        cudaGetLastError();
        *p = nullptr;
        if (pinned) set_error("pinned staging of %zu bytes failed: %s", bytes, cudaGetErrorString(e));
        else set_error("cudaMalloc(%zu bytes) failed: %s", bytes, cudaGetErrorString(e));
        return WK_ERR_CUDA;
    }
    live_.push_back({*p, bytes, pinned});
    g_live_bytes[pinned].fetch_add((int64_t)bytes);
    if (zero) {
        if (pinned) memset(*p, 0, bytes);
        else if ((e = cudaMemset(*p, 0, bytes)) != cudaSuccess) { set_error("cudaMemset failed: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    }
    return WK_OK;
}

static void free_buffer(void* p, size_t bytes, bool pinned) {
    if (pinned) cudaFreeHost(p);
    else cudaFree(p);
    g_live_bytes[pinned].fetch_sub((int64_t)bytes);
}

wk_status Buffers::regrow(void** p, size_t bytes, bool pinned, cudaStream_t drain, bool* moved) {
    if (moved) *moved = false;
    auto it = std::find_if(live_.begin(), live_.end(), [&](const Buf& b) { return *p && b.p == *p; });
    if ((it == live_.end() ? 0 : it->bytes) >= bytes) return WK_OK;
    if (moved) *moved = true;
    if (it != live_.end()) {
        if (drain) WK_CUDA_CHECK(cudaStreamSynchronize(drain));
        free_buffer(it->p, it->bytes, it->pinned);
        live_.erase(it);
    }
    return alloc(p, bytes, pinned, false);
}

void Buffers::release_all() {
    for (const Buf& b : live_) free_buffer(b.p, b.bytes, b.pinned);
    live_.clear();
}

int choose_splits(int tiles, int total_kb, int num_sms) {
    // Split-K depth of a decoder swap-AB GEMM: the deepest split that still fits ONE wave of CTAs (tiles * s <= SMs), so every SM that
    // takes part streams its share of the weights exactly once: one SM alone cannot pull HBM bandwidth, so too few CTAs starve, while a
    // second wave costs more than the extra parallelism saves (tools/microbench_cold.py times the choices with HBM-cold weights).
    int best = 1;
    for (int s = 1; s <= total_kb && s <= 20; ++s) {   // 20 = kMaxSplits of the fused reduce kernels
        if (total_kb % s) continue;
        if (tiles * s <= num_sms) best = s;
    }
    return best;
}

size_t esize(int dtype) { return dtype == WK_DTYPE_F32 || dtype == WK_DTYPE_I32 ? 4 : 2; }

static wk_status alloc_ln(Buffers& b, LayerNormW& ln, int d) {
    WK_CHECK(b.dmalloc(&ln.g, d));
    WK_CHECK(b.dmalloc(&ln.b, d));
    return WK_OK;
}

static wk_status model_alloc(wk_model* m) {
    const wk_model_config& c = m->cfg;
    const int d = c.d_model, L = c.enc_layers, Ld = c.dec_layers;
    const size_t T = c.n_audio_ctx;
    Buffers& b = m->mem;
    WK_CHECK(b.alloc16(&m->conv1_w, (size_t)d * 3 * 128));
    WK_CHECK(b.dmalloc(&m->conv1_b, d));
    WK_CHECK(b.alloc16(&m->conv2_w, (size_t)d * 3 * d));
    WK_CHECK(b.dmalloc(&m->conv2_b, d));
    WK_CHECK(b.dmalloc(&m->enc_pos, T * d));
    m->enc.resize(L);
    for (auto& l : m->enc) {
        WK_CHECK(alloc_ln(b, l.ln1, d)); WK_CHECK(alloc_ln(b, l.ln2, d));
        WK_CHECK(b.alloc16(&l.wqkv, (size_t)3 * d * d)); WK_CHECK(b.dmalloc(&l.bqkv, 3 * d));
        WK_CHECK(b.alloc16(&l.wo, (size_t)d * d)); WK_CHECK(b.dmalloc(&l.bo, d));
        WK_CHECK(b.alloc16(&l.w1, (size_t)4 * d * d)); WK_CHECK(b.dmalloc(&l.b1, 4 * d));
        WK_CHECK(b.alloc16(&l.w2, (size_t)4 * d * d)); WK_CHECK(b.dmalloc(&l.b2, d));
    }
    WK_CHECK(alloc_ln(b, m->enc_ln, d));
    // embedding rows padded to a multiple of 128 so the last TMA tile never leaves the allocation
    WK_CHECK(b.alloc16(&m->emb, (size_t)round_up(c.vocab, 128) * d));
    WK_CHECK(b.dmalloc(&m->dec_pos, (size_t)c.n_text_ctx * d));
    m->dec.resize(Ld);
    for (auto& l : m->dec) {
        WK_CHECK(alloc_ln(b, l.ln1, d)); WK_CHECK(alloc_ln(b, l.lnx, d)); WK_CHECK(alloc_ln(b, l.ln3, d));
        WK_CHECK(b.alloc16(&l.wqkv, (size_t)3 * d * d)); WK_CHECK(b.dmalloc(&l.bq, d)); WK_CHECK(b.dmalloc(&l.bv, d));
        WK_CHECK(b.alloc16(&l.wo, (size_t)d * d)); WK_CHECK(b.dmalloc(&l.bo, d));
        WK_CHECK(b.alloc16(&l.wcq, (size_t)d * d)); WK_CHECK(b.dmalloc(&l.bcq, d));
        WK_CHECK(b.alloc16(&l.wco, (size_t)d * d)); WK_CHECK(b.dmalloc(&l.bco, d));
        WK_CHECK(b.alloc16(&l.w1, (size_t)4 * d * d)); WK_CHECK(b.dmalloc(&l.b1, 4 * d));
        WK_CHECK(b.alloc16(&l.w2, (size_t)4 * d * d)); WK_CHECK(b.dmalloc(&l.b2, d));
    }
    WK_CHECK(alloc_ln(b, m->dec_ln, d));
    WK_CHECK(b.alloc16(&m->wckv, (size_t)2 * Ld * d * d));
    WK_CHECK(b.dmalloc(&m->bckv, (size_t)2 * Ld * d));
    return WK_OK;
}

wk_status enc_ws_ensure(wk_model* m, EncWorkspace* ws, int max_batch) {
    if (ws->max_batch >= max_batch) return WK_OK;
    *ws = EncWorkspace();   // releases a smaller workspace
    const wk_model_config& c = m->cfg;
    const int d = c.d_model, Bm = max_batch;
    const size_t T = c.n_audio_ctx;
    Buffers& b = ws->mem;
    WK_CHECK(b.dmalloc(&ws->pcm_dev, (size_t)Bm * kWindowSamples, false));
    WK_CHECK(b.dmalloc(&ws->nvalid_dev, Bm));
    WK_CHECK(b.dmalloc(&ws->gmax, Bm));
    WK_CHECK(b.alloc16(&ws->mel, (size_t)Bm * kMelRows * kMelCols));
    WK_CHECK(b.alloc16(&ws->h1, (size_t)Bm * kMelRows * d));
    const size_t M = (size_t)Bm * T;
    WK_CHECK(b.dmalloc(&ws->x, M * d, false));
    WK_CHECK(b.alloc16(&ws->xn, M * d));
    WK_CHECK(b.alloc16(&ws->qkv, M * 3 * d));
    WK_CHECK(b.alloc16(&ws->attn, M * d));
    WK_CHECK(b.alloc16(&ws->ffn, M * 4 * d));
    WK_CHECK(b.alloc16(&ws->enc_out, M * d));
    ws->max_batch = Bm;
    return WK_OK;
}

// ---------------------------------------------------------------------------------------------- weight ingestion
__global__ void conv_w_rearrange_kernel(const float* __restrict__ src, __half* __restrict__ dst, int co, int ci, int ci_pad) {
    // src [co][ci][3] f32 -> dst [co][3][ci_pad] f16
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long n = (long long)co * 3 * ci_pad;
    if (idx >= n) return;
    const int c = (int)(idx % ci_pad);
    const int tap = (int)((idx / ci_pad) % 3);
    const int o = (int)(idx / (3LL * ci_pad));
    dst[idx] = c < ci ? __float2half_rn(src[((long long)o * ci + c) * 3 + tap]) : __float2half_rn(0.f);
}

struct Dest { void* p; int dtype; size_t numel; int special; };  // special: 1 conv1, 2 conv2

// The decoder's HF parameter names (model.decoder.*, proj_out.weight) into decoder weight set w: the model's own decoder or its draft
static bool resolve_decoder_name(const wk_model* m, const DecoderWeights& w, const std::string& name, Dest* out) {
    const int d = m->cfg.d_model, dt = m->cfg.dtype;
    auto W = [&](void* p, size_t rows_off, size_t n) { *out = {(char*)p + rows_off * (size_t)d * 2, dt, n, 0}; return true; };
    auto F = [&](float* p, size_t n) { *out = {p, WK_DTYPE_F32, n, 0}; return true; };
    int i = -1;
    char rest[128];
    if (name == "model.decoder.embed_tokens.weight" || name == "proj_out.weight") { *out = {w.emb, dt, (size_t)m->cfg.vocab * d, 0}; return true; }
    if (name == "model.decoder.embed_positions.weight") return F(w.pos, (size_t)m->cfg.n_text_ctx * d);
    if (name == "model.decoder.layer_norm.weight") return F(w.ln.g, d);
    if (name == "model.decoder.layer_norm.bias") return F(w.ln.b, d);
    if (sscanf(name.c_str(), "model.decoder.layers.%d.%127s", &i, rest) == 2 && i >= 0 && i < w.n_layers) {
        DecLayer& l = w.layers[i];
        const std::string r = rest;
        const size_t dd = (size_t)d * d;
        if (r == "self_attn.q_proj.weight") return W(l.wqkv, 0, dd);
        if (r == "self_attn.k_proj.weight") return W(l.wqkv, d, dd);
        if (r == "self_attn.v_proj.weight") return W(l.wqkv, 2 * (size_t)d, dd);
        if (r == "self_attn.q_proj.bias") return F(l.bq, d);
        if (r == "self_attn.v_proj.bias") return F(l.bv, d);
        if (r == "self_attn.out_proj.weight") return W(l.wo, 0, dd);
        if (r == "self_attn.out_proj.bias") return F(l.bo, d);
        if (r == "self_attn_layer_norm.weight") return F(l.ln1.g, d);
        if (r == "self_attn_layer_norm.bias") return F(l.ln1.b, d);
        if (r == "encoder_attn.q_proj.weight") return W(l.wcq, 0, dd);
        if (r == "encoder_attn.q_proj.bias") return F(l.bcq, d);
        if (r == "encoder_attn.k_proj.weight") return W(w.wckv, (size_t)(2 * i) * d, dd);
        if (r == "encoder_attn.v_proj.weight") return W(w.wckv, (size_t)(2 * i + 1) * d, dd);
        if (r == "encoder_attn.v_proj.bias") return F(w.bckv + (size_t)(2 * i + 1) * d, d);
        if (r == "encoder_attn.out_proj.weight") return W(l.wco, 0, dd);
        if (r == "encoder_attn.out_proj.bias") return F(l.bco, d);
        if (r == "encoder_attn_layer_norm.weight") return F(l.lnx.g, d);
        if (r == "encoder_attn_layer_norm.bias") return F(l.lnx.b, d);
        if (r == "final_layer_norm.weight") return F(l.ln3.g, d);
        if (r == "final_layer_norm.bias") return F(l.ln3.b, d);
        if (r == "fc1.weight") return W(l.w1, 0, 4 * dd);
        if (r == "fc1.bias") return F(l.b1, 4 * (size_t)d);
        if (r == "fc2.weight") return W(l.w2, 0, 4 * dd);
        if (r == "fc2.bias") return F(l.b2, d);
        return false;
    }
    return false;
}

static bool resolve_name(wk_model* m, const std::string& name, Dest* out) {
    const int d = m->cfg.d_model, dt = m->cfg.dtype;
    auto W = [&](void* p, size_t rows_off, size_t n) { *out = {(char*)p + rows_off * (size_t)d * 2, dt, n, 0}; return true; };
    auto F = [&](float* p, size_t n) { *out = {p, WK_DTYPE_F32, n, 0}; return true; };
    int i = -1;
    char rest[128];
    if (name == "model.encoder.conv1.weight") { *out = {m->conv1_w, WK_DTYPE_F16, (size_t)d * m->cfg.n_mels * 3, 1}; return true; }
    if (name == "model.encoder.conv1.bias") return F(m->conv1_b, d);
    if (name == "model.encoder.conv2.weight") { *out = {m->conv2_w, WK_DTYPE_F16, (size_t)d * d * 3, 2}; return true; }
    if (name == "model.encoder.conv2.bias") return F(m->conv2_b, d);
    if (name == "model.encoder.embed_positions.weight") return F(m->enc_pos, (size_t)m->cfg.n_audio_ctx * d);
    if (name == "model.encoder.layer_norm.weight") return F(m->enc_ln.g, d);
    if (name == "model.encoder.layer_norm.bias") return F(m->enc_ln.b, d);
    if (resolve_decoder_name(m, m->main_decoder(), name, out)) return true;
    if (sscanf(name.c_str(), "model.encoder.layers.%d.%127s", &i, rest) == 2 && i >= 0 && i < (int)m->enc.size()) {
        EncLayer& l = m->enc[i];
        const std::string r = rest;
        const size_t dd = (size_t)d * d;
        if (r == "self_attn.q_proj.weight") return W(l.wqkv, 0, dd);
        if (r == "self_attn.k_proj.weight") return W(l.wqkv, d, dd);
        if (r == "self_attn.v_proj.weight") return W(l.wqkv, 2 * (size_t)d, dd);
        if (r == "self_attn.q_proj.bias") return F(l.bqkv, d);
        if (r == "self_attn.k_proj.bias") return F(l.bqkv + d, d);
        if (r == "self_attn.v_proj.bias") return F(l.bqkv + 2 * d, d);
        if (r == "self_attn.out_proj.weight") return W(l.wo, 0, dd);
        if (r == "self_attn.out_proj.bias") return F(l.bo, d);
        if (r == "self_attn_layer_norm.weight") return F(l.ln1.g, d);
        if (r == "self_attn_layer_norm.bias") return F(l.ln1.b, d);
        if (r == "final_layer_norm.weight") return F(l.ln2.g, d);
        if (r == "final_layer_norm.bias") return F(l.ln2.b, d);
        if (r == "fc1.weight") return W(l.w1, 0, 4 * dd);
        if (r == "fc1.bias") return F(l.b1, 4 * (size_t)d);
        if (r == "fc2.weight") return W(l.w2, 0, 4 * dd);
        if (r == "fc2.bias") return F(l.b2, d);
        return false;
    }
    return false;
}

// ---------------------------------------------------------------------------------------------- mel + encoder schedule
GemmDesc plain_gemm(const void* a, int64_t M, int K, const void* w, int N, int dtype, int mode, void* out, int64_t ld_out,
                    const float* bias, int gelu) {
    GemmDesc g;
    memset(&g, 0, sizeof(g));
    g.a = a; g.a_rows = M; g.a_cols = K; g.a_ld = K; g.a_batches = 1;
    g.b = w; g.b_rows = N; g.b_ld = K; g.in_dtype = dtype;
    g.m_rows_per_batch = (int)M; g.n = N; g.k = K; g.taps = 1;
    g.bn = N >= 256 ? 256 : round_up(N, 16);
    g.splits = 1; g.mode = mode; g.gelu = gelu; g.out = out; g.ld_out = ld_out; g.out_rows_per_batch = M; g.bias = bias;
    return g;
}

wk_status mel_stage(EncWorkspace* ws, const float* pcm, int64_t n, int64_t stride, cudaStream_t stream, const float** src, int64_t* src_stride) {
    cudaPointerAttributes at;
    const bool on_device = cudaPointerGetAttributes(&at, pcm) == cudaSuccess && at.type == cudaMemoryTypeDevice;
    cudaGetLastError();
    *src = pcm;
    *src_stride = stride;
    if (on_device && stride >= kWindowSamples) return WK_OK;
    // host PCM, or short rows: stage (padOrTrimAudio, AudioProcessor.swift:151-174)
    if (stride < kWindowSamples) WK_CUDA_CHECK(cudaMemsetAsync(ws->pcm_dev, 0, (size_t)n * kWindowSamples * 4, stream));
    WK_CUDA_CHECK(cudaMemcpy2DAsync(ws->pcm_dev, kWindowSamples * 4, pcm, stride * 4, std::min<int64_t>(stride, kWindowSamples) * 4, n,
                                    cudaMemcpyDefault, stream));
    *src = ws->pcm_dev;
    *src_stride = kWindowSamples;
    return WK_OK;
}

wk_status mel_run(wk_model* m, EncWorkspace* ws, const float* pcm, int64_t n, int64_t stride, const int32_t* samples_per_window,
                  void* mel_out, cudaStream_t stream) {
    if (n < 1 || n > ws->max_batch) { set_error("log-mel: %lld windows outside [1, %d]", (long long)n, ws->max_batch); return WK_ERR_AUDIO_PROCESSING_FAILED; }
    if (stride < kWindowSamples && !samples_per_window) { set_error("log-mel: stride %lld < 480000 requires samples_per_window", (long long)stride); return WK_ERR_AUDIO_PROCESSING_FAILED; }
    const float* src;
    int64_t src_stride;
    WK_CHECK(mel_stage(ws, pcm, n, stride, stream, &src, &src_stride));
    const int32_t* nv = nullptr;
    if (samples_per_window) {
        for (int64_t i = 0; i < n; ++i)
            if (samples_per_window[i] < 0 || samples_per_window[i] > kWindowSamples) { set_error("log-mel: samples_per_window[%lld] out of range", (long long)i); return WK_ERR_AUDIO_PROCESSING_FAILED; }
        WK_CUDA_CHECK(cudaMemcpyAsync(ws->nvalid_dev, samples_per_window, n * 4, cudaMemcpyHostToDevice, stream));
        nv = ws->nvalid_dev;
    }
    return mel_forward(&m->mel_tables, src, n, src_stride, nv, mel_out, ws->gmax, stream);
}

// an FP8 GEMM of the encoder: A = E4M3 codes [M][K] with block scales a_scale [K / 128][ld], W = E4M3 [N][K] with channel scales
static GemmDesc fp8_gemm(const uint8_t* a, const float* a_scale, int64_t ld, int64_t M, int K, const uint8_t* w, const float* w_scale, int N,
                         int dtype, int mode, void* out, float* out_scale, const float* bias, int gelu) {
    GemmDesc g = plain_gemm(a, M, K, w, N, dtype, mode, out, N, bias, gelu);
    g.a_ld = K; g.b_ld = K;   // bytes: one per code
    g.a_scale = a_scale; g.a_scale_ld = ld; g.w_scale = w_scale; g.out_scale = out_scale;
    return g;
}

// The encoder layers under the FP8 policy: LayerNorms write E4M3 codes + block scales into xn, the QKV / FC1 / FC2 GEMMs run on the FP8
// tensor cores (FC1 quantizes its GELU output into ffn for FC2); attention, the out-projection and the residual stream are as in the
// 16-bit schedule.  Every scale comes from its own row, so a window's result does not depend on the batch it is encoded in.
static wk_status encode_layers_fp8(wk_model* m, EncWorkspace* ws, int B, void* enc_out, cudaStream_t s) {
    const wk_model_config& c = m->cfg;
    const int d = c.d_model, T = c.n_audio_ctx, dt = c.dtype;
    const int64_t M = (int64_t)B * T;
    const int64_t ld = round_up(ws->max_batch * T, 128);
    if (!ws->xn_scale) {
        WK_CHECK(ws->mem.dmalloc(&ws->xn_scale, (size_t)(d / kFp8Block) * ld));
        WK_CHECK(ws->mem.dmalloc(&ws->ffn_scale, (size_t)(4 * d / kFp8Block) * ld));
    }
    uint8_t* xn8 = static_cast<uint8_t*>(ws->xn);
    uint8_t* ffn8 = static_cast<uint8_t*>(ws->ffn);
    for (int li = 0; li < c.enc_layers; ++li) {
        EncLayer& l = m->enc[li];
        WK_CHECK(layernorm_f32_to_fp8(ws->x, l.ln1.g, l.ln1.b, xn8, ws->xn_scale, ld, M, d, s));
        WK_CHECK(gemm_wgmma_fp8(fp8_gemm(xn8, ws->xn_scale, ld, M, d, l.wqkv8, l.sqkv, 3 * d, dt, GEMM_OUT_T16, ws->qkv, nullptr, l.bqkv, 0),
                                m->num_sms, s));
        WK_CHECK(encoder_attention(ws->qkv, ws->attn, B, T, c.n_heads, dt, s));
        WK_CHECK(gemm_wgmma(plain_gemm(ws->attn, M, d, l.wo, d, dt, GEMM_OUT_F32_ADD, ws->x, d, l.bo, 0), m->num_sms, s));
        WK_CHECK(layernorm_f32_to_fp8(ws->x, l.ln2.g, l.ln2.b, xn8, ws->xn_scale, ld, M, d, s));
        WK_CHECK(gemm_wgmma_fp8(fp8_gemm(xn8, ws->xn_scale, ld, M, d, l.w18, l.s1, 4 * d, dt, GEMM_OUT_FP8_BLOCKS, ffn8, ws->ffn_scale, l.b1, 1),
                                m->num_sms, s));
        WK_CHECK(gemm_wgmma_fp8(fp8_gemm(ffn8, ws->ffn_scale, ld, M, 4 * d, l.w28, l.s2, d, dt, GEMM_OUT_F32_ADD, ws->x, nullptr, l.b2, 0),
                                m->num_sms, s));
    }
    WK_CHECK(layernorm_f32_to_16(ws->x, m->enc_ln.g, m->enc_ln.b, enc_out, M, d, dt, s));
    return WK_OK;
}

// E4M3 copies of encoder layer li's QKV / FC1 / FC2 weights (the FP8 policy), from the 16-bit weights, on the model stream
static wk_status quantize_enc_layer(wk_model* m, int li) {
    const int d = m->cfg.d_model, dt = m->cfg.dtype;
    EncLayer& l = m->enc[li];
    WK_CHECK(quantize_weight_rows_fp8(l.wqkv, dt, l.wqkv8, l.sqkv, 3 * d, d, m->stream));
    WK_CHECK(quantize_weight_rows_fp8(l.w1, dt, l.w18, l.s1, 4 * d, d, m->stream));
    WK_CHECK(quantize_weight_rows_fp8(l.w2, dt, l.w28, l.s2, d, 4 * d, m->stream));
    return WK_OK;
}

static wk_status quantize_enc_weights(wk_model* m) {
    for (size_t li = 0; li < m->enc.size(); ++li) WK_CHECK(quantize_enc_layer(m, (int)li));
    WK_CUDA_CHECK(cudaStreamSynchronize(m->stream));
    return WK_OK;
}

wk_status encode_chunk(wk_model* m, EncWorkspace* ws, const void* mel, int B, void* enc_out, cudaStream_t s) {
    const wk_model_config& c = m->cfg;
    const int d = c.d_model, T = c.n_audio_ctx, dt = c.dtype;
    const int64_t M = (int64_t)B * T;
    if (B < 1 || B > ws->max_batch) { set_error("encoder: %d windows outside [1, %d]", B, ws->max_batch); return WK_ERR_INVALID_ARGUMENT; }
    // conv1 (k=3, pad 1) + GELU as implicit GEMM over the time-major mel: taps = 3 row shifts of the same tensor map
    {
        GemmDesc g;
        memset(&g, 0, sizeof(g));
        g.a = mel; g.a_rows = kMelRows; g.a_cols = kMelCols; g.a_ld = kMelCols; g.a_batch_stride = (int64_t)kMelRows * kMelCols;
        g.a_batches = B; g.a_3d = 1;
        g.b = m->conv1_w; g.b_rows = d; g.b_ld = 3 * kMelCols; g.in_dtype = WK_DTYPE_F16;
        g.m_rows_per_batch = 2 * T; g.n = d; g.k = kMelCols; g.taps = 3;
        for (int t = 0; t < 3; ++t) { g.tap_row_shift[t] = t; g.tap_col_off[t] = 0; }
        g.bn = d >= 256 ? 256 : round_up(d, 16);
        g.splits = 1; g.mode = GEMM_OUT_T16; g.gelu = 1;
        g.out = (char*)ws->h1 + (size_t)d * 2;  // row 0 of every window is the zero pad
        g.ld_out = d; g.out_rows_per_batch = kMelRows; g.bias = m->conv1_b;
        WK_CHECK(gemm_wgmma(g, m->num_sms, s));
    }
    // conv2 (k=3, stride 2, pad 1) + GELU + positional embedding -> residual stream x (f32)
    {
        GemmDesc g;
        memset(&g, 0, sizeof(g));
        g.a = ws->h1; g.a_rows = kMelRows / 2; g.a_cols = 2 * d; g.a_ld = 2 * d; g.a_batch_stride = (int64_t)kMelRows * d;
        g.a_batches = B; g.a_3d = 1;
        g.b = m->conv2_w; g.b_rows = d; g.b_ld = 3 * d; g.in_dtype = WK_DTYPE_F16;
        g.m_rows_per_batch = T; g.n = d; g.k = d; g.taps = 3;
        g.tap_row_shift[0] = 0; g.tap_col_off[0] = 0;
        g.tap_row_shift[1] = 0; g.tap_col_off[1] = d;
        g.tap_row_shift[2] = 1; g.tap_col_off[2] = 0;
        g.bn = d >= 256 ? 256 : round_up(d, 16);
        g.splits = 1; g.mode = GEMM_OUT_F32_GELU_POS; g.gelu = 1;
        g.out = ws->x; g.ld_out = d; g.out_rows_per_batch = T; g.bias = m->conv2_b; g.pos = m->enc_pos; g.ld_pos = d;
        WK_CHECK(gemm_wgmma(g, m->num_sms, s));
    }
    if (m->enc_fp8) return encode_layers_fp8(m, ws, B, enc_out, s);
    for (int li = 0; li < c.enc_layers; ++li) {
        EncLayer& l = m->enc[li];
        WK_CHECK(layernorm_f32_to_16(ws->x, l.ln1.g, l.ln1.b, ws->xn, M, d, dt, s));
        WK_CHECK(gemm_wgmma(plain_gemm(ws->xn, M, d, l.wqkv, 3 * d, dt, GEMM_OUT_T16, ws->qkv, 3 * d, l.bqkv, 0), m->num_sms, s));
        WK_CHECK(encoder_attention(ws->qkv, ws->attn, B, T, c.n_heads, dt, s));
        WK_CHECK(gemm_wgmma(plain_gemm(ws->attn, M, d, l.wo, d, dt, GEMM_OUT_F32_ADD, ws->x, d, l.bo, 0), m->num_sms, s));
        WK_CHECK(layernorm_f32_to_16(ws->x, l.ln2.g, l.ln2.b, ws->xn, M, d, dt, s));
        WK_CHECK(gemm_wgmma(plain_gemm(ws->xn, M, d, l.w1, 4 * d, dt, GEMM_OUT_T16, ws->ffn, 4 * d, l.b1, 1), m->num_sms, s));
        WK_CHECK(gemm_wgmma(plain_gemm(ws->ffn, M, 4 * d, l.w2, d, dt, GEMM_OUT_F32_ADD, ws->x, d, l.b2, 0), m->num_sms, s));
    }
    WK_CHECK(layernorm_f32_to_16(ws->x, m->enc_ln.g, m->enc_ln.b, enc_out, M, d, dt, s));
    return WK_OK;
}

}  // namespace wk

using namespace wk;

// =====================================================================================================
// C ABI
// =====================================================================================================
extern "C" {

const char* wk_last_error(void) { return wk::last_error_cstr(); }
const char* wk_version(void) { return "wkb200 0.3 (sm_90a)"; }

int32_t wk_device_available(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) return 0;
    cudaDeviceProp p;
    if (cudaGetDeviceProperties(&p, 0) != cudaSuccess) return 0;
    return p.major == 9 ? 1 : 0;   // the kernels are built for sm_90a only (wgmma, TMA, setmaxnreg)
}

void wk_default_config(const char* variant, wk_model_config* c) {
    memset(c, 0, sizeof(*c));
    c->n_audio_ctx = 1500; c->n_text_ctx = 448; c->dtype = WK_DTYPE_BF16; c->max_batch = 16;
    std::string v = variant ? variant : "large-v3";
    // OpenAI Whisper dimensions (external facts; the reference reads them off the CoreML model descriptions)
    struct Dim { const char* name; int mels, d, heads, enc, dec, vocab; };
    static const Dim dims[] = {
        {"tiny", 80, 384, 6, 4, 4, 51865},       {"tiny.en", 80, 384, 6, 4, 4, 51864},       {"base", 80, 512, 8, 6, 6, 51865},
        {"base.en", 80, 512, 8, 6, 6, 51864},    {"small", 80, 768, 12, 12, 12, 51865},      {"small.en", 80, 768, 12, 12, 12, 51864},
        {"medium", 80, 1024, 16, 24, 24, 51865}, {"medium.en", 80, 1024, 16, 24, 24, 51864}, {"large", 80, 1280, 20, 32, 32, 51865},
        {"large-v2", 80, 1280, 20, 32, 32, 51865}, {"large-v3", 128, 1280, 20, 32, 32, 51866}, {"large-v3-turbo", 128, 1280, 20, 32, 4, 51866},
        {"distil-large-v3", 128, 1280, 20, 32, 2, 51866}, {"toy", 80, 128, 2, 2, 2, 1024},   {"toy128", 128, 256, 4, 2, 2, 2048},
        {"toy512", 80, 512, 8, 2, 2, 2048}, {"toy768", 80, 768, 12, 2, 2, 2048},
    };
    const Dim* d = &dims[10];
    for (const Dim& e : dims) if (v == e.name) d = &e;
    c->n_mels = d->mels; c->d_model = d->d; c->n_heads = d->heads; c->enc_layers = d->enc; c->dec_layers = d->dec; c->vocab = d->vocab;
}

// ModelUtilities.detectVariant (ModelUtilities.swift:128-173) and tokenizerNameForVariant (:175-205)
wk_status wk_detect_variant(int32_t logits_dim, int32_t encoder_dim, const char** variant, const char** tokenizer_repo, int32_t* is_multilingual) {
    const char* v = "base";
    if (logits_dim == 51865) {
        switch (encoder_dim) { case 384: v = "tiny"; break; case 512: v = "base"; break; case 768: v = "small"; break; case 1024: v = "medium"; break;
                               case 1280: v = "large-v2"; break; default: v = "base"; }
    } else if (logits_dim == 51864) {
        switch (encoder_dim) { case 384: v = "tiny.en"; break; case 512: v = "base.en"; break; case 768: v = "small.en"; break; case 1024: v = "medium.en"; break;
                               default: v = "base.en"; }
    } else if (logits_dim == 51866) {
        v = "large-v3";
    }
    static const char* names[][2] = {{"tiny", "openai/whisper-tiny"}, {"tiny.en", "openai/whisper-tiny.en"}, {"base", "openai/whisper-base"},
                                     {"base.en", "openai/whisper-base.en"}, {"small", "openai/whisper-small"}, {"small.en", "openai/whisper-small.en"},
                                     {"medium", "openai/whisper-medium"}, {"medium.en", "openai/whisper-medium.en"},
                                     {"large-v2", "openai/whisper-large-v2"}, {"large-v3", "openai/whisper-large-v3"}};
    if (variant) *variant = v;
    if (tokenizer_repo) for (auto& n : names) if (!strcmp(n[0], v)) *tokenizer_repo = n[1];
    if (is_multilingual) *is_multilingual = logits_dim != 51864;   // ModelUtilities.isModelMultilingual (:124-126)
    return WK_OK;
}

wk_status wk_model_create(const wk_model_config* cfg, int32_t device, wk_model** out) {
    if (!cfg || !out) { set_error("wk_model_create: null argument"); return WK_ERR_INVALID_ARGUMENT; }
    if (!wk_device_available()) {
        set_error("no sm_90 (Hopper) CUDA device visible: libwkb200 has no CPU fallback");
        return WK_ERR_MODELS_UNAVAILABLE;
    }
    if (cfg->d_model != cfg->n_heads * 64 || cfg->d_model % 128 != 0 || (cfg->n_mels != 80 && cfg->n_mels != 128) ||
        cfg->n_audio_ctx != 1500 || cfg->max_batch < 1 || cfg->vocab < 16 ||
        (cfg->dtype != WK_DTYPE_BF16 && cfg->dtype != WK_DTYPE_F16)) {
        set_error("wk_model_create: unsupported configuration (d_model %d heads %d mels %d ctx %d dtype %d)", cfg->d_model,
                  cfg->n_heads, cfg->n_mels, cfg->n_audio_ctx, cfg->dtype);
        return WK_ERR_INVALID_ARGUMENT;
    }
    WK_CUDA_CHECK(cudaSetDevice(device));
    std::unique_ptr<wk_model> m(new wk_model());   // released on any failure below
    m->cfg = *cfg;
    wk_model_set_alignment_heads(m.get(), nullptr, 0);
    m->device = device;
    cudaDeviceProp prop;
    WK_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
    m->num_sms = prop.multiProcessorCount;
    WK_CUDA_CHECK(cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking));
    for (auto& e : m->ev) WK_CUDA_CHECK(cudaEventCreate(&e));
    WK_CHECK(model_alloc(m.get()));
    WK_CHECK(mel_tables_create(cfg->n_mels, m->mem, &m->mel_tables));
    WK_CUDA_CHECK(cudaDeviceSynchronize());  // setup memsets / table uploads ran on the legacy default stream
    *out = m.release();
    return WK_OK;
}

// host tensor `data` (dtype, shape) converted into the weight buffer dst resolved from `name`
static wk_status store_tensor(wk_model* m, const Dest& dst, const char* name, const void* data, int32_t dtype, const int64_t* shape, int32_t ndim) {
    size_t numel = 1;
    for (int i = 0; i < ndim; ++i) numel *= (size_t)shape[i];
    if (numel != dst.numel) {
        set_error("wk_model_set_tensor: '%s' has %zu elements, expected %zu", name, numel, dst.numel);
        return WK_ERR_INVALID_ARGUMENT;
    }
    Buffers scratch;
    uint8_t* tmp = nullptr;
    WK_CHECK(scratch.dmalloc(&tmp, numel * esize(dtype), false));
    // stream-ordered copy: a pageable-host cudaMemcpy may return before its DMA lands, and the library stream is
    // non-blocking (it does not order against the legacy default stream)
    WK_CUDA_CHECK(cudaMemcpyAsync(tmp, data, numel * esize(dtype), cudaMemcpyDefault, m->stream));
    wk_status st = WK_OK;
    if (dst.special) {
        float* f = nullptr;
        WK_CHECK(scratch.dmalloc(&f, numel, false));
        st = convert_to_16(tmp, dtype, f, WK_DTYPE_F32, (int64_t)numel, m->stream);
        const int co = m->cfg.d_model, ci = dst.special == 1 ? m->cfg.n_mels : m->cfg.d_model, cip = dst.special == 1 ? kMelCols : m->cfg.d_model;
        const long long n = (long long)co * 3 * cip;
        conv_w_rearrange_kernel<<<(unsigned)((n + 255) / 256), 256, 0, m->stream>>>(f, (__half*)dst.p, co, ci, cip);
        cudaStreamSynchronize(m->stream);
    } else {
        st = convert_to_16(tmp, dtype, dst.p, dst.dtype, (int64_t)numel, m->stream);
        cudaStreamSynchronize(m->stream);
    }
    return st;
}

wk_status wk_model_set_tensor(wk_model* m, const char* name, const void* data, int32_t dtype, const int64_t* shape, int32_t ndim) {
    if (!m || !name || !data) { set_error("wk_model_set_tensor: null argument"); return WK_ERR_INVALID_ARGUMENT; }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    Dest dst;
    if (!resolve_name(m, name, &dst)) {
        if (strstr(name, "k_proj.bias")) return WK_OK;  // Whisper has no key bias; tolerate zero tensors
        set_error("wk_model_set_tensor: unknown parameter '%s'", name);
        return WK_ERR_INVALID_ARGUMENT;
    }
    wk_status st = store_tensor(m, dst, name, data, dtype, shape, ndim);
    int li = -1;
    char rest[128];
    if (st == WK_OK && m->enc_fp8 && sscanf(name, "model.encoder.layers.%d.%127s", &li, rest) == 2) {
        const std::string r = rest;   // a QKV / FC1 / FC2 weight of an FP8 encoder: refresh the layer's E4M3 copies
        if (r == "self_attn.q_proj.weight" || r == "self_attn.k_proj.weight" || r == "self_attn.v_proj.weight" || r == "fc1.weight" ||
            r == "fc2.weight") {
            st = quantize_enc_layer(m, li);
            const cudaError_t e = cudaStreamSynchronize(m->stream);
            if (st == WK_OK && e != cudaSuccess) { set_error("wk_model_set_tensor: %s", cudaGetErrorString(e)); st = WK_ERR_CUDA; }
        }
    }
    return st;
}

// ---------------------------------------------------------------------------------------------- safetensors loader
// HuggingFace checkpoint directory: config.json + *.safetensors (8-byte LE header length, JSON header, raw tensors).
// The reference loads CoreML bundles instead (WhisperKit.swift:358-442); here weights come from safetensors.
namespace {
struct JsonScan {
    const char* p; const char* end;
    void ws() { while (p < end && (*p == ' ' || *p == '\n' || *p == '\t' || *p == '\r' || *p == ',')) ++p; }
    bool str(std::string* out) {
        ws();
        if (p >= end || *p != '"') return false;
        ++p; out->clear();
        while (p < end && *p != '"') { if (*p == '\\' && p + 1 < end) ++p; out->push_back(*p++); }
        if (p < end) ++p;
        return true;
    }
    void skip_value() {   // skips any JSON value
        ws();
        if (p >= end) return;
        if (*p == '"') { std::string t; str(&t); return; }
        if (*p == '{' || *p == '[') {
            const char open = *p, close = open == '{' ? '}' : ']';
            int depth = 0;
            while (p < end) {
                if (*p == '"') { std::string t; str(&t); continue; }
                if (*p == open) ++depth;
                else if (*p == close) { if (--depth == 0) { ++p; return; } }
                ++p;
            }
            return;
        }
        while (p < end && *p != ',' && *p != '}' && *p != ']') ++p;
    }
};
static bool json_int(const std::string& js, const char* key, long long* out) {
    const std::string k = std::string("\"") + key + "\"";
    size_t pos = js.find(k);
    if (pos == std::string::npos) return false;
    pos = js.find(':', pos + k.size());
    if (pos == std::string::npos) return false;
    *out = atoll(js.c_str() + pos + 1);
    return true;
}
static bool read_file(const std::string& path, std::vector<char>* buf) {
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) return false;
    fseek(f, 0, SEEK_END);
    const long n = ftell(f);
    fseek(f, 0, SEEK_SET);
    buf->resize((size_t)n);
    const size_t got = fread(buf->data(), 1, (size_t)n, f);
    fclose(f);
    return got == (size_t)n;
}
}  // namespace

// draft: the file's decoder tensors go to the model's draft decoder (wk_model_set_draft_tensor); everything else is skipped
static wk_status load_safetensors_file(wk_model* m, const std::string& path, int* n_loaded, bool draft = false) {
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) { set_error("cannot open %s", path.c_str()); return WK_ERR_MODELS_UNAVAILABLE; }
    uint64_t hlen = 0;
    if (fread(&hlen, 8, 1, f) != 1 || hlen > (1ull << 28)) { fclose(f); set_error("%s: bad safetensors header", path.c_str()); return WK_ERR_MODELS_UNAVAILABLE; }
    std::vector<char> hdr((size_t)hlen);
    if (fread(hdr.data(), 1, (size_t)hlen, f) != (size_t)hlen) { fclose(f); set_error("%s: truncated header", path.c_str()); return WK_ERR_MODELS_UNAVAILABLE; }
    const long long data0 = 8 + (long long)hlen;
    JsonScan js{hdr.data(), hdr.data() + hdr.size()};
    js.ws();
    if (js.p < js.end && *js.p == '{') ++js.p;
    std::vector<char> buf;
    std::string name;
    while (js.str(&name)) {
        js.ws();
        if (js.p < js.end && *js.p == ':') ++js.p;
        if (name == "__metadata__") { js.skip_value(); continue; }
        const char* v0 = js.p;
        js.skip_value();
        const std::string obj(v0, js.p);
        // {"dtype":"F32","shape":[a,b],"data_offsets":[s,e]}
        size_t dp = obj.find("\"dtype\"");
        size_t sp = obj.find("\"shape\"");
        size_t op = obj.find("\"data_offsets\"");
        if (dp == std::string::npos || sp == std::string::npos || op == std::string::npos) continue;
        const size_t dq = obj.find('"', obj.find(':', dp) + 1);
        const std::string dts = obj.substr(dq + 1, obj.find('"', dq + 1) - dq - 1);
        int dt = -1;
        if (dts == "F32") dt = WK_DTYPE_F32; else if (dts == "F16") dt = WK_DTYPE_F16; else if (dts == "BF16") dt = WK_DTYPE_BF16;
        int64_t shape[8]; int nd = 0;
        { const char* q = obj.c_str() + obj.find('[', sp) + 1;
          while (*q && *q != ']' && nd < 8) { while (*q == ' ' || *q == ',') ++q; if (*q == ']') break; shape[nd++] = atoll(q); while (*q && *q != ',' && *q != ']') ++q; } }
        long long off[2] = {0, 0};
        { const char* q = obj.c_str() + obj.find('[', op) + 1; off[0] = atoll(q); while (*q && *q != ',') ++q; if (*q) off[1] = atoll(q + 1); }
        Dest d;
        if (dt < 0 || !(draft ? resolve_decoder_name(m, m->draft->view(), name, &d) : resolve_name(m, name, &d))) continue;   // not a hot-path parameter (or unsupported dtype)
        const size_t bytes = (size_t)(off[1] - off[0]);
        buf.resize(bytes);
        if (fseek(f, data0 + off[0], SEEK_SET) != 0 || fread(buf.data(), 1, bytes, f) != bytes) { fclose(f); set_error("%s: truncated tensor %s", path.c_str(), name.c_str()); return WK_ERR_MODELS_UNAVAILABLE; }
        wk_status st = draft ? wk_model_set_draft_tensor(m, name.c_str(), buf.data(), dt, shape, nd) : wk_model_set_tensor(m, name.c_str(), buf.data(), dt, shape, nd);
        if (st != WK_OK) { fclose(f); return st; }
        ++*n_loaded;
    }
    fclose(f);
    return WK_OK;
}

static std::vector<std::string> safetensors_files(const std::string& dir) {
    std::vector<std::string> files;
    if (DIR* d = opendir(dir.c_str())) {
        while (dirent* e = readdir(d)) {
            const std::string fn = e->d_name;
            if (fn.size() > 12 && fn.substr(fn.size() - 12) == ".safetensors") files.push_back(dir + "/" + fn);
        }
        closedir(d);
    }
    std::sort(files.begin(), files.end());
    return files;
}

wk_status wk_model_load(const char* weights_dir, int32_t device, int32_t max_batch, int32_t dtype, wk_model** out) {
    if (!weights_dir || !out) { set_error("wk_model_load: null argument"); return WK_ERR_INVALID_ARGUMENT; }
    const std::string dir = weights_dir;
    std::vector<char> cfgbuf;
    if (!read_file(dir + "/config.json", &cfgbuf)) { set_error("wk_model_load: %s/config.json not found", weights_dir); return WK_ERR_MODELS_UNAVAILABLE; }
    const std::string cj(cfgbuf.begin(), cfgbuf.end());
    wk_model_config c;
    memset(&c, 0, sizeof(c));
    long long v;
    c.n_mels = json_int(cj, "num_mel_bins", &v) ? (int)v : 80;
    c.d_model = json_int(cj, "d_model", &v) ? (int)v : 0;
    c.n_heads = json_int(cj, "encoder_attention_heads", &v) ? (int)v : 0;
    c.enc_layers = json_int(cj, "encoder_layers", &v) ? (int)v : 0;
    c.dec_layers = json_int(cj, "decoder_layers", &v) ? (int)v : 0;
    c.vocab = json_int(cj, "vocab_size", &v) ? (int)v : 0;
    c.n_audio_ctx = json_int(cj, "max_source_positions", &v) ? (int)v : 1500;
    c.n_text_ctx = json_int(cj, "max_target_positions", &v) ? (int)v : 448;
    c.dtype = dtype ? dtype : WK_DTYPE_BF16;
    c.max_batch = max_batch > 0 ? max_batch : 16;
    wk_model* m = nullptr;
    WK_CHECK(wk_model_create(&c, device, &m));
    // every *.safetensors in the directory (single file or HF shards)
    int n_loaded = 0;
    const std::vector<std::string> files = safetensors_files(dir);
    if (files.empty()) { wk_model_free(m); set_error("wk_model_load: no *.safetensors in %s", weights_dir); return WK_ERR_MODELS_UNAVAILABLE; }
    for (const auto& fp : files) {
        wk_status st = load_safetensors_file(m, fp, &n_loaded);
        if (st != WK_OK) { wk_model_free(m); return st; }
    }
    const int expected = 4 + 1 + 2 + c.enc_layers * 15 + 1 + 1 + 2 + c.dec_layers * 24;
    if (n_loaded < expected) { wk_model_free(m); set_error("wk_model_load: only %d of %d expected tensors found in %s", n_loaded, expected, weights_dir); return WK_ERR_MODELS_UNAVAILABLE; }
    // generation_config.json "alignment_heads": [[layer, head], ...] - the checkpoint's own word-timestamp heads, which the reference's
    // decoder model bakes into its alignment_heads_weights output (TextDecoder.swift:310,414)
    std::vector<char> gbuf;
    if (read_file(dir + "/generation_config.json", &gbuf)) {
        const std::string gj(gbuf.begin(), gbuf.end());
        size_t pos = gj.find("\"alignment_heads\"");
        if (pos != std::string::npos && (pos = gj.find('[', pos)) != std::string::npos) {
            std::vector<int32_t> pairs;
            int depth = 0;
            for (size_t i = pos; i < gj.size(); ++i) {
                const char ch = gj[i];
                if (ch == '[') ++depth;
                else if (ch == ']') { if (--depth == 0) break; }
                else if (ch >= '0' && ch <= '9') {
                    pairs.push_back((int32_t)atol(gj.c_str() + i));
                    while (i + 1 < gj.size() && gj[i + 1] >= '0' && gj[i + 1] <= '9') ++i;
                }
            }
            if (!pairs.empty() && pairs.size() % 2 == 0) {
                wk_status st = wk_model_set_alignment_heads(m, pairs.data(), (int32_t)pairs.size() / 2);
                if (st != WK_OK) { wk_model_free(m); return st; }
            }
        }
    }
    WK_CHECK(wk_model_finalize(m));
    *out = m;
    return WK_OK;
}

wk_status wk_model_finalize(wk_model* m) {
    if (!m) return WK_ERR_INVALID_ARGUMENT;
    WK_CUDA_CHECK(cudaStreamSynchronize(m->stream));
    m->finalized = true;
    return WK_OK;
}

// seeded synthetic weights of decoder weight set w (the model's decoder or its draft); *k numbers the fills
static wk_status init_decoder_random(wk_model* m, const DecoderWeights& w, uint64_t* k, float std) {
    const wk_model_config& c = m->cfg;
    const int d = c.d_model, dt = c.dtype;
    cudaStream_t s = m->stream;
    auto W = [&](void* p, size_t n, int dtype) { return fill_random_16(p, (int64_t)n, ++*k, std, 0.f, dtype, s); };
    auto F = [&](float* p, size_t n, float mean) { return fill_random_f32(p, (int64_t)n, ++*k, std, mean, s); };
    auto LN = [&](const LayerNormW& l) { wk_status r = F(l.g, d, 1.f); return r != WK_OK ? r : F(l.b, d, 0.f); };
    WK_CHECK(W(w.emb, (size_t)c.vocab * d, dt));
    WK_CHECK(F(w.pos, (size_t)c.n_text_ctx * d, 0.f));
    for (int i = 0; i < w.n_layers; ++i) {
        const DecLayer& l = w.layers[i];
        WK_CHECK(LN(l.ln1)); WK_CHECK(LN(l.lnx)); WK_CHECK(LN(l.ln3));
        WK_CHECK(W(l.wqkv, (size_t)3 * d * d, dt)); WK_CHECK(F(l.bq, d, 0.f)); WK_CHECK(F(l.bv, d, 0.f));
        WK_CHECK(W(l.wo, (size_t)d * d, dt)); WK_CHECK(F(l.bo, d, 0.f));
        WK_CHECK(W(l.wcq, (size_t)d * d, dt)); WK_CHECK(F(l.bcq, d, 0.f));
        WK_CHECK(W(l.wco, (size_t)d * d, dt)); WK_CHECK(F(l.bco, d, 0.f));
        WK_CHECK(W(l.w1, (size_t)4 * d * d, dt)); WK_CHECK(F(l.b1, 4 * d, 0.f));
        WK_CHECK(W(l.w2, (size_t)4 * d * d, dt)); WK_CHECK(F(l.b2, d, 0.f));
    }
    WK_CHECK(LN(w.ln));
    WK_CHECK(W(w.wckv, (size_t)2 * w.n_layers * d * d, dt));
    WK_CHECK(F(w.bckv, (size_t)2 * w.n_layers * d, 0.f));
    for (int i = 0; i < w.n_layers; ++i) WK_CUDA_CHECK(cudaMemsetAsync(w.bckv + 2 * (size_t)i * d, 0, d * 4, s));  // no key bias
    return WK_OK;
}

wk_status wk_model_init_random(wk_model* m, uint64_t seed, float std) {
    if (!m) return WK_ERR_INVALID_ARGUMENT;
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    const wk_model_config& c = m->cfg;
    const int d = c.d_model, dt = c.dtype;
    cudaStream_t s = m->stream;
    uint64_t k = seed * 1000003ull;
    auto W = [&](void* p, size_t n, int dtype) { return fill_random_16(p, (int64_t)n, ++k, std, 0.f, dtype, s); };
    auto F = [&](float* p, size_t n, float mean) { return fill_random_f32(p, (int64_t)n, ++k, std, mean, s); };
    auto LN = [&](LayerNormW& l) { wk_status r = F(l.g, d, 1.f); return r != WK_OK ? r : F(l.b, d, 0.f); };
    WK_CHECK(W(m->conv1_w, (size_t)d * 3 * 128, WK_DTYPE_F16));
    if (c.n_mels < kMelCols) {  // zero the padded input channels (keeps the padded GEMM exact)
        std::vector<float> w((size_t)d * c.n_mels * 3);
        srand((unsigned)seed);
        for (auto& v : w) v = std * ((rand() / (float)RAND_MAX) * 2.f - 1.f) * 1.7f;
        int64_t shp[3] = {d, c.n_mels, 3};
        WK_CHECK(wk_model_set_tensor(m, "model.encoder.conv1.weight", w.data(), WK_DTYPE_F32, shp, 3));
    }
    WK_CHECK(F(m->conv1_b, d, 0.f));
    WK_CHECK(W(m->conv2_w, (size_t)d * 3 * d, WK_DTYPE_F16));
    WK_CHECK(F(m->conv2_b, d, 0.f));
    {
        std::vector<float> pe((size_t)c.n_audio_ctx * d);
        const int half = d / 2;
        const double inc = log(10000.0) / (half - 1);
        for (int t = 0; t < c.n_audio_ctx; ++t)
            for (int i = 0; i < half; ++i) {
                const double a = t * exp(-inc * i);
                pe[(size_t)t * d + i] = (float)sin(a);
                pe[(size_t)t * d + half + i] = (float)cos(a);
            }
        WK_CUDA_CHECK(cudaMemcpyAsync(m->enc_pos, pe.data(), pe.size() * 4, cudaMemcpyHostToDevice, s));
        WK_CUDA_CHECK(cudaStreamSynchronize(s));
    }
    for (auto& l : m->enc) {
        WK_CHECK(LN(l.ln1)); WK_CHECK(LN(l.ln2));
        WK_CHECK(W(l.wqkv, (size_t)3 * d * d, dt)); WK_CHECK(F(l.bqkv, 3 * d, 0.f));
        WK_CUDA_CHECK(cudaMemsetAsync(l.bqkv + d, 0, d * 4, s));  // no key bias
        WK_CHECK(W(l.wo, (size_t)d * d, dt)); WK_CHECK(F(l.bo, d, 0.f));
        WK_CHECK(W(l.w1, (size_t)4 * d * d, dt)); WK_CHECK(F(l.b1, 4 * d, 0.f));
        WK_CHECK(W(l.w2, (size_t)4 * d * d, dt)); WK_CHECK(F(l.b2, d, 0.f));
    }
    WK_CHECK(LN(m->enc_ln));
    WK_CHECK(init_decoder_random(m, m->main_decoder(), &k, std));
    WK_CUDA_CHECK(cudaStreamSynchronize(s));
    if (m->enc_fp8) WK_CHECK(quantize_enc_weights(m));
    m->finalized = true;
    return WK_OK;
}

wk_status wk_model_info_get(const wk_model* m, wk_model_info* o) {
    if (!m || !o) return WK_ERR_INVALID_ARGUMENT;
    const wk_model_config& c = m->cfg;
    o->n_mels = c.n_mels; o->n_audio_ctx = c.n_audio_ctx; o->d_model = c.d_model; o->n_heads = c.n_heads;
    o->enc_layers = c.enc_layers; o->dec_layers = c.dec_layers; o->vocab = c.vocab;
    o->kv_embed_dim = c.dec_layers * c.d_model; o->kv_max_len = kKvMaxLen; o->window_samples = kWindowSamples;
    // the reference derives supportsWordTimestamps from the presence of the alignment_heads_weights output (TextDecoder.swift:309-311);
    // here: checkpoint-specific heads were supplied (generation_config.json or wk_model_set_alignment_heads)
    o->has_alignment_heads = m->has_alignment_heads;
    o->is_multilingual = c.vocab != 51864;
    o->dtype = c.dtype; o->max_batch = c.max_batch;
    o->cross_kv_dtype = m->cross_kv_fp8 ? WK_DTYPE_FP8_E4M3 : c.dtype;
    return WK_OK;
}

wk_status wk_model_set_cross_kv_dtype(wk_model* m, int32_t dtype) {
    if (!m) return WK_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> lock(m->api_mu);   // wk_session_create reads the policy and marks the model under the same lock
    if (m->session_created) { set_error("wk_model_set_cross_kv_dtype: the cross K/V storage is fixed once a session exists"); return WK_ERR_INVALID_ARGUMENT; }
    if (dtype != WK_DTYPE_FP8_E4M3 && dtype != m->cfg.dtype) {
        set_error("wk_model_set_cross_kv_dtype: dtype %d is neither WK_DTYPE_FP8_E4M3 nor the model's dtype %d", dtype, m->cfg.dtype);
        return WK_ERR_INVALID_ARGUMENT;
    }
    if (dtype == WK_DTYPE_FP8_E4M3 && m->cfg.n_audio_ctx % 500 != 0) {   // the FP8 cross-attention kernel streams 250-row stages
        set_error("wk_model_set_cross_kv_dtype: the FP8 cache needs n_audio_ctx to be a multiple of 500 (%d)", m->cfg.n_audio_ctx);
        return WK_ERR_INVALID_ARGUMENT;
    }
    m->cross_kv_fp8 = dtype == WK_DTYPE_FP8_E4M3;
    return WK_OK;
}

wk_status wk_model_set_encoder_dtype(wk_model* m, int32_t dtype) {
    if (!m) return WK_ERR_INVALID_ARGUMENT;
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    std::lock_guard<std::mutex> lock(m->api_mu);   // wk_session_create and wk_encode mark the model under the same lock
    if (m->session_created || m->encoded) {
        set_error("wk_model_set_encoder_dtype: the encoder precision is fixed once a session exists or wk_encode has run");
        return WK_ERR_INVALID_ARGUMENT;
    }
    if (dtype != WK_DTYPE_FP8_E4M3 && dtype != m->cfg.dtype) {
        set_error("wk_model_set_encoder_dtype: dtype %d is neither WK_DTYPE_FP8_E4M3 nor the model's dtype %d", dtype, m->cfg.dtype);
        return WK_ERR_INVALID_ARGUMENT;
    }
    if (dtype == WK_DTYPE_FP8_E4M3 && !m->enc_fp8) {
        const size_t d = m->cfg.d_model;
        for (EncLayer& l : m->enc) {
            if (l.wqkv8) continue;   // kept from an earlier FP8 setting
            WK_CHECK(m->mem.dmalloc(&l.wqkv8, 3 * d * d, false)); WK_CHECK(m->mem.dmalloc(&l.sqkv, 3 * d, false));
            WK_CHECK(m->mem.dmalloc(&l.w18, 4 * d * d, false)); WK_CHECK(m->mem.dmalloc(&l.s1, 4 * d, false));
            WK_CHECK(m->mem.dmalloc(&l.w28, 4 * d * d, false)); WK_CHECK(m->mem.dmalloc(&l.s2, d, false));
        }
        WK_CHECK(quantize_enc_weights(m));
    }
    m->enc_fp8 = dtype == WK_DTYPE_FP8_E4M3;
    return WK_OK;
}

wk_status wk_model_encoder_dtype(const wk_model* m, int32_t* dtype) {
    if (!m || !dtype) return WK_ERR_INVALID_ARGUMENT;
    *dtype = m->enc_fp8 ? WK_DTYPE_FP8_E4M3 : m->cfg.dtype;
    return WK_OK;
}

wk_status wk_fp8_quantize_blocks(const float* x, int64_t rows, int64_t cols, int64_t block, uint8_t* codes, float* scales) {
    if (!x || !codes || !scales || rows < 0 || block < 1 || cols < 0 || cols % block != 0) {
        set_error("wk_fp8_quantize_blocks: bad arguments");
        return WK_ERR_INVALID_ARGUMENT;
    }
    const int64_t nb = cols / block;
    for (int64_t r = 0; r < rows; ++r)
        for (int64_t b = 0; b < nb; ++b) fp8_quantize_row(x + r * cols + b * block, (int)block, codes + r * cols + b * block, scales + r * nb + b);
    return WK_OK;
}

wk_status wk_cross_kv_quantize_rows(const float* x, int64_t rows, uint8_t* codes, float* scales) {
    if (!x || !codes || !scales || rows < 0) { set_error("wk_cross_kv_quantize_rows: bad arguments"); return WK_ERR_INVALID_ARGUMENT; }
    for (int64_t r = 0; r < rows; ++r) fp8_quantize_row(x + r * 64, 64, codes + r * 64, scales + r);
    return WK_OK;
}

wk_model::~wk_model() {
    for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
    if (stream) cudaStreamDestroy(stream);
}

// ---------------------------------------------------------------------------------------------- draft decoder (speculative decoding)
// Refuses once a session exists: sessions size their draft buffers from the draft decoder they first see.  Called under api_mu.
static wk_status draft_settable(wk_model* m, const char* fn) {
    if (m->session_created) { set_error("%s: the draft decoder is fixed once a session exists", fn); return WK_ERR_INVALID_ARGUMENT; }
    return WK_OK;
}

wk_status wk_model_create_draft(wk_model* m, int32_t dec_layers) {
    if (!m) return WK_ERR_INVALID_ARGUMENT;
    if (dec_layers < 1 || dec_layers > 64) { set_error("wk_model_create_draft: %d decoder layers outside [1, 64]", dec_layers); return WK_ERR_INVALID_ARGUMENT; }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    std::lock_guard<std::mutex> lock(m->api_mu);
    WK_CHECK(draft_settable(m, "wk_model_create_draft"));
    const wk_model_config& c = m->cfg;
    const int d = c.d_model;
    std::unique_ptr<DraftDecoder> dr(new DraftDecoder());
    Buffers& b = dr->mem;
    WK_CHECK(b.alloc16(&dr->emb, (size_t)round_up(c.vocab, 128) * d));   // padded like the model's: the logits GEMM's last TMA tile
    WK_CHECK(b.dmalloc(&dr->pos, (size_t)c.n_text_ctx * d));
    dr->dec.resize(dec_layers);
    for (auto& l : dr->dec) {
        WK_CHECK(alloc_ln(b, l.ln1, d)); WK_CHECK(alloc_ln(b, l.lnx, d)); WK_CHECK(alloc_ln(b, l.ln3, d));
        WK_CHECK(b.alloc16(&l.wqkv, (size_t)3 * d * d)); WK_CHECK(b.dmalloc(&l.bq, d)); WK_CHECK(b.dmalloc(&l.bv, d));
        WK_CHECK(b.alloc16(&l.wo, (size_t)d * d)); WK_CHECK(b.dmalloc(&l.bo, d));
        WK_CHECK(b.alloc16(&l.wcq, (size_t)d * d)); WK_CHECK(b.dmalloc(&l.bcq, d));
        WK_CHECK(b.alloc16(&l.wco, (size_t)d * d)); WK_CHECK(b.dmalloc(&l.bco, d));
        WK_CHECK(b.alloc16(&l.w1, (size_t)4 * d * d)); WK_CHECK(b.dmalloc(&l.b1, 4 * d));
        WK_CHECK(b.alloc16(&l.w2, (size_t)4 * d * d)); WK_CHECK(b.dmalloc(&l.b2, d));
    }
    WK_CHECK(alloc_ln(b, dr->ln, d));
    WK_CHECK(b.alloc16(&dr->wckv, (size_t)2 * dec_layers * d * d));
    WK_CHECK(b.dmalloc(&dr->bckv, (size_t)2 * dec_layers * d));
    WK_CUDA_CHECK(cudaDeviceSynchronize());   // the zero fills ran on the legacy default stream
    m->draft = std::move(dr);
    return WK_OK;
}

wk_status wk_model_set_draft_tensor(wk_model* m, const char* name, const void* data, int32_t dtype, const int64_t* shape, int32_t ndim) {
    if (!m || !name || !data) { set_error("wk_model_set_draft_tensor: null argument"); return WK_ERR_INVALID_ARGUMENT; }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    {
        std::lock_guard<std::mutex> lock(m->api_mu);
        WK_CHECK(draft_settable(m, "wk_model_set_draft_tensor"));
    }
    if (!m->draft) { set_error("wk_model_set_draft_tensor: the model has no draft decoder (wk_model_create_draft)"); return WK_ERR_INVALID_ARGUMENT; }
    Dest dst;
    if (!resolve_decoder_name(m, m->draft->view(), name, &dst)) {
        if (strstr(name, "k_proj.bias")) return WK_OK;
        set_error("wk_model_set_draft_tensor: unknown draft decoder parameter '%s'", name);
        return WK_ERR_INVALID_ARGUMENT;
    }
    return store_tensor(m, dst, name, data, dtype, shape, ndim);
}

wk_status wk_model_init_draft_random(wk_model* m, uint64_t seed, float std) {
    if (!m) return WK_ERR_INVALID_ARGUMENT;
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    {
        std::lock_guard<std::mutex> lock(m->api_mu);
        WK_CHECK(draft_settable(m, "wk_model_init_draft_random"));
    }
    if (!m->draft) { set_error("wk_model_init_draft_random: the model has no draft decoder (wk_model_create_draft)"); return WK_ERR_INVALID_ARGUMENT; }
    uint64_t k = seed * 1000003ull;
    WK_CHECK(init_decoder_random(m, m->draft->view(), &k, std));
    WK_CUDA_CHECK(cudaStreamSynchronize(m->stream));
    return WK_OK;
}

wk_status wk_model_load_draft(wk_model* m, const char* weights_dir) {
    if (!m || !weights_dir) { set_error("wk_model_load_draft: null argument"); return WK_ERR_INVALID_ARGUMENT; }
    const std::string dir = weights_dir;
    std::vector<char> cfgbuf;
    if (!read_file(dir + "/config.json", &cfgbuf)) { set_error("wk_model_load_draft: %s/config.json not found", weights_dir); return WK_ERR_MODELS_UNAVAILABLE; }
    const std::string cj(cfgbuf.begin(), cfgbuf.end());
    const wk_model_config& c = m->cfg;
    long long dm = 0, heads = 0, vocab = 0, layers = 0, ctx = 1500;
    json_int(cj, "d_model", &dm);
    if (!json_int(cj, "decoder_attention_heads", &heads)) json_int(cj, "encoder_attention_heads", &heads);
    json_int(cj, "vocab_size", &vocab);
    json_int(cj, "decoder_layers", &layers);
    json_int(cj, "max_source_positions", &ctx);
    if (dm != c.d_model || heads != c.n_heads || vocab != c.vocab || ctx != c.n_audio_ctx) {
        set_error("wk_model_load_draft: the draft (d_model %lld, heads %lld, vocab %lld, n_audio_ctx %lld) does not match the model (%d, %d, %d, %d)",
                  dm, heads, vocab, ctx, c.d_model, c.n_heads, c.vocab, c.n_audio_ctx);
        return WK_ERR_INVALID_ARGUMENT;
    }
    const std::vector<std::string> files = safetensors_files(dir);
    if (files.empty()) { set_error("wk_model_load_draft: no *.safetensors in %s", weights_dir); return WK_ERR_MODELS_UNAVAILABLE; }
    WK_CHECK(wk_model_create_draft(m, (int32_t)layers));
    int n_loaded = 0;
    wk_status st = WK_OK;
    for (const auto& fp : files) if (st == WK_OK) st = load_safetensors_file(m, fp, &n_loaded, true);
    const int expected = 4 + (int)layers * 24;
    if (st == WK_OK && n_loaded < expected) {
        set_error("wk_model_load_draft: only %d of %d expected decoder tensors found in %s", n_loaded, expected, weights_dir);
        st = WK_ERR_MODELS_UNAVAILABLE;
    }
    if (st != WK_OK) {
        std::lock_guard<std::mutex> lock(m->api_mu);
        m->draft.reset();   // a half-loaded draft is never used
    }
    return st;
}

wk_status wk_model_draft_layers(const wk_model* m, int32_t* n) {
    if (!m || !n) return WK_ERR_INVALID_ARGUMENT;
    *n = m->draft ? (int32_t)m->draft->dec.size() : 0;
    return WK_OK;
}

void wk_model_free(wk_model* m) {
    if (!m) return;
    cudaSetDevice(m->device);
    cudaDeviceSynchronize();
    delete m;
}

void* wk_model_stream(wk_model* m) { return m ? (void*)m->stream : nullptr; }

// ---------------------------------------------------------------------------------------------- tensors
// A wk_tensor owns its device buffer (stream-ordered allocation on the model stream): the MLMultiArray a Swift host gets back from
// logMelSpectrogram / encodeFeatures stays valid until it is released, whatever the host does with the model in between.
static wk_status tensor_new(wk_model* m, int kind, int dtype, int64_t batch, size_t bytes, wk_tensor** out) {
    wk_tensor* t = new wk_tensor();
    t->kind = kind; t->dtype = dtype; t->batch = batch; t->owner = m; t->data = nullptr;
    cudaEvent_t ready = nullptr;
    cudaError_t e = cudaMallocAsync(&t->data, bytes, m->stream);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ready, cudaEventDisableTiming);
    if (e == cudaSuccess) t->events.push_back(ready);
    if (e != cudaSuccess) { set_error("tensor allocation of %zu bytes failed: %s", bytes, cudaGetErrorString(e)); delete t; return WK_ERR_CUDA; }
    *out = t;
    return WK_OK;
}

wk_status wk_tensor_shape(const wk_tensor* t, int64_t* shape4, int32_t* ndim, int32_t* dtype) {
    if (!t) return WK_ERR_INVALID_ARGUMENT;
    const wk_model_config& c = t->owner->cfg;
    if (t->kind == 0) { shape4[0] = t->batch; shape4[1] = c.n_mels; shape4[2] = 1; shape4[3] = 3000; }
    else { shape4[0] = t->batch; shape4[1] = c.d_model; shape4[2] = 1; shape4[3] = c.n_audio_ctx; }
    if (ndim) *ndim = 4;
    if (dtype) *dtype = t->dtype;
    return WK_OK;
}

wk_status wk_tensor_to_host_strided(const wk_tensor* t, float* dst, int64_t stride_b, int64_t stride_c, int64_t stride_t, int64_t dst_elems) {
    if (!t || !dst) return WK_ERR_INVALID_ARGUMENT;
    wk_model* m = t->owner;
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    const wk_model_config& c = m->cfg;
    const int64_t rows = t->kind == 0 ? 3000 : c.n_audio_ctx, cols = t->kind == 0 ? c.n_mels : c.d_model;
    const int64_t n = t->batch * rows * cols;
    const bool packed = stride_t == 1 && stride_c == rows && stride_b == rows * cols;
    const int64_t span = (t->batch - 1) * stride_b + (cols - 1) * stride_c + (rows - 1) * stride_t + 1;
    if (stride_b < 1 || stride_c < 1 || stride_t < 1 || dst_elems < span) {
        set_error("wk_tensor_to_host: destination too small or bad strides (%lld elements, need %lld)", (long long)dst_elems, (long long)span);
        return WK_ERR_INVALID_ARGUMENT;
    }
    std::lock_guard<std::mutex> lock(m->api_mu);
    float* tmp = nullptr;
    WK_CUDA_CHECK(cudaMallocAsync((void**)&tmp, n * 4, m->stream));
    wk_status s = t->kind == 0
        ? transpose_to_host_layout(t->data, tmp, t->batch, rows, cols, kMelRows, 1, kMelCols, WK_DTYPE_F16, m->stream)
        : transpose_to_host_layout(t->data, tmp, t->batch, rows, cols, rows, 0, cols, t->dtype, m->stream);
    if (s == WK_OK) {
        cudaError_t e;
        if (packed) {
            e = cudaMemcpyAsync(dst, tmp, n * 4, cudaMemcpyDeviceToHost, m->stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(m->stream);
        } else {
            // padded MLMultiArray rows (IOSurface-backed Float16/Float32 arrays, MLMultiArrayExtensions.swift:11-21): element strides
            std::vector<float> host((size_t)n);
            e = cudaMemcpyAsync(host.data(), tmp, n * 4, cudaMemcpyDeviceToHost, m->stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(m->stream);
            if (e == cudaSuccess)
                for (int64_t b = 0; b < t->batch; ++b)
                    for (int64_t ch = 0; ch < cols; ++ch)
                        for (int64_t r = 0; r < rows; ++r) dst[b * stride_b + ch * stride_c + r * stride_t] = host[(size_t)((b * cols + ch) * rows + r)];
        }
        if (e != cudaSuccess) { set_error("wk_tensor_to_host: %s", cudaGetErrorString(e)); s = WK_ERR_CUDA; }
    }
    cudaFreeAsync(tmp, m->stream);
    return s;
}

wk_status wk_tensor_to_host(const wk_tensor* t, float* dst, int64_t dst_elems) {
    if (!t) return WK_ERR_INVALID_ARGUMENT;
    const wk_model_config& c = t->owner->cfg;
    const int64_t rows = t->kind == 0 ? 3000 : c.n_audio_ctx, cols = t->kind == 0 ? c.n_mels : c.d_model;
    return wk_tensor_to_host_strided(t, dst, rows * cols, rows, 1, dst_elems);
}

void wk_tensor_free(wk_tensor* t) {
    if (!t) return;
    wk_model* m = t->owner;
    cudaSetDevice(m->device);
    {
        std::lock_guard<std::mutex> lock(m->api_mu);
        for (cudaEvent_t e : t->events) cudaStreamWaitEvent(m->stream, e, 0);   // readers on session streams (cross-KV projection) finish first
        cudaFreeAsync(t->data, m->stream);
    }
    for (cudaEvent_t e : t->events) cudaEventDestroy(e);
    delete t;
}

// ---------------------------------------------------------------------------------------------- mel / encode
wk_status wk_mel(wk_model* m, const float* pcm, int64_t n_windows, int64_t stride, const int32_t* samples_per_window, wk_tensor** mel_out) {
    if (!m || !pcm || !mel_out) { set_error("wk_mel: null argument"); return WK_ERR_INVALID_ARGUMENT; }
    if (n_windows < 1 || n_windows > m->cfg.max_batch) { set_error("wk_mel: n_windows %lld outside [1, max_batch=%d]", (long long)n_windows, m->cfg.max_batch); return WK_ERR_AUDIO_PROCESSING_FAILED; }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    std::lock_guard<std::mutex> lock(m->api_mu);
    WK_CHECK(enc_ws_ensure(m, &m->ws, m->cfg.max_batch));
    wk_tensor* t = nullptr;
    WK_CHECK(tensor_new(m, 0, WK_DTYPE_F16, n_windows, (size_t)n_windows * kMelRows * kMelCols * 2, &t));
    // rows 0 / 3001 (the conv stem's zero padding) and the channels past n_mels are never written by the mel kernels
    WK_CUDA_CHECK(cudaMemsetAsync(t->data, 0, (size_t)n_windows * kMelRows * kMelCols * 2, m->stream));
    wk_status s = mel_run(m, &m->ws, pcm, n_windows, stride, samples_per_window, t->data, m->stream);
    if (s != WK_OK) { cudaFreeAsync(t->data, m->stream); cudaEventDestroy(t->events[0]); delete t; return s; }
    WK_CUDA_CHECK(cudaEventRecord(t->events[0], m->stream));
    *mel_out = t;
    return WK_OK;
}

wk_status wk_encode(wk_model* m, const wk_tensor* mel, wk_tensor** enc_out) {
    if (!m || !mel || !enc_out) { set_error("wk_encode: null argument"); return WK_ERR_INVALID_ARGUMENT; }
    if (!m->finalized) { set_error("wk_encode: model weights not finalized"); return WK_ERR_MODELS_UNAVAILABLE; }
    if (mel->kind != 0 || mel->owner != m) { set_error("wk_encode: input is not this model's mel tensor"); return WK_ERR_INVALID_ARGUMENT; }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    std::lock_guard<std::mutex> lock(m->api_mu);
    WK_CHECK(enc_ws_ensure(m, &m->ws, m->cfg.max_batch));
    m->encoded = true;
    wk_tensor* t = nullptr;
    WK_CHECK(tensor_new(m, 1, m->cfg.dtype, mel->batch, (size_t)mel->batch * m->cfg.n_audio_ctx * m->cfg.d_model * 2, &t));
    wk_status s = encode_chunk(m, &m->ws, mel->data, (int)mel->batch, t->data, m->stream);
    if (s != WK_OK) { cudaFreeAsync(t->data, m->stream); cudaEventDestroy(t->events[0]); delete t; return s; }
    WK_CUDA_CHECK(cudaEventRecord(t->events[0], m->stream));   // (the mel tensor is read and released on this same stream: ordered)
    *enc_out = t;
    return WK_OK;
}

wk_status wk_filter_sample(wk_model* m, const wk_special_tokens* st, const wk_decode_opts* opts, int32_t is_multilingual,
                           const float* logits, int32_t batch, int32_t vocab, const int32_t* tokens, int32_t ld_tokens,
                           const int32_t* n_tokens, int32_t sample_begin_ts, int32_t sample_begin_blank,
                           const int32_t* language_tokens, int32_t n_language_tokens, int32_t language_sample_begin,
                           int32_t* token_out, float* logprob_out, float* filtered_out) {
    if (!m || !st || !opts || !logits || !n_tokens || batch < 1 || vocab < 2) { set_error("wk_filter_sample: bad arguments"); return WK_ERR_INVALID_ARGUMENT; }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    std::lock_guard<std::mutex> lock(m->api_mu);
    cudaStream_t s = m->stream;
    float *dlog = nullptr, *dfil = nullptr, *dlp = nullptr;
    int32_t *dtok = nullptr, *dn = nullptr, *dout = nullptr, *dsup = nullptr, *dlang = nullptr;
    const int ldt = ld_tokens > 0 ? ld_tokens : 1;
    Buffers scratch;
    WK_CHECK(scratch.dmalloc(&dlog, (size_t)batch * vocab, false));
    WK_CHECK(scratch.dmalloc(&dfil, (size_t)batch * vocab, false));
    WK_CHECK(scratch.dmalloc(&dlp, batch, false));
    WK_CHECK(scratch.dmalloc(&dtok, (size_t)batch * ldt, false));
    WK_CHECK(scratch.dmalloc(&dn, batch, false));
    WK_CHECK(scratch.dmalloc(&dout, batch, false));
    WK_CHECK(scratch.dmalloc(&dsup, 4096, false));
    WK_CHECK(scratch.dmalloc(&dlang, 4096, false));
    WK_CUDA_CHECK(cudaMemcpyAsync(dlog, logits, (size_t)batch * vocab * 4, cudaMemcpyDefault, s));
    if (tokens && ld_tokens > 0) WK_CUDA_CHECK(cudaMemcpyAsync(dtok, tokens, (size_t)batch * ldt * 4, cudaMemcpyDefault, s));
    WK_CUDA_CHECK(cudaMemcpyAsync(dn, n_tokens, batch * 4, cudaMemcpyDefault, s));
    SamplerParams p;
    memset(&p, 0, sizeof(p));
    p.st = *st; p.vocab = vocab; p.is_multilingual = is_multilingual; p.loop_mode = 0;
    p.sample_begin_ts = sample_begin_ts; p.sample_begin_blank = sample_begin_blank;
    std::vector<int32_t> sup;
    for (int i = 0; i < opts->n_suppress_tokens; ++i)
        if (opts->suppress_tokens[i] >= 0 && opts->suppress_tokens[i] < vocab) sup.push_back(opts->suppress_tokens[i]);
    if (sup.size() > 4096 || n_language_tokens > 4096) { set_error("wk_filter_sample: list too long"); return WK_ERR_INVALID_ARGUMENT; }
    if (!sup.empty()) WK_CUDA_CHECK(cudaMemcpyAsync(dsup, sup.data(), sup.size() * 4, cudaMemcpyHostToDevice, s));
    p.suppress = dsup; p.n_suppress = (int)sup.size();
    if (language_tokens && n_language_tokens > 0) {
        WK_CUDA_CHECK(cudaMemcpyAsync(dlang, language_tokens, n_language_tokens * 4, cudaMemcpyHostToDevice, s));
        p.language_tokens = dlang; p.n_language_tokens = n_language_tokens; p.language_sample_begin = language_sample_begin;
    }
    p.temperature = opts->temperature; p.top_k = opts->top_k; p.seed = opts->seed;
    p.max_ctx = kKvMaxLen;
    DecodeState none;
    memset(&none, 0, sizeof(none));
    wk_status r = sampler_filter_sample(dlog, vocab, p, none, dtok, ldt, dn, dout, dlp, dfil, batch, s);
    if (r == WK_OK) {
        cudaError_t e = cudaSuccess;
        if (token_out) e = cudaMemcpyAsync(token_out, dout, batch * 4, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess && logprob_out) e = cudaMemcpyAsync(logprob_out, dlp, batch * 4, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess && filtered_out) e = cudaMemcpyAsync(filtered_out, dfil, (size_t)batch * vocab * 4, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e != cudaSuccess) { set_error("wk_filter_sample: %s", cudaGetErrorString(e)); r = WK_ERR_CUDA; }
    }
    return r;
}

static void default_alignment_heads(wk_model* m) {
    // openai-whisper's default when a checkpoint names no alignment heads: every head of the last half of the decoder layers
    const int L = m->cfg.dec_layers, H = m->cfg.n_heads;
    m->align_mask.assign(L, 0u);
    m->align_base.assign(L, 0);
    int slots = 0;
    for (int l = 0; l < L; ++l) {
        m->align_base[l] = slots;
        if (l >= L / 2) { m->align_mask[l] = H >= 32 ? 0xffffffffu : ((1u << H) - 1u); slots += H; }
    }
    m->n_align_slots = slots;
}

wk_status wk_model_set_alignment_heads(wk_model* m, const int32_t* layer_head_pairs, int32_t n_pairs) {
    if (!m || n_pairs < 0 || (n_pairs > 0 && !layer_head_pairs)) { set_error("wk_model_set_alignment_heads: bad arguments"); return WK_ERR_INVALID_ARGUMENT; }
    if (n_pairs == 0) { default_alignment_heads(m); m->has_alignment_heads = 0; return WK_OK; }
    const int L = m->cfg.dec_layers, H = m->cfg.n_heads;
    std::vector<uint32_t> mask(L, 0u);
    for (int i = 0; i < n_pairs; ++i) {
        const int l = layer_head_pairs[2 * i], h = layer_head_pairs[2 * i + 1];
        if (l < 0 || l >= L || h < 0 || h >= H || h >= 32) { set_error("wk_model_set_alignment_heads: (layer %d, head %d) out of range", l, h); return WK_ERR_INVALID_ARGUMENT; }
        mask[l] |= 1u << h;
    }
    m->align_mask = mask;
    m->align_base.assign(L, 0);
    int slots = 0;
    for (int l = 0; l < L; ++l) { m->align_base[l] = slots; slots += __builtin_popcount(mask[l]); }
    m->n_align_slots = slots;
    m->has_alignment_heads = 1;
    return WK_OK;
}

int64_t wk_kernel_launch_count(int32_t reset) {
    const long long v = wk::launch_counter_load();
    if (reset) wk::launch_counter_sub(v);
    return v;
}

wk_status wk_debug_live_bytes(int64_t* device_bytes, int64_t* pinned_bytes) {
    if (!device_bytes || !pinned_bytes) return WK_ERR_INVALID_ARGUMENT;
    *device_bytes = g_live_bytes[0].load();
    *pinned_bytes = g_live_bytes[1].load();
    return WK_OK;
}

wk_status wk_last_timings(wk_model* m, float* ms6) {
    if (!m || !ms6) return WK_ERR_INVALID_ARGUMENT;
    memcpy(ms6, m->timings, sizeof(m->timings));
    return WK_OK;
}

// ---------------------------------------------------------------------------------------------- kernel-level hooks
wk_status wk_test_gemm(wk_model* m, const void* a, const void* w, const float* bias, void* out, int32_t M, int32_t N, int32_t K,
                       int32_t in_dtype, int32_t out_dtype, int32_t gelu) {
    if (!m) return WK_ERR_INVALID_ARGUMENT;
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    std::lock_guard<std::mutex> lock(m->api_mu);
    const int mode = out_dtype == WK_DTYPE_F32 ? GEMM_OUT_F32 : GEMM_OUT_T16;
    WK_CHECK(gemm_wgmma(plain_gemm(a, M, K, w, N, in_dtype, mode, out, N, bias, gelu), m->num_sms, m->stream));
    WK_CUDA_CHECK(cudaStreamSynchronize(m->stream));
    return WK_OK;
}

// out[M, N] (f32, in place) += A W^T + bias: the residual-update epilogue of the encoder's out-proj / FC2 (GEMM_OUT_F32_ADD)
wk_status wk_test_gemm_residual(wk_model* m, const void* a, const void* w, const float* bias, float* out, int32_t M, int32_t N, int32_t K, int32_t in_dtype) {
    if (!m || !a || !w || !out) return WK_ERR_INVALID_ARGUMENT;
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    std::lock_guard<std::mutex> lock(m->api_mu);
    WK_CHECK(gemm_wgmma(plain_gemm(a, M, K, w, N, in_dtype, GEMM_OUT_F32_ADD, out, N, bias, 0), m->num_sms, m->stream));
    WK_CUDA_CHECK(cudaStreamSynchronize(m->stream));
    return WK_OK;
}

// The FP8 encoder GEMM alone: kind 0 QKV (16-bit out), 1 FC1 (GELU, E4M3 codes + block scales out), 2 FC2 (f32 residual in place)
wk_status wk_test_gemm_fp8(wk_model* m, int32_t kind, const uint8_t* a, const float* a_scale, const uint8_t* w, const float* w_scale,
                           const float* bias, void* out, float* out_scale, int32_t M, int32_t N, int32_t K, int32_t dtype) {
    if (!m || !a || !a_scale || !w || !w_scale || !out || kind < 0 || kind > 2 || (kind == 1 && !out_scale) || M < 1) {
        set_error("wk_test_gemm_fp8: bad arguments");
        return WK_ERR_INVALID_ARGUMENT;
    }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    std::lock_guard<std::mutex> lock(m->api_mu);
    static const int modes[3] = {GEMM_OUT_T16, GEMM_OUT_FP8_BLOCKS, GEMM_OUT_F32_ADD};
    WK_CHECK(gemm_wgmma_fp8(fp8_gemm(a, a_scale, round_up(M, 128), M, K, w, w_scale, N, dtype, modes[kind], out, out_scale, bias, kind == 1),
                            m->num_sms, m->stream));
    WK_CUDA_CHECK(cudaStreamSynchronize(m->stream));
    return WK_OK;
}

__global__ void reduce_partials_kernel(const float* __restrict__ partial, int splits, int Bp, int N, int rows, float* __restrict__ out) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)rows * N) return;
    const int b = (int)(idx / N), i = (int)(idx % N);
    float a = 0.f;
    for (int s = 0; s < splits; ++s) a += partial[((long long)s * Bp + b) * N + i];
    out[idx] = a;
}

wk_status wk_test_gemm_splitk(wk_model* m, const void* w, const void* x, float* out, int32_t N, int32_t rows_x, int32_t K, int32_t in_dtype, int32_t splits) {
    if (!m) return WK_ERR_INVALID_ARGUMENT;
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    std::lock_guard<std::mutex> lock(m->api_mu);
    if (rows_x % 16 != 0 || rows_x > 256) { set_error("wk_test_gemm_splitk: rows_x must be a multiple of 16 <= 256"); return WK_ERR_INVALID_ARGUMENT; }
    const int tiles = (N + 127) / 128;
    const int sp = splits > 0 ? splits : choose_splits(tiles, K / 64, m->num_sms);
    Buffers scratch;
    float* partial = nullptr;
    WK_CHECK(scratch.dmalloc(&partial, (size_t)sp * rows_x * N, false));
    GemmDesc g;
    memset(&g, 0, sizeof(g));
    g.a = w; g.a_rows = N; g.a_cols = K; g.a_ld = K; g.a_batches = 1;
    g.b = x; g.b_rows = rows_x; g.b_ld = K; g.in_dtype = in_dtype;
    g.m_rows_per_batch = N; g.n = rows_x; g.k = K; g.taps = 1; g.bn = rows_x; g.splits = sp;
    g.mode = GEMM_OUT_PARTIAL_T; g.out = partial; g.ld_out = N; g.out_rows_per_batch = N; g.partial_cols = rows_x;
    wk_status r = gemm_wgmma(g, m->num_sms, m->stream);
    if (r == WK_OK) {
        const long long n = (long long)rows_x * N;
        reduce_partials_kernel<<<(unsigned)((n + 255) / 256), 256, 0, m->stream>>>(partial, sp, rows_x, N, rows_x, out);
        cudaError_t e = cudaStreamSynchronize(m->stream);
        if (e != cudaSuccess) { set_error("wk_test_gemm_splitk: %s", cudaGetErrorString(e)); r = WK_ERR_CUDA; }
    }
    return r;
}

wk_status wk_test_attention(wk_model* m, const void* qkv, void* out, int32_t B, int32_t T, int32_t n_heads, int32_t dtype) {
    if (!m) return WK_ERR_INVALID_ARGUMENT;
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    std::lock_guard<std::mutex> lock(m->api_mu);
    WK_CHECK(encoder_attention(qkv, out, B, T, n_heads, dtype, m->stream));
    WK_CUDA_CHECK(cudaStreamSynchronize(m->stream));
    return WK_OK;
}

// decoder_cross_attention_kernel alone: q [B][H*64] f32 (the un-reduced query, bias included), K/V [B][H][T][64] 16-bit -> out [B][H*64]
wk_status wk_test_cross_attention(wk_model* m, const float* q, const void* kcross, const void* vcross, void* out, int32_t B, int32_t H,
                                  int32_t T, int32_t dtype, const int32_t* done) {
    if (!m || !q || !kcross || !vcross || !out || B < 1 || H < 1 || H > 32) { set_error("wk_test_cross_attention: bad arguments"); return WK_ERR_INVALID_ARGUMENT; }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    std::lock_guard<std::mutex> lock(m->api_mu);
    Buffers scratch;
    float* zero = nullptr;
    WK_CHECK(scratch.dmalloc(&zero, (size_t)H * 64));
    wk_status r = decoder_cross_attention(q, 1, B, zero, kcross, vcross, out, B, H, T, dtype, m->stream, done);
    cudaError_t e = cudaStreamSynchronize(m->stream);
    if (r == WK_OK && e != cudaSuccess) { set_error("wk_test_cross_attention: %s", cudaGetErrorString(e)); r = WK_ERR_CUDA; }
    return r;
}

// the beam-search form: B rows in groups of kv_div adjacent rows that share one K/V block ([B / kv_div][H][T][64])
wk_status wk_test_cross_attention_shared(wk_model* m, const float* q, const void* kcross, const void* vcross, void* out, int32_t B, int32_t H,
                                         int32_t T, int32_t dtype, const int32_t* done, int32_t kv_div) {
    if (!m || !q || !kcross || !vcross || !out || B < 1 || H < 1 || H > 32 || kv_div < 1) { set_error("wk_test_cross_attention_shared: bad arguments"); return WK_ERR_INVALID_ARGUMENT; }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    std::lock_guard<std::mutex> lock(m->api_mu);
    Buffers scratch;
    float* zero = nullptr;
    WK_CHECK(scratch.dmalloc(&zero, (size_t)H * 64));
    wk_status r = decoder_cross_attention(q, 1, B, zero, kcross, vcross, out, B, H, T, dtype, m->stream, done, nullptr, 0, kv_div);
    cudaError_t e = cudaStreamSynchronize(m->stream);
    if (r == WK_OK && e != cudaSuccess) { set_error("wk_test_cross_attention_shared: %s", cudaGetErrorString(e)); r = WK_ERR_CUDA; }
    return r;
}

// the FP8 cache form of both: K/V codes [B / kv_div][H][T][64] u8 with row scales [B / kv_div][H][T] f32 (kv_div = 1: the single-query
// kernel; 2..8: the beam kernel).  align_out != nullptr: every head exports its softmax row into align_out [H][B][T] (single-query kernel)
wk_status wk_test_cross_attention_fp8(wk_model* m, const float* q, const uint8_t* kcodes, const uint8_t* vcodes, const float* kscale, const float* vscale,
                                      void* out, int32_t B, int32_t H, int32_t T, int32_t dtype, const int32_t* done, int32_t kv_div,
                                      float* align_out) {
    if (!m || !q || !kcodes || !vcodes || !kscale || !vscale || !out || B < 1 || H < 1 || H > 32 || kv_div < 1) {
        set_error("wk_test_cross_attention_fp8: bad arguments");
        return WK_ERR_INVALID_ARGUMENT;
    }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    std::lock_guard<std::mutex> lock(m->api_mu);
    Buffers scratch;
    float* zero = nullptr;
    WK_CHECK(scratch.dmalloc(&zero, (size_t)H * 64));
    const uint32_t all_heads = H == 32 ? 0xffffffffu : (1u << H) - 1u;
    wk_status r = decoder_cross_attention(q, 1, B, zero, kcodes, vcodes, out, B, H, T, dtype, m->stream, done, align_out, align_out ? all_heads : 0u,
                                          kv_div, kscale, vscale);
    cudaError_t e = cudaStreamSynchronize(m->stream);
    if (r == WK_OK && e != cudaSuccess) { set_error("wk_test_cross_attention_fp8: %s", cudaGetErrorString(e)); r = WK_ERR_CUDA; }
    return r;
}

wk_status wk_test_cross_kv_project(wk_model* m, const void* x, const void* w, const float* bias, int32_t windows, int32_t T, int32_t H,
                                   int32_t packed, void* out, uint8_t* hdr) {
    if (!m || !x || !w || !out || (packed && !hdr) || windows < 1 || T < 1 || H < 1) { set_error("wk_test_cross_kv_project: bad arguments"); return WK_ERR_INVALID_ARGUMENT; }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    std::lock_guard<std::mutex> lock(m->api_mu);
    const int d = H * 64;
    GemmDesc g = plain_gemm(x, (int64_t)windows * T, d, w, d, WK_DTYPE_BF16, packed ? GEMM_OUT_PACKED_HEADS : GEMM_OUT_T16_HEADS, out, 0, bias, 0);
    g.heads_T = T; g.heads_B = windows; g.heads_H = H; g.heads_dmodel = d;
    g.out_hdr = packed ? hdr : nullptr;
    wk_status r = gemm_wgmma(g, m->num_sms, m->stream);
    cudaError_t e = cudaStreamSynchronize(m->stream);
    if (r == WK_OK && e != cudaSuccess) { set_error("wk_test_cross_kv_project: %s", cudaGetErrorString(e)); r = WK_ERR_CUDA; }
    return r;
}

wk_status wk_test_cross_attention_packed(wk_model* m, const float* q, const void* kc, const void* vc, const uint8_t* khdr, const uint8_t* vhdr,
                                         void* out, int32_t B, int32_t H, int32_t T, const int32_t* done, int32_t kv_div, float* align_out) {
    if (!m || !q || !kc || !vc || !khdr || !vhdr || !out || B < 1 || H < 1 || H > 32 || kv_div < 1) {
        set_error("wk_test_cross_attention_packed: bad arguments");
        return WK_ERR_INVALID_ARGUMENT;
    }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    std::lock_guard<std::mutex> lock(m->api_mu);
    Buffers scratch;
    float* zero = nullptr;
    WK_CHECK(scratch.dmalloc(&zero, (size_t)H * 64));
    const uint32_t all_heads = H == 32 ? 0xffffffffu : (1u << H) - 1u;
    wk_status r = decoder_cross_attention(q, 1, B, zero, kc, vc, out, B, H, T, WK_DTYPE_BF16, m->stream, done, align_out, align_out ? all_heads : 0u,
                                          kv_div, nullptr, nullptr, false, khdr, vhdr);
    cudaError_t e = cudaStreamSynchronize(m->stream);
    if (r == WK_OK && e != cudaSuccess) { set_error("wk_test_cross_attention_packed: %s", cudaGetErrorString(e)); r = WK_ERR_CUDA; }
    return r;
}

wk_status wk_test_align_cross_attention(wk_model* m, const void* q, const void* kc, const void* vc, const uint8_t* khdr, const uint8_t* vhdr,
                                        const int32_t* seq_len, int32_t nw, int32_t H, int32_t T, uint32_t mask, void* out, float* acc) {
    if (!m || !q || !kc || !vc || !seq_len || !out || !acc || nw < 1 || H < 1 || H > 32 || (!khdr != !vhdr)) {
        set_error("wk_test_align_cross_attention: bad arguments");
        return WK_ERR_INVALID_ARGUMENT;
    }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    std::lock_guard<std::mutex> lock(m->api_mu);
    const int64_t rows = (int64_t)nw * 224;
    Buffers scratch;
    float* stats = nullptr;
    WK_CHECK(scratch.dmalloc(&stats, (size_t)2 * H * rows));
    wk_status r = align_cross_attention(q, kc, vc, nullptr, nullptr, seq_len, 0, out, stats, rows, nw, H, T, WK_DTYPE_BF16, m->stream, khdr, vhdr);
    if (r == WK_OK && mask) r = align_export(q, kc, nullptr, stats, rows, seq_len, 0, mask, 1, acc, nw, H, T, WK_DTYPE_BF16, m->stream, khdr);
    cudaError_t e = cudaStreamSynchronize(m->stream);
    if (r == WK_OK && e != cudaSuccess) { set_error("wk_test_align_cross_attention: %s", cudaGetErrorString(e)); r = WK_ERR_CUDA; }
    return r;
}

// decoder_self_attention_kernel alone: qkv [B][3*H*64] f32 (q | k | v of the new token, biases included), caches [B][H][224][64] 16-bit
// holding positions < pos[b]; appends the new K/V row at pos[b] and writes out [B][H*64]
wk_status wk_test_self_attention(wk_model* m, const float* qkv, void* kcache, void* vcache, const int32_t* pos, void* out, int32_t B,
                                 int32_t H, int32_t dtype, const int32_t* done) {
    if (!m || !qkv || !kcache || !vcache || !pos || !out || B < 1 || H < 1) { set_error("wk_test_self_attention: bad arguments"); return WK_ERR_INVALID_ARGUMENT; }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    std::lock_guard<std::mutex> lock(m->api_mu);
    Buffers scratch;
    float* zero = nullptr;
    WK_CHECK(scratch.dmalloc(&zero, (size_t)H * 64));
    wk_status r = decoder_self_attention(qkv, 1, B, zero, zero, kcache, vcache, pos, done, out, B, H, kKvMaxLen, dtype, m->stream);
    cudaError_t e = cudaStreamSynchronize(m->stream);
    if (r == WK_OK && e != cudaSuccess) { set_error("wk_test_self_attention: %s", cudaGetErrorString(e)); r = WK_ERR_CUDA; }
    return r;
}

// The swap-AB split-K GEMM configured as dec_gemm (partial_cols = rows_x) or the logits GEMM (partial_cols = B < rows_x, splits = 1) configure
// it, its raw partials [splits][partial_cols][N] f32 written to the caller's buffer
wk_status wk_test_gemm_partial(wk_model* m, const void* w, const void* x, float* partial_out, int32_t N, int32_t rows_x, int32_t partial_cols,
                               int32_t K, int32_t dtype, int32_t splits) {
    if (!m || !w || !x || !partial_out || N < 1 || rows_x < 16 || rows_x > 256 || rows_x % 16 != 0 || partial_cols < 1 || partial_cols > rows_x ||
        splits < 1) {
        set_error("wk_test_gemm_partial: bad arguments");
        return WK_ERR_INVALID_ARGUMENT;
    }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    std::lock_guard<std::mutex> lock(m->api_mu);
    GemmDesc g;
    memset(&g, 0, sizeof(g));
    g.a = w; g.a_rows = N; g.a_cols = K; g.a_ld = K; g.a_batches = 1;
    g.b = x; g.b_rows = rows_x; g.b_ld = K; g.in_dtype = dtype;
    g.m_rows_per_batch = N; g.n = rows_x; g.k = K; g.taps = 1; g.bn = rows_x; g.splits = splits;
    g.mode = GEMM_OUT_PARTIAL_T; g.out = partial_out; g.ld_out = N; g.out_rows_per_batch = N; g.partial_cols = partial_cols;
    g.pdl = 1; g.a_static = 1;
    wk_status r = gemm_wgmma(g, m->num_sms, m->stream);
    cudaError_t e = cudaStreamSynchronize(m->stream);
    if (r == WK_OK && e != cudaSuccess) { set_error("wk_test_gemm_partial: %s", cudaGetErrorString(e)); r = WK_ERR_CUDA; }
    return r;
}

// The split-K consumers of the FC / out-projection GEMMs on caller-made partials [splits][Bp][n]: kind 0 decoder_reduce_resid_ln (x [B][n]
// f32 updated in place, out16 = LN(x)), kind 1 decoder_reduce_bias_gelu (out16 = gelu(bias + sum), x / gamma / beta unused)
wk_status wk_test_decoder_reduce(wk_model* m, int32_t kind, const float* partial, int32_t splits, int32_t Bp, const float* bias, const float* gamma,
                                 const float* beta, float* x, void* out16, int32_t B, int32_t n, int32_t dtype) {
    if (!m || !partial || !out16 || B < 1 || Bp < B || splits < 1 || n < 4 || n % 4 != 0 || (kind == 0 && (!gamma || !beta || !x)) ||
        (kind == 1 && !bias) || kind < 0 || kind > 1) {
        set_error("wk_test_decoder_reduce: bad arguments");
        return WK_ERR_INVALID_ARGUMENT;
    }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    std::lock_guard<std::mutex> lock(m->api_mu);
    wk_status r = kind == 0 ? decoder_reduce_resid_ln(partial, splits, Bp, bias, gamma, beta, x, out16, B, n, dtype, m->stream)
                            : decoder_reduce_bias_gelu(partial, splits, Bp, bias, out16, B, n, dtype, m->stream);
    cudaError_t e = cudaStreamSynchronize(m->stream);
    if (r == WK_OK && e != cudaSuccess) { set_error("wk_test_decoder_reduce: %s", cudaGetErrorString(e)); r = WK_ERR_CUDA; }
    return r;
}

// decoder_self_attention_kernel as the decode step runs it: q|k|v split-K partials [splits][Bp][3*H*64] plus the q / v biases, beam cache
// ancestry anc [B][224] (may be NULL: every row reads its own cache row)
wk_status wk_test_self_attention_splitk(wk_model* m, const float* partial, int32_t splits, int32_t Bp, const float* bq, const float* bv, void* kcache,
                                        void* vcache, const int32_t* pos, const int32_t* done, const int32_t* anc, void* out, int32_t B, int32_t H,
                                        int32_t dtype) {
    if (!m || !partial || !bq || !bv || !kcache || !vcache || !pos || !out || B < 1 || Bp < B || splits < 1 || H < 1) {
        set_error("wk_test_self_attention_splitk: bad arguments");
        return WK_ERR_INVALID_ARGUMENT;
    }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    std::lock_guard<std::mutex> lock(m->api_mu);
    wk_status r = decoder_self_attention(partial, splits, Bp, bq, bv, kcache, vcache, pos, done, out, B, H, kKvMaxLen, dtype, m->stream, anc);
    cudaError_t e = cudaStreamSynchronize(m->stream);
    if (r == WK_OK && e != cudaSuccess) { set_error("wk_test_self_attention_splitk: %s", cudaGetErrorString(e)); r = WK_ERR_CUDA; }
    return r;
}

wk_status wk_test_kv_append(wk_model* m, const float* partial, int32_t splits, int32_t Bp, const float* bv, void* kcache, void* vcache,
                            const int32_t* pos, const int32_t* done, int32_t B, int32_t H, int32_t dtype) {
    if (!m || !partial || !bv || !kcache || !vcache || !pos || B < 1 || Bp < B || splits < 1 || H < 1) {
        set_error("wk_test_kv_append: bad arguments");
        return WK_ERR_INVALID_ARGUMENT;
    }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    std::lock_guard<std::mutex> lock(m->api_mu);
    wk_status r = decoder_kv_append(partial, splits, Bp, bv, kcache, vcache, pos, done, B, H, kKvMaxLen, dtype, m->stream);
    cudaError_t e = cudaStreamSynchronize(m->stream);
    if (r == WK_OK && e != cudaSuccess) { set_error("wk_test_kv_append: %s", cudaGetErrorString(e)); r = WK_ERR_CUDA; }
    return r;
}

// decoder cross-attention as the decode step runs it: q split-K partials [splits][Bp][H*64] plus bq; K/V [B / kv_div][H][T][64] 16-bit, or
// E4M3 codes with row scales [B / kv_div][H][T] when kscale / vscale are given (kv_div = 1: the single-query kernel, 2..8: the beam kernel)
wk_status wk_test_cross_attention_splitk(wk_model* m, const float* partial, int32_t splits, int32_t Bp, const float* bq, const void* kcross,
                                         const void* vcross, const float* kscale, const float* vscale, void* out, int32_t B, int32_t H, int32_t T,
                                         int32_t dtype, const int32_t* done, int32_t kv_div) {
    if (!m || !partial || !bq || !kcross || !vcross || !out || B < 1 || Bp < B || splits < 1 || H < 1 || H > 32 || kv_div < 1 || kv_div > 8 ||
        (kscale == nullptr) != (vscale == nullptr)) {
        set_error("wk_test_cross_attention_splitk: bad arguments");
        return WK_ERR_INVALID_ARGUMENT;
    }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    std::lock_guard<std::mutex> lock(m->api_mu);
    wk_status r = decoder_cross_attention(partial, splits, Bp, bq, kcross, vcross, out, B, H, T, dtype, m->stream, done, nullptr, 0u, kv_div,
                                          kscale, vscale);
    cudaError_t e = cudaStreamSynchronize(m->stream);
    if (r == WK_OK && e != cudaSuccess) { set_error("wk_test_cross_attention_splitk: %s", cudaGetErrorString(e)); r = WK_ERR_CUDA; }
    return r;
}

}  // extern "C"
