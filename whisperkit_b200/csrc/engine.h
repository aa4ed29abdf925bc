// Internal object layouts of libwkb200 shared by engine.cu (model, weights, mel + encoder schedule, kernel hooks) and
// session.cu (decode sessions, the device-resident token loop, the window scheduler).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <memory>
#include <mutex>
#include <vector>

#include "kernels.h"

namespace wk {

constexpr int kKvMaxLen = 224;        // Constants.maxTokenContext (Models.swift:1334)
constexpr int kWindowSamples = 480000;  // Constants.defaultWindowSamples (Models.swift:1457)

static inline int round_up(int a, int b) { return (a + b - 1) / b * b; }

struct LayerNormW { float* g = nullptr; float* b = nullptr; };
struct EncLayer {
    LayerNormW ln1, ln2;
    void* wqkv = nullptr; float* bqkv = nullptr;  // [3d, d]
    void* wo = nullptr; float* bo = nullptr;
    void* w1 = nullptr; float* b1 = nullptr;      // [4d, d]
    void* w2 = nullptr; float* b2 = nullptr;      // [d, 4d]
    // FP8 encoder policy (wk_model_set_encoder_dtype): E4M3 copies of wqkv / w1 / w2 with one f32 scale per output channel
    uint8_t* wqkv8 = nullptr; float* sqkv = nullptr;
    uint8_t* w18 = nullptr; float* s1 = nullptr;
    uint8_t* w28 = nullptr; float* s2 = nullptr;
};
struct DecLayer {
    LayerNormW ln1, lnx, ln3;
    void* wqkv = nullptr; float* bq = nullptr; float* bv = nullptr;
    void* wo = nullptr; float* bo = nullptr;
    void* wcq = nullptr; float* bcq = nullptr;
    void* wco = nullptr; float* bco = nullptr;
    void* w1 = nullptr; float* b1 = nullptr;
    void* w2 = nullptr; float* b2 = nullptr;
};

// One decoder's weights as the decode step reads them: the model's own decoder, or its draft decoder (speculative decoding)
struct DecoderWeights {
    void* emb = nullptr;                 // [V][d], tied output projection
    float* pos = nullptr;                // [n_text_ctx][d]
    DecLayer* layers = nullptr; int n_layers = 0;
    LayerNormW ln;                       // final LayerNorm
    void* wckv = nullptr; float* bckv = nullptr;   // cross-attention K/V projection [2L*d][d], [2L*d]
};

// A draft decoder (wk_model_create_draft / wk_model_load_draft): its own embedding, positional table, layers, final LayerNorm and
// cross-K/V projection, with the main model's d_model, heads, vocabulary and n_audio_ctx.  It reads the main model's encoder output.
struct DraftDecoder {
    Buffers mem;
    void* emb = nullptr; float* pos = nullptr;
    std::vector<DecLayer> dec;
    LayerNormW ln;
    void* wckv = nullptr; float* bckv = nullptr;
    DecoderWeights view() { return DecoderWeights{emb, pos, dec.data(), (int)dec.size(), ln, wckv, bckv}; }
};

// Mel + encoder activations for up to max_batch windows.  The model keeps one for the piecewise API (wk_mel / wk_encode, serialised by
// wk_model::api_mu); every session allocates its own on first use, so sessions on different host threads encode concurrently.
struct EncWorkspace {
    Buffers mem;
    int max_batch = 0;
    float* pcm_dev = nullptr; int32_t* nvalid_dev = nullptr; int32_t* gmax = nullptr;
    void* mel = nullptr;       // f16 [Bm][3002][128]
    void* h1 = nullptr;        // f16 [Bm][3002][d]
    float* x = nullptr;        // f32 [Bm*1500][d]
    void* xn = nullptr; void* qkv = nullptr; void* attn = nullptr; void* ffn = nullptr;
    void* enc_out = nullptr;   // 16-bit [Bm*1500][d]
    // FP8 encoder policy: xn / ffn then hold E4M3 codes; their block scales [d / 128][ld] and [4d / 128][ld], ld = Bm*1500 rounded up to
    // 128 (allocated by the first FP8 encode)
    float* xn_scale = nullptr; float* ffn_scale = nullptr;
};

}  // namespace wk

struct wk_tensor {
    void* data;
    int kind;      // 0 = mel [B,3002,128] f16 ; 1 = encoder output [B*1500, d] model dtype
    int dtype;
    int64_t batch;
    wk_model* owner;
    std::vector<cudaEvent_t> events;   // [0] producer done (model stream), then one per reader on another stream (guarded by owner->api_mu):
                                       // readers wait on them, wk_tensor_free orders the release after them
};

struct wk_model {
    ~wk_model();   // destroys the stream and events; the caller has made the model's device current and drained it
    wk::Buffers mem;                 // weights and mel tables
    wk_model_config cfg;
    int device = 0;
    int num_sms = 132;
    cudaStream_t stream = nullptr;   // the piecewise API (wk_mel, wk_encode, wk_filter_sample, readbacks) is enqueued here
    std::mutex api_mu;               // ... one host thread at a time: the handle itself is immutable once finalized
    bool finalized = false;
    int esz = 2;
    // weights
    void* conv1_w = nullptr; float* conv1_b = nullptr;   // f16 [d][3][128]
    void* conv2_w = nullptr; float* conv2_b = nullptr;   // f16 [d][3][d]
    float* enc_pos = nullptr;                            // [1500][d]
    std::vector<wk::EncLayer> enc;
    wk::LayerNormW enc_ln;
    void* emb = nullptr;                                 // [V][d]
    float* dec_pos = nullptr;                            // [448][d]
    std::vector<wk::DecLayer> dec;
    wk::LayerNormW dec_ln;
    void* wckv = nullptr; float* bckv = nullptr;         // [2L*d][d], [2L*d]
    wk::MelTables mel_tables = {};
    wk::EncWorkspace ws;                                 // allocated on the first wk_mel / wk_encode
    // alignment heads (word timestamps): per decoder layer a head bit mask and the first scratch slot of the layer
    std::vector<uint32_t> align_mask; std::vector<int> align_base; int n_align_slots = 0; int has_alignment_heads = 0;
    float timings[6] = {0, 0, 0, 0, 0, 0};
    cudaEvent_t ev[8] = {};
    // cross-attention K/V cache storage: the model dtype, or FP8 E4M3 with per-row scales (wk_model_set_cross_kv_dtype); fixed once the
    // first session exists.  Both fields are read and written under api_mu.
    bool cross_kv_fp8 = false;
    bool session_created = false;
    // encoder QKV / FC1 / FC2 GEMMs on E4M3 operands (wk_model_set_encoder_dtype); fixed once a session exists or wk_encode has run
    bool enc_fp8 = false;
    bool encoded = false;
    // speculative decoding (wk_model_create_draft / wk_model_load_draft): null = the model has no draft decoder; fixed once a session exists
    std::unique_ptr<wk::DraftDecoder> draft;
    wk::DecoderWeights main_decoder() { return wk::DecoderWeights{emb, dec_pos, dec.data(), (int)dec.size(), dec_ln, wckv, bckv}; }
};

namespace wk {

wk_status enc_ws_ensure(wk_model* m, EncWorkspace* ws, int max_batch);
// the staging half of mel_run: host PCM, or rows shorter than a window, copied into ws->pcm_dev (zero-padded) on `stream`; *src /
// *src_stride are the rows the mel kernel reads
wk_status mel_stage(EncWorkspace* ws, const float* pcm, int64_t n, int64_t stride, cudaStream_t stream, const float** src, int64_t* src_stride);
// PCM rows (host or device) -> staged in ws->pcm_dev when needed -> log-mel into mel_out ([n][3002][128] f16), all on `stream`
wk_status mel_run(wk_model* m, EncWorkspace* ws, const float* pcm, int64_t n, int64_t stride, const int32_t* samples_per_window_host,
                  void* mel_out, cudaStream_t stream);
// conv stem + encoder layers over B windows of `mel` into enc_out ([B*1500][d], model dtype), activations in ws, on `stream`
wk_status encode_chunk(wk_model* m, EncWorkspace* ws, const void* mel, int B, void* enc_out, cudaStream_t stream);
GemmDesc plain_gemm(const void* a, int64_t M, int K, const void* w, int N, int dtype, int mode, void* out, int64_t ld_out,
                    const float* bias, int gelu);
int choose_splits(int tiles, int total_kb, int num_sms);
// audio.cu: a session's audio-loading workspace (pinned staging, device buffers), created on its first wk_audio_* call
struct AudioWs;
void audio_ws_free(AudioWs* w);
AudioWs** session_audio_ws(wk_session* s);   // session.cu
cudaStream_t session_stream(wk_session* s);
int session_device(wk_session* s);
size_t esize(int dtype);
long long launch_counter_load();
void launch_counter_sub(long long n);

}  // namespace wk
