// Internal launcher declarations shared by the .cu files of libwkb200.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

#include "../../include/wkb200.h"

namespace wk {

void set_error(const char* fmt, ...);
const char* last_error_cstr();
void count_launch(int n = 1);

#define WK_CHECK(expr)                    \
    do {                                  \
        wk_status _s = (expr);            \
        if (_s != WK_OK) return _s;       \
    } while (0)

// Owner of device (cudaMalloc) and pinned host (cudaHostAlloc) buffers: everything allocated through it is released when it is
// destroyed, so an object that holds one frees its memory on every path, a half-built one included.  Structs handed to kernels keep raw
// pointers into it.  Releasing does not synchronise: the holder drains the streams that use the buffers first.  Every byte it holds is
// counted in the process-wide totals of wk_debug_live_bytes.
class Buffers {
public:
    Buffers() = default;
    Buffers(const Buffers&) = delete;
    Buffers& operator=(const Buffers&) = delete;
    Buffers(Buffers&& o) noexcept { live_.swap(o.live_); }
    Buffers& operator=(Buffers&& o) noexcept {
        if (this != &o) { release_all(); live_.swap(o.live_); }
        return *this;
    }
    ~Buffers() { release_all(); }

    // n elements of T on the device, zero-filled unless zero == false; alloc16: n elements of a 16-bit dtype, zero-filled
    template <typename T>
    wk_status dmalloc(T** p, size_t n, bool zero = true) { return alloc(reinterpret_cast<void**>(p), n * sizeof(T), false, zero); }
    wk_status alloc16(void** p, size_t n) { return alloc(p, n * 2, false, true); }
    // n elements of T in pinned host memory, zero-filled
    template <typename T>
    wk_status pinned(T** p, size_t n) { return alloc(reinterpret_cast<void**>(p), n * sizeof(T), true, true); }
    // *p (null or a buffer of this owner) holds at least n elements of T afterwards.  A smaller buffer is released, after `drain` (when not
    // null) has finished, and replaced by one that is not zero-filled; *moved tells whether that happened.
    template <typename T>
    wk_status grow(T** p, size_t n, cudaStream_t drain = nullptr, bool* moved = nullptr) {
        return regrow(reinterpret_cast<void**>(p), n * sizeof(T), false, drain, moved);
    }
    template <typename T>
    wk_status grow_pinned(T** p, size_t n) { return regrow(reinterpret_cast<void**>(p), n * sizeof(T), true, nullptr, nullptr); }

private:
    struct Buf { void* p; size_t bytes; bool pinned; };
    std::vector<Buf> live_;
    wk_status alloc(void** p, size_t bytes, bool pinned, bool zero);
    wk_status regrow(void** p, size_t bytes, bool pinned, cudaStream_t drain, bool* moved);
    void release_all();
};

// ---------------------------------------------------------------- GEMM (gemm_wgmma.cu)
enum GemmMode {
    GEMM_OUT_T16 = 0,        // out16[row, col] = act(acc + bias[col])
    GEMM_OUT_F32_ADD = 1,    // out32[row, col] += acc + bias[col]           (residual update in place)
    GEMM_OUT_F32_GELU_POS = 2,  // out32[row, col] = gelu(acc + bias[col]) + pos[row_in_batch, col]
    GEMM_OUT_PARTIAL_T = 3,  // out32[split][col][row] = acc                  (swap-AB split-K partials)
    GEMM_OUT_T16_HEADS = 4,  // out16[which][b][h][t][64] head-major scatter  (cross-attention K/V cache)
    GEMM_OUT_F32 = 5,        // out32[row, col] = acc + bias[col]
    GEMM_OUT_FP8_HEADS = 6,  // out8[which][b][h][t][64] E4M3 codes + out_scale[which][b][h][t] f32 (FP8 cross-attention K/V cache)
    GEMM_OUT_FP8_BLOCKS = 7, // out8[row, col] E4M3 codes of act(acc + bias[col]) + out_scale[col / 128][row] f32 (FP8 encoder FC1)
    GEMM_OUT_PACKED_HEADS = 8,  // packed bf16 rows in the [which][b][h] blocks of T x 128 bytes + out_hdr[which][b][h][round_up(T, 16)] (common.cuh)
};

struct GemmDesc {
    // A operand: [a_rows, K] 16-bit, K contiguous.  If a_batches > 1 it is a 3-D tensor
    // [a_batches][a_rows_per_batch][a_cols] addressed per batch (conv-as-GEMM with taps).
    const void* a;
    int64_t a_rows;          // rows (per batch if a_batches > 1)
    int64_t a_cols;          // row length in elements (>= K for tap addressing)
    int64_t a_ld;            // row stride in elements
    int64_t a_batch_stride;  // elements between batches (3-D only)
    int a_batches;           // 1 = plain 2-D
    int a_3d;                // address A through a 3-D tensor map [a_batches][a_rows][a_cols]
    // B operand: [b_rows, K_total] 16-bit, K contiguous (weights [N,K] or, swap-AB, activations)
    const void* b;
    int64_t b_rows;
    int64_t b_ld;
    int in_dtype;            // WK_DTYPE_BF16 / WK_DTYPE_F16
    // problem
    int m_rows_per_batch;    // output rows per batch (== valid A rows per batch for this op)
    int n;                   // valid output columns (<= b_rows)
    int k;                   // K per tap (multiple of 64)
    int taps;                // 1, or 3 for the conv stem
    int tap_row_shift[3];    // A row offset per tap
    int tap_col_off[3];      // A column offset per tap (elements)
    int bn;                  // tile N (multiple of 16, <= 256)
    int splits;              // split-K (GEMM_OUT_PARTIAL_T only), divides taps*k/64
    // epilogue
    int mode;
    int gelu;
    void* out;
    int64_t ld_out;          // row stride of out (elements); PARTIAL_T: elements per [col] row = total M
    int64_t out_rows_per_batch;  // global out row = batch*out_rows_per_batch + row_in_batch
    int64_t partial_cols;    // PARTIAL_T: number of col rows per split (padded batch)
    const float* bias;       // indexed by col (row for PARTIAL_T is not biased)
    const float* pos;        // GELU_POS: [m_rows_per_batch, ld_pos]
    int64_t ld_pos;
    // HEADS scatter
    int heads_T, heads_B, heads_H, heads_dmodel;
    float* out_scale;        // FP8_HEADS: one scale per 64-value row
    uint8_t* out_hdr;        // PACKED_HEADS: one header byte per 64-value row
    int pdl;                // launch with programmatic dependent launch (decode-step chain)
    int max_stages;          // 0 = as many smem stages as fit; >0 caps the ring (lets other kernels co-reside on the SM)
    int a_static;            // A operand (weights) does not depend on the upstream kernel: with PDL its first tiles are fetched before griddepcontrol.wait
    // FP8 operands (gemm_wgmma_fp8 only): a / b hold E4M3 codes, a_scale [K / 128][a_scale_ld] one f32 per (row, 128-column block),
    // w_scale [n] one f32 per output channel; FP8_BLOCKS writes its scales to out_scale with the same layout and ld (a_scale_ld)
    const float* a_scale;
    int64_t a_scale_ld;      // a multiple of 128 >= the rows: a tile's 128 row scales of one k-block are one 512-byte copy
    const float* w_scale;
};

wk_status gemm_wgmma(const GemmDesc& d, int num_sms, cudaStream_t stream);
// The FP8 encoder GEMMs: D = sum over 128-wide k-blocks kb of (A8 W8^T)[kb] * a_scale[kb][row], times w_scale[col] in the epilogue;
// plain 2-D operands, n and k multiples of 128, modes GEMM_OUT_T16 (QKV), GEMM_OUT_FP8_BLOCKS (FC1) and GEMM_OUT_F32_ADD (FC2).
// in_dtype is the model's 16-bit type (the type of a T16 output)
wk_status gemm_wgmma_fp8(const GemmDesc& d, int num_sms, cudaStream_t stream);
// the wgmma tile width (N) a GEMM with bn output columns per tile runs with: bn rounded up to a power of two >= 16
int wgmma_tile_n(int bn);

// ---------------------------------------------------------------- mel (mel.cu)
namespace mel { struct cf; }
struct MelTables {   // device tables of the log-mel kernel, which takes them by value
    int n_mels;
    float* win;        // [400] window
    mel::cf* tw400;    // [25][9] twiddles
    mel::cf* tw25;     // [5][5]
    float* wts;        // [kMaxTaps][128] sparse filterbank
    int* start;        // [128]
};
// uploads the tables for n_mels channels into buffers of `mem`
wk_status mel_tables_create(int n_mels, Buffers& mem, MelTables* out);
// pcm [n_windows, stride] f32 device; out [n_windows, 3002, 128] f16 (rows 0 and 3001 are the conv zero pad, mel
// channels >= n_mels zero); gmax scratch [n_windows] int32
wk_status mel_forward(const MelTables* t, const float* pcm, int64_t n_windows, int64_t stride, const int32_t* n_valid,
                      void* out_f16, int32_t* gmax_scratch, cudaStream_t stream);
constexpr int kMelRows = 3002;
constexpr int kMelCols = 128;

// ---------------------------------------------------------------- encoder ops (encoder_ops.cu)
wk_status layernorm_f32_to_16(const float* x, const float* gamma, const float* beta, void* out, int64_t rows, int d, int dtype,
                              cudaStream_t stream);
wk_status layernorm_f32_to_f32(const float* x, const float* gamma, const float* beta, float* out, int64_t rows, int d,
                               cudaStream_t stream);
// LayerNorm straight from f32 to E4M3: codes [rows][d], one scale per (row, 128-column block) in scales [d / 128][scale_ld]
wk_status layernorm_f32_to_fp8(const float* x, const float* gamma, const float* beta, uint8_t* codes, float* scales, int64_t scale_ld,
                               int64_t rows, int d, cudaStream_t stream);
// 16-bit weights [rows][k] -> E4M3 codes [rows][k] with one scale per row (output channel) over the whole row
wk_status quantize_weight_rows_fp8(const void* w, int dtype, uint8_t* codes, float* scales, int64_t rows, int k, cudaStream_t stream);
wk_status encoder_attention(const void* qkv, void* out, int B, int T, int n_heads, int dtype, cudaStream_t stream);
// TMA + wgmma implementation (attention_wgmma.cu) behind encoder_attention()
wk_status encoder_attention_wgmma(const void* qkv, void* out, int B, int T, int n_heads, int dtype, cudaStream_t stream);
wk_status transpose_to_host_layout(const void* src, float* dst, int64_t B, int64_t rows, int64_t cols, int64_t src_rows_alloc,
                                   int64_t src_row_off, int64_t src_ld, int dtype, cudaStream_t stream);
wk_status fill_random_16(void* dst, int64_t n, uint64_t seed, float std, float mean, int dtype, cudaStream_t stream);
wk_status fill_random_f32(float* dst, int64_t n, uint64_t seed, float std, float mean, cudaStream_t stream);
wk_status convert_to_16(const void* src, int src_dtype, void* dst, int dst_dtype, int64_t n, cudaStream_t stream);

// ---------------------------------------------------------------- decoder ops (decoder_ops.cu)
// Per-row decode options, device-resident: what differs between the items of transcribeWithOptions' decodeOptionsArray
// (WhisperKit.swift:716-735) and between the rungs of the temperature ladder (TranscribeTask.swift:316-411).
struct RowParams {
    int32_t prompt_len;          // initialPrompt.count
    int32_t sample_begin_ts;     // TimestampRulesFilter.sampleBegin, <0 = filter absent
    int32_t sample_begin_blank;  // SuppressBlankFilter.sampleBegin, <0 = absent
    int32_t max_steps;           // min(sampleLength, 223): loop bound (TextDecoder.swift:566)
    float temperature; int32_t top_k;
    int32_t has_first_thr; float first_thr;
    uint64_t seed;
    int32_t suppress_off, n_suppress;   // slice of the session's suppress-token pool
    // DecodingOptions.detectLanguage (TranscribeTask.swift:340-365): 0 off; 1 the row's step 0 is the detection forward ([SOT] at
    // position 0); 2 the prompt does not start with SOT, so one leading detection step runs before step 0
    int32_t detect;
    int32_t lang_pos;            // prompt slot of <|xx|> rewritten with the detected language, <0 = report only
    int32_t n_lang;              // entries of SamplerParams.detect_tokens
    int32_t lead_token;          // <|startoftranscript|>: what the leading detection step feeds at position 0
    // DecodingResult.noSpeechProb: the step (= index of the prompt's first SOT) whose raw logits give it, <0 = off
    int32_t no_speech_pos;
    int32_t mode;                // kRowSingle / kRowBeam / kRowSample: how the row's rung decodes (one step mixes groups at different rungs)
    // DecodingOptions.biasPhrases: the window's phrase set in the session's bias pool (DecodeState.bias_pool + bias_off), bias_n phrases
    // of bias_len tokens in all (0 = no bias), boost λ
    int32_t bias_off, bias_n, bias_len;
    float bias_boost;
};
// RowParams.mode.  Single and sample rows run the per-row sampler and bookkeeping (a sample row is one of best_of independent draws of its
// group); beam rows only rank candidates, and beam_update_kernel does their bookkeeping per group
constexpr int kRowSingle = 0, kRowBeam = 1, kRowSample = 2;

struct DecodeState {
    // all device pointers; one entry per decode row (slot).  A slot with done != 0 is skipped by every kernel of the step.
    int32_t* tokens;      // [Bmax, 224] currentTokens
    int32_t* n_tokens;    // [Bmax]
    float* logprobs;      // [Bmax, 224]
    int32_t* next_token;  // [Bmax]
    int32_t* done;        // [Bmax]
    int32_t* first_low;   // [Bmax]
    int32_t* steps;       // [Bmax] forward passes consumed = tokenIndex of the step about to run = KV-cache position
    int32_t* input_ids;   // [Bmax] token fed at this step (written by embed)
    int32_t* error;       // [Bmax] 1 = the sampler saw no finite logit (WhisperError.decodingLogitsFailed)
    const RowParams* rp;  // [Bmax]
    int32_t* lang_token;  // [Bmax] language detected in the loop, -1 = none
    float* lang_logprob;  // [Bmax]
    int32_t* lang_state;  // [Bmax] kLangLead: the leading detection step is next; kLangLeadRan: it was this step's; 0 otherwise
    float* no_speech;     // [Bmax] softmax(raw logits)[no_speech_token] at step RowParams.no_speech_pos; NaN = not computed
    // contextual biasing: the phrase pool of the call's sets (nullptr = no set attached: the loop never reads the two arrays below),
    // each row's KMP match length per phrase and the sum of g(v) - G over its appended tokens (the bonus it banked, in units of λ)
    const int32_t* bias_pool;
    uint8_t* bias_m;      // [Bmax][kMaxBiasPhrases]
    int32_t* bias_acc;    // [Bmax]
};
constexpr int kLangLead = 2, kLangLeadRan = 3;
// A bias set: up to 256 phrases of 1..16 token ids each, 1024 tokens in all.  Its pool record is [n] descriptors (start | len << 16),
// [total] phrase tokens, [total] failure links (f(k) for k = 1..len of a phrase at its start + k - 1)
constexpr int kMaxBiasPhrases = 256, kMaxBiasLen = 16, kMaxBiasTotal = 1024;
// DecodingOptions.topLogProbs: k in [0, 20] (OpenAI's top_logprobs limit)
constexpr int kMaxTopLogprobs = 20;

// Beam search (SURVEY 8f row 2; semantics restated from openai/whisper BeamSearchDecoder in oracle/beam_ref.py - the reference's
// BeamSearchTokenSampler is a fatalError stub, TokenSampler.swift:254-290).  Decode rows come in groups of `group` consecutive rows per
// window (G = max(beam_size, best_of)); a beam-mode group uses its first `beam` rows, a best-of group its first best_of rows.
constexpr int kMaxBeam = 8;
constexpr int kMaxCand = 8;        // maxCandidates = Int(Float(beamSize) * patience) (TokenSampler.swift:266)
struct BeamState {
    int beam;                      // beams of a beam-mode group; <= 1 = the call has no beam rows, every pointer below unused
    int max_candidates;
    int group;                     // decode rows per window (<= 1: one)
    float* sum_lp;                 // [rows] cumulative log-prob of the sampled tokens of the beam
    int32_t* cand_tok; float* cand_lp;   // [rows][kMaxBeam + 1] best tokens of the step's filtered log-softmax, best first (-1 = none)
    float* cand_sc;                // [rows][kMaxBeam + 1] the candidates' score increments: cand_lp plus the phrase bonus (= cand_lp unbiased)
    int32_t* anc;                  // [rows][224] physical cache row that holds position t of this beam's self K/V
    int32_t* fin_tokens; float* fin_lps;   // [groups][kMaxCand][224] finished sequences (EOT included), per-token log-probs (EOT -> 0)
    int32_t* fin_len; float* fin_score;    // [groups][kMaxCand]
    int32_t* n_fin;                // [groups]
    int use_anc;                   // the loop's rows read their self K/V through anc (beam search, or draft verification)
};

struct SamplerParams {
    wk_special_tokens st;
    int vocab;
    int is_multilingual;
    int loop_mode;           // 1: decode loop (per-row options from DecodeState.rp); 0: stateless (wk_filter_sample / detectLanguage)
    const int32_t* suppress; // loop mode: the pool RowParams.suppress_off indexes; stateless: the list itself
    const int32_t* language_tokens; int n_language_tokens; int language_sample_begin;
    int max_ctx;             // 224
    const int32_t* detect_tokens;   // loop mode: allLanguageTokens of the rows with RowParams.detect (in-loop language detection)
    BeamState beam;         // loop mode: rows with RowParams.mode == kRowBeam only rank candidates; beam_update() does their bookkeeping
    int rng_div;            // loop mode: decode rows per Philox subsequence (a draft call's G, so that row 0 of slot q draws as row q of a
                            // draft-less call); 0 or 1 = every row its own
    // loop mode, DecodingOptions.topLogProbs: the top_n best (token, log-prob) candidates of every sampled position, [rows][224][top_n]
    // at the position DecodeState.logprobs uses, best first, padded with (-1, -inf); top_n = 0: off, the sampler has no top-k pass
    int32_t* top_tok; float* top_lp; int top_n;
    // stateless mode only
    int sample_begin_ts, sample_begin_blank, n_suppress;
    float temperature; int top_k; uint64_t seed;
};

// pos: explicit per-row positions (wk_decode_step) or nullptr = DecodeState.steps
wk_status decoder_embed_ln(const void* emb16, const float* pos, const float* gamma, const float* beta, DecodeState st, int vocab,
                           int ts_begin, float* x, void* xn, int B, int d, int dtype, const int32_t* explicit_pos, cudaStream_t stream);
// x[b,:] += bias + sum_s partial[s][b][:]; xn = LN(x) (16-bit).  partial layout [S][Bp][d]
wk_status decoder_reduce_resid_ln(const float* partial, int splits, int Bp, const float* bias, const float* gamma,
                                  const float* beta, float* x, void* xn, int B, int d, int dtype, cudaStream_t stream);
// h = gelu(bias + sum partial) 16-bit [B, n]
wk_status decoder_reduce_bias_gelu(const float* partial, int splits, int Bp, const float* bias, void* out, int B, int n,
                                   int dtype, cudaStream_t stream);
// self attention for one new token per sequence; reduces qkv partials [S][Bp][3d], appends K/V at pos[b].  done != nullptr: rows with
// done[b] != 0 are skipped (their window has ended: no cache traffic)
// anc != nullptr (beam search): position t of row b is read from cache row anc[b][t]; the new row is written to row b itself
wk_status decoder_self_attention(const float* partial, int splits, int Bp, const float* bq, const float* bv, void* kcache,
                                 void* vcache, const int32_t* pos, const int32_t* done, void* out, int B, int H,
                                 int max_len, int dtype, cudaStream_t stream, const int32_t* anc = nullptr);
// the K/V half of decoder_self_attention alone: reduces the k / v partials of every live row and appends them at pos[b] of its own cache
// row, with the same arithmetic and rounding.  Run before decoder_self_attention(anc) when rows of one step read each other's new
// positions (draft verification: row j attends to rows 0..j-1 of its window at this step); the attention kernel's own append then
// writes the same bits again
wk_status decoder_kv_append(const float* partial, int splits, int Bp, const float* bv, void* kcache, void* vcache, const int32_t* pos,
                            const int32_t* done, int B, int H, int max_len, int dtype, cudaStream_t stream);
// cross attention over T encoder positions; reduces q partials [S][Bp][d]; K/V [B][H][T][64]
// align_scratch != nullptr: heads h with bit h of align_mask set also write their softmax row (f32, [slot][B][T], slot = rank of h in
// the mask) - the alignment heads behind the reference decoder's `alignment_heads_weights` output (TextDecoder.swift:310,414)
// kscale / vscale != nullptr: the FP8 cache - K/V are E4M3 codes [B][H][T][64] with one f32 scale per row ([B][H][T]); dtype is then only
// the type of `out`
wk_status decoder_cross_attention(const float* partial, int splits, int Bp, const float* bq, const void* kcross,
                                  const void* vcross, void* out, int B, int H, int T, int dtype, cudaStream_t stream,
                                  const int32_t* done = nullptr, float* align_scratch = nullptr, uint32_t align_mask = 0, int kv_div = 1,
                                  const float* kscale = nullptr, const float* vscale = nullptr, bool single_query = false,
                                  const uint8_t* khdr = nullptr, const uint8_t* vhdr = nullptr);
// khdr / vhdr != nullptr: the packed bf16 cache (common.cuh), header vectors [B / kv_div][H][round_up(T, 16)]
// rows [0, blocks * T) of packed blocks -> the 16-bit [blocks][T][64] layout
wk_status cross_kv_unpack(const void* packed, const uint8_t* hdr, void* out, int64_t blocks, int T, cudaStream_t stream);
// kv_div > 1 (beam search): row b reads the K/V block of window b / kv_div; the CTAs of one (window, head) are adjacent in the grid so that
// their K/V stream is shared through L2.  single_query: never the tensor-core form below (its arithmetic differs): every row computes
// exactly what it would as the only row of its window
// tensor-core variant for nq = 2..8 rows per K/V block (cross_attention_mq.cu): one K/V stream per (window, head) serves all nq beams
wk_status decoder_cross_attention_mq(const float* partial, int splits, int Bp, const float* bq, const void* kcross, const void* vcross, void* out, int B, int H,
                                     int Tlen, int dtype, cudaStream_t stream, const int32_t* done, int nq,
                                     const float* kscale = nullptr, const float* vscale = nullptr, const uint8_t* khdr = nullptr,
                                     const uint8_t* vhdr = nullptr);
// alignment row of the step just sampled (run AFTER the sampler advanced steps[b] to tokenIndex + 1): out[b][steps[b]][t] =
// Float16(mean over n_slots of scratch[slot][b][t]) unless done[b] (TextDecoder.updateAlignmentWeights, TextDecoder.swift:272-296:
// the slice of step tokenIndex lands in row tokenIndex + 1; a completed segment breaks out before the update, :668-674)
// A row whose step was the leading language-detection step (lang_state, may be NULL) gets no row either.
wk_status decoder_align_mean(const float* scratch, int n_slots, const int32_t* steps, const int32_t* done, const int32_t* lang_state,
                             void* out_f16, int B, int T, int max_rows, cudaStream_t stream);
wk_status sampler_filter_sample(const float* logits, int64_t ld_logits, SamplerParams p, DecodeState st, const int32_t* tokens,
                                int ld_tokens, const int32_t* n_tokens, int32_t* token_out, float* logprob_out,
                                float* filtered_out, int B, cudaStream_t stream);
// (re)starts the decode of n slots: slot_ids[i] gets prompt row i of prompts [n][224] (length rp[i].prompt_len) and RowParams rp[i]
wk_status decode_slots_init(DecodeState st, RowParams* rp_dev, const int32_t* slot_ids, const int32_t* prompts, const RowParams* rp_new,
                            int n, cudaStream_t stream, BeamState beam = BeamState());
// the beam-search step after the sampler ranked every row's candidates: per window, merge the beams' candidates, move finished sequences
// to the finished list, permute token / log-prob histories and cache ancestry to the surviving beams, advance the loop state.  One CTA per
// group of beam.group rows; groups whose rung is not in beam mode return at once
wk_status beam_update(DecodeState st, BeamState beam, wk_special_tokens sp, int max_ctx, int groups, cudaStream_t stream);

// ---- speculative greedy decoding (session.cu's draft rounds).  A window holds G = k + 1 decode rows; the draft decoder has one row per
// window slot with its own DecodeState (history = the window's, plus its proposals).  One round: draft_round_begin; k + 1 times
// draft_feed + draft forward + draft sampler (a step either catches the draft up on a committed token or makes proposal i); verify_setup;
// the main step over every row; draft_accept.
struct DraftRound {
    int k, group, slots;
    int32_t* fed;        // [S] the draft's self K/V holds positions 0 .. fed - 1 of the window's committed tokens
    int32_t* p0;         // [S] the window's committed position (main row 0's steps) at the round start, -1 = no live window
    int32_t* verify;     // [S] 1: the window verifies proposals this round (past its prompt, live, temperature 0)
    int32_t* prop;       // [S][8] proposals of the round
    int32_t* nprop;      // [S] proposals made
    int32_t* rows;       // [S] verification rows 1..rows set up this round (row j runs step p0 + j)
    int32_t* cur;        // [S] proposal index the draft step just run makes, -1 = none
    unsigned long long* counters;   // [3] rounds that verified, proposals verified, proposals accepted
};
constexpr int kMaxDraftTokens = 7;
// main row 0 of every slot -> the round's plan; the draft's history and options from the window's
wk_status draft_round_begin(DecodeState st, DecodeState ds, RowParams* drp, DraftRound R, cudaStream_t stream);
// the previous draft step's proposal recorded; the next draft step's token and position (or the draft row idle); collect_only: record only
wk_status draft_feed(DecodeState st, DecodeState ds, DraftRound R, int collect_only, cudaStream_t stream);
// rows 1..nv of each verifying window: history = row 0's + proposals 0..j-1, input = proposal j-1 at position p0 + j, ancestry through
// the rows of this step
wk_status draft_verify_setup(DecodeState st, RowParams* rp, int32_t* anc, DraftRound R, cudaStream_t stream);
// proposal i is accepted when it equals the token row 0 holds after taking over rows 1..i (the model's sample at step p0 + i); row 0
// takes over row i + 1 while the window runs on; rows 1..G-1 end
wk_status draft_accept(DecodeState st, int32_t* anc, DraftRound R, cudaStream_t stream);

// ---- teacher-forced alignment pass (align_pass.cu): rows are (window, position) pairs, 224 rows per window, row w * 224 + t = position t.
// seq_len[w] = the window's token count (0 = skipped); cross K/V of window w sit in cache block slot0 + w ([slot][H][T][64])
// x[row] = embedding[row_tok[row]] + positional embedding[t] (f32), 0 where row_tok[row] < 0
wk_status align_embed(const void* emb, const float* pos_emb, const int32_t* row_tok, float* x, int64_t rows, int d, int dtype, cudaStream_t stream);
// causal self-attention over the [rows][3d] QKV output (biases already added) -> out [rows][d]
wk_status align_self_attention(const void* qkv, const int32_t* seq_len, void* out, int nw, int H, int dtype, cudaStream_t stream);
// q [rows][d] (16-bit) against the layer's cache block; kscale / vscale != nullptr: the FP8 cache, khdr / vhdr: the packed bf16 cache.  stats != nullptr: each row's final softmax
// (max, sum) per head as float pairs [H][stat_rows]
wk_status align_cross_attention(const void* q, const void* kc, const void* vc, const float* kscale, const float* vscale, const int32_t* seq_len,
                                int slot0, void* out, float* stats, int64_t stat_rows, int nw, int H, int Tlen, int dtype, cudaStream_t stream,
                                const uint8_t* khdr = nullptr, const uint8_t* vhdr = nullptr);
// acc[row][T] (f32) += the normalised softmax rows of the heads in `mask`, ascending (first != 0: acc starts at 0)
wk_status align_export(const void* q, const void* kc, const float* kscale, const float* stats, int64_t stat_rows, const int32_t* seq_len, int slot0,
                       uint32_t mask, int first, float* acc, int nw, int H, int Tlen, int dtype, cudaStream_t stream, const uint8_t* khdr = nullptr);
// Float16 alignmentWeights [nw][store_rows][T]: row t + 1 = acc[position t] / n_slots, row 0 and rows past the sequence 0
wk_status align_rows_f16(const float* acc, const int32_t* seq_len, int n_slots, void* out, int nw, int Tlen, int store_rows, cudaStream_t stream);
// logits rows [r0, r0 + rows) of the pass ([rows][ld] f32): out[r + 1] = log softmax(logits[r][:eot])[row_tok[r + 1]], NaN for targets >= eot
wk_status align_token_logprobs(const float* logits, int64_t ld, int64_t r0, int64_t rows, const int32_t* row_tok, const int32_t* seq_len, int eot,
                               float* out, cudaStream_t stream);

// ---- AudioStreamTranscriber.shouldStopEarly (AudioStreamTranscriber.swift:208-227) as a deterministic window stop (session.cu)
// A window ends at its first appended, non-prefill token t whose history currentTokens = tokens[0..t] meets either rule:
//   count > window and compressionRatio(last `window` tokens) > compression_threshold (compressionRatioThreshold ?? 0.0), or
//   has_logprob and avg(logProbs[0..t]) < logprob_threshold (prompt log-probs are 0).
// The result is the history cut after t, then finalize and the usual DecodingFallback; unlike a progress-callback stop, the window
// walks the fallback ladder when its DecodingFallback asks for it.
struct StopRule {
    int window;
    float compression_threshold;
    int has_logprob;
    float logprob_threshold;
};
// wk_transcribe_windows_ex with the stop rule applied to every window (stop == nullptr: wk_transcribe_windows_ex).  Single-row windows
// only (no beam search, no best-of).
// draft: speculative decoding's proposals per round (wk_transcribe_windows_draft), 0 = none
wk_status transcribe_windows_stop(wk_model* m, wk_session* s, const float* pcm_host, int64_t n_windows, int64_t stride,
                                  const int32_t* samples_per_window, const wk_special_tokens* st, const wk_batch_opts* bo,
                                  wk_decode_result* results, const StopRule* stop, int draft = 0);
// bias sets attached with wk_session_set_bias (0 = none), and the set each window of the session's next calls uses (empty: the plain
// rule, set i for window i or set 0 for every window)
int64_t session_bias_sets(const wk_session* s);
void session_bias_map(wk_session* s, std::vector<int> map);
int session_top_logprobs(const wk_session* s);   // the k of wk_session_set_top_logprobs

}  // namespace wk
