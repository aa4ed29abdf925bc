// libwkb200 decode sessions: per-worker decoder state (TextDecoding.prepareDecoderInputs, TextDecoder.swift:109-161), one decoder
// forward (predictLogits, :361-418), the device-resident token loop (decodeText, :541-855) and the window scheduler behind
// wk_transcribe_windows (the per-window body of TranscribeTask.run, TranscribeTask.swift:116-278, fanned out like
// WhisperKit.transcribeWithOptions, WhisperKit.swift:716-812, with decodeWithFallback's temperature ladder, TranscribeTask.swift:316-411).
//
// Scheduling model.  A session owns `max_batch` decode SLOTS.  Every slot carries its own position, prompt and options on the device
// (DecodeState / RowParams), so one CUDA graph of the step serves any mix of windows; a slot whose window has ended is skipped by every
// kernel of the step (no cross-KV stream, no cache traffic, no logits row).  The host polls the done flags every few steps, finalises the
// windows that ended (sampler.finalize, slicing, avgLogProb, compressionRatio, DecodingFallback) and hands their slots to the next
// encoded windows - or back to the same window at the next ladder temperature.  The mel + encoder pass of the next chunk runs on a
// second stream while the current slots decode (tensor-bound under HBM-bound).
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <zlib.h>

#include <algorithm>
#include <memory>
#include <string>
#include <vector>

#include "common.cuh"
#include "engine.h"

using namespace wk;

struct wk_session {
    ~wk_session();   // drains and destroys the streams, events and graphs; the owners release the buffers after it
    Buffers mem;              // every device and pinned buffer below
    wk_model* m = nullptr;
    int max_batch = 0;        // decode slots
    int batch = 0;            // rows the step runs over: slots [0, batch / G), G = max(beam, best_of) rows per slot
    int bound_windows = 0;    // windows bound by wk_session_set_encoder_output (cross K/V blocks 0 .. bound_windows - 1)
    int bp = 16;              // batch padded to a multiple of 16 (the GEMM tile N granule)
    cudaStream_t stream = nullptr;      // decode stream
    cudaStream_t enc_stream = nullptr;  // mel + encoder of the batched entry
    EncWorkspace ws;                    // this session's mel / encoder activations (allocated on first use)
    void* cross_kv = nullptr;   // [2L][S][H][T][64] model dtype, or E4M3 codes when ckv_fp8
    float* cross_scale = nullptr;   // ckv_fp8: [2L][S][H][T] row scales
    bool ckv_fp8 = false;
    // bf16 models (no FP8 cache): the cache holds packed rows (common.cuh) with their headers [2L][S][H][round_up(T, 16)]
    bool ckv_packed = false;
    uint8_t* cross_hdr = nullptr;
    void* self_k = nullptr;     // [L][S][H][224][64]
    void* self_v = nullptr;
    float* partial = nullptr; size_t partial_elems = 0;
    float* x = nullptr; void* xn = nullptr; void* attn = nullptr; void* ffn = nullptr;
    float* logits = nullptr;
    DecodeState st;
    RowParams* rp_dev = nullptr;
    // lang_dev: allLanguageTokens of wk_detect_language and of in-loop detection.  Fixed at the 4096-entry limit, so its pointer (baked
    // into the step graphs through SamplerParams.detect_tokens) never changes
    int32_t* pos_dev = nullptr; int32_t* lang_dev = nullptr;
    int32_t* suppress_dev = nullptr; size_t suppress_cap = 0;
    // slot admission staging (pinned host + device)
    int32_t *h_adm_slots = nullptr, *h_adm_prompts = nullptr; RowParams* h_adm_rp = nullptr;
    int32_t *d_adm_slots = nullptr, *d_adm_prompts = nullptr; RowParams* d_adm_rp = nullptr;
    // pinned readback of the decode state
    int32_t *h_tokens = nullptr, *h_n_tokens = nullptr, *h_done = nullptr, *h_first_low = nullptr, *h_steps = nullptr, *h_error = nullptr;
    float* h_logprobs = nullptr;
    int32_t* h_lang_token = nullptr; float* h_lang_logprob = nullptr; float* h_no_speech = nullptr;
    // language detected per window of the last batched call (wk_session_languages): -1 / 0 where a window did not detect
    std::vector<int32_t> win_lang; std::vector<float> win_lang_logprob;
    std::vector<float> win_no_speech;   // noSpeechProb per window of the last batched call (wk_session_no_speech_probs), NaN = none
    // step graph, cached across calls: the step depends on the call only through the rows it covers, the alignment export and the
    // special-token ids baked into the sampler's parameters
    cudaGraphExec_t graph_exec = nullptr, graph_exec_live = nullptr;   // the step with / without the ended-row checks in the attention kernels
    int graph_batch = 0; bool graph_align = false; wk_special_tokens graph_st; long long launches_per_step = 0;
    bool warmed = false;
    // word timestamps: per-head softmax rows of the current step, the [S][224][T] Float16 alignmentWeights of the slots, and the per-window
    // copies handed out by wk_session_alignment_weights
    float* align_scratch = nullptr; void* align_w = nullptr; int align_slots = 0; bool align_on = false;
    // align_store_rows rows per window: 224 after a decode, 225 after an align call (row t + 1 = position t)
    uint8_t* align_store = nullptr; int64_t align_store_n = 0; int align_store_rows = kKvMaxLen;
    // teacher-forced alignment pass (wk_align_tokens / wk_align_windows): buffers for the windows of one chunk, 224 rows each - the f32
    // alignment accumulator [rows][T], per-head softmax (max, sum) [H][rows][2], row tokens, sequence lengths, token log-probs, the QKV
    // biases [L][3d]; and the log-probs of the last call on the host, 224 per window
    float *al_acc = nullptr, *al_stats = nullptr, *al_lp = nullptr, *al_bqkv = nullptr;
    int32_t *al_tok = nullptr, *al_seq = nullptr;
    std::vector<float> win_align_lp;
    cudaEvent_t ev_enc = nullptr, ev_adm = nullptr, ev_stage = nullptr, ev_t[10] = {};
    // beam search (allocated on the first call that asks for it)
    BeamState bs = BeamState(); int bs_cap_rows = 0;
    int32_t *h_n_fin = nullptr, *h_fin_len = nullptr, *h_fin_tokens = nullptr; float *h_fin_score = nullptr, *h_fin_lps = nullptr, *h_sum_lp = nullptr;
    int graph_beam = 1;
    int64_t stats[4] = {0, 0, 0, 0};   // of the last batched call: step launches, sum of live rows over them, admissions, ladder re-admissions
    AudioWs* audio = nullptr;          // wk_audio_load / wk_audio_convert workspace (audio.cu)
    int32_t* pos100 = nullptr;         // wk_bench_kernel's self-attention positions (all 100)
    // speculative decoding (wk_transcribe_windows_draft), allocated on first use when the model has a draft decoder: the draft's self K/V
    // (one row per slot) and cross K/V (the session's storage policy), its decode state, and the rounds' device bookkeeping
    int draft_k = 0;                   // proposals per round of the current call, 0 = no draft
    bool draft_ready = false;
    void* dr_self_k = nullptr; void* dr_self_v = nullptr; void* dr_cross_kv = nullptr; float* dr_cross_scale = nullptr; uint8_t* dr_cross_hdr = nullptr;
    DecodeState dst; RowParams* drp = nullptr;
    DraftRound dr = DraftRound();
    int64_t draft_stats[3] = {0, 0, 0};   // of the last batched call: rounds that verified, proposals verified, proposals accepted
    int graph_draft = 0;
    // contextual biasing (wk_session_set_bias): the attached sets' records in one device pool, where each set sits in it (n = 0: a
    // window without bias), and the per-window set indices a long-form round uses (empty: set i for window i, or set 0 for all)
    struct BiasSlot { int off = 0, n = 0, len = 0; float boost = 0.f; };
    int32_t* bias_pool = nullptr; size_t bias_cap = 0;
    std::vector<BiasSlot> bias_sets;
    std::vector<int> bias_map;
    int32_t* h_bias_acc = nullptr;
    const int32_t* graph_bias = nullptr;
    // DecodingOptions.topLogProbs (wk_session_set_top_logprobs): the setting for the next calls and the k of the running call; the
    // sampler's pairs [S][224][k] on the device (allocated for k = 20 on first use) and their pinned readback; per window of the last
    // call, the pairs of its result tokens [n_tokens][k] (top_store_k = the call's k)
    int top_k = 0, top_n = 0, graph_top = 0, top_store_k = 0;
    int32_t *top_tok = nullptr, *h_top_tok = nullptr; float *top_lp = nullptr, *h_top_lp = nullptr;
    std::vector<std::vector<int32_t>> win_top_tok;
    std::vector<std::vector<float>> win_top_lp;
};

// a phrase set as wk_bias_create validated it: its pool record (kernels.h) and boost
struct wk_bias {
    std::vector<int32_t> rec;
    int n = 0, len = 0;
    float boost = 0.f;
};

// The cached step graphs bake in the call's shape and the session's buffer pointers: dropped, they are captured again on the next step
static void drop_graphs(wk_session* s) {
    if (s->graph_exec) { cudaGraphExecDestroy(s->graph_exec); s->graph_exec = nullptr; }
    if (s->graph_exec_live) { cudaGraphExecDestroy(s->graph_exec_live); s->graph_exec_live = nullptr; }
}

wk_session::~wk_session() {
    if (stream) cudaStreamSynchronize(stream);
    if (enc_stream) cudaStreamSynchronize(enc_stream);
    drop_graphs(this);
    audio_ws_free(audio);
    for (cudaEvent_t e : {ev_enc, ev_adm, ev_stage}) if (e) cudaEventDestroy(e);
    for (cudaEvent_t e : ev_t) if (e) cudaEventDestroy(e);
    if (stream) cudaStreamDestroy(stream);
    if (enc_stream) cudaStreamDestroy(enc_stream);
}

namespace wk {

AudioWs** session_audio_ws(wk_session* s) { return &s->audio; }
cudaStream_t session_stream(wk_session* s) { return s->stream; }
int session_device(wk_session* s) { return s->m->device; }
int64_t session_bias_sets(const wk_session* s) { return (int64_t)s->bias_sets.size(); }
int session_top_logprobs(const wk_session* s) { return s->top_k; }
void session_bias_map(wk_session* s, std::vector<int> map) { s->bias_map = std::move(map); }

// ---------------------------------------------------------------------------------------------- decoder schedule
static wk_status dec_gemm(wk_session* s, const void* w, int N, int K, const void* act, int* splits_out, int bp = 0) {
    wk_model* m = s->m;
    if (bp == 0) bp = s->bp;
    GemmDesc g;
    memset(&g, 0, sizeof(g));
    // swap-AB: A = weights [N, K] (128 output features per tile), B = activations [Bp, K]
    g.a = w; g.a_rows = N; g.a_cols = K; g.a_ld = K; g.a_batches = 1;
    g.b = act; g.b_rows = bp; g.b_ld = K; g.in_dtype = m->cfg.dtype;
    g.m_rows_per_batch = N; g.n = bp; g.k = K; g.taps = 1; g.bn = bp;
    const int tiles = (N + 127) / 128;
    g.splits = choose_splits(tiles, K / 64, m->num_sms);
    g.mode = GEMM_OUT_PARTIAL_T; g.out = s->partial; g.ld_out = N; g.out_rows_per_batch = N; g.partial_cols = bp;
    g.pdl = 1; g.a_static = 1;
    if ((size_t)g.splits * bp * N > s->partial_elems) { set_error("partial workspace too small"); return WK_ERR_DECODING_FAILED; }
    *splits_out = g.splits;
    return gemm_wgmma(g, m->num_sms, s->stream);
}

// Bytes of one cross K/V element, and the projection of `cnt` windows of encoder output `src` ([cnt * T][d]) into slots [q0, q0 + cnt) of
// the cache in the session's storage policy: the model's decoder's cache, or (draft) the draft decoder's
static size_t ckv_esize(const wk_session* s) { return s->ckv_fp8 ? 1 : 2; }
// the draft decoder's buffers hold one row per window slot; a draft call has at most max_batch / 2 (G = k + 1 >= 2 rows per window)
static int draft_slots(const wk_session* s) { return s->max_batch / 2; }
static GemmDesc cross_kv_gemm(const wk_session* s, const void* src, int cnt, int q0, bool draft = false) {
    const wk_model_config& c = s->m->cfg;
    const int T = c.n_audio_ctx, H = c.n_heads;
    const DecoderWeights w = draft ? s->m->draft->view() : s->m->main_decoder();
    void* cache = draft ? s->dr_cross_kv : s->cross_kv;
    float* scale = draft ? s->dr_cross_scale : s->cross_scale;
    GemmDesc g = plain_gemm(src, (int64_t)cnt * T, c.d_model, w.wckv, 2 * w.n_layers * c.d_model, c.dtype,
                            s->ckv_fp8 ? GEMM_OUT_FP8_HEADS : s->ckv_packed ? GEMM_OUT_PACKED_HEADS : GEMM_OUT_T16_HEADS, (char*)cache + (size_t)q0 * H * T * 64 * ckv_esize(s), 0,
                            w.bckv, 0);
    g.heads_T = T; g.heads_B = draft ? draft_slots(s) : s->max_batch; g.heads_H = H; g.heads_dmodel = c.d_model;
    if (s->ckv_fp8) g.out_scale = scale + (size_t)q0 * H * T;
    if (s->ckv_packed) g.out_hdr = (draft ? s->dr_cross_hdr : s->cross_hdr) + (size_t)q0 * H * packed_hdr_stride(T);
    return g;
}

// One decoder forward: which decoder (the model's or its draft), its caches (every layer strided by the session's max_batch rows or slots),
// the decode state and the rows.  kv_div: rows per cross K/V block (window); anc: rows read their self K/V through the cache ancestry;
// verify: the rows of a window are consecutive positions of one step (draft verification) - every row's K/V is appended before any row
// attends, and the cross-attention keeps its single-query form so that each row computes what it would alone
struct DecPass {
    DecoderWeights w;
    int cap;                       // rows (or window slots) the caches hold per layer
    void* self_k; void* self_v; void* cross_kv; float* cross_scale; uint8_t* cross_hdr;
    DecodeState st;
    int B, Bp, kv_div;
    const int32_t* anc;
    bool verify, align;
};

// explicit_pos == nullptr: loop mode (token / position from the pass's DecodeState, ended rows skipped)
static wk_status decoder_pass(wk_session* s, const DecPass& P, int ts_begin, const int32_t* explicit_pos, bool check_done) {
    wk_model* m = s->m;
    const wk_model_config& c = m->cfg;
    const int d = c.d_model, H = c.n_heads, dt = c.dtype, B = P.B, Bp = P.Bp, T = c.n_audio_ctx;
    cudaStream_t st = s->stream;
    const size_t self_layer = (size_t)P.cap * H * kKvMaxLen * 64 * 2;   // bytes per layer
    const size_t cross_rows = (size_t)P.cap * H * T;                    // rows of 64 per (layer, k|v)
    const size_t cross_block = cross_rows * 64 * ckv_esize(s);                 // bytes per (layer, k|v)
    const int32_t* pos = explicit_pos ? explicit_pos : P.st.steps;
    // ended rows are skipped by the attention kernels; a burst that starts with every slot live runs the variant without the checks (a
    // row that ends inside it just keeps computing until the next poll, as harmlessly as before it ended)
    const int32_t* done = (explicit_pos || !check_done) ? nullptr : P.st.done;
    const int n_layers = P.w.n_layers;
    int sp = 1;
    WK_CHECK(decoder_embed_ln(P.w.emb, P.w.pos, P.w.layers[0].ln1.g, P.w.layers[0].ln1.b, P.st, c.vocab, ts_begin, s->x, s->xn, B, d, dt, explicit_pos, st));
    auto self_attn = [&](int li, const DecLayer& l) {
        char* kc = (char*)P.self_k + li * self_layer;
        char* vc = (char*)P.self_v + li * self_layer;
        if (P.verify) WK_CHECK(decoder_kv_append(s->partial, sp, Bp, l.bv, kc, vc, pos, done, B, H, kKvMaxLen, dt, st));
        return decoder_self_attention(s->partial, sp, Bp, l.bq, l.bv, kc, vc, pos, done, s->attn, B, H, kKvMaxLen, dt, st, P.anc);
    };
    const size_t hdr_block = (size_t)P.cap * H * packed_hdr_stride(T);   // header bytes per (layer, k|v)
    auto cross_attn = [&](int li, const DecLayer& l) {
        const bool align = P.align && m->align_mask[li] != 0;
        const char* kc = (const char*)P.cross_kv + (size_t)(2 * li) * cross_block;
        const char* vc = (const char*)P.cross_kv + (size_t)(2 * li + 1) * cross_block;
        const uint8_t* kh = s->ckv_packed ? P.cross_hdr + (2 * li) * hdr_block : nullptr;
        const uint8_t* vh = s->ckv_packed ? P.cross_hdr + (2 * li + 1) * hdr_block : nullptr;
        return decoder_cross_attention(s->partial, sp, Bp, l.bcq, kc, vc, s->attn, B, H, T, dt, st, done,
                                       align ? s->align_scratch + (size_t)m->align_base[li] * B * T : nullptr, align ? m->align_mask[li] : 0u,
                                       P.kv_div, s->ckv_fp8 ? P.cross_scale + (2 * li) * cross_rows : nullptr,
                                       s->ckv_fp8 ? P.cross_scale + (2 * li + 1) * cross_rows : nullptr, P.verify, kh, vh);
    };
    for (int li = 0; li < n_layers; ++li) {
        const DecLayer& l = P.w.layers[li];
        WK_CHECK(dec_gemm(s, l.wqkv, 3 * d, d, s->xn, &sp, Bp));
        WK_CHECK(self_attn(li, l));
        WK_CHECK(dec_gemm(s, l.wo, d, d, s->attn, &sp, Bp));
        WK_CHECK(decoder_reduce_resid_ln(s->partial, sp, Bp, l.bo, l.lnx.g, l.lnx.b, s->x, s->xn, B, d, dt, st));
        WK_CHECK(dec_gemm(s, l.wcq, d, d, s->xn, &sp, Bp));
        WK_CHECK(cross_attn(li, l));
        WK_CHECK(dec_gemm(s, l.wco, d, d, s->attn, &sp, Bp));
        WK_CHECK(decoder_reduce_resid_ln(s->partial, sp, Bp, l.bco, l.ln3.g, l.ln3.b, s->x, s->xn, B, d, dt, st));
        WK_CHECK(dec_gemm(s, l.w1, 4 * d, d, s->xn, &sp, Bp));
        WK_CHECK(decoder_reduce_bias_gelu(s->partial, sp, Bp, l.b1, s->ffn, B, 4 * d, dt, st));
        WK_CHECK(dec_gemm(s, l.w2, d, 4 * d, s->ffn, &sp, Bp));
        const LayerNormW& nxt = (li + 1 < n_layers) ? P.w.layers[li + 1].ln1 : P.w.ln;
        WK_CHECK(decoder_reduce_resid_ln(s->partial, sp, Bp, l.b2, nxt.g, nxt.b, s->x, s->xn, B, d, dt, st));
    }
    // logits = xn . E^T  (tied embedding), written [B][V] f32 by the transposed-store epilogue (splits = 1)
    {
        GemmDesc g;
        memset(&g, 0, sizeof(g));
        g.a = P.w.emb; g.a_rows = c.vocab; g.a_cols = d; g.a_ld = d; g.a_batches = 1;
        g.b = s->xn; g.b_rows = Bp; g.b_ld = d; g.in_dtype = dt;
        g.m_rows_per_batch = c.vocab; g.n = Bp; g.k = d; g.taps = 1; g.bn = Bp; g.splits = 1;
        g.mode = GEMM_OUT_PARTIAL_T; g.out = s->logits; g.ld_out = c.vocab; g.out_rows_per_batch = c.vocab; g.partial_cols = B;
        g.pdl = 1; g.a_static = 1;
        WK_CHECK(gemm_wgmma(g, m->num_sms, st));
    }
    return WK_OK;
}

// one forward of the model's decoder for every row of the step.  explicit_pos == nullptr: loop mode
static wk_status decoder_forward(wk_session* s, int ts_begin, const int32_t* explicit_pos, bool check_done = true) {
    const bool loop = !explicit_pos;
    // loop mode: the window's G rows share one cross K/V block; beam rows and draft verification rows read the self K/V through the
    // cache ancestry
    DecPass P{s->m->main_decoder(), s->max_batch, s->self_k, s->self_v, s->cross_kv, s->cross_scale, s->cross_hdr, s->st, s->batch, s->bp,
              loop ? std::max(1, s->bs.group) : 1, loop && s->bs.use_anc ? s->bs.anc : nullptr, loop && s->draft_k > 0, loop && s->align_on};
    return decoder_pass(s, P, ts_begin, explicit_pos, check_done);
}

static SamplerParams loop_sampler_params(wk_session* s, const wk_special_tokens* st) {
    SamplerParams p;
    memset(&p, 0, sizeof(p));
    p.st = *st;
    p.vocab = s->m->cfg.vocab;
    p.is_multilingual = s->m->cfg.vocab != 51864;
    p.loop_mode = 1;
    p.suppress = s->suppress_dev;
    p.max_ctx = kKvMaxLen;
    p.detect_tokens = s->lang_dev;
    p.beam = s->bs;
    p.rng_div = s->draft_k > 0 ? s->bs.group : 1;
    p.top_tok = s->top_tok; p.top_lp = s->top_lp; p.top_n = s->top_n;
    return p;
}

// TextUtilities.compressionRatio(of: [Int]) (TextUtilities.swift:14-28): raw DEFLATE of the Int32 LE bytes, on one deflate state kept
// across the windows of a call (deflateReset gives the output of a fresh deflateInit2 without its allocation) - the stream stop rule
// evaluates it once per decoded token
namespace {
struct Deflater {
    z_stream zs;
    bool ok = false;
    std::vector<unsigned char> out;
    Deflater() { memset(&zs, 0, sizeof(zs)); ok = deflateInit2(&zs, 5, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY) == Z_OK; }
    ~Deflater() { if (ok) deflateEnd(&zs); }
    Deflater(const Deflater&) = delete;
    Deflater& operator=(const Deflater&) = delete;
    float ratio(const int32_t* toks, int n) {
        if (n <= 0 || !ok || deflateReset(&zs) != Z_OK) return INFINITY;
        const uLong bytes = (uLong)n * 4;
        out.resize(deflateBound(&zs, bytes) + 64);
        zs.next_in = (Bytef*)toks; zs.avail_in = (uInt)bytes;
        zs.next_out = out.data(); zs.avail_out = (uInt)out.size();
        const int r = deflate(&zs, Z_FINISH);
        const uLong clen = zs.total_out;
        if (r != Z_STREAM_END || clen == 0) return INFINITY;
        return (float)bytes / (float)clen;
    }
};
}  // namespace

// AudioStreamTranscriber.shouldStopEarly (AudioStreamTranscriber.swift:208-227) over history entries [from, n): the first index t >= P
// (a token the loop appended, so a callback that may stop, TextDecoder.swift:732-751) whose history tokens[0..t] meets the rule, else -1.
// *sum carries logProbs.reduce(0, +) over [0, from) and is advanced in the same order
static int stop_rule_index(const StopRule& rule, Deflater& z, const int32_t* tok, const float* lp, int from, int n, int P, float* sum) {
    for (int i = from; i < n; ++i) {
        *sum += lp[i];
        if (i < P) continue;
        const int count = i + 1;
        if (count > rule.window && z.ratio(tok + count - rule.window, rule.window) > rule.compression_threshold) return i;
        if (rule.has_logprob && *sum / (float)count < rule.logprob_threshold) return i;
    }
    return -1;
}

// finalisation of one window on the host: finalize + slicing + averages (TextDecoder.swift:776-853).  Returns the history index of the
// result's first token
static size_t finalize_result(wk_decode_result& r, const int32_t* tokens, const float* lps, int n_tok, int steps, int first_low,
                              const wk_special_tokens* st, const wk_decode_opts* o, float temperature, float no_speech_prob, Deflater& z) {
    memset(&r, 0, sizeof(r));
    std::vector<int32_t> seg(tokens, tokens + n_tok);
    std::vector<float> slp(lps, lps + n_tok);
    r.n_current_tokens = n_tok;
    r.steps = steps;
    r.first_token_logprob_too_low = first_low;
    if (seg.empty() || seg.back() != st->end_token) { seg.push_back(st->end_token); slp.push_back(0.f); }  // sampler.finalize
    size_t start = 0, end = seg.size();
    for (size_t i = 0; i < seg.size(); ++i) if (seg[i] == st->start_of_transcript_token) { start = i; break; }
    for (size_t i = 0; i < seg.size(); ++i) if (seg[i] == st->end_token) { end = i; break; }
    if (end >= seg.size()) end = seg.size() - 1;
    if (end < start) start = 0;
    float sum = 0.f;
    std::vector<int32_t> words;
    r.n_tokens = 0;
    for (size_t i = start; i <= end && r.n_tokens < 226; ++i) {
        r.tokens[r.n_tokens] = seg[i];
        r.token_logprobs[r.n_tokens] = slp[i];
        sum += slp[i];
        if (seg[i] < st->special_token_begin) words.push_back(seg[i]);
        ++r.n_tokens;
    }
    r.avg_logprob = sum / (float)r.n_tokens;
    r.compression_ratio = z.ratio(words.data(), (int)words.size());
    r.temperature = roundf(temperature * 1000.f) / 1000.f;
    // DecodingFallback (Models.swift:357-381); noSpeechProb is 0 unless the window computes it (the reference's is always 0,
    // TextDecoder.swift:802)
    r.needs_fallback = 0; r.fallback_reason = 0;
    if (first_low) { r.needs_fallback = 1; r.fallback_reason = 1; }
    else if (o->has_no_speech_threshold && no_speech_prob > o->no_speech_threshold) { r.needs_fallback = 0; r.fallback_reason = 2; }
    else if (o->has_compression_ratio_threshold && r.compression_ratio > o->compression_ratio_threshold) { r.needs_fallback = 1; r.fallback_reason = 3; }
    else if (o->has_logprob_threshold && r.avg_logprob < o->logprob_threshold) { r.needs_fallback = 1; r.fallback_reason = 4; }
    return start;
}

// prefillDecoderInputs (TextDecoder.swift:163-216)
static void build_prompt(const wk_model* m, const wk_special_tokens* st, const wk_decode_opts* o, int use_options, std::vector<int32_t>& p) {
    p.clear();
    p.push_back(st->start_of_transcript_token);
    if (use_options && o) {
        const bool multilingual = m->cfg.vocab != 51864;
        if (multilingual) {
            p.push_back(o->language_token >= 0 ? o->language_token : st->english_token);
            p.push_back(o->task_translate ? st->translate_token : st->transcribe_token);
        }
        p.push_back(o->without_timestamps ? st->no_timestamps_token : st->time_token_begin);
        if (o->n_prompt_tokens >= 0 && (o->prompt_tokens || o->n_prompt_tokens == 0)) {
            const int maxlen = kKvMaxLen / 2 - 1;
            std::vector<int32_t> q;
            const int start = o->n_prompt_tokens > maxlen ? o->n_prompt_tokens - maxlen : 0;
            q.push_back(st->start_of_previous_token);
            for (int i = start; i < o->n_prompt_tokens; ++i)
                if (o->prompt_tokens[i] < st->special_token_begin) q.push_back(o->prompt_tokens[i]);
            q.insert(q.end(), p.begin(), p.end());
            p.swap(q);
        }
        if (o->n_prefix_tokens >= 0 && (o->prefix_tokens || o->n_prefix_tokens == 0)) {
            const int maxlen = kKvMaxLen / 2;
            const int start = o->n_prefix_tokens > maxlen ? o->n_prefix_tokens - maxlen : 0;
            for (int i = start; i < o->n_prefix_tokens; ++i)
                if (o->prefix_tokens[i] < st->special_token_begin) p.push_back(o->prefix_tokens[i]);
        }
    }
}

// ---------------------------------------------------------------------------------------------- the step and its graph
// A draft call's step is a round (kernels.h, DraftRound): k + 1 draft steps over the window slots - each catches the draft up on a
// committed token or makes a proposal - then the verification rows are set up; the model's step over every row and the acceptance follow
static wk_status enqueue_draft_steps(wk_session* s, const wk_special_tokens* st) {
    wk_model* m = s->m;
    const int slots = s->dr.slots;
    WK_CHECK(draft_round_begin(s->st, s->dst, s->drp, s->dr, s->stream));
    DecPass P{m->draft->view(), draft_slots(s), s->dr_self_k, s->dr_self_v, s->dr_cross_kv, s->dr_cross_scale, s->dr_cross_hdr, s->dst, slots, round_up(slots, 16), 1, nullptr, false, false};
    SamplerParams sp = loop_sampler_params(s, st);
    sp.beam = BeamState();
    sp.rng_div = 1;
    for (int i = 0; i <= s->draft_k; ++i) {
        WK_CHECK(draft_feed(s->st, s->dst, s->dr, 0, s->stream));
        WK_CHECK(decoder_pass(s, P, st->time_token_begin, nullptr, true));
        WK_CHECK(sampler_filter_sample(s->logits, m->cfg.vocab, sp, s->dst, nullptr, 0, nullptr, nullptr, nullptr, nullptr, slots, s->stream));
    }
    WK_CHECK(draft_feed(s->st, s->dst, s->dr, 1, s->stream));
    return draft_verify_setup(s->st, s->rp_dev, s->bs.anc, s->dr, s->stream);
}

static wk_status enqueue_step(wk_session* s, const wk_special_tokens* st, bool check_done) {
    wk_model* m = s->m;
    if (s->draft_k > 0) WK_CHECK(enqueue_draft_steps(s, st));
    WK_CHECK(decoder_forward(s, st->time_token_begin, nullptr, check_done));
    WK_CHECK(sampler_filter_sample(s->logits, m->cfg.vocab, loop_sampler_params(s, st), s->st, nullptr, 0, nullptr, nullptr, nullptr, nullptr, s->batch, s->stream));
    if (s->bs.beam > 1) WK_CHECK(beam_update(s->st, s->bs, *st, kKvMaxLen, s->batch / s->bs.group, s->stream));
    if (s->draft_k > 0) WK_CHECK(draft_accept(s->st, s->bs.anc, s->dr, s->stream));
    if (s->align_on)
        WK_CHECK(decoder_align_mean(s->align_scratch, m->n_align_slots, s->st.steps, s->st.done, s->st.lang_state, s->align_w, s->batch, m->cfg.n_audio_ctx,
                                    kKvMaxLen, s->stream));
    return WK_OK;
}

// runs `n` decode steps on the session stream (CUDA graph replay; the first step of a session runs eagerly so that lazily loaded
// kernels and function attributes exist before a capture)
static wk_status run_steps(wk_session* s, const wk_special_tokens* st, int n, bool all_live) {
    const bool check_done = !all_live;
    int done = 0;
    if (!s->warmed) {
        WK_CHECK(enqueue_step(s, st, check_done));
        ++done;
        s->warmed = true;
    }
    if (done >= n) return WK_OK;
    // the step's shape depends on the rows per window (cross K/V sharing) and on whether the call has beam rows (ancestry, beam_update)
    // and on the bias pool the sampler reads (nullptr: no set attached)
    const int beam_key = (std::max(1, s->bs.group) * 16 + std::max(1, s->bs.beam)) * 16 + s->bs.max_candidates;
    const bool stale = s->graph_batch != s->batch || s->graph_align != s->align_on || s->graph_beam != beam_key ||
                       s->graph_draft != s->draft_k || s->graph_bias != s->st.bias_pool || s->graph_top != s->top_n ||
                       memcmp(&s->graph_st, st, sizeof(*st)) != 0;
    if (stale) {
        drop_graphs(s);
        s->graph_batch = s->batch; s->graph_align = s->align_on; s->graph_st = *st; s->graph_beam = beam_key; s->graph_draft = s->draft_k;
        s->graph_bias = s->st.bias_pool; s->graph_top = s->top_n;
    }
    cudaGraphExec_t& exec = check_done ? s->graph_exec : s->graph_exec_live;
    if (!exec) {
        for (int attempt = 0; attempt < 2; ++attempt) {
            cudaGraph_t graph = nullptr;
            const long long before = launch_counter_load();
            WK_CUDA_CHECK(cudaStreamBeginCapture(s->stream, cudaStreamCaptureModeThreadLocal));
            wk_status r = enqueue_step(s, st, check_done);
            cudaError_t e = cudaStreamEndCapture(s->stream, &graph);
            s->launches_per_step = launch_counter_load() - before;
            launch_counter_sub(s->launches_per_step);  // captured, not executed
            if (r != WK_OK) { if (graph) cudaGraphDestroy(graph); return r; }
            if (e != cudaSuccess) { set_error("graph capture failed: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
            e = cudaGraphInstantiate(&exec, graph, 0);
            cudaGraphDestroy(graph);
            if (e == cudaSuccess) break;
            exec = nullptr;
            if (attempt == 0 && pdl_enabled()) {   // programmatic edges rejected by this driver: plain serialisation, capture again
                cudaGetLastError();
                pdl_disable();
                continue;
            }
            set_error("graph instantiate failed: %s", cudaGetErrorString(e));
            return WK_ERR_CUDA;
        }
    }
    for (; done < n; ++done) {
        WK_CUDA_CHECK(cudaGraphLaunch(exec, s->stream));
        count_launch((int)s->launches_per_step);
    }
    return WK_OK;
}

// ---------------------------------------------------------------------------------------------- the window scheduler
struct CoreArgs {
    const float* pcm; int64_t n; int64_t stride; const int32_t* spw;   // pcm == nullptr: windows are the session's bound rows (decodeText)
    const wk_special_tokens* st; const wk_batch_opts* bo; wk_decode_result* results;
    bool ladder;
    const StopRule* stop = nullptr;   // stream stop rule (transcribe_windows_stop); nullptr: windows end on their own or by callback
    int draft = 0;                    // speculative decoding: proposals per round, 0 = none
};

static const wk_decode_opts& opts_of(const wk_batch_opts* bo, int64_t w) { return bo->n_opts == 1 ? bo->opts[0] : bo->opts[w]; }

// the per-window alignmentWeights handed out by wk_session_alignment_weights: n_windows x rows x T Float16
static wk_status ensure_align_store(wk_session* s, int64_t n_windows, int rows) {
    WK_CHECK(s->mem.grow(&s->align_store, (size_t)n_windows * rows * s->m->cfg.n_audio_ctx * 2, s->stream));
    s->align_store_n = n_windows;
    s->align_store_rows = rows;
    return WK_OK;
}

static wk_status ensure_align(wk_session* s, int64_t n_windows) {
    wk_model* m = s->m;
    const size_t T = m->cfg.n_audio_ctx;
    if (!s->align_w) WK_CHECK(s->mem.alloc16(&s->align_w, (size_t)s->max_batch * kKvMaxLen * T));
    bool moved = false;
    WK_CHECK(s->mem.grow(&s->align_scratch, (size_t)std::max(1, m->n_align_slots) * s->max_batch * T, s->stream, &moved));
    if (moved || s->align_slots != m->n_align_slots) drop_graphs(s);   // the scratch pointer and the head slots are baked into the graphs
    s->align_slots = m->n_align_slots;
    return ensure_align_store(s, n_windows, kKvMaxLen);
}

static wk_status ensure_beam(wk_session* s) {
    if (s->bs_cap_rows >= s->max_batch) return WK_OK;
    const int S = s->max_batch, G = S / 2 + 1;
    Buffers& b = s->mem;
    WK_CHECK(b.dmalloc(&s->bs.sum_lp, S));
    WK_CHECK(b.dmalloc(&s->bs.cand_tok, (size_t)S * (kMaxBeam + 1)));
    WK_CHECK(b.dmalloc(&s->bs.cand_lp, (size_t)S * (kMaxBeam + 1)));
    WK_CHECK(b.dmalloc(&s->bs.cand_sc, (size_t)S * (kMaxBeam + 1)));
    WK_CHECK(b.dmalloc(&s->bs.anc, (size_t)S * kKvMaxLen));
    WK_CHECK(b.dmalloc(&s->bs.fin_tokens, (size_t)G * kMaxCand * kKvMaxLen));
    WK_CHECK(b.dmalloc(&s->bs.fin_lps, (size_t)G * kMaxCand * kKvMaxLen));
    WK_CHECK(b.dmalloc(&s->bs.fin_len, (size_t)G * kMaxCand));
    WK_CHECK(b.dmalloc(&s->bs.fin_score, (size_t)G * kMaxCand));
    WK_CHECK(b.dmalloc(&s->bs.n_fin, G));
    WK_CHECK(b.pinned(&s->h_n_fin, G));
    WK_CHECK(b.pinned(&s->h_fin_len, (size_t)G * kMaxCand));
    WK_CHECK(b.pinned(&s->h_fin_score, (size_t)G * kMaxCand));
    WK_CHECK(b.pinned(&s->h_fin_tokens, (size_t)G * kMaxCand * kKvMaxLen));
    WK_CHECK(b.pinned(&s->h_fin_lps, (size_t)G * kMaxCand * kKvMaxLen));
    WK_CHECK(b.pinned(&s->h_sum_lp, S));
    s->bs_cap_rows = S;
    return WK_OK;
}

// the draft decoder's buffers (speculative decoding), for draft_slots(s) windows: self K/V and cross K/V, decode state, the rounds'
// bookkeeping
static wk_status ensure_draft(wk_session* s) {
    if (s->draft_ready) return WK_OK;
    const wk_model_config& c = s->m->cfg;
    const int S = draft_slots(s), H = c.n_heads, T = c.n_audio_ctx, Ld = (int)s->m->draft->dec.size();
    Buffers& b = s->mem;
    if (s->ckv_fp8) {
        uint8_t* codes = nullptr;
        WK_CHECK(b.dmalloc(&codes, (size_t)2 * Ld * S * H * T * 64));
        s->dr_cross_kv = codes;
        WK_CHECK(b.dmalloc(&s->dr_cross_scale, (size_t)2 * Ld * S * H * T));
    } else {
        WK_CHECK(b.alloc16(&s->dr_cross_kv, (size_t)2 * Ld * S * H * T * 64));
        if (s->ckv_packed) WK_CHECK(b.dmalloc(&s->dr_cross_hdr, (size_t)2 * Ld * S * H * packed_hdr_stride(T)));
    }
    WK_CHECK(b.alloc16(&s->dr_self_k, (size_t)Ld * S * H * kKvMaxLen * 64));
    WK_CHECK(b.alloc16(&s->dr_self_v, (size_t)Ld * S * H * kKvMaxLen * 64));
    DecodeState& d = s->dst;
    WK_CHECK(b.dmalloc(&d.tokens, (size_t)S * kKvMaxLen));
    WK_CHECK(b.dmalloc(&d.logprobs, (size_t)S * kKvMaxLen));
    for (int32_t** p : {&d.n_tokens, &d.next_token, &d.done, &d.first_low, &d.steps, &d.input_ids, &d.error, &d.lang_token, &d.lang_state})
        WK_CHECK(b.dmalloc(p, S));
    WK_CHECK(b.dmalloc(&d.lang_logprob, S));
    WK_CHECK(b.dmalloc(&d.no_speech, S));
    WK_CHECK(b.dmalloc(&s->drp, S));
    d.rp = s->drp;
    DraftRound& R = s->dr;
    for (int32_t** p : {&R.fed, &R.p0, &R.verify, &R.nprop, &R.rows, &R.cur}) WK_CHECK(b.dmalloc(p, S));
    WK_CHECK(b.dmalloc(&R.prop, (size_t)S * 8));
    WK_CHECK(b.dmalloc(&R.counters, 3));
    s->draft_ready = true;
    return WK_OK;
}

// the sampler's top-k pairs and their readback (DecodingOptions.topLogProbs), sized for k = 20: their pointers never change
static wk_status ensure_top(wk_session* s) {
    if (s->top_tok) return WK_OK;
    const size_t n = (size_t)s->max_batch * kKvMaxLen * kMaxTopLogprobs;
    Buffers& b = s->mem;
    WK_CHECK(b.dmalloc(&s->top_tok, n));
    WK_CHECK(b.dmalloc(&s->top_lp, n));
    WK_CHECK(b.pinned(&s->h_top_tok, n));
    WK_CHECK(b.pinned(&s->h_top_lp, n));
    return WK_OK;
}

// One window as the call decodes it: its prompt, the index of the prompt's first <|startoftranscript|> (-1: none) and whether the window
// detects its language in the loop
struct WindowPlan { const int32_t* p = nullptr; int np = 0, sot = -1; bool detects = false; };

// What a call decodes, worked out on the host before any CUDA work
struct CallPlan {
    int beam = 1, best_of = 0, G = 1, max_cand = 0;   // G = max(beam, best_of), or draft + 1: decode rows per window
    int draft = 0;                                    // proposals per round (wk_transcribe_windows_draft), 0 = no draft
    std::vector<WindowPlan> win;
    std::vector<std::vector<int32_t>> built;          // the prompts built from the options, when the call passes none
    std::vector<int32_t> sup_pool;                    // suppress ids of every option set: set i's at [sup_off[i], sup_off[i] + sup_n[i])
    std::vector<int> sup_off, sup_n;
    std::vector<int32_t> lang_list, lang_sorted;      // the call's allLanguageTokens: one list for every detecting window (one device buffer)
    std::vector<wk_status> st_local;
    wk_status* status = nullptr;                      // per window: bo->status, or st_local
    std::string first_err;                            // the message of the first window that failed
    std::vector<int> bias_of;                         // per window: its entry of the session's bias sets (empty: no set attached)
    bool any_words = false, any_detect = false, any_nsp = false;
    void fail(int64_t w, wk_status code, wk_decode_result* results) {
        status[w] = code;
        if (first_err.empty()) first_err = last_error_cstr();
        memset(&results[w], 0, sizeof(wk_decode_result));
    }
};

// Checks the call's options and windows and builds its plan; resets the session's per-window outputs of the last call.  A bad window
// fails alone (WhisperKit.swift:775-790); a call without a status array returns the first failure in the order of the passes below
static wk_status plan_call(wk_session* s, const CoreArgs& a, CallPlan& p) {
    const wk_model_config& c = s->m->cfg;
    const wk_batch_opts* bo = a.bo;
    const wk_special_tokens* st = a.st;
    const int64_t n = a.n;
    // beam search / best-of: every window takes G = max(beam, best_of) consecutive decode rows; one setting per call (it shapes the step
    // graph).  best_of == 0 keeps the plain rule: beam search (no ladder) or one row; best_of >= 1 picks the rows per ladder rung
    const int beam = p.beam = bo->opts[0].beam_size > 1 ? bo->opts[0].beam_size : 1;
    const int best_of = p.best_of = bo->best_of;
    for (int i = 0; i < bo->n_opts; ++i)
        if ((bo->opts[i].beam_size > 1 ? bo->opts[i].beam_size : 1) != beam || (beam > 1 && bo->opts[i].beam_patience != bo->opts[0].beam_patience)) {
            set_error("beam size / patience must be the same for every window of a call"); return WK_ERR_INVALID_ARGUMENT;
        }
    if (best_of < 0 || best_of > kMaxBeam) { set_error("best_of %d outside [0, %d]", best_of, kMaxBeam); return WK_ERR_INVALID_ARGUMENT; }
    // speculative decoding: greedy single-row windows only; the window's rows verify the draft's proposals
    const int draft = p.draft = a.draft;
    if (draft != 0) {
        if (draft < 1 || draft > kMaxDraftTokens) { set_error("draft_tokens %d outside [1, %d]", draft, kMaxDraftTokens); return WK_ERR_INVALID_ARGUMENT; }
        if (!s->m->draft) { set_error("draft_tokens %d: the model has no draft decoder", draft); return WK_ERR_INVALID_ARGUMENT; }
        if (beam > 1 || best_of != 0) { set_error("draft_tokens does not combine with beam search or best_of"); return WK_ERR_INVALID_ARGUMENT; }
        if (a.stop) { set_error("draft_tokens is not supported in streams"); return WK_ERR_INVALID_ARGUMENT; }
        for (int i = 0; i < bo->n_opts; ++i)
            if (bo->opts[i].word_timestamps) { set_error("draft_tokens does not combine with word timestamps"); return WK_ERR_INVALID_ARGUMENT; }
    }
    // contextual biasing: one attached set for every window, one per window, or the long-form round's per-window choice
    if (!s->bias_sets.empty()) {
        const int64_t ns = (int64_t)s->bias_sets.size();
        if (draft != 0) { set_error("a bias set does not combine with draft_tokens"); return WK_ERR_INVALID_ARGUMENT; }
        if (!s->bias_map.empty() ? (int64_t)s->bias_map.size() != n : (ns != 1 && ns != n)) {
            set_error("%lld bias sets attached for a call of %lld windows (1 or one per window)", (long long)ns, (long long)n);
            return WK_ERR_INVALID_ARGUMENT;
        }
        p.bias_of.resize((size_t)n);
        for (int64_t w = 0; w < n; ++w) p.bias_of[w] = !s->bias_map.empty() ? s->bias_map[w] : (ns == 1 ? 0 : (int)w);
    }
    const int G = p.G = draft > 0 ? draft + 1 : std::max(beam, std::max(best_of, 1));
    if (G > s->max_batch) {
        set_error("%d rows per window (beam size %d, best_of %d, draft_tokens %d) exceed the session's %d rows", G, beam, best_of, draft, s->max_batch);
        return WK_ERR_INVALID_ARGUMENT;
    }
    if (a.stop && (G != 1 || a.stop->window < 1)) { set_error("the stream stop rule needs single-row windows and a check window >= 1"); return WK_ERR_INVALID_ARGUMENT; }
    // top log-probs: the rows of greedy, sampling and best-of windows (a beam's history is reordered through its cache ancestry)
    if (s->top_k > 0 && (beam > 1 || draft > 0 || a.stop)) {
        set_error("topLogProbs %d does not combine with beam search, draft_tokens or streams", s->top_k);
        return WK_ERR_INVALID_ARGUMENT;
    }
    if (beam > 1) {
        const float patience = bo->opts[0].beam_patience > 0.f ? bo->opts[0].beam_patience : 1.f;
        p.max_cand = (int)((float)beam * patience);                                  // TokenSampler.swift:266
        if (beam > kMaxBeam || p.max_cand < 1 || p.max_cand > kMaxCand || s->max_batch < beam) {
            set_error("beam size %d / patience %.2f unsupported (beam <= %d, candidates in [1, %d], session rows %d)", beam, patience, kMaxBeam, kMaxCand, s->max_batch);
            return WK_ERR_INVALID_ARGUMENT;
        }
        for (int i = 0; i < bo->n_opts; ++i)
            if (bo->opts[i].word_timestamps) { set_error("wordTimestamps with beam search is not supported"); return WK_ERR_INVALID_ARGUMENT; }
    }
    if (!a.pcm && n > s->max_batch / G) { set_error("wk_decode_text: %lld bound windows x %d rows exceed the session's %d rows", (long long)n, G, s->max_batch); return WK_ERR_PREPARE_DECODER_INPUTS; }
    p.st_local.assign((size_t)n, WK_OK);
    p.status = bo->status ? bo->status : p.st_local.data();
    for (int64_t w = 0; w < n; ++w) p.status[w] = WK_OK;
    // ---- per-window prompts, options, suppress lists
    if (!bo->prompts && !bo->prompt) {
        p.built.resize(bo->n_opts == 1 ? 1 : (size_t)n);
        for (size_t i = 0; i < p.built.size(); ++i) {
            const wk_decode_opts& o = opts_of(bo, (int64_t)i);
            build_prompt(s->m, st, &o, o.use_prefill_prompt, p.built[i]);
        }
    }
    p.sup_off.resize(bo->n_opts);
    p.sup_n.resize(bo->n_opts);
    for (int i = 0; i < bo->n_opts; ++i) {
        const wk_decode_opts& o = bo->opts[i];
        p.any_words |= o.word_timestamps != 0;
        p.sup_off[i] = (int)p.sup_pool.size();
        for (int k = 0; k < o.n_suppress_tokens; ++k)   // SuppressTokensFilter gets the (< specialTokenBegin) ids only (TextDecoder.swift:876-879)
            if (o.suppress_tokens[k] >= 0 && o.suppress_tokens[k] < st->special_token_begin) p.sup_pool.push_back(o.suppress_tokens[k]);
        p.sup_n[i] = (int)p.sup_pool.size() - p.sup_off[i];
    }
    p.win.resize((size_t)n);
    for (int64_t w = 0; w < n; ++w) {
        WindowPlan& wp = p.win[w];
        if (bo->prompts) { wp.p = bo->prompts[w]; wp.np = bo->prompt_lens[w]; }
        else if (bo->prompt) { wp.p = bo->prompt; wp.np = bo->n_prompt; }
        else { const auto& v = p.built[bo->n_opts == 1 ? 0 : (size_t)w]; wp.p = v.data(); wp.np = (int)v.size(); }
        if (!wp.p || wp.np < 1 || wp.np >= kKvMaxLen) { set_error("window %lld: prompt length %d out of range", (long long)w, wp.np); p.fail(w, WK_ERR_PREPARE_DECODER_INPUTS, a.results); continue; }
        bool ok = true;
        for (int i = 0; i < wp.np && ok; ++i)
            if (wp.p[i] < 0 || wp.p[i] >= c.vocab) { set_error("window %lld: prompt token %d out of range", (long long)w, wp.p[i]); ok = false; }
        if (!ok) { p.fail(w, WK_ERR_PREPARE_DECODER_INPUTS, a.results); continue; }
        const int32_t* sot = std::find(wp.p, wp.p + wp.np, st->start_of_transcript_token);
        wp.sot = sot == wp.p + wp.np ? -1 : (int)(sot - wp.p);
        if (a.pcm && a.spw && (a.spw[w] < 0 || a.spw[w] > kWindowSamples)) {
            set_error("window %lld: samples_per_window %d out of range", (long long)w, a.spw[w]);
            p.fail(w, WK_ERR_AUDIO_PROCESSING_FAILED, a.results);
        }
    }
    // ---- in-loop language detection (DecodingOptions.detectLanguage): a multilingual model, no language set (TranscribeTask.swift:341)
    const bool multilingual = c.vocab != 51864;
    for (int64_t w = 0; w < n; ++w) {
        const wk_decode_opts& o = opts_of(bo, w);
        p.win[w].detects = o.detect_language != 0 && multilingual && o.language_token < 0;
        if (p.status[w] != WK_OK || !p.win[w].detects) continue;
        if (!o.language_tokens || o.n_language_tokens < 1 || o.n_language_tokens > 4096) {
            set_error("window %lld: detectLanguage needs 1..4096 language tokens (got %d)", (long long)w, o.language_tokens ? o.n_language_tokens : 0);
            p.fail(w, WK_ERR_INVALID_ARGUMENT, a.results);
            continue;
        }
        bool ok = true;
        for (int i = 0; i < o.n_language_tokens && ok; ++i)
            if (o.language_tokens[i] < 0 || o.language_tokens[i] >= c.vocab) {
                set_error("window %lld: language token %d outside the vocabulary (%d)", (long long)w, o.language_tokens[i], c.vocab);
                ok = false;
            }
        if (ok && p.any_detect &&
            ((int)p.lang_list.size() != o.n_language_tokens || !std::equal(p.lang_list.begin(), p.lang_list.end(), o.language_tokens))) {
            set_error("window %lld: every detecting window of a call must carry the same language tokens", (long long)w);
            ok = false;
        }
        if (!ok) { p.fail(w, WK_ERR_INVALID_ARGUMENT, a.results); continue; }
        if (!p.any_detect) p.lang_list.assign(o.language_tokens, o.language_tokens + o.n_language_tokens);
        p.any_detect = true;
    }
    p.lang_sorted = p.lang_list;
    std::sort(p.lang_sorted.begin(), p.lang_sorted.end());
    // ---- noSpeechProb (compute_no_speech_prob): the value comes from the step that feeds the prompt's first SOT, so that SOT must exist
    for (int64_t w = 0; w < n; ++w) {
        if (p.status[w] != WK_OK || !opts_of(bo, w).compute_no_speech_prob) continue;
        if (p.win[w].sot < 0) {
            set_error("window %lld: computeNoSpeechProb needs <|startoftranscript|> (token %d) in the prompt, which has none", (long long)w,
                      st->start_of_transcript_token);
            p.fail(w, WK_ERR_PREPARE_DECODER_INPUTS, a.results);
            continue;
        }
        p.any_nsp = true;
    }
    s->win_lang.assign((size_t)n, -1);
    s->win_lang_logprob.assign((size_t)n, 0.f);
    s->win_no_speech.assign((size_t)n, NAN);
    s->win_top_tok.assign((size_t)n, {});
    s->win_top_lp.assign((size_t)n, {});
    s->top_store_k = s->top_k;
    if (a.pcm && a.stride < kWindowSamples && !a.spw) { set_error("wk_transcribe_windows: stride < 480000 requires samples_per_window"); return WK_ERR_AUDIO_PROCESSING_FAILED; }
    if (!bo->status)
        for (int64_t w = 0; w < n; ++w) if (p.status[w] != WK_OK) { set_error("%s", p.first_err.c_str()); return p.status[w]; }
    return WK_OK;
}

// the plan's suppress pool and language list on the device
static wk_status upload_plan(wk_session* s, const CallPlan& p) {
    if (p.sup_pool.size() > s->suppress_cap) {
        const size_t cap = std::max<size_t>(4096, p.sup_pool.size() * 2);
        WK_CHECK(s->mem.grow(&s->suppress_dev, cap, s->stream));
        s->suppress_cap = cap;
        drop_graphs(s);   // pool pointer is baked into the graphs
    }
    if (!p.sup_pool.empty()) WK_CUDA_CHECK(cudaMemcpyAsync(s->suppress_dev, p.sup_pool.data(), p.sup_pool.size() * 4, cudaMemcpyHostToDevice, s->stream));
    if (p.any_detect) WK_CUDA_CHECK(cudaMemcpyAsync(s->lang_dev, p.lang_list.data(), p.lang_list.size() * 4, cudaMemcpyHostToDevice, s->stream));
    WK_CUDA_CHECK(cudaStreamSynchronize(s->stream));   // the host lists are pageable
    return WK_OK;
}

// temperature of ladder rung i, computed in Float16 like the reference (TranscribeTask.swift:327)
static float rung_temperature(const wk_decode_opts& o, int i) {
    if (i == 0) return o.temperature;
    const float f16_t = __half2float(__float2half(o.temperature));
    const float f16_step = __half2float(__float2half(__half2float(__float2half((float)i)) * __half2float(__float2half(o.temperature_increment_on_fallback))));
    return __half2float(__float2half(f16_t + f16_step));
}

// the rows a rung decodes with (openai/whisper decode_with_fallback): best_of == 0 - beam search on every row of a beam call, else one
// row; best_of >= 1 - beam search at temperature 0 when beam > 1, best_of independent samples at temperature > 0 when best_of > 1,
// else one row.  The group's other rows stay ended
static int rung_mode(int beam, int best_of, float temperature, int* active) {
    if (beam > 1 && (best_of == 0 || temperature == 0.f)) { *active = beam; return kRowBeam; }
    if (best_of > 1 && temperature > 0.f) { *active = best_of; return kRowSample; }
    *active = 1;
    return kRowSingle;
}

// the decode rows of window w at ladder rung `rung`; *active: how many of its G rows the rung decodes with
static RowParams row_params(const CallPlan& p, const wk_batch_opts* bo, const wk_special_tokens* st, int64_t w, int rung, int* active) {
    const wk_decode_opts& o = opts_of(bo, w);
    const int oi = bo->n_opts == 1 ? 0 : (int)w;
    const WindowPlan& wp = p.win[w];
    RowParams R;
    memset(&R, 0, sizeof(R));
    R.prompt_len = wp.np;
    // createLogitsFilters (TextDecoder.swift:857-899): SuppressBlank(sampleBegin = prefilledIndex = 0), TimestampRules(sampleBegin = initialPrompt.count)
    R.sample_begin_ts = o.without_timestamps ? -1 : wp.np;
    R.sample_begin_blank = o.suppress_blank ? 0 : -1;
    R.max_steps = std::max(1, std::min(o.sample_length, kKvMaxLen - 1));   // TextDecoder.swift:566
    R.temperature = rung_temperature(o, rung); R.top_k = o.top_k;
    R.has_first_thr = o.has_first_token_logprob_threshold; R.first_thr = o.first_token_logprob_threshold;
    R.seed = o.seed + (uint64_t)rung;
    R.suppress_off = p.sup_off[oi]; R.n_suppress = p.sup_n[oi];
    // every rung detects again at its own temperature (detectLanguage runs inside decodeWithFallback's loop, TranscribeTask.swift:333-365)
    R.lead_token = st->start_of_transcript_token;
    R.lang_pos = -1;
    R.no_speech_pos = o.compute_no_speech_prob ? wp.sot : -1;   // the same step at every rung
    if (wp.detects) {
        R.detect = wp.p[0] == st->start_of_transcript_token ? 1 : 2;
        R.n_lang = (int32_t)p.lang_list.size();
        // usePrefillPrompt: the prompt is rebuilt with the detected language - prefillDecoderInputs puts <|xx|> right after the first
        // SOT (TextDecoder.swift:176-186); a prompt without a language token there only reports the language
        const int i = wp.sot + 1;
        if (o.use_prefill_prompt && wp.sot >= 0 && i < wp.np && std::binary_search(p.lang_sorted.begin(), p.lang_sorted.end(), wp.p[i])) R.lang_pos = i;
    }
    R.mode = rung_mode(p.beam, p.best_of, R.temperature, active);
    return R;
}

// the bias set of window w (RowParams.bias_*), none when the call has no set attached
static void row_bias(const wk_session* s, const CallPlan& p, int64_t w, RowParams& R) {
    if (p.bias_of.empty()) return;
    const wk_session::BiasSlot& b = s->bias_sets[p.bias_of[w]];
    R.bias_off = b.off; R.bias_n = b.n; R.bias_len = b.len; R.bias_boost = b.boost;
}

// The decode slots of a call: the window each holds (-1: free), its ladder rung, and the stream stop rule's progress through the window's
// history (entries checked, their log-prob sum).  admit() stages the window's rows in the session's pinned buffers, flush() sends what
// is staged to the device in one go
struct Slots {
    wk_session* s; const CallPlan& p; const CoreArgs& a;
    std::vector<int> window, rung, stop_checked;
    std::vector<float> stop_sum;
    int live = 0, staged = 0;   // slots holding a window; rows staged since the last flush
    Slots(wk_session* s, const CallPlan& p, const CoreArgs& a, int S) : s(s), p(p), a(a), window(S, -1), rung(S, 0), stop_checked(S, 0), stop_sum(S, 0.f) {}

    // window w into free slot q at rung 0, or back into its slot at the next rung
    wk_status admit(int q, int64_t w, int r) {
        int active = 1;
        RowParams R = row_params(p, a.bo, a.st, w, r, &active);
        row_bias(s, p, w, R);
        if (staged == 0) WK_CUDA_CHECK(cudaEventSynchronize(s->ev_stage));   // the previous round's copies out of the pinned staging have landed
        for (int j = 0; j < active; ++j) {                                     // beam search / best-of: `active` identical rows start the window
            s->h_adm_slots[staged] = q * p.G + j;
            memset(s->h_adm_prompts + (size_t)staged * kKvMaxLen, 0, kKvMaxLen * 4);
            memcpy(s->h_adm_prompts + (size_t)staged * kKvMaxLen, p.win[w].p, (size_t)p.win[w].np * 4);
            s->h_adm_rp[staged] = R;
            ++staged;
        }
        if (r == 0) { ++live; ++s->stats[2]; } else { ++s->stats[3]; }
        window[q] = (int)w; rung[q] = r; stop_checked[q] = 0; stop_sum[q] = 0.f;
        return WK_OK;
    }
    wk_status flush() {
        if (staged == 0) return WK_OK;
        const int T = s->m->cfg.n_audio_ctx;
        WK_CUDA_CHECK(cudaMemcpyAsync(s->d_adm_slots, s->h_adm_slots, (size_t)staged * 4, cudaMemcpyHostToDevice, s->stream));
        WK_CUDA_CHECK(cudaMemcpyAsync(s->d_adm_prompts, s->h_adm_prompts, (size_t)staged * kKvMaxLen * 4, cudaMemcpyHostToDevice, s->stream));
        WK_CUDA_CHECK(cudaMemcpyAsync(s->d_adm_rp, s->h_adm_rp, (size_t)staged * sizeof(RowParams), cudaMemcpyHostToDevice, s->stream));
        if (s->align_on)
            for (int i = 0; i < staged; ++i)   // row 0 and unreached rows of alignmentWeights stay 0
                WK_CUDA_CHECK(cudaMemsetAsync((char*)s->align_w + (size_t)s->h_adm_slots[i] * kKvMaxLen * T * 2, 0, (size_t)kKvMaxLen * T * 2, s->stream));
        WK_CHECK(decode_slots_init(s->st, s->rp_dev, s->d_adm_slots, s->d_adm_prompts, s->d_adm_rp, staged, s->stream, s->bs));
        WK_CUDA_CHECK(cudaEventRecord(s->ev_stage, s->stream));
        staged = 0;
        return WK_OK;
    }
};

// samples_per_window of windows [w0, w0 + cnt), those that failed validation masked to 0: encoded as silence, they never reach a slot
template <typename Status>
static const int32_t* mask_failed(const int32_t* spw, const Status* status, int64_t w0, int64_t cnt, std::vector<int32_t>& buf) {
    if (!spw) return nullptr;
    buf.assign(spw + w0, spw + w0 + cnt);
    for (int64_t i = 0; i < cnt; ++i) if (status[w0 + i] != WK_OK) buf[i] = 0;
    return buf.data();
}

// The encoder side of a call: chunks of windows through mel + encoder on the encoder stream while the decode stream runs, and the
// cross-attention K/V of the windows admitted from the chunk in enc_out.  acc: the stage times of wk_last_timings
struct EncoderFeed {
    wk_session* s; const CoreArgs& a; const wk_status* status; int Ec;
    int64_t next = 0, w0 = 0, n = 0, adm = 0;   // the next window to encode; the chunk in enc_out - windows [w0, w0 + n), adm of them handled
    bool waited = true;                         // the decode stream waits for the chunk's encoder output
    bool pending = false, ckv_timing = false;   // the chunk's stage times are unread; ev_t[4..5] hold an unread projection region
    float acc[6] = {0, 0, 0, 0, 0, 0};

    wk_status encode() {
        const int64_t nc = std::min<int64_t>(Ec, a.n - next);
        std::vector<int32_t> spw_buf;
        const int32_t* spw = mask_failed(a.spw, status, next, nc, spw_buf);
        cudaStream_t es = s->enc_stream;
        WK_CUDA_CHECK(cudaStreamWaitEvent(es, s->ev_adm, 0));   // the previous chunk's cross-KV projections have read enc_out
        WK_CUDA_CHECK(cudaEventRecord(s->ev_t[0], es));
        const float* src;
        int64_t src_stride;
        WK_CHECK(mel_stage(&s->ws, a.pcm + next * a.stride, nc, a.stride, es, &src, &src_stride));   // timed apart from the mel kernel
        WK_CUDA_CHECK(cudaEventRecord(s->ev_t[1], es));
        WK_CHECK(mel_run(s->m, &s->ws, src, nc, src_stride, spw, s->ws.mel, es));
        WK_CUDA_CHECK(cudaEventRecord(s->ev_t[2], es));
        WK_CHECK(encode_chunk(s->m, &s->ws, s->ws.mel, (int)nc, s->ws.enc_out, es));
        WK_CUDA_CHECK(cudaEventRecord(s->ev_t[3], es));
        WK_CUDA_CHECK(cudaEventRecord(s->ev_enc, es));
        w0 = next; n = nc; adm = 0; next += nc; waited = false; pending = true;
        return WK_OK;
    }
    // the chunk's windows into the free slots among the first `slots`, passing over the windows that failed validation; windows going
    // to consecutive slots share one projection GEMM, and the round's first one opens the timed region unless one is still unread
    wk_status admit(Slots& sl, int slots) {
        const size_t win_bytes = (size_t)s->m->cfg.n_audio_ctx * s->m->cfg.d_model * 2;
        bool first = true;
        for (int q = 0;;) {
            while (adm < n && status[w0 + adm] != WK_OK) ++adm;
            while (q < slots && sl.window[q] >= 0) ++q;
            if (adm == n || q == slots) break;
            const int q0 = q;
            const int64_t run0 = adm;
            for (; q < slots && adm < n && sl.window[q] < 0 && status[w0 + adm] == WK_OK; ++q, ++adm) WK_CHECK(sl.admit(q, w0 + adm, 0));
            if (!waited) { WK_CUDA_CHECK(cudaStreamWaitEvent(s->stream, s->ev_enc, 0)); waited = true; }
            if (first && !ckv_timing) WK_CUDA_CHECK(cudaEventRecord(s->ev_t[4], s->stream));
            first = false;
            WK_CHECK(gemm_wgmma(cross_kv_gemm(s, (const char*)s->ws.enc_out + run0 * win_bytes, q - q0, q0), s->m->num_sms, s->stream));
            if (s->draft_k > 0)   // the draft's cross K/V from the same encoder output
                WK_CHECK(gemm_wgmma(cross_kv_gemm(s, (const char*)s->ws.enc_out + run0 * win_bytes, q - q0, q0, true), s->m->num_sms, s->stream));
        }
        if (!first && !ckv_timing) { WK_CUDA_CHECK(cudaEventRecord(s->ev_t[5], s->stream)); ckv_timing = true; }
        if (adm == n) WK_CUDA_CHECK(cudaEventRecord(s->ev_adm, s->stream));
        return sl.flush();
    }
    // the stage times of finished work: after a burst's readback the burst (ev_t[6..7]) and the projections before it, then the chunk's
    // staging, mel and encoder once they have run
    void collect(bool after_burst) {
        float t;
        if (after_burst) {
            cudaEventElapsedTime(&t, s->ev_t[6], s->ev_t[7]); acc[3] += t;
            if (ckv_timing) { cudaEventElapsedTime(&t, s->ev_t[4], s->ev_t[5]); acc[2] += t; ckv_timing = false; }
        }
        if (!pending || cudaEventQuery(s->ev_t[3]) != cudaSuccess) return;
        cudaEventElapsedTime(&t, s->ev_t[0], s->ev_t[1]); acc[4] += t;
        cudaEventElapsedTime(&t, s->ev_t[1], s->ev_t[2]); acc[0] += t;
        cudaEventElapsedTime(&t, s->ev_t[2], s->ev_t[3]); acc[1] += t;
        pending = false;
    }
};

// the decode state of the step's rows back in the session's pinned buffers, in one synchronisation
static wk_status read_back(wk_session* s, const CallPlan& p) {
    const int rows = s->batch, slots = s->batch / p.G;
    WK_CUDA_CHECK(cudaMemcpyAsync(s->h_done, s->st.done, rows * 4, cudaMemcpyDeviceToHost, s->stream));
    WK_CUDA_CHECK(cudaMemcpyAsync(s->h_n_tokens, s->st.n_tokens, rows * 4, cudaMemcpyDeviceToHost, s->stream));
    WK_CUDA_CHECK(cudaMemcpyAsync(s->h_steps, s->st.steps, rows * 4, cudaMemcpyDeviceToHost, s->stream));
    WK_CUDA_CHECK(cudaMemcpyAsync(s->h_first_low, s->st.first_low, rows * 4, cudaMemcpyDeviceToHost, s->stream));
    WK_CUDA_CHECK(cudaMemcpyAsync(s->h_error, s->st.error, rows * 4, cudaMemcpyDeviceToHost, s->stream));
    WK_CUDA_CHECK(cudaMemcpyAsync(s->h_tokens, s->st.tokens, (size_t)rows * kKvMaxLen * 4, cudaMemcpyDeviceToHost, s->stream));
    WK_CUDA_CHECK(cudaMemcpyAsync(s->h_logprobs, s->st.logprobs, (size_t)rows * kKvMaxLen * 4, cudaMemcpyDeviceToHost, s->stream));
    if (p.any_detect) {
        WK_CUDA_CHECK(cudaMemcpyAsync(s->h_lang_token, s->st.lang_token, rows * 4, cudaMemcpyDeviceToHost, s->stream));
        WK_CUDA_CHECK(cudaMemcpyAsync(s->h_lang_logprob, s->st.lang_logprob, rows * 4, cudaMemcpyDeviceToHost, s->stream));
    }
    if (p.any_nsp) WK_CUDA_CHECK(cudaMemcpyAsync(s->h_no_speech, s->st.no_speech, rows * 4, cudaMemcpyDeviceToHost, s->stream));
    if (!p.bias_of.empty() && p.best_of > 1) WK_CUDA_CHECK(cudaMemcpyAsync(s->h_bias_acc, s->st.bias_acc, rows * 4, cudaMemcpyDeviceToHost, s->stream));
    if (p.beam > 1) {
        WK_CUDA_CHECK(cudaMemcpyAsync(s->h_sum_lp, s->bs.sum_lp, rows * 4, cudaMemcpyDeviceToHost, s->stream));
        WK_CUDA_CHECK(cudaMemcpyAsync(s->h_n_fin, s->bs.n_fin, slots * 4, cudaMemcpyDeviceToHost, s->stream));
        WK_CUDA_CHECK(cudaMemcpyAsync(s->h_fin_len, s->bs.fin_len, (size_t)slots * kMaxCand * 4, cudaMemcpyDeviceToHost, s->stream));
        WK_CUDA_CHECK(cudaMemcpyAsync(s->h_fin_score, s->bs.fin_score, (size_t)slots * kMaxCand * 4, cudaMemcpyDeviceToHost, s->stream));
        WK_CUDA_CHECK(cudaMemcpyAsync(s->h_fin_tokens, s->bs.fin_tokens, (size_t)slots * kMaxCand * kKvMaxLen * 4, cudaMemcpyDeviceToHost, s->stream));
        WK_CUDA_CHECK(cudaMemcpyAsync(s->h_fin_lps, s->bs.fin_lps, (size_t)slots * kMaxCand * kKvMaxLen * 4, cudaMemcpyDeviceToHost, s->stream));
    }
    const cudaError_t e = cudaStreamSynchronize(s->stream);
    if (e != cudaSuccess) { set_error("decode loop: %s", cudaGetErrorString(e)); return WK_ERR_DECODING_FAILED; }
    return WK_OK;
}

// The sequence the window in slot q returns, from the readback of its rows (first row q * G) decoded in rung mode `mode`: the row's own
// history, the best-ranked best-of sample or the beam search winner (P: prompt length); cut after the token the stream stop rule stops
// at when stop_at >= 0.  Points into the session's pinned readback buffers
struct Choice { int row; const int32_t* tok; const float* lp; int n; };
static Choice select_result(const wk_session* s, int q, int G, int mode, int beam, int best_of, int P, int stop_at, float bias_boost) {
    const int r0 = q * G;
    int rc = r0;                              // the row whose result the window returns
    if (mode == kRowSample) {
        // best-of: MaximumLikelihoodRanker without length penalty over the samples (oracle/best_of_ref.py rank_best_of) - the sum of
        // the row's recorded log-probs over max(sampled tokens, 1); ties go to the lowest row.  With a bias set the sum carries the
        // bonus the row banked (bias_boost > 0)
        float best_rank = -INFINITY;
        for (int j = 0; j < best_of; ++j) {
            const int rr = r0 + j;
            const float* lp = s->h_logprobs + (size_t)rr * kKvMaxLen;
            float sum = 0.f;
            for (int i = 0; i < s->h_n_tokens[rr]; ++i) sum += lp[i];
            if (bias_boost != 0.f) sum += bias_boost * (float)s->h_bias_acc[rr];
            const float rk = sum / (float)std::max(s->h_n_tokens[rr] - P, 1);
            if (j == 0 || rk > best_rank) { rc = rr; best_rank = rk; }
        }
    }
    Choice ch{rc, s->h_tokens + (size_t)rc * kKvMaxLen, s->h_logprobs + (size_t)rc * kKvMaxLen, s->h_n_tokens[rc]};
    if (mode == kRowBeam) {
        // BeamSearchDecoder.finalize + MaximumLikelihoodRanker (oracle/beam_ref.py): the finished list, topped up with the live beams
        // (best sum first) to `beam` entries; the winner maximises sum_logprob / sampled tokens
        struct Cand { const int32_t* tok; const float* lp; int len; float score; bool live; };
        std::vector<Cand> cands;
        const int nf = std::min(s->h_n_fin[q], kMaxCand);
        for (int f = 0; f < nf; ++f) {
            const size_t slot = (size_t)q * kMaxCand + f;
            cands.push_back(Cand{s->h_fin_tokens + slot * kKvMaxLen, s->h_fin_lps + slot * kKvMaxLen, s->h_fin_len[slot], s->h_fin_score[slot], false});
        }
        if ((int)cands.size() < beam) {
            std::vector<int> order(beam);
            for (int j = 0; j < beam; ++j) order[j] = j;
            std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return s->h_sum_lp[r0 + x] > s->h_sum_lp[r0 + y]; });
            for (int j : order) {
                const int rr = r0 + j;
                cands.push_back(Cand{s->h_tokens + (size_t)rr * kKvMaxLen, s->h_logprobs + (size_t)rr * kKvMaxLen, s->h_n_tokens[rr] + 1, s->h_sum_lp[rr], true});
                if ((int)cands.size() >= beam) break;
            }
        }
        int best = 0; float best_rank = -INFINITY;
        for (size_t i = 0; i < cands.size(); ++i) {
            const float rk = cands[i].score / (float)std::max(cands[i].len - P - 1, 1);
            if (i == 0 || rk > best_rank) { best = (int)i; best_rank = rk; }
        }
        const Cand& cd = cands[best];
        ch = Choice{r0, cd.tok, cd.lp, cd.live ? cd.len - 1 : cd.len};   // live beams carry no EOT yet: finalize_result appends it
    }
    // stream stop rule: the history cut after the stopping token (appended at step stop_at - 1), then the usual finalize
    if (stop_at >= 0) ch.n = stop_at + 1;
    return ch;
}

static wk_status transcribe_core(wk_session* s, const CoreArgs& a) {
    wk_model* m = s->m;
    const wk_batch_opts* bo = a.bo;
    const bool bound = a.pcm == nullptr;
    const int64_t n = a.n;
    const int T = m->cfg.n_audio_ctx;
    const int poll = bo->progress_every > 0 ? bo->progress_every : 16;
    CallPlan p;
    WK_CHECK(plan_call(s, a, p));
    const int beam = p.beam, best_of = p.best_of, G = p.G;
    if (beam > 1 || p.draft > 0) WK_CHECK(ensure_beam(s));
    if (p.draft > 0) WK_CHECK(ensure_draft(s));
    s->bs.beam = beam; s->bs.max_candidates = p.max_cand; s->bs.group = G; s->bs.use_anc = beam > 1 || p.draft > 0;
    s->draft_k = p.draft;
    s->st.bias_pool = p.bias_of.empty() ? nullptr : s->bias_pool;
    s->top_n = s->top_k;
    if (s->top_n > 0) WK_CHECK(ensure_top(s));
    WK_CHECK(upload_plan(s, p));
    s->align_on = p.any_words;
    s->win_align_lp.clear();   // the log-probs belong to the last align call only
    if (p.any_words) WK_CHECK(ensure_align(s, n));

    // ---- slots
    const int S = s->max_batch / G;                    // decode slots (windows in flight)
    const int Brun = (int)std::min<int64_t>(S, n);     // slots in use; the step covers Brun * G rows
    s->batch = Brun * G;
    s->bp = round_up(s->batch, 16);
    Slots slots(s, p, a, S);
    Deflater z;   // the compression ratios of the call's windows and of the stream stop rule
    {   // every slot starts free: done = 1 keeps its rows out of the step until a window is admitted
        std::vector<int32_t> ones(s->max_batch, 1);
        WK_CUDA_CHECK(cudaMemcpyAsync(s->st.done, ones.data(), s->max_batch * 4, cudaMemcpyHostToDevice, s->stream));
        if (p.draft > 0) {
            s->dr.k = p.draft; s->dr.group = G; s->dr.slots = Brun;
            WK_CUDA_CHECK(cudaMemsetAsync(s->dr.fed, 0, draft_slots(s) * 4, s->stream));
            WK_CUDA_CHECK(cudaMemsetAsync(s->dr.counters, 0, 3 * sizeof(unsigned long long), s->stream));
        }
        WK_CUDA_CHECK(cudaStreamSynchronize(s->stream));
    }
    memset(s->draft_stats, 0, sizeof(s->draft_stats));
    const int Ec = bound ? 0 : std::max(1, std::min(bo->encoder_chunk > 0 ? bo->encoder_chunk : m->cfg.max_batch, m->cfg.max_batch));
    EncoderFeed feed{s, a, p.status, Ec};
    if (!bound) WK_CHECK(enc_ws_ensure(m, &s->ws, m->cfg.max_batch));
    int64_t finished = 0;
    for (int64_t w = 0; w < n; ++w) if (p.status[w] != WK_OK) ++finished;
    memset(s->stats, 0, sizeof(s->stats));
    if (bound) {
        // decodeText on the bound rows: window w sits in slot w with its cross K/V already projected
        for (int64_t w = 0; w < n; ++w) if (p.status[w] == WK_OK) WK_CHECK(slots.admit((int)w, w, 0));
        WK_CHECK(slots.flush());
    }
    while (finished < n) {
        // (A) next chunk through mel + encoder as soon as the previous chunk has left enc_out
        if (!bound && feed.adm == feed.n && feed.next < n) WK_CHECK(feed.encode());
        // (B) admit encoded windows into free slots
        if (!bound && feed.adm < feed.n) WK_CHECK(feed.admit(slots, Brun));
        if (slots.live == 0) {
            if (!bound && (feed.adm < feed.n || feed.next < n)) continue;
            break;
        }
        // (C) a burst of decode steps, then the state comes back in one go
        WK_CUDA_CHECK(cudaEventRecord(s->ev_t[6], s->stream));
        WK_CHECK(run_steps(s, a.st, poll, slots.live == Brun && p.draft == 0));   // a draft call's rows 1..G-1 end every round
        s->stats[0] += poll; s->stats[1] += (int64_t)poll * slots.live;
        WK_CUDA_CHECK(cudaEventRecord(s->ev_t[7], s->stream));
        WK_CHECK(read_back(s, p));
        feed.collect(true);
        // (D) retire ended windows; progress callback / early stop for the live ones
        struct TopCopy { int64_t w; int row; size_t start; int np, n; };
        std::vector<TopCopy> top_copies;   // returned windows whose top log-probs come back after the loop
        for (int q = 0; q < Brun; ++q) {
            const int w = slots.window[q];
            if (w < 0) continue;
            const int r0 = q * G;                     // first decode row of the slot (the only one of a single-row rung)
            const wk_decode_opts& o = opts_of(bo, w);
            bool ended = true, stopped = false;       // a group has ended when all its rows have (best-of samples end one by one)
            for (int j = 0; j < G; ++j) ended &= s->h_done[r0 + j] != 0;
            int stop_at = -1;                         // stream stop rule: history index of the token the window stops at
            if (a.stop) {
                // every history entry since the last check (the history is causal: steps run past the stopping token are only lost time)
                const int nt = s->h_n_tokens[r0];
                stop_at = stop_rule_index(*a.stop, z, s->h_tokens + (size_t)r0 * kKvMaxLen, s->h_logprobs + (size_t)r0 * kKvMaxLen,
                                          slots.stop_checked[q], nt, p.win[w].np, &slots.stop_sum[q]);
                slots.stop_checked[q] = nt;
                if (stop_at >= 0 && !ended) {
                    const int32_t one = 1;
                    WK_CUDA_CHECK(cudaMemcpyAsync(s->st.done + r0, &one, 4, cudaMemcpyHostToDevice, s->stream));
                    WK_CUDA_CHECK(cudaStreamSynchronize(s->stream));
                    ended = true;
                }
            }
            if (!ended && bo->progress) {
                const int nt = s->h_n_tokens[r0];
                float sum = 0.f;
                for (int i = 0; i < nt; ++i) sum += s->h_logprobs[(size_t)r0 * kKvMaxLen + i];
                if (!bo->progress(bo->progress_user, w, s->h_tokens + (size_t)r0 * kKvMaxLen, nt, nt > 0 ? sum / nt : 0.f)) {
                    // callback -> false: the reference's early-stop flag ends the loop at the next token (TextDecoder.swift:733-762)
                    std::vector<int32_t> ones(G, 1);
                    WK_CUDA_CHECK(cudaMemcpyAsync(s->st.done + r0, ones.data(), G * 4, cudaMemcpyHostToDevice, s->stream));
                    WK_CUDA_CHECK(cudaStreamSynchronize(s->stream));
                    stopped = true;              // an early-stopped window does not walk the ladder
                    ended = true;
                }
            }
            if (!ended) continue;
            const float temperature = rung_temperature(o, slots.rung[q]);
            int active = 1;
            const float boost = p.bias_of.empty() ? 0.f : s->bias_sets[p.bias_of[w]].boost;
            const Choice ch = select_result(s, q, G, rung_mode(beam, best_of, temperature, &active), beam, best_of, p.win[w].np, stop_at, boost);
            // beam search: every beam of the window is the same forced copy through the prefill, so row r0 holds the value
            const float nsp = o.compute_no_speech_prob ? s->h_no_speech[r0] : NAN;
            wk_decode_result r;
            const size_t start = finalize_result(r, ch.tok, ch.lp, ch.n, stop_at >= 0 ? stop_at : s->h_steps[ch.row], s->h_first_low[ch.row], a.st,
                                                 &o, temperature, isnan(nsp) ? 0.f : nsp, z);
            int err_row = -1;                         // a row of the rung without a finite logit fails the window
            for (int j = 0; j < active && err_row < 0; ++j) if (s->h_error[r0 + j]) err_row = r0 + j;
            if (err_row >= 0) {
                set_error("window %d: no finite logit at decoder step %d", w, s->h_steps[err_row] - 1);
                p.fail(w, WK_ERR_DECODING_LOGITS_FAILED, a.results);
            } else if (a.ladder && (beam == 1 || best_of >= 1) && !stopped && r.needs_fallback && slots.rung[q] < o.temperature_fallback_count) {
                // decodeWithFallback (TranscribeTask.swift:316-411): same encoder output (the slot keeps its cross K/V), next temperature
                WK_CHECK(slots.admit(q, w, slots.rung[q] + 1));
                continue;
            } else {
                a.results[w] = r;
                if (p.any_detect) { s->win_lang[w] = s->h_lang_token[r0]; s->win_lang_logprob[w] = s->h_lang_logprob[r0]; }   // the returned rung's
                s->win_no_speech[w] = nsp;
                const int np = p.win[w].np;
                if (s->top_n > 0 && ch.n > np) {   // the sampled positions [np, n) of the returned row, before a re-admission reuses it
                    const size_t off = ((size_t)ch.row * kKvMaxLen + np) * s->top_n, cnt = (size_t)(ch.n - np) * s->top_n;
                    WK_CUDA_CHECK(cudaMemcpyAsync(s->h_top_tok + off, s->top_tok + off, cnt * 4, cudaMemcpyDeviceToHost, s->stream));
                    WK_CUDA_CHECK(cudaMemcpyAsync(s->h_top_lp + off, s->top_lp + off, cnt * 4, cudaMemcpyDeviceToHost, s->stream));
                }
                if (s->top_n > 0) top_copies.push_back(TopCopy{w, ch.row, start, np, ch.n});
            }
            if (s->align_on && p.status[w] == WK_OK && stop_at >= 0)   // rows of the steps run past the stopping token: the reference never ran them
                WK_CUDA_CHECK(cudaMemsetAsync((char*)s->align_w + ((size_t)ch.row * kKvMaxLen + stop_at + 1) * T * 2, 0,
                                              (size_t)(kKvMaxLen - stop_at - 1) * T * 2, s->stream));
            if (s->align_on && p.status[w] == WK_OK)
                WK_CUDA_CHECK(cudaMemcpyAsync((char*)s->align_store + (size_t)w * kKvMaxLen * T * 2, (char*)s->align_w + (size_t)ch.row * kKvMaxLen * T * 2,
                                              (size_t)kKvMaxLen * T * 2, cudaMemcpyDeviceToDevice, s->stream));
            slots.window[q] = -1;
            --slots.live;
            ++finished;
        }
        if (!top_copies.empty()) {
            WK_CUDA_CHECK(cudaStreamSynchronize(s->stream));
            const int k = s->top_n;
            for (const TopCopy& c : top_copies) {   // result token i is history entry start + i; forced entries and the closing EOT stay padded
                const int nr = a.results[c.w].n_tokens;
                std::vector<int32_t>& tt = s->win_top_tok[c.w];
                std::vector<float>& tl = s->win_top_lp[c.w];
                tt.assign((size_t)nr * k, -1);
                tl.assign((size_t)nr * k, -INFINITY);
                for (int t = std::max<int>(c.np, (int)c.start); t < c.n && t - (int)c.start < nr; ++t) {
                    const size_t src = ((size_t)c.row * kKvMaxLen + t) * k, dst = (size_t)(t - c.start) * k;
                    memcpy(tt.data() + dst, s->h_top_tok + src, (size_t)k * 4);
                    memcpy(tl.data() + dst, s->h_top_lp + src, (size_t)k * 4);
                }
            }
        }
        WK_CHECK(slots.flush());   // ladder re-admissions
    }
    if (p.draft > 0) {
        unsigned long long c[3];
        WK_CUDA_CHECK(cudaMemcpyAsync(c, s->dr.counters, sizeof(c), cudaMemcpyDeviceToHost, s->stream));
        WK_CUDA_CHECK(cudaStreamSynchronize(s->stream));
        for (int i = 0; i < 3; ++i) s->draft_stats[i] = (int64_t)c[i];
    }
    WK_CUDA_CHECK(cudaStreamSynchronize(s->stream));
    if (!bound) {
        WK_CUDA_CHECK(cudaStreamSynchronize(s->enc_stream));
        feed.collect(false);
        memcpy(m->timings, feed.acc, sizeof(feed.acc));
    }
    if (!bo->status)
        for (int64_t w = 0; w < n; ++w) if (p.status[w] != WK_OK) { set_error("%s", p.first_err.c_str()); return p.status[w]; }
    return WK_OK;
}

// ---------------------------------------------------------------------------------------------- teacher-forced alignment pass
// openai-whisper's find_alignment forward (timing.py): every position of a known token sequence through the decoder in one pass, the
// alignment heads' cross-attention rows and the text tokens' log-probs out of it.  Row w * 224 + t of the encoder workspace is position t
// of window w; the decoder GEMMs are the encoder's plain wgmma GEMMs over all rows, the attention / export / log-prob kernels are in
// align_pass.cu.
static constexpr int kAlignRows = kKvMaxLen + 1;   // alignment rows per window: row t + 1 for input position t, t < 224

static wk_status ensure_align_pass(wk_session* s, int nw) {
    const wk_model_config& c = s->m->cfg;
    const size_t R = (size_t)nw * kKvMaxLen;
    Buffers& b = s->mem;
    WK_CHECK(b.grow(&s->al_acc, R * c.n_audio_ctx, s->stream));
    WK_CHECK(b.grow(&s->al_stats, R * c.n_heads * 2, s->stream));
    WK_CHECK(b.grow(&s->al_lp, R, s->stream));
    WK_CHECK(b.grow(&s->al_bqkv, (size_t)c.dec_layers * 3 * c.d_model, s->stream));
    WK_CHECK(b.grow(&s->al_tok, R, s->stream));
    WK_CHECK(b.grow(&s->al_seq, (size_t)nw, s->stream));
    return WK_OK;
}

// windows [w_first, w_first + nw) of the call, their cross K/V in cache slots [slot0, slot0 + nw); seq / len: each window's tokens
// (len 0 = a window that failed validation: no rows, zero alignment rows)
static wk_status align_chunk(wk_session* s, const wk_special_tokens* st, int slot0, int nw, int64_t w_first, const int32_t* const* seq, const int* len) {
    wk_model* m = s->m;
    const wk_model_config& c = m->cfg;
    const int d = c.d_model, H = c.n_heads, T = c.n_audio_ctx, dt = c.dtype;
    const int64_t R = (int64_t)nw * kKvMaxLen;
    cudaStream_t stm = s->stream;
    EncWorkspace& ws = s->ws;
    std::vector<int32_t> tok((size_t)R, -1), n(nw);
    for (int i = 0; i < nw; ++i) {
        n[i] = len[i];
        for (int t = 0; t < len[i]; ++t) tok[(size_t)i * kKvMaxLen + t] = seq[i][t];
    }
    WK_CUDA_CHECK(cudaMemcpyAsync(s->al_tok, tok.data(), (size_t)R * 4, cudaMemcpyHostToDevice, stm));
    WK_CUDA_CHECK(cudaMemcpyAsync(s->al_seq, n.data(), (size_t)nw * 4, cudaMemcpyHostToDevice, stm));
    const size_t cross_rows = (size_t)s->max_batch * H * T;
    const size_t cross_block = cross_rows * 64 * ckv_esize(s);
    auto gemm = [&](const void* a, int K, const void* w, int N, int mode, void* out, const float* bias, int gelu) {
        return gemm_wgmma(plain_gemm(a, R, K, w, N, dt, mode, out, N, bias, gelu), m->num_sms, stm);
    };
    WK_CHECK(align_embed(m->emb, m->dec_pos, s->al_tok, ws.x, R, d, dt, stm));
    int first_align = 1;
    for (int li = 0; li < c.dec_layers; ++li) {
        const DecLayer& l = m->dec[li];
        WK_CHECK(layernorm_f32_to_16(ws.x, l.ln1.g, l.ln1.b, ws.xn, R, d, dt, stm));
        WK_CHECK(gemm(ws.xn, d, l.wqkv, 3 * d, GEMM_OUT_T16, ws.qkv, s->al_bqkv + (size_t)li * 3 * d, 0));
        WK_CHECK(align_self_attention(ws.qkv, s->al_seq, ws.attn, nw, H, dt, stm));
        WK_CHECK(gemm(ws.attn, d, l.wo, d, GEMM_OUT_F32_ADD, ws.x, l.bo, 0));
        WK_CHECK(layernorm_f32_to_16(ws.x, l.lnx.g, l.lnx.b, ws.xn, R, d, dt, stm));
        WK_CHECK(gemm(ws.xn, d, l.wcq, d, GEMM_OUT_T16, ws.qkv, l.bcq, 0));   // cross-attention queries [R][d]
        const uint32_t mask = m->align_mask[li];
        const char* kc = (const char*)s->cross_kv + (size_t)(2 * li) * cross_block;
        const char* vc = (const char*)s->cross_kv + (size_t)(2 * li + 1) * cross_block;
        const float* ksc = s->ckv_fp8 ? s->cross_scale + (size_t)(2 * li) * cross_rows : nullptr;
        const float* vsc = s->ckv_fp8 ? s->cross_scale + (size_t)(2 * li + 1) * cross_rows : nullptr;
        const size_t hb = (size_t)s->max_batch * H * packed_hdr_stride(T);
        const uint8_t* kh = s->ckv_packed ? s->cross_hdr + (2 * li) * hb : nullptr;
        const uint8_t* vh = s->ckv_packed ? s->cross_hdr + (2 * li + 1) * hb : nullptr;
        WK_CHECK(align_cross_attention(ws.qkv, kc, vc, ksc, vsc, s->al_seq, slot0, ws.attn, mask ? s->al_stats : nullptr, R, nw, H, T, dt, stm, kh, vh));
        if (mask) {
            WK_CHECK(align_export(ws.qkv, kc, ksc, s->al_stats, R, s->al_seq, slot0, mask, first_align, s->al_acc, nw, H, T, dt, stm, kh));
            first_align = 0;
        }
        WK_CHECK(gemm(ws.attn, d, l.wco, d, GEMM_OUT_F32_ADD, ws.x, l.bco, 0));
        WK_CHECK(layernorm_f32_to_16(ws.x, l.ln3.g, l.ln3.b, ws.xn, R, d, dt, stm));
        WK_CHECK(gemm(ws.xn, d, l.w1, 4 * d, GEMM_OUT_T16, ws.ffn, l.b1, 1));
        WK_CHECK(gemm(ws.ffn, 4 * d, l.w2, d, GEMM_OUT_F32_ADD, ws.x, l.b2, 0));
    }
    WK_CHECK(align_rows_f16(s->al_acc, s->al_seq, first_align ? 0 : m->n_align_slots, (char*)s->align_store + (size_t)w_first * kAlignRows * T * 2, nw, T,
                            kAlignRows, stm));
    // token log-probs: final LayerNorm, then the tied-embedding GEMM over the rows in chunks that fit the (now free) FC1 buffer, so that the
    // [rows][vocab] logits never exist whole.  Columns [vocab, Vp) come out 0 (TMA zero-fills the weight rows past the vocabulary).
    WK_CHECK(layernorm_f32_to_16(ws.x, m->dec_ln.g, m->dec_ln.b, ws.xn, R, d, dt, stm));
    const int Vp = round_up(c.vocab, 32);
    const int eot = std::min(st->end_token, c.vocab);
    const int64_t chunk = std::max<int64_t>(1, (int64_t)ws.max_batch * T * 4 * d * 2 / ((int64_t)Vp * 4));
    for (int64_t r0 = 0; r0 < R; r0 += chunk) {
        const int64_t rc = std::min(chunk, R - r0);
        GemmDesc g = plain_gemm((const char*)ws.xn + (size_t)r0 * d * 2, rc, d, m->emb, Vp, dt, GEMM_OUT_F32, ws.ffn, Vp, nullptr, 0);
        g.b_rows = c.vocab;
        WK_CHECK(gemm_wgmma(g, m->num_sms, stm));
        WK_CHECK(align_token_logprobs((const float*)ws.ffn, Vp, r0, rc, s->al_tok, s->al_seq, eot, s->al_lp, stm));
    }
    std::vector<float> lp((size_t)R);
    WK_CUDA_CHECK(cudaMemcpyAsync(lp.data(), s->al_lp, (size_t)R * 4, cudaMemcpyDeviceToHost, stm));
    cudaError_t e = cudaStreamSynchronize(stm);
    if (e != cudaSuccess) { set_error("alignment pass: %s", cudaGetErrorString(e)); return WK_ERR_DECODING_FAILED; }
    for (int i = 0; i < nw; ++i)
        for (int t = 1; t < len[i]; ++t) s->win_align_lp[(size_t)(w_first + i) * kKvMaxLen + t] = lp[(size_t)i * kKvMaxLen + t];
    return WK_OK;
}

// wk_align_tokens (pcm == nullptr: windows are the bound rows) and wk_align_windows (PCM -> mel -> encoder -> cross K/V per chunk)
static wk_status align_core(wk_session* s, const wk_special_tokens* st, const float* pcm, int64_t n, int64_t stride, const int32_t* spw,
                            const int32_t* tokens, const int32_t* offsets, int32_t* status_out) {
    wk_model* m = s->m;
    const wk_model_config& c = m->cfg;
    std::vector<int32_t> st_local((size_t)n, WK_OK);
    int32_t* status = status_out ? status_out : st_local.data();
    std::vector<int> len((size_t)n, 0);
    std::string first_err;
    for (int64_t w = 0; w < n; ++w) {
        status[w] = WK_OK;
        const int64_t cnt = (int64_t)offsets[w + 1] - offsets[w];
        wk_status code = WK_OK;
        if (cnt < 1) { set_error("window %lld: empty token sequence", (long long)w); code = WK_ERR_PREPARE_DECODER_INPUTS; }
        else if (cnt > kKvMaxLen) { set_error("window %lld: %lld tokens exceed the %d-token decoder context", (long long)w, (long long)cnt, kKvMaxLen); code = WK_ERR_PREPARE_DECODER_INPUTS; }
        else if (offsets[w] < 0) { set_error("window %lld: negative token offset %d", (long long)w, offsets[w]); code = WK_ERR_INVALID_ARGUMENT; }
        else {
            for (int64_t i = 0; i < cnt; ++i) {
                const int32_t v = tokens[offsets[w] + i];
                if (v < 0 || v >= c.vocab) {
                    set_error("window %lld: token %d at position %lld outside the vocabulary (%d)", (long long)w, v, (long long)i, c.vocab);
                    code = WK_ERR_PREPARE_DECODER_INPUTS;
                    break;
                }
            }
        }
        if (code == WK_OK && pcm && spw && (spw[w] < 0 || spw[w] > kWindowSamples)) {
            set_error("window %lld: samples_per_window %d out of range", (long long)w, spw[w]);
            code = WK_ERR_AUDIO_PROCESSING_FAILED;
        }
        if (code != WK_OK) {
            status[w] = code;
            if (first_err.empty()) first_err = last_error_cstr();
            if (!status_out) return code;
            continue;
        }
        len[w] = (int)cnt;
    }
    if (pcm && stride < kWindowSamples && !spw) { set_error("wk_align_windows: stride < 480000 requires samples_per_window"); return WK_ERR_AUDIO_PROCESSING_FAILED; }
    s->align_on = false;
    WK_CHECK(enc_ws_ensure(m, &s->ws, c.max_batch));
    WK_CHECK(ensure_align_store(s, n, kAlignRows));
    s->win_align_lp.assign((size_t)n * kKvMaxLen, NAN);
    // chunk size: the encoder's batch (PCM) or the rows the encoder workspace holds (bound windows), and the session's slots
    const int Wc = (int)std::min<int64_t>(n, pcm ? std::min(s->max_batch, s->ws.max_batch) : (int64_t)s->ws.max_batch * c.n_audio_ctx / kKvMaxLen);
    WK_CHECK(ensure_align_pass(s, Wc));
    for (int li = 0; li < c.dec_layers; ++li) {   // the self-attention QKV bias [bq | 0 | bv]: the decoder's k projection has none
        float* b = s->al_bqkv + (size_t)li * 3 * c.d_model;
        WK_CUDA_CHECK(cudaMemcpyAsync(b, m->dec[li].bq, (size_t)c.d_model * 4, cudaMemcpyDeviceToDevice, s->stream));
        WK_CUDA_CHECK(cudaMemsetAsync(b + c.d_model, 0, (size_t)c.d_model * 4, s->stream));
        WK_CUDA_CHECK(cudaMemcpyAsync(b + 2 * c.d_model, m->dec[li].bv, (size_t)c.d_model * 4, cudaMemcpyDeviceToDevice, s->stream));
    }
    std::vector<const int32_t*> seq((size_t)Wc);
    for (int64_t w0 = 0; w0 < n; w0 += Wc) {
        const int cnt = (int)std::min<int64_t>(Wc, n - w0);
        int slot0 = (int)w0;
        if (pcm) {
            std::vector<int32_t> spw_buf;
            WK_CHECK(mel_run(m, &s->ws, pcm + w0 * stride, cnt, stride, mask_failed(spw, status, w0, cnt, spw_buf), s->ws.mel, s->stream));
            WK_CHECK(encode_chunk(m, &s->ws, s->ws.mel, cnt, s->ws.enc_out, s->stream));
            WK_CHECK(gemm_wgmma(cross_kv_gemm(s, s->ws.enc_out, cnt, 0), m->num_sms, s->stream));
            slot0 = 0;
        }
        for (int i = 0; i < cnt; ++i) seq[i] = tokens + (len[w0 + i] > 0 ? offsets[w0 + i] : 0);
        WK_CHECK(align_chunk(s, st, slot0, cnt, w0, seq.data(), len.data() + w0));
    }
    s->align_on = true;
    if (!first_err.empty()) set_error("%s", first_err.c_str());   // per-window failures are in status_out; the message of the first one
    return WK_OK;
}

}  // namespace wk

// =====================================================================================================
// C ABI
// =====================================================================================================
extern "C" {

wk_status wk_session_create(wk_model* m, int32_t max_batch, wk_session** out) {
    if (!m || !out || max_batch < 1 || max_batch > 256) { set_error("wk_session_create: bad arguments (max_batch %d, limit 256)", max_batch); return WK_ERR_INVALID_ARGUMENT; }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    const wk_model_config& c = m->cfg;
    const int d = c.d_model, H = c.n_heads, L = c.dec_layers, T = c.n_audio_ctx, S = max_batch;
    std::unique_ptr<wk_session> s(new wk_session());   // released on any failure below
    s->m = m;
    s->max_batch = S;
    WK_CUDA_CHECK(cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking));
    WK_CUDA_CHECK(cudaStreamCreateWithFlags(&s->enc_stream, cudaStreamNonBlocking));
    const int bpm = round_up(S, 16);
    {
        std::lock_guard<std::mutex> lock(m->api_mu);   // against a concurrent wk_model_set_cross_kv_dtype
        m->session_created = true;
        s->ckv_fp8 = m->cross_kv_fp8;
    }
    Buffers& b = s->mem;
    if (s->ckv_fp8) {
        uint8_t* codes = nullptr;
        WK_CHECK(b.dmalloc(&codes, (size_t)2 * L * S * H * T * 64));
        s->cross_kv = codes;
        WK_CHECK(b.dmalloc(&s->cross_scale, (size_t)2 * L * S * H * T));
    } else {
        WK_CHECK(b.alloc16(&s->cross_kv, (size_t)2 * L * S * H * T * 64));
        s->ckv_packed = c.dtype == WK_DTYPE_BF16;
        if (s->ckv_packed) WK_CHECK(b.dmalloc(&s->cross_hdr, (size_t)2 * L * S * H * packed_hdr_stride(T)));
    }
    WK_CHECK(b.alloc16(&s->self_k, (size_t)L * S * H * kKvMaxLen * 64));
    WK_CHECK(b.alloc16(&s->self_v, (size_t)L * S * H * kKvMaxLen * 64));
    // split-K partial workspace: max over the decoder GEMM shapes of splits * N
    size_t pe = 0;
    const int shapes[4][2] = {{3 * d, d}, {d, d}, {4 * d, d}, {d, 4 * d}};
    for (auto& sh : shapes) {
        const int sp = choose_splits((sh[0] + 127) / 128, sh[1] / 64, m->num_sms);
        pe = std::max(pe, (size_t)sp * sh[0]);
    }
    s->partial_elems = pe * bpm;
    WK_CHECK(b.dmalloc(&s->partial, s->partial_elems));
    WK_CHECK(b.dmalloc(&s->x, (size_t)bpm * d));
    WK_CHECK(b.alloc16(&s->xn, (size_t)bpm * d));
    WK_CHECK(b.alloc16(&s->attn, (size_t)bpm * d));
    WK_CHECK(b.alloc16(&s->ffn, (size_t)bpm * 4 * d));
    WK_CHECK(b.dmalloc(&s->logits, (size_t)S * c.vocab));
    WK_CHECK(b.dmalloc(&s->st.tokens, (size_t)S * kKvMaxLen));
    WK_CHECK(b.dmalloc(&s->st.n_tokens, S));
    WK_CHECK(b.dmalloc(&s->st.logprobs, (size_t)S * kKvMaxLen));
    WK_CHECK(b.dmalloc(&s->st.next_token, S));
    WK_CHECK(b.dmalloc(&s->st.done, S));
    WK_CHECK(b.dmalloc(&s->st.first_low, S));
    WK_CHECK(b.dmalloc(&s->st.steps, S));
    WK_CHECK(b.dmalloc(&s->st.input_ids, S));
    WK_CHECK(b.dmalloc(&s->st.error, S));
    WK_CHECK(b.dmalloc(&s->st.lang_token, S));
    WK_CHECK(b.dmalloc(&s->st.lang_logprob, S));
    WK_CHECK(b.dmalloc(&s->st.lang_state, S));
    WK_CHECK(b.dmalloc(&s->st.no_speech, S));
    WK_CHECK(b.dmalloc(&s->rp_dev, S));
    s->st.rp = s->rp_dev;
    WK_CHECK(b.dmalloc(&s->pos_dev, S));
    WK_CHECK(b.dmalloc(&s->lang_dev, 4096));
    s->suppress_cap = 4096;
    WK_CHECK(b.dmalloc(&s->suppress_dev, s->suppress_cap));
    WK_CHECK(b.dmalloc(&s->d_adm_slots, S));
    WK_CHECK(b.dmalloc(&s->d_adm_prompts, (size_t)S * kKvMaxLen));
    WK_CHECK(b.dmalloc(&s->d_adm_rp, S));
    WK_CHECK(b.pinned(&s->h_adm_slots, S));
    WK_CHECK(b.pinned(&s->h_adm_prompts, (size_t)S * kKvMaxLen));
    WK_CHECK(b.pinned(&s->h_adm_rp, S));
    WK_CHECK(b.pinned(&s->h_tokens, (size_t)S * kKvMaxLen));
    WK_CHECK(b.pinned(&s->h_logprobs, (size_t)S * kKvMaxLen));
    WK_CHECK(b.pinned(&s->h_n_tokens, S));
    WK_CHECK(b.pinned(&s->h_done, S));
    WK_CHECK(b.pinned(&s->h_first_low, S));
    WK_CHECK(b.pinned(&s->h_steps, S));
    WK_CHECK(b.pinned(&s->h_error, S));
    WK_CHECK(b.pinned(&s->h_lang_token, S));
    WK_CHECK(b.pinned(&s->h_lang_logprob, S));
    WK_CHECK(b.pinned(&s->h_no_speech, S));
    WK_CHECK(b.dmalloc(&s->st.bias_m, (size_t)S * kMaxBiasPhrases));
    WK_CHECK(b.dmalloc(&s->st.bias_acc, S));
    WK_CHECK(b.pinned(&s->h_bias_acc, S));
    WK_CUDA_CHECK(cudaEventCreateWithFlags(&s->ev_enc, cudaEventDisableTiming));
    WK_CUDA_CHECK(cudaEventCreateWithFlags(&s->ev_adm, cudaEventDisableTiming));
    WK_CUDA_CHECK(cudaEventCreateWithFlags(&s->ev_stage, cudaEventDisableTiming));
    for (auto& e : s->ev_t) WK_CUDA_CHECK(cudaEventCreate(&e));
    WK_CUDA_CHECK(cudaDeviceSynchronize());  // setup memsets ran on the legacy default stream
    WK_CUDA_CHECK(cudaEventRecord(s->ev_adm, s->stream));
    WK_CUDA_CHECK(cudaEventRecord(s->ev_stage, s->stream));
    *out = s.release();
    return WK_OK;
}

void wk_session_free(wk_session* s) {
    if (!s) return;
    cudaSetDevice(s->m->device);
    delete s;
}

wk_status wk_session_reset(wk_session* s) {
    if (!s) return WK_ERR_INVALID_ARGUMENT;
    WK_CUDA_CHECK(cudaSetDevice(s->m->device));
    const wk_model_config& c = s->m->cfg;
    const size_t n = (size_t)c.dec_layers * s->max_batch * c.n_heads * kKvMaxLen * 64 * 2;
    WK_CUDA_CHECK(cudaMemsetAsync(s->self_k, 0, n, s->stream));
    WK_CUDA_CHECK(cudaMemsetAsync(s->self_v, 0, n, s->stream));
    return WK_OK;
}

wk_status wk_bias_create(const int32_t* tokens, const int32_t* phrase_lens, int32_t n_phrases, float boost, int32_t special_token_begin, wk_bias** out) {
    if (!out || !phrase_lens || !tokens) { set_error("wk_bias_create: null argument"); return WK_ERR_INVALID_ARGUMENT; }
    *out = nullptr;
    if (n_phrases < 1 || n_phrases > kMaxBiasPhrases) { set_error("wk_bias_create: %d phrases outside [1, %d]", n_phrases, kMaxBiasPhrases); return WK_ERR_INVALID_ARGUMENT; }
    if (!(boost >= 0.f) || !isfinite(boost)) { set_error("wk_bias_create: boost %g is not a finite value >= 0", boost); return WK_ERR_INVALID_ARGUMENT; }
    if (special_token_begin < 1) { set_error("wk_bias_create: special_token_begin %d", special_token_begin); return WK_ERR_INVALID_ARGUMENT; }
    int total = 0;
    for (int p = 0; p < n_phrases; ++p) {
        if (phrase_lens[p] < 1 || phrase_lens[p] > kMaxBiasLen) { set_error("wk_bias_create: phrase %d has %d tokens (1..%d)", p, phrase_lens[p], kMaxBiasLen); return WK_ERR_INVALID_ARGUMENT; }
        total += phrase_lens[p];
        if (total > kMaxBiasTotal) { set_error("wk_bias_create: more than %d phrase tokens in all", kMaxBiasTotal); return WK_ERR_INVALID_ARGUMENT; }
    }
    for (int i = 0; i < total; ++i)
        if (tokens[i] < 0 || tokens[i] >= special_token_begin) {
            set_error("wk_bias_create: token %d is not a text token (ids below %d)", tokens[i], special_token_begin);
            return WK_ERR_INVALID_ARGUMENT;
        }
    std::unique_ptr<wk_bias> B(new wk_bias());
    B->n = n_phrases; B->len = total; B->boost = boost;
    B->rec.assign((size_t)n_phrases + 2 * total, 0);
    int32_t* tok = B->rec.data() + n_phrases;
    int32_t* fail = tok + total;
    for (int p = 0, start = 0; p < n_phrases; start += phrase_lens[p], ++p) {
        const int L = phrase_lens[p];
        B->rec[p] = start | L << 16;
        memcpy(tok + start, tokens + start, (size_t)L * 4);
        // KMP failure links: fail[k - 1] = the longest proper border of w[0..k)
        const int32_t* w = tokens + start;
        int32_t* f = fail + start;
        f[0] = 0;
        for (int k = 1, b = 0; k < L; ++k) {
            while (b > 0 && w[k] != w[b]) b = f[b - 1];
            if (w[k] == w[b]) ++b;
            f[k] = b;
        }
    }
    *out = B.release();
    return WK_OK;
}

void wk_bias_free(wk_bias* b) { delete b; }

wk_status wk_session_set_bias(wk_session* s, const wk_bias* const* sets, int64_t n_sets) {
    if (!s || n_sets < 0 || (n_sets > 0 && !sets)) { set_error("wk_session_set_bias: bad arguments"); return WK_ERR_INVALID_ARGUMENT; }
    std::vector<wk_session::BiasSlot> slots((size_t)n_sets);
    std::vector<int32_t> pool;
    for (int64_t i = 0; i < n_sets; ++i) {
        const wk_bias* b = sets[i];
        if (!b) continue;                                 // a window without bias
        int64_t same = -1;                                // a set passed again shares its record
        for (int64_t j = 0; j < i && same < 0; ++j) if (sets[j] == b) same = j;
        if (same >= 0) { slots[i] = slots[same]; continue; }
        slots[i].off = (int)pool.size(); slots[i].n = b->n; slots[i].len = b->len; slots[i].boost = b->boost;
        pool.insert(pool.end(), b->rec.begin(), b->rec.end());
    }
    WK_CUDA_CHECK(cudaSetDevice(s->m->device));
    if (pool.size() > s->bias_cap) {
        const size_t cap = std::max<size_t>(4096, pool.size());
        WK_CHECK(s->mem.grow(&s->bias_pool, cap, s->stream));   // a new pointer makes the next step capture its graph again
        s->bias_cap = cap;
    }
    if (!pool.empty()) {
        WK_CUDA_CHECK(cudaMemcpyAsync(s->bias_pool, pool.data(), pool.size() * 4, cudaMemcpyHostToDevice, s->stream));
        WK_CUDA_CHECK(cudaStreamSynchronize(s->stream));   // the host record is pageable
    }
    s->bias_sets = std::move(slots);
    s->bias_map.clear();
    return WK_OK;
}

wk_status wk_session_set_top_logprobs(wk_session* s, int32_t k) {
    if (!s || k < 0 || k > kMaxTopLogprobs) { set_error("wk_session_set_top_logprobs: k %d outside [0, %d]", k, kMaxTopLogprobs); return WK_ERR_INVALID_ARGUMENT; }
    s->top_k = k;
    return WK_OK;
}

wk_status wk_session_top_logprobs(const wk_session* s, int32_t window, int32_t n, int32_t* tokens, float* logprobs) {
    if (!s || window < 0 || (size_t)window >= s->win_top_tok.size() || n < 0 || (n > 0 && s->top_store_k > 0 && (!tokens || !logprobs))) {
        set_error("wk_session_top_logprobs: window %d / %d tokens outside the last call's %zu windows", window, n, s ? s->win_top_tok.size() : (size_t)0);
        return WK_ERR_INVALID_ARGUMENT;
    }
    const size_t want = (size_t)n * s->top_store_k;
    const std::vector<int32_t>& tt = s->win_top_tok[window];
    const std::vector<float>& tl = s->win_top_lp[window];
    for (size_t i = 0; i < want; ++i) {
        tokens[i] = i < tt.size() ? tt[i] : -1;
        logprobs[i] = i < tl.size() ? tl[i] : -INFINITY;
    }
    return WK_OK;
}

wk_status wk_session_set_encoder_output(wk_session* s, const wk_tensor* enc) {
    if (!s || !enc) { set_error("wk_session_set_encoder_output: null argument"); return WK_ERR_INVALID_ARGUMENT; }
    wk_model* m = s->m;
    if (enc->kind != 1 || enc->owner != m) { set_error("encoder output does not belong to this model"); return WK_ERR_INVALID_ARGUMENT; }
    if (enc->batch < 1 || enc->batch > s->max_batch) { set_error("encoder batch %lld exceeds session max_batch %d", (long long)enc->batch, s->max_batch); return WK_ERR_PREPARE_DECODER_INPUTS; }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    s->batch = (int)enc->batch;
    s->bound_windows = s->batch;
    s->bs.beam = 1; s->bs.group = 1;
    s->bp = round_up(s->batch, 16);
    // the encoder ran on the model stream; the projection reads its output on the session stream and the tensor remembers the reader
    std::lock_guard<std::mutex> lock(m->api_mu);
    for (cudaEvent_t e : enc->events) WK_CUDA_CHECK(cudaStreamWaitEvent(s->stream, e, 0));
    WK_CHECK(gemm_wgmma(cross_kv_gemm(s, enc->data, s->batch, 0), m->num_sms, s->stream));
    // a model with a draft decoder binds the draft's cross K/V too (wk_decode_text_draft), when the windows fit a draft call: the session
    // does not keep the encoder output, so binding is the one time it can be projected
    if (m->draft && s->batch <= draft_slots(s)) {
        WK_CHECK(ensure_draft(s));
        WK_CHECK(gemm_wgmma(cross_kv_gemm(s, enc->data, s->batch, 0, true), m->num_sms, s->stream));
    }
    cudaEvent_t ev;
    WK_CUDA_CHECK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    WK_CUDA_CHECK(cudaEventRecord(ev, s->stream));
    const_cast<wk_tensor*>(enc)->events.push_back(ev);
    return WK_OK;
}

wk_status wk_build_prompt(const wk_model* m, const wk_special_tokens* st, const wk_decode_opts* o, int32_t use_options, int32_t* out, int32_t cap, int32_t* n) {
    if (!m || !st || !out || !n) return WK_ERR_INVALID_ARGUMENT;
    std::vector<int32_t> p;
    build_prompt(m, st, o, use_options, p);
    if ((int)p.size() > cap) { set_error("wk_build_prompt: capacity %d < %zu", cap, p.size()); return WK_ERR_PREPARE_DECODER_INPUTS; }
    memcpy(out, p.data(), p.size() * 4);
    *n = (int)p.size();
    return WK_OK;
}

wk_status wk_decode_step(wk_session* s, const int32_t* input_ids, const int32_t* cache_length, float* logits_out) {
    if (!s || !input_ids || !cache_length) { set_error("wk_decode_step: null argument"); return WK_ERR_INVALID_ARGUMENT; }
    wk_model* m = s->m;
    if (s->batch < 1) { set_error("wk_decode_step: no encoder output bound"); return WK_ERR_PREPARE_DECODER_INPUTS; }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    for (int i = 0; i < s->batch; ++i) {
        if (cache_length[i] < 0 || cache_length[i] >= kKvMaxLen) { set_error("wk_decode_step: cache_length[%d]=%d out of range", i, cache_length[i]); return WK_ERR_DECODING_LOGITS_FAILED; }
        if (input_ids[i] < 0 || input_ids[i] >= m->cfg.vocab) { set_error("wk_decode_step: input_ids[%d]=%d out of range", i, input_ids[i]); return WK_ERR_DECODING_LOGITS_FAILED; }
    }
    WK_CUDA_CHECK(cudaMemcpyAsync(s->st.input_ids, input_ids, s->batch * 4, cudaMemcpyHostToDevice, s->stream));
    WK_CUDA_CHECK(cudaMemcpyAsync(s->pos_dev, cache_length, s->batch * 4, cudaMemcpyHostToDevice, s->stream));
    WK_CHECK(decoder_forward(s, 0, s->pos_dev));
    if (logits_out)
        WK_CUDA_CHECK(cudaMemcpyAsync(logits_out, s->logits, (size_t)s->batch * m->cfg.vocab * 4, cudaMemcpyDeviceToHost, s->stream));
    cudaError_t e = cudaStreamSynchronize(s->stream);
    if (e != cudaSuccess) { set_error("wk_decode_step: %s", cudaGetErrorString(e)); return WK_ERR_DECODING_LOGITS_FAILED; }
    return WK_OK;
}

wk_status wk_session_last_logits(wk_session* s, float* logits_out) {
    if (!s || !logits_out) return WK_ERR_INVALID_ARGUMENT;
    WK_CUDA_CHECK(cudaSetDevice(s->m->device));
    WK_CUDA_CHECK(cudaMemcpyAsync(logits_out, s->logits, (size_t)s->batch * s->m->cfg.vocab * 4, cudaMemcpyDeviceToHost, s->stream));
    WK_CUDA_CHECK(cudaStreamSynchronize(s->stream));
    return WK_OK;
}

// TextDecoder.detectLanguage (TextDecoder.swift:420-539): one decoder step on [SOT] at position 0, LanguageLogitsFilter
// (keep only the language tokens), GreedyTokenSampler -> language token id + logprob for every bound window.
wk_status wk_detect_language(wk_session* s, const wk_special_tokens* st, const int32_t* language_tokens, int32_t n_language_tokens,
                             float temperature, int32_t* token_out, float* logprob_out) {
    if (!s || !st || !language_tokens || n_language_tokens < 1 || n_language_tokens > 4096 || !token_out) {
        set_error("wk_detect_language: bad arguments");
        return WK_ERR_INVALID_ARGUMENT;
    }
    wk_model* m = s->m;
    if (s->batch < 1) { set_error("wk_detect_language: no encoder output bound"); return WK_ERR_PREPARE_DECODER_INPUTS; }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    const int B = s->batch;
    std::vector<int32_t> ids(B, st->start_of_transcript_token), zeros(B, 0), ones(B, 1);
    WK_CUDA_CHECK(cudaMemcpyAsync(s->st.input_ids, ids.data(), B * 4, cudaMemcpyHostToDevice, s->stream));
    WK_CUDA_CHECK(cudaMemcpyAsync(s->pos_dev, zeros.data(), B * 4, cudaMemcpyHostToDevice, s->stream));
    WK_CHECK(decoder_forward(s, 0, s->pos_dev));
    // currentTokens = [SOT] for every window: reuse the decode-state arrays as the stateless token history
    WK_CUDA_CHECK(cudaMemcpyAsync(s->st.tokens, ids.data(), B * 4, cudaMemcpyHostToDevice, s->stream));   // ld_tokens = 1
    WK_CUDA_CHECK(cudaMemcpyAsync(s->st.n_tokens, ones.data(), B * 4, cudaMemcpyHostToDevice, s->stream));
    WK_CUDA_CHECK(cudaMemcpyAsync(s->lang_dev, language_tokens, n_language_tokens * 4, cudaMemcpyHostToDevice, s->stream));
    SamplerParams p;
    memset(&p, 0, sizeof(p));
    p.st = *st; p.vocab = m->cfg.vocab; p.is_multilingual = 1; p.loop_mode = 0;
    p.sample_begin_ts = -1; p.sample_begin_blank = -1;
    p.language_tokens = s->lang_dev; p.n_language_tokens = n_language_tokens; p.language_sample_begin = 0;
    p.temperature = temperature; p.top_k = 5; p.seed = 0;
    p.max_ctx = kKvMaxLen;
    DecodeState none;
    memset(&none, 0, sizeof(none));
    WK_CHECK(sampler_filter_sample(s->logits, m->cfg.vocab, p, none, s->st.tokens, 1, s->st.n_tokens, s->st.next_token, s->st.logprobs, nullptr, B, s->stream));
    WK_CUDA_CHECK(cudaMemcpyAsync(token_out, s->st.next_token, B * 4, cudaMemcpyDeviceToHost, s->stream));
    if (logprob_out) WK_CUDA_CHECK(cudaMemcpyAsync(logprob_out, s->st.logprobs, B * 4, cudaMemcpyDeviceToHost, s->stream));
    cudaError_t e = cudaStreamSynchronize(s->stream);
    if (e != cudaSuccess) { set_error("wk_detect_language: %s", cudaGetErrorString(e)); return WK_ERR_DECODING_FAILED; }
    return WK_OK;
}

wk_status wk_decode_text_ex(wk_session* s, const wk_special_tokens* st, const wk_batch_opts* bo, wk_decode_result* results) {
    return wk_decode_text_draft(s, st, bo, 0, results);
}

wk_status wk_decode_text_draft(wk_session* s, const wk_special_tokens* st, const wk_batch_opts* bo, int32_t draft_tokens, wk_decode_result* results) {
    if (!s || !st || !bo || !bo->opts || bo->n_opts < 1 || !results) { set_error("wk_decode_text: null argument"); return WK_ERR_INVALID_ARGUMENT; }
    if (s->bound_windows < 1) { set_error("wk_decode_text: no encoder output bound"); return WK_ERR_PREPARE_DECODER_INPUTS; }
    if (bo->n_opts != 1 && bo->n_opts != s->bound_windows) { set_error("wk_decode_text: %d option sets for %d windows", bo->n_opts, s->bound_windows); return WK_ERR_INVALID_ARGUMENT; }
    WK_CUDA_CHECK(cudaSetDevice(s->m->device));
    CoreArgs a{nullptr, s->bound_windows, 0, nullptr, st, bo, results, false, nullptr, draft_tokens};
    return transcribe_core(s, a);
}

wk_status wk_decode_text(wk_session* s, const wk_special_tokens* st, const wk_decode_opts* o, const int32_t* prompt, int32_t n_prompt,
                         wk_decode_result* results) {
    if (!s || !st || !o || !prompt || !results) { set_error("wk_decode_text: null argument"); return WK_ERR_INVALID_ARGUMENT; }
    wk_batch_opts bo;
    memset(&bo, 0, sizeof(bo));
    bo.opts = o; bo.n_opts = 1; bo.prompt = prompt; bo.n_prompt = n_prompt;
    return wk_decode_text_ex(s, st, &bo, results);
}

wk_status wk_transcribe_windows_ex(wk_model* m, wk_session* s, const float* pcm_host, int64_t n_windows, int64_t stride,
                                   const int32_t* samples_per_window, const wk_special_tokens* st, const wk_batch_opts* bo,
                                   wk_decode_result* results) {
    return wk::transcribe_windows_stop(m, s, pcm_host, n_windows, stride, samples_per_window, st, bo, results, nullptr);
}

wk_status wk_transcribe_windows_draft(wk_model* m, wk_session* s, const float* pcm_host, int64_t n_windows, int64_t stride,
                                      const int32_t* samples_per_window, const wk_special_tokens* st, const wk_batch_opts* bo,
                                      int32_t draft_tokens, wk_decode_result* results) {
    return wk::transcribe_windows_stop(m, s, pcm_host, n_windows, stride, samples_per_window, st, bo, results, nullptr, draft_tokens);
}

}  // extern "C"

wk_status wk::transcribe_windows_stop(wk_model* m, wk_session* s, const float* pcm_host, int64_t n_windows, int64_t stride,
                                      const int32_t* samples_per_window, const wk_special_tokens* st, const wk_batch_opts* bo,
                                      wk_decode_result* results, const StopRule* stop, int draft) {
    if (!m || !s || !pcm_host || !st || !bo || !bo->opts || bo->n_opts < 1 || !results || n_windows < 1) { set_error("wk_transcribe_windows: null argument"); return WK_ERR_INVALID_ARGUMENT; }
    if (s->m != m) { set_error("wk_transcribe_windows: session belongs to another model"); return WK_ERR_INVALID_ARGUMENT; }
    if (bo->n_opts != 1 && bo->n_opts != n_windows) { set_error("wk_transcribe_windows: %d option sets for %lld windows", bo->n_opts, (long long)n_windows); return WK_ERR_INVALID_ARGUMENT; }
    if (bo->prompts && !bo->prompt_lens) { set_error("wk_transcribe_windows: prompts without prompt_lens"); return WK_ERR_INVALID_ARGUMENT; }
    if (!m->finalized) { set_error("wk_transcribe_windows: model weights not finalized"); return WK_ERR_MODELS_UNAVAILABLE; }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    CoreArgs a{pcm_host, n_windows, stride, samples_per_window, st, bo, results, true, stop, draft};
    return transcribe_core(s, a);
}

extern "C" {

wk_status wk_transcribe_windows(wk_model* m, wk_session* s, const float* pcm_host, int64_t n_windows, int64_t stride,
                                const int32_t* samples_per_window, const wk_special_tokens* st, const wk_decode_opts* opts,
                                const int32_t* prompt, int32_t n_prompt, wk_decode_result* results) {
    if (!opts || !prompt) { set_error("wk_transcribe_windows: null argument"); return WK_ERR_INVALID_ARGUMENT; }
    wk_batch_opts bo;
    memset(&bo, 0, sizeof(bo));
    bo.opts = opts; bo.n_opts = 1; bo.prompt = prompt; bo.n_prompt = n_prompt;
    return wk_transcribe_windows_ex(m, s, pcm_host, n_windows, stride, samples_per_window, st, &bo, results);
}

wk_status wk_session_stats(const wk_session* s, int64_t* out4) {
    if (!s || !out4) return WK_ERR_INVALID_ARGUMENT;
    memcpy(out4, s->stats, sizeof(s->stats));
    return WK_OK;
}

wk_status wk_session_draft_stats(const wk_session* s, int64_t* out3) {
    if (!s || !out3) return WK_ERR_INVALID_ARGUMENT;
    memcpy(out3, s->draft_stats, sizeof(s->draft_stats));
    return WK_OK;
}

wk_status wk_session_languages(const wk_session* s, int32_t first, int32_t n, int32_t* tokens, float* logprobs) {
    if (!s || first < 0 || n < 0 || (int64_t)first + n > (int64_t)s->win_lang.size()) {
        set_error("wk_session_languages: windows [%d, %d) outside the last call's %zu", first, first + n, s ? s->win_lang.size() : (size_t)0);
        return WK_ERR_INVALID_ARGUMENT;
    }
    if (tokens && n > 0) memcpy(tokens, s->win_lang.data() + first, (size_t)n * 4);
    if (logprobs && n > 0) memcpy(logprobs, s->win_lang_logprob.data() + first, (size_t)n * 4);
    return WK_OK;
}

wk_status wk_session_no_speech_probs(const wk_session* s, int32_t first, int32_t n, float* out) {
    if (!s || !out || first < 0 || n < 0 || (int64_t)first + n > (int64_t)s->win_no_speech.size()) {
        set_error("wk_session_no_speech_probs: windows [%d, %d) outside the last call's %zu", first, first + n, s ? s->win_no_speech.size() : (size_t)0);
        return WK_ERR_INVALID_ARGUMENT;
    }
    if (n > 0) memcpy(out, s->win_no_speech.data() + first, (size_t)n * 4);
    return WK_OK;
}

wk_status wk_session_alignment_weights(wk_session* s, int32_t window, int32_t rows, float* out) {
    if (!s || !out || window < 0 || rows < 0 || rows > s->align_store_rows) { set_error("wk_session_alignment_weights: bad arguments"); return WK_ERR_INVALID_ARGUMENT; }
    if (!s->align_on || !s->align_store || window >= s->align_store_n) { set_error("wk_session_alignment_weights: the last decode did not ask for word timestamps (or window %d is outside it)", window); return WK_ERR_INVALID_ARGUMENT; }
    WK_CUDA_CHECK(cudaSetDevice(s->m->device));
    const size_t T = s->m->cfg.n_audio_ctx;
    std::vector<__half> h((size_t)rows * T);
    WK_CUDA_CHECK(cudaMemcpyAsync(h.data(), (const __half*)s->align_store + (size_t)window * s->align_store_rows * T, h.size() * 2, cudaMemcpyDeviceToHost, s->stream));
    WK_CUDA_CHECK(cudaStreamSynchronize(s->stream));
    for (size_t i = 0; i < h.size(); ++i) out[i] = __half2float(h[i]);
    return WK_OK;
}

wk_status wk_session_alignment_weights_f16(wk_session* s, int32_t window, int32_t rows, uint16_t* out, int32_t sync) {
    if (!s || !out || window < 0 || rows < 0 || rows > s->align_store_rows) { set_error("wk_session_alignment_weights_f16: bad arguments"); return WK_ERR_INVALID_ARGUMENT; }
    if (!s->align_on || !s->align_store || window >= s->align_store_n) { set_error("wk_session_alignment_weights_f16: the last decode did not ask for word timestamps (or window %d is outside it)", window); return WK_ERR_INVALID_ARGUMENT; }
    WK_CUDA_CHECK(cudaSetDevice(s->m->device));
    const size_t T = s->m->cfg.n_audio_ctx;
    if (rows > 0)
        WK_CUDA_CHECK(cudaMemcpyAsync(out, (const __half*)s->align_store + (size_t)window * s->align_store_rows * T, (size_t)rows * T * 2, cudaMemcpyDeviceToHost, s->stream));
    if (sync) WK_CUDA_CHECK(cudaStreamSynchronize(s->stream));
    return WK_OK;
}

wk_status wk_align_tokens(wk_session* s, const wk_special_tokens* st, const int32_t* tokens, const int32_t* offsets, int64_t n_windows, int32_t* status) {
    if (!s || !st || !tokens || !offsets || n_windows < 1) { set_error("wk_align_tokens: null argument"); return WK_ERR_INVALID_ARGUMENT; }
    if (s->bound_windows < 1) { set_error("wk_align_tokens: no encoder output bound"); return WK_ERR_PREPARE_DECODER_INPUTS; }
    if (n_windows > s->bound_windows) {
        set_error("wk_align_tokens: %lld token sequences for %d bound windows", (long long)n_windows, s->bound_windows);
        return WK_ERR_INVALID_ARGUMENT;
    }
    WK_CUDA_CHECK(cudaSetDevice(s->m->device));
    return align_core(s, st, nullptr, n_windows, 0, nullptr, tokens, offsets, status);
}

wk_status wk_align_windows(wk_model* m, wk_session* s, const float* pcm_host, int64_t n_windows, int64_t stride, const int32_t* samples_per_window,
                           const wk_special_tokens* st, const int32_t* tokens, const int32_t* offsets, int32_t* status) {
    if (!m || !s || !pcm_host || !st || !tokens || !offsets || n_windows < 1) { set_error("wk_align_windows: null argument"); return WK_ERR_INVALID_ARGUMENT; }
    if (s->m != m) { set_error("wk_align_windows: session belongs to another model"); return WK_ERR_INVALID_ARGUMENT; }
    if (!m->finalized) { set_error("wk_align_windows: model weights not finalized"); return WK_ERR_MODELS_UNAVAILABLE; }
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    return align_core(s, st, pcm_host, n_windows, stride, samples_per_window, tokens, offsets, status);
}

wk_status wk_session_aligned_logprobs(const wk_session* s, int32_t window, int32_t n, float* out) {
    if (!s || !out || window < 0 || n < 0 || n > kKvMaxLen || (int64_t)(window + 1) * kKvMaxLen > (int64_t)s->win_align_lp.size()) {
        set_error("wk_session_aligned_logprobs: window %d / %d tokens outside the last align call", window, n);
        return WK_ERR_INVALID_ARGUMENT;
    }
    if (n > 0) memcpy(out, s->win_align_lp.data() + (size_t)window * kKvMaxLen, (size_t)n * 4);
    return WK_OK;
}

// Average device time (ms) of one launch of a named hot kernel on the session's buffers (CUDA events on the stream the kernel runs on;
// decoder-side kernels are replayed `iters` times as one CUDA graph so that host launch cost stays out, as in the real step):
//   0 decoder cross-attention (one layer, `batch` live rows)      1 encoder FC1+GELU GEMM (M = batch*1500)   2 log-mel
//   3 encoder attention      4 decoder QKV swap-AB GEMM      5 encoder QKV GEMM      6/7 decoder d x d / FC2 GEMM (L2-warm weights)
//   8 split-K reduce + LN    9 decoder self-attention at position 100      10 sampler (V-long rows)
//   14-17 decoder GEMMs with the weights rotating over the layers (HBM-cold: d x d, FC1, FC2, QKV)
// Also returns the algorithmic bytes (HBM-bound kernels) or FLOPs (tensor-bound) of one launch.
wk_status wk_bench_kernel(wk_model* m, wk_session* s, int32_t which, int32_t batch, int32_t iters, float* ms_out, double* work_out) {
    if (!m || !s || s->m != m || !ms_out || !work_out || iters < 1) return WK_ERR_INVALID_ARGUMENT;
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    const wk_model_config& c = m->cfg;
    const int d = c.d_model, T = c.n_audio_ctx, H = c.n_heads, dt = c.dtype;
    const bool enc_side = which == 1 || which == 2 || which == 3 || which == 5;
    int B = batch;
    if (B < 1 || B > (enc_side ? c.max_batch : s->max_batch)) { set_error("wk_bench_kernel: bad batch"); return WK_ERR_INVALID_ARGUMENT; }
    if (enc_side) WK_CHECK(enc_ws_ensure(m, &s->ws, c.max_batch));
    const int64_t M = (int64_t)B * T;
    cudaStream_t st = enc_side ? s->enc_stream : s->stream;
    const int saved_batch = s->batch, saved_bp = s->bp;
    if (!enc_side) { s->batch = B; s->bp = round_up(B, 16); }
    const size_t cross_rows = (size_t)s->max_batch * H * T;
    const size_t cross_block = cross_rows * 64 * ckv_esize(s);
    const float* ksc = s->ckv_fp8 ? s->cross_scale : nullptr;
    const float* vsc = s->ckv_fp8 ? s->cross_scale + cross_rows : nullptr;
    const size_t hs = packed_hdr_stride(T);
    const uint8_t* kh = s->ckv_packed ? s->cross_hdr : nullptr;
    const uint8_t* vh = s->ckv_packed ? s->cross_hdr + (size_t)s->max_batch * H * hs : nullptr;
    if (which == 9 && !s->pos100) {
        std::vector<int32_t> h(256, 100);
        WK_CHECK(s->mem.dmalloc(&s->pos100, 256, false));
        WK_CUDA_CHECK(cudaMemcpy(s->pos100, h.data(), 256 * 4, cudaMemcpyHostToDevice));
    }
    int rot = 0;
    auto run = [&]() -> wk_status {
        int sp;
        switch (which) {
            case 0: return decoder_cross_attention(s->partial, 1, s->bp, m->dec[0].bcq, s->cross_kv, (char*)s->cross_kv + cross_block, s->attn, B, H, T, dt, st,
                                                   nullptr, nullptr, 0, 1, ksc, vsc, false, kh, vh);
            case 1: return gemm_wgmma(plain_gemm(s->ws.xn, M, d, m->enc[0].w1, 4 * d, dt, GEMM_OUT_T16, s->ws.ffn, 4 * d, m->enc[0].b1, 1), m->num_sms, st);
            case 2: return mel_forward(&m->mel_tables, s->ws.pcm_dev, B, kWindowSamples, nullptr, s->ws.mel, s->ws.gmax, st);
            case 3: return encoder_attention(s->ws.qkv, s->ws.attn, B, T, H, dt, st);
            case 4: return dec_gemm(s, m->dec[0].wqkv, 3 * d, d, s->xn, &sp);
            case 5: return gemm_wgmma(plain_gemm(s->ws.xn, M, d, m->enc[0].wqkv, 3 * d, dt, GEMM_OUT_T16, s->ws.qkv, 3 * d, m->enc[0].bqkv, 0), m->num_sms, st);
            case 6: return dec_gemm(s, m->dec[0].wo, d, d, s->attn, &sp);
            case 7: return dec_gemm(s, m->dec[0].w2, d, 4 * d, s->ffn, &sp);
            case 8: return decoder_reduce_resid_ln(s->partial, choose_splits((d + 127) / 128, d / 64, m->num_sms), s->bp, m->dec[0].bo, m->dec[0].lnx.g, m->dec[0].lnx.b, s->x, s->xn, B, d, dt, st);
            case 9: return decoder_self_attention(s->partial, 1, s->bp, m->dec[0].bq, m->dec[0].bv, s->self_k, s->self_v, s->pos100, nullptr, s->attn, B, H, kKvMaxLen, dt, st);
            case 14: case 15: case 16: case 17: {
                const int r = rot++;
                const DecLayer& l = m->dec[r % c.dec_layers];
                if (which == 14) { const void* w3[3] = {l.wo, l.wcq, l.wco}; return dec_gemm(s, w3[(r / c.dec_layers) % 3], d, d, s->attn, &sp); }
                if (which == 15) return dec_gemm(s, l.w1, 4 * d, d, s->xn, &sp);
                if (which == 16) return dec_gemm(s, l.w2, d, 4 * d, s->ffn, &sp);
                return dec_gemm(s, l.wqkv, 3 * d, d, s->xn, &sp);
            }
            default: set_error("wk_bench_kernel: unknown kernel %d", which); return WK_ERR_INVALID_ARGUMENT;
        }
    };
    switch (which) {
        case 0:   // K + V bytes (+ FP8 row scales; packed: primary slots, header vectors and the secondary slots of raw rows)
            *work_out = (double)B * H * T * (64 * (double)ckv_esize(s) + (s->ckv_fp8 ? 4 : 0)) * 2;
            if (s->ckv_packed) {
                std::vector<uint8_t> hk((size_t)B * H * hs), hv(hk.size());
                WK_CUDA_CHECK(cudaMemcpy(hk.data(), kh, hk.size(), cudaMemcpyDeviceToHost));
                WK_CUDA_CHECK(cudaMemcpy(hv.data(), vh, hv.size(), cudaMemcpyDeviceToHost));
                size_t raw = 0;
                for (size_t blk = 0; blk < (size_t)B * H; ++blk)
                    for (int t = 0; t < T; ++t) raw += (hk[blk * hs + t] == kPackedRaw) + (hv[blk * hs + t] == kPackedRaw);
                *work_out = (double)B * H * (T * (double)kPackedRowBytes + hs) * 2 + 32.0 * raw;
            }
            break;
        case 1: *work_out = 2.0 * (double)M * d * 4 * d; break;                            // FLOPs
        case 2: *work_out = (double)B * (kWindowSamples * 4.0 + c.n_mels * 3000 * 2.0); break;  // bytes (SURVEY 8d)
        case 3: *work_out = 4.0 * (double)B * H * T * T * 64; break;                       // FLOPs
        case 4: case 17: *work_out = 3.0 * d * d * 2; break;                               // weight bytes
        case 5: *work_out = 2.0 * (double)M * d * 3 * d; break;
        case 6: case 14: *work_out = 1.0 * d * d * 2; break;
        case 7: case 15: case 16: *work_out = 4.0 * d * d * 2; break;
        case 9: *work_out = (double)B * H * 100 * 64 * 2 * 2; break;                       // K + V rows read at position 100
        default: *work_out = 0; break;
    }
    wk_status rs = WK_OK;
    for (int i = 0; i < 2 && rs == WK_OK; ++i) rs = run();
    float t = 0.f;
    if (rs == WK_OK && !enc_side) {
        cudaGraph_t graph = nullptr;
        cudaGraphExec_t exec = nullptr;
        WK_CUDA_CHECK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
        for (int i = 0; i < iters && rs == WK_OK; ++i) rs = run();
        WK_CUDA_CHECK(cudaStreamEndCapture(st, &graph));
        if (rs == WK_OK) {
            WK_CUDA_CHECK(cudaGraphInstantiate(&exec, graph, 0));
            WK_CUDA_CHECK(cudaGraphLaunch(exec, st));
            WK_CUDA_CHECK(cudaEventRecord(s->ev_t[8], st));
            WK_CUDA_CHECK(cudaGraphLaunch(exec, st));
            WK_CUDA_CHECK(cudaEventRecord(s->ev_t[9], st));
            WK_CUDA_CHECK(cudaEventSynchronize(s->ev_t[9]));
            cudaEventElapsedTime(&t, s->ev_t[8], s->ev_t[9]);
            cudaGraphExecDestroy(exec);
        }
        if (graph) cudaGraphDestroy(graph);
    } else if (rs == WK_OK) {
        WK_CUDA_CHECK(cudaEventRecord(s->ev_t[8], st));
        for (int i = 0; i < iters && rs == WK_OK; ++i) rs = run();
        WK_CUDA_CHECK(cudaEventRecord(s->ev_t[9], st));
        WK_CUDA_CHECK(cudaEventSynchronize(s->ev_t[9]));
        cudaEventElapsedTime(&t, s->ev_t[8], s->ev_t[9]);
    }
    s->batch = saved_batch; s->bp = saved_bp;
    *ms_out = t / iters;
    return rs;
}

// Debug readback of an internal buffer as f32 (tests/tools only).  which: session encoder workspace 0 mel[Bm,3002,128] 1 h1[Bm,3002,d]
// 2 x[M,d] 3 xn[M,d] 4 qkv[M,3d] 5 attn[M,d] 6 ffn[M,4d] 7 enc_out[M,d]; decode 10 x[Bp,d] 11 xn[Bp,d] 12 attn[Bp,d]
// 13 ffn[Bp,4d] 14 logits[S,V] 15 cross_kv (all; an FP8 cache is returned dequantized, code * row scale) 16 self_k (all) 17 self_v (all)
// 18 partial; 20.. weights
wk_status wk_debug_read(wk_model* m, wk_session* s, int32_t which, int64_t offset_elems, float* dst, int64_t n) {
    if (!m || !dst) return WK_ERR_INVALID_ARGUMENT;
    WK_CUDA_CHECK(cudaSetDevice(m->device));
    const EncWorkspace* ws = s ? &s->ws : &m->ws;
    const void* src = nullptr;
    int dt = m->cfg.dtype;
    switch (which) {
        case 0: src = ws->mel; dt = WK_DTYPE_F16; break;
        case 1: src = ws->h1; dt = WK_DTYPE_F16; break;
        case 2: src = ws->x; dt = WK_DTYPE_F32; break;
        case 3: src = ws->xn; break;
        case 4: src = ws->qkv; break;
        case 5: src = ws->attn; break;
        case 6: src = ws->ffn; break;
        case 7: src = ws->enc_out; break;
        case 10: src = s ? s->x : nullptr; dt = WK_DTYPE_F32; break;
        case 11: src = s ? s->xn : nullptr; break;
        case 12: src = s ? s->attn : nullptr; break;
        case 13: src = s ? s->ffn : nullptr; break;
        case 14: src = s ? s->logits : nullptr; dt = WK_DTYPE_F32; break;
        case 15: src = s ? s->cross_kv : nullptr; break;
        case 16: src = s ? s->self_k : nullptr; break;
        case 17: src = s ? s->self_v : nullptr; break;
        case 18: src = s ? s->partial : nullptr; dt = WK_DTYPE_F32; break;
        case 20: src = m->enc[0].wqkv; break;
        case 21: src = m->emb; break;
        case 22: src = m->enc[0].w1; break;
        case 23: src = m->wckv; break;
        case 24: src = m->enc[0].b1; dt = WK_DTYPE_F32; break;
        case 25: src = m->enc[0].bqkv; dt = WK_DTYPE_F32; break;
        default: break;
    }
    if (!src) { set_error("wk_debug_read: unknown or unallocated buffer %d", which); return WK_ERR_INVALID_ARGUMENT; }
    std::lock_guard<std::mutex> lock(m->api_mu);
    if (which == 15 && s->ckv_fp8) {   // codes [offset, offset + n) and the scales of their rows, dequantized here
        if (n < 1) return WK_OK;
        const int64_t r0 = offset_elems / 64, r1 = (offset_elems + n - 1) / 64;
        std::vector<uint8_t> codes(n);
        std::vector<float> sc(r1 - r0 + 1);
        WK_CUDA_CHECK(cudaDeviceSynchronize());
        WK_CUDA_CHECK(cudaMemcpy(codes.data(), (const uint8_t*)s->cross_kv + offset_elems, n, cudaMemcpyDeviceToHost));
        WK_CUDA_CHECK(cudaMemcpy(sc.data(), s->cross_scale + r0, sc.size() * 4, cudaMemcpyDeviceToHost));
        for (int64_t i = 0; i < n; ++i) dst[i] = fp8_decode(codes[i]) * sc[(offset_elems + i) / 64 - r0];
        return WK_OK;
    }
    Buffers scratch;
    float* tmp = nullptr;
    WK_CHECK(scratch.dmalloc(&tmp, n, false));
    WK_CUDA_CHECK(cudaDeviceSynchronize());
    if (which == 15 && s->ckv_packed && n > 0) {   // the packed blocks holding [offset, offset + n), unpacked here
        const int T = m->cfg.n_audio_ctx;
        const int64_t b0 = offset_elems / ((int64_t)T * 64), b1 = (offset_elems + n - 1) / ((int64_t)T * 64);
        void* raw = nullptr;
        WK_CHECK(scratch.alloc16(&raw, (size_t)(b1 - b0 + 1) * T * 64));
        WK_CHECK(cross_kv_unpack((const char*)s->cross_kv + b0 * T * 128, s->cross_hdr + b0 * packed_hdr_stride(T), raw, b1 - b0 + 1, T, m->stream));
        src = (const char*)raw - b0 * T * 128;
    }
    wk_status r = convert_to_16((const char*)src + offset_elems * esize(dt), dt, tmp, WK_DTYPE_F32, n, m->stream);
    if (r == WK_OK) {
        cudaError_t e = cudaMemcpyAsync(dst, tmp, n * 4, cudaMemcpyDeviceToHost, m->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(m->stream);
        if (e != cudaSuccess) { set_error("wk_debug_read: %s", cudaGetErrorString(e)); r = WK_ERR_CUDA; }
    }
    return r;
}

}  // extern "C"
