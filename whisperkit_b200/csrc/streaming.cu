// Live transcription of many audio streams at once: AudioStreamTranscriber (Sources/WhisperKit/Core/Audio/AudioStreamTranscriber.swift)
// for N caller-fed streams, in host C++ like longform.cu.  A round takes every stream whose new audio passes the reference's gates
// (more than 1 s, AudioProcessor.isVoiceDetected) and runs all of them through ONE batched pass of the seek loop, with the stream's
// shouldStopEarly rule applied inside the window scheduler; then each stream applies the reference's segment confirmation.
//   transcribeCurrentBuffer        AudioStreamTranscriber.swift:126-193
//   transcribeAudioSamples         :195-206 (clipTimestamps = [lastConfirmedSegmentEndSeconds])
//   shouldStopEarly                :208-227 (session.cu, StopRule)
//   processBuffer / relativeEnergy AudioProcessor.swift:907-917, calculateRelativeEnergy :724-741, calculateAverageEnergy :698-702
//   isVoiceDetected                AudioProcessor.swift:636-655
// Memory: a stream keeps its audio from the current clip start round(lastConfirmedSegmentEndSeconds * 16000) on, i.e. its unconfirmed
// plus not yet transcribed audio.  A stream whose segments never confirm keeps everything, as the reference does.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "kernels.h"
#include "longform.h"

using namespace wk;

namespace {
constexpr int kSampleRate = 16000;     // WhisperKit.sampleRate
constexpr int kBlock = 1600;           // AudioProcessor.minBufferLength: one energy value per 100 ms block
constexpr int kRefBlocks = 20;         // processBuffer's reference level: the lowest RMS of the previous 20 blocks
constexpr int64_t kChunk = 16000;      // audio storage granule: 1 s, never reallocated once allocated

float swift_min(float x, float y) { return y < x ? y : x; }    // Swift.min(_:_:) on Float
float swift_max(float x, float y) { return y >= x ? y : x; }   // Swift.max(_:_:) on Float

// vDSP_rmsqv
float block_rms(const float* x, int64_t n) {
    double acc = 0.0;
    for (int64_t i = 0; i < n; ++i) acc += (double)x[i] * (double)x[i];
    return n > 0 ? (float)sqrt(acc / (double)n) : 0.f;
}

// calculateRelativeEnergy(of:relativeTo:) with reference = min RMS of the previous blocks (+inf when there is none)
float relative_energy(float rms, float reference) {
    const float ref = swift_max(1e-8f, reference);
    const float db = 20.f * (float)log10((double)rms);
    const float ref_db = 20.f * (float)log10((double)ref);
    const float normalized = (db - ref_db) / (0.f - ref_db);
    return swift_max(0.f, swift_min(normalized, 1.f));   // NaN (first block: inf / inf) -> 0
}

bool voice_detected(const float* e, int64_t n, float next_buffer_seconds, float silence_threshold) {
    const float q = next_buffer_seconds / 0.1f;
    int64_t k = 0;
    if (q > 0.f) k = q >= 9.0e18f ? INT64_MAX : (int64_t)q;   // max(0, Int(nextBufferInSeconds / 0.1))
    const int64_t m = std::min(k, n);                        // relativeEnergy.suffix(k)
    const int64_t check = std::min(m, std::max<int64_t>(10, m - 10));   // .prefix(max(10, count - 10))
    for (int64_t i = 0; i < check; ++i)
        if (e[n - m + i] > silence_threshold) return true;
    return false;
}

struct StreamSegment {
    wk_segment seg;
    std::vector<int32_t> tokens;
    std::vector<float> logprobs;
    std::vector<OutWord> words;   // .segment unused
    bool same(const StreamSegment& o) const {
        return seg.seek == o.seg.seek && seg.start == o.seg.start && seg.end == o.seg.end && tokens == o.tokens && logprobs == o.logprobs;
    }
};

struct Stream {
    // audio: absolute samples [held_from, pushed) in fixed chunks; chunk c holds samples [(chunk0 + c) * kChunk, ... + kChunk).  A push
    // writes only past `pushed` and never moves a chunk, so a round can copy [base, n) of its snapshot without the streamer's lock
    std::deque<std::unique_ptr<float[]>> chunks;
    int64_t chunk0 = 0;
    int64_t held_from = 0, pushed = 0;
    int64_t duplicate_confirmations = 0;   // rounds whose confirmation candidates were already confirmed (:178)
    // energies: one relative energy per complete block; values of blocks [energy_from, n_blocks) are held
    std::vector<float> energy;
    int64_t energy_from = 0, n_blocks = 0;
    std::vector<float> recent_rms;   // RMS of the last <= 20 complete blocks
    std::vector<float> partial;      // samples of the incomplete trailing block
    // AudioStreamTranscriber.State
    int64_t last_buffer_size = 0;
    float last_confirmed = 0.f;
    std::vector<StreamSegment> confirmed, unconfirmed;
    bool transcribed = false;

    void add_block(const float* x) {
        const float rms = block_rms(x, kBlock);
        float ref = INFINITY;
        for (float r : recent_rms) ref = swift_min(ref, r);
        energy.push_back(relative_energy(rms, ref));
        ++n_blocks;
        recent_rms.push_back(rms);
        if ((int)recent_rms.size() > kRefBlocks) recent_rms.erase(recent_rms.begin());
    }
    // the chunk pointers covering absolute samples [a, b) (taken under the streamer's lock, read after it)
    std::vector<const float*> chunk_ptrs(int64_t a, int64_t b) const {
        std::vector<const float*> p;
        if (b > a)
            for (int64_t c = a / kChunk; c <= (b - 1) / kChunk; ++c) p.push_back(chunks[c - chunk0].get());
        return p;
    }
    void push(const float* x, int64_t n) {
        for (int64_t done = 0; done < n;) {
            const int64_t at = pushed + done, c = at / kChunk - chunk0, off = at % kChunk;
            if (c >= (int64_t)chunks.size()) chunks.emplace_back(new float[kChunk]);
            const int64_t take = std::min(n - done, kChunk - off);
            memcpy(chunks[c].get() + off, x + done, (size_t)take * sizeof(float));
            done += take;
        }
        pushed += n;
        int64_t i = 0;
        if (!partial.empty()) {
            const int64_t take = std::min<int64_t>(n, kBlock - (int64_t)partial.size());
            partial.insert(partial.end(), x, x + take);
            i = take;
            if ((int64_t)partial.size() == kBlock) { add_block(partial.data()); partial.clear(); }
        }
        for (; i + kBlock <= n; i += kBlock) add_block(x + i);
        if (i < n) partial.assign(x + i, x + n);
    }
    // drop what no later round reads: audio before the clip start, energies older than the audio since lastBufferSize
    void trim(int64_t clip_start) {
        const int64_t keep = std::min(clip_start, pushed);
        if (keep > held_from) held_from = keep;
        while (!chunks.empty() && (chunk0 + 1) * kChunk <= held_from) { chunks.pop_front(); ++chunk0; }
        // isVoiceDetected reads the last Int((n - lastBufferSize) / 1600) values at most: blocks from lastBufferSize / 1600 - 1 on
        // (two blocks of slack for the f32 division)
        const int64_t keep_blocks = std::max<int64_t>(0, last_buffer_size / kBlock - 2);
        if (keep_blocks > energy_from) { energy.erase(energy.begin(), energy.begin() + (keep_blocks - energy_from)); energy_from = keep_blocks; }
    }
};

// prepareSeekClips([lastConfirmedSegmentEndSeconds], n): the clip start, Swift round() of seconds * 16000 in f32
int64_t clip_start_of(float last_confirmed) { return (int64_t)roundf(last_confirmed * (float)kSampleRate); }
}  // namespace

struct wk_streamer {
    wk_model* m; wk_session* s;
    wk_special_tokens st;
    wk_decode_opts opts;
    std::vector<int32_t> suppress, prompt_tokens, prefix_tokens, language_tokens;   // storage behind opts' pointers
    std::vector<int32_t> prompt;
    wk_stream_config cfg;
    wk_tokenizer_hooks hooks; bool has_hooks = false;
    std::mutex mu;         // streams and their state (pushes, rounds' snapshot and commit)
    std::mutex round_mu;   // one round at a time
    std::map<int32_t, std::shared_ptr<Stream>> streams;
    int32_t next_id = 0;
};

extern "C" {

wk_status wk_stream_relative_energy(const float* pcm, int64_t n, float* out, int64_t cap, int64_t* n_blocks) {
    if (n < 0 || (n > 0 && !pcm) || !n_blocks) { set_error("wk_stream_relative_energy: bad arguments"); return WK_ERR_INVALID_ARGUMENT; }
    Stream x;
    x.push(pcm, n);
    if ((int64_t)x.energy.size() > cap || (!out && !x.energy.empty())) { set_error("wk_stream_relative_energy: capacity %lld < %zu", (long long)cap, x.energy.size()); return WK_ERR_INVALID_ARGUMENT; }
    if (!x.energy.empty()) memcpy(out, x.energy.data(), x.energy.size() * sizeof(float));
    *n_blocks = (int64_t)x.energy.size();
    return WK_OK;
}

wk_status wk_stream_voice_detected(const float* energies, int64_t n, float next_buffer_seconds, float silence_threshold, int32_t* out) {
    if (n < 0 || (n > 0 && !energies) || !out) { set_error("wk_stream_voice_detected: bad arguments"); return WK_ERR_INVALID_ARGUMENT; }
    *out = voice_detected(energies, n, next_buffer_seconds, silence_threshold) ? 1 : 0;
    return WK_OK;
}

wk_status wk_streamer_create(wk_model* m, wk_session* s, const wk_special_tokens* st, const wk_decode_opts* o, const int32_t* prompt,
                             int32_t n_prompt, const wk_stream_config* cfg, const wk_tokenizer_hooks* hooks, wk_streamer** out) {
    if (!m || !s || !st || !o || !prompt || n_prompt < 1 || !cfg || !out) { set_error("wk_streamer_create: bad arguments"); return WK_ERR_INVALID_ARGUMENT; }
    if (o->beam_size > 1) { set_error("wk_streamer_create: beam search is not supported in streams (beam_size %d)", o->beam_size); return WK_ERR_INVALID_ARGUMENT; }
    if (session_top_logprobs(s) > 0) { set_error("wk_streamer_create: topLogProbs is not supported in streams"); return WK_ERR_INVALID_ARGUMENT; }
    if (o->word_timestamps && (!hooks || !hooks->split_to_word_tokens)) { set_error("wk_streamer_create: wordTimestamps needs the tokenizer's split_to_word_tokens hook"); return WK_ERR_INVALID_ARGUMENT; }
    if (cfg->required_segments_for_confirmation < 0 || cfg->compression_check_window < 1) {
        set_error("wk_streamer_create: required_segments_for_confirmation %d must be >= 0 and compression_check_window %d >= 1",
                  cfg->required_segments_for_confirmation, cfg->compression_check_window);
        return WK_ERR_INVALID_ARGUMENT;
    }
    wk_streamer* t = new wk_streamer();
    t->m = m; t->s = s; t->st = *st; t->opts = *o; t->cfg = *cfg;
    auto own = [](std::vector<int32_t>& v, const int32_t* p, int32_t n) -> const int32_t* {
        if (!p || n <= 0) return p;
        v.assign(p, p + n);
        return v.data();
    };
    t->opts.suppress_tokens = const_cast<int32_t*>(own(t->suppress, o->suppress_tokens, o->n_suppress_tokens));
    t->opts.prompt_tokens = const_cast<int32_t*>(own(t->prompt_tokens, o->prompt_tokens, o->n_prompt_tokens));
    t->opts.prefix_tokens = const_cast<int32_t*>(own(t->prefix_tokens, o->prefix_tokens, o->n_prefix_tokens));
    t->opts.language_tokens = const_cast<int32_t*>(own(t->language_tokens, o->language_tokens, o->n_language_tokens));
    t->prompt.assign(prompt, prompt + n_prompt);
    if (hooks) { t->hooks = *hooks; t->has_hooks = true; }
    *out = t;
    return WK_OK;
}

wk_status wk_streamer_add_stream(wk_streamer* t, int32_t* id) {
    if (!t || !id) { set_error("wk_streamer_add_stream: bad arguments"); return WK_ERR_INVALID_ARGUMENT; }
    std::lock_guard<std::mutex> lock(t->mu);
    *id = t->next_id++;
    t->streams[*id] = std::make_shared<Stream>();
    return WK_OK;
}

wk_status wk_streamer_remove_stream(wk_streamer* t, int32_t id) {
    if (!t) { set_error("wk_streamer_remove_stream: bad arguments"); return WK_ERR_INVALID_ARGUMENT; }
    std::lock_guard<std::mutex> lock(t->mu);
    if (!t->streams.erase(id)) { set_error("wk_streamer_remove_stream: unknown stream %d", id); return WK_ERR_INVALID_ARGUMENT; }
    return WK_OK;
}

wk_status wk_streamer_push(wk_streamer* t, int32_t id, const float* pcm, int64_t n) {
    if (!t || n < 0 || (n > 0 && !pcm)) { set_error("wk_streamer_push: bad arguments"); return WK_ERR_INVALID_ARGUMENT; }
    std::lock_guard<std::mutex> lock(t->mu);
    auto it = t->streams.find(id);
    if (it == t->streams.end()) { set_error("wk_streamer_push: unknown stream %d", id); return WK_ERR_INVALID_ARGUMENT; }
    it->second->push(pcm, n);
    return WK_OK;
}

wk_status wk_streamer_round(wk_streamer* t, int32_t* ids, int32_t cap, int32_t* n_out) {
    if (!t || !n_out || cap < 0 || (cap > 0 && !ids)) { set_error("wk_streamer_round: bad arguments"); return WK_ERR_INVALID_ARGUMENT; }
    if (session_bias_sets(t->s) > 0) { set_error("wk_streamer_round: the session has a bias set attached"); return WK_ERR_INVALID_ARGUMENT; }
    std::lock_guard<std::mutex> round_lock(t->round_mu);
    struct Ready { int32_t id; std::shared_ptr<Stream> stream; int64_t n; std::vector<float> audio; int64_t base; std::vector<const float*> src; };
    std::vector<Ready> ready;
    std::vector<int32_t> all_ids;
    {   // snapshot: the gates of transcribeCurrentBuffer (:126-158) and where each ready stream's [clip start, n) lies
        std::lock_guard<std::mutex> lock(t->mu);
        for (auto& kv : t->streams) {
            Stream& x = *kv.second;
            all_ids.push_back(kv.first);
            const int64_t n = x.pushed;
            const float next_seconds = (float)(n - x.last_buffer_size) / (float)kSampleRate;
            if (!(next_seconds > 1.f)) continue;
            if (t->cfg.use_vad) {
                // relativeEnergy as it stands at n: one value per complete block
                const int64_t nb = x.n_blocks, have = nb - x.energy_from;
                if (!voice_detected(x.energy.data(), have, next_seconds, t->cfg.silence_threshold)) continue;
            }
            Ready r;
            r.id = kv.first; r.stream = kv.second; r.n = n;
            r.base = std::min(std::max(clip_start_of(x.last_confirmed), x.held_from), n);
            r.src = x.chunk_ptrs(r.base, n);
            ready.push_back(std::move(r));
        }
    }
    // the copies, outside the lock: pushes only write past each snapshot's n, and only this round frees chunks (when it trims)
    for (Ready& r : ready) {
        r.audio.resize((size_t)(r.n - r.base));
        for (int64_t a = r.base; a < r.n;) {
            const int64_t c = a / kChunk - r.base / kChunk, off = a % kChunk, take = std::min(r.n - a, kChunk - off);
            memcpy(r.audio.data() + (a - r.base), r.src[c] + off, (size_t)take * sizeof(float));
            a += take;
        }
    }
    if ((int32_t)ready.size() > cap) { set_error("wk_streamer_round: %zu streams ready, capacity %d", ready.size(), cap); return WK_ERR_INVALID_ARGUMENT; }
    std::vector<std::vector<StreamSegment>> segs(ready.size());
    if (!ready.empty()) {
        std::vector<Unit> units;
        for (size_t i = 0; i < ready.size(); ++i) {
            Ready& r = ready[i];
            Unit u;
            u.stream = (int)i; u.audio = r.audio.data(); u.n = r.n; u.offset = 0; u.base = r.base;
            const float lc = r.stream->last_confirmed;   // written only by rounds, which this one excludes
            u.clips.resize(2 * 2);
            int nc = 0;
            wk_status rc = wk_prepare_seek_clips(&lc, 1, r.n, u.clips.data(), 2, &nc);
            if (rc != WK_OK) return rc;
            u.clips.resize(2 * nc);
            units.push_back(std::move(u));
        }
        StopRule stop;
        stop.window = t->cfg.compression_check_window;
        stop.compression_threshold = t->opts.has_compression_ratio_threshold ? t->opts.compression_ratio_threshold : 0.f;   // ?? 0.0
        stop.has_logprob = t->opts.has_logprob_threshold;
        stop.logprob_threshold = t->opts.logprob_threshold;
        wk_transcription* T = nullptr;
        wk_status rc = seek_loop_units(t->m, t->s, units, (int)ready.size(), &t->st, &t->opts, t->prompt.data(), (int32_t)t->prompt.size(), 1.0f, -1,
                                       t->has_hooks ? &t->hooks : nullptr, 0, 0, &stop, false, &T);
        if (rc != WK_OK) return rc;
        std::vector<size_t> local(T->segments.size());   // index of each result segment inside its stream's list
        for (size_t g = 0; g < T->segments.size(); ++g) {
            const wk_segment& sg = T->segments[g];
            local[g] = segs[sg.stream].size();
            StreamSegment x;
            x.seg = sg;
            x.tokens.assign(T->tokens.begin() + sg.token_offset, T->tokens.begin() + sg.token_offset + sg.n_tokens);
            x.logprobs.assign(T->logprobs.begin() + sg.token_offset, T->logprobs.begin() + sg.token_offset + sg.n_tokens);
            segs[sg.stream].push_back(std::move(x));
        }
        for (const OutWord& w : T->words) segs[T->segments[w.segment].stream][local[w.segment]].words.push_back(w);
        wk_transcription_free(T);
    }
    // commit: lastBufferSize, the confirmation logic (:164-192), trimming
    std::lock_guard<std::mutex> lock(t->mu);
    for (int32_t id : all_ids) {
        auto it = t->streams.find(id);
        if (it != t->streams.end()) it->second->transcribed = false;
    }
    const size_t R = (size_t)t->cfg.required_segments_for_confirmation;
    for (size_t i = 0; i < ready.size(); ++i) {
        Stream& x = *ready[i].stream;
        x.transcribed = true;
        x.last_buffer_size = ready[i].n;
        std::vector<StreamSegment>& sg = segs[i];
        for (StreamSegment& g : sg) g.seg.stream = ready[i].id;
        if (sg.size() > R) {
            const size_t k = sg.size() - R;
            if (sg[k - 1].seg.end > x.last_confirmed) {
                x.last_confirmed = sg[k - 1].seg.end;
                // !confirmedSegments.contains(confirmedSegmentsArray): a contiguous run of equal segments
                bool contained = false;
                for (size_t a = 0; a + k <= x.confirmed.size() && !contained; ++a) {
                    bool eq = true;
                    for (size_t b = 0; b < k && eq; ++b) eq = x.confirmed[a + b].same(sg[b]);
                    contained = eq;
                }
                if (contained) ++x.duplicate_confirmations;
                else x.confirmed.insert(x.confirmed.end(), sg.begin(), sg.begin() + k);
            }
            x.unconfirmed.assign(std::make_move_iterator(sg.begin() + k), std::make_move_iterator(sg.end()));
        } else {
            x.unconfirmed = std::move(sg);
        }
        x.trim(clip_start_of(x.last_confirmed));
    }
    for (size_t i = 0; i < ready.size(); ++i) ids[i] = ready[i].id;
    *n_out = (int32_t)ready.size();
    return WK_OK;
}

wk_status wk_streamer_state(wk_streamer* t, int32_t id, wk_stream_state* out) {
    if (!t || !out) { set_error("wk_streamer_state: bad arguments"); return WK_ERR_INVALID_ARGUMENT; }
    std::lock_guard<std::mutex> lock(t->mu);
    auto it = t->streams.find(id);
    if (it == t->streams.end()) { set_error("wk_streamer_state: unknown stream %d", id); return WK_ERR_INVALID_ARGUMENT; }
    const Stream& x = *it->second;
    memset(out, 0, sizeof(*out));
    out->last_buffer_size = x.last_buffer_size;
    out->last_confirmed_segment_end_seconds = x.last_confirmed;
    out->n_confirmed_segments = (int32_t)x.confirmed.size();
    out->n_unconfirmed_segments = (int32_t)x.unconfirmed.size();
    out->transcribed = x.transcribed ? 1 : 0;
    out->pushed_samples = x.pushed;
    out->held_samples = x.pushed - x.held_from;
    out->held_from = x.held_from;
    out->duplicate_confirmations = x.duplicate_confirmations;
    return WK_OK;
}

wk_status wk_streamer_result(wk_streamer* t, int32_t id, wk_transcription** out) {
    if (!t || !out) { set_error("wk_streamer_result: bad arguments"); return WK_ERR_INVALID_ARGUMENT; }
    std::lock_guard<std::mutex> lock(t->mu);
    auto it = t->streams.find(id);
    if (it == t->streams.end()) { set_error("wk_streamer_result: unknown stream %d", id); return WK_ERR_INVALID_ARGUMENT; }
    const Stream& x = *it->second;
    wk_transcription* T = new wk_transcription();
    T->lang.assign(1, -1); T->lang_logprob.assign(1, 0.f); T->lang_at.assign(1, -1);
    for (const auto* list : {&x.confirmed, &x.unconfirmed})
        for (const StreamSegment& g : *list) {
            wk_segment sg = g.seg;
            sg.token_offset = (int64_t)T->tokens.size();
            sg.n_tokens = (int32_t)g.tokens.size();
            T->tokens.insert(T->tokens.end(), g.tokens.begin(), g.tokens.end());
            T->logprobs.insert(T->logprobs.end(), g.logprobs.begin(), g.logprobs.end());
            for (OutWord w : g.words) { w.segment = (int)T->segments.size(); T->words.push_back(std::move(w)); }
            T->segments.push_back(sg);
        }
    *out = T;
    return WK_OK;
}

void wk_streamer_free(wk_streamer* t) { delete t; }

}  // extern "C"
