// The batched seek loop's internal interface (longform.cu), shared with the stream transcriber (streaming.cu).
#pragma once
#include <stdint.h>

#include <string>
#include <vector>

#include "kernels.h"

struct OutWord {
    std::string word;
    std::vector<int32_t> tokens;
    float start, end, probability;
    int segment;
};

struct wk_transcription {
    std::vector<wk_segment> segments;
    std::vector<OutWord> words;   // .segment indexes `segments`
    std::vector<int32_t> tokens;
    std::vector<float> logprobs;
    // DecodingOptions.topLogProbs: top_k pairs per entry of `tokens` (padded with -1 / -inf), empty when top_k = 0
    int top_k = 0;
    std::vector<int32_t> top_tok;
    std::vector<float> top_lp;
    int windows = 0;
    // per stream: the detected language of its latest window (in stream time) that detected one, and where that window started
    std::vector<int32_t> lang; std::vector<float> lang_logprob; std::vector<int64_t> lang_at;
};

namespace wk {

struct Unit {                 // one independently advancing cursor: a stream, or one VAD chunk of a stream
    int stream;
    const float* audio;       // the unit's samples from `base` on: sample j of the unit sits at audio[j - base]
    int64_t n;                // samples in the unit (contentFrames); seeks and clips are unit sample indices in [base, n]
    int64_t offset;           // unit start inside the stream (seekOffsetIndex)
    int64_t base = 0;         // first sample held: a stream that dropped its confirmed prefix keeps absolute seeks, so segment times
                              // are computed from the same seek values as on the whole buffer (no f32 offset add)
    std::vector<int64_t> clips;
    int clip = 0;
    int64_t seek = 0;
    bool done = false;
    std::vector<wk_segment> segs;
    std::vector<OutWord> words;   // word timings; .segment indexes `segs`
};

// TranscribeTask.run's seek loop over `units` (each with its own clips), batched across them; the result lists streams in order, units
// in order, with chunk offsets applied.  stop (may be nullptr) is applied to every window (transcribe_windows_stop).  renumber_ids:
// segment ids count 0, 1, ... per stream over its units; otherwise they stay findSeekPointAndSegments' allSegments.count + index,
// which keeps the gaps the reference leaves where word timing drops a zero-length segment (one unit per stream).
wk_status seek_loop_units(wk_model* m, wk_session* s, std::vector<Unit>& units, int n_streams, const wk_special_tokens* st,
                          const wk_decode_opts* o, const int32_t* prompt, int32_t n_prompt, float window_clip_time, int64_t max_window_seek,
                          const wk_tokenizer_hooks* hooks, int32_t best_of, int32_t draft_tokens, const StopRule* stop, bool renumber_ids,
                          wk_transcription** out);

}  // namespace wk
