/*
 * wkb200.h - C ABI of libwkb200.so: the Hopper (sm_90a) implementation of WhisperKit's hot path
 *            PCM -> log-mel -> audio encoder -> KV-cached text decoder -> logits filters -> sampler.
 *
 * Every entry point is what a Swift (or Python ctypes) host binds to replace one member of the
 * reference's protocol surface (paths relative to the WhisperKit repo):
 *
 *   wk_mel                  FeatureExtracting.logMelSpectrogram   Sources/WhisperKit/Core/FeatureExtractor.swift:13-17,40-56
 *   wk_encode               AudioEncoding.encodeFeatures          Sources/WhisperKit/Core/AudioEncoder.swift:10-18,50-63
 *   wk_session_create/reset TextDecoding.prepareDecoderInputs     Sources/WhisperKit/Core/TextDecoder.swift:109-161
 *   wk_build_prompt         TextDecoding.prefillDecoderInputs     Sources/WhisperKit/Core/TextDecoder.swift:163-216
 *   wk_decode_step          TextDecoding.predictLogits            Sources/WhisperKit/Core/TextDecoder.swift:361-418
 *   wk_detect_language      TextDecoding.detectLanguage           Sources/WhisperKit/Core/TextDecoder.swift:420-539
 *   wk_filter_sample        LogitsFiltering.filterLogits (x4) +   Sources/WhisperKit/Core/Text/LogitsFilter.swift:8-276
 *                           TokenSampling.update                  Sources/WhisperKit/Core/Text/TokenSampler.swift:8-11,215-240
 *   wk_decode_text          TextDecoding.decodeText (+ sampler    Sources/WhisperKit/Core/TextDecoder.swift:541-855
 *                           finalize, DecodingFallback)           Sources/WhisperKit/Core/Models.swift:357-381
 *   wk_transcribe_windows   the per-window body of                Sources/WhisperKit/Core/TranscribeTask.swift:116-278
 *                           TranscribeTask.run, batched like      Sources/WhisperKit/Core/WhisperKit.swift:716-812
 *                           WhisperKit.transcribeWithOptions
 *   wk_model_info           melCount/windowSamples/embedSize/     FeatureExtractor.swift:24-38, AudioEncoder.swift:24-38,
 *                           logitsSize/kvCache* properties        TextDecoder.swift:313-331
 *
 * Conventions: plain C types only; every function returns a wk_status (0 = ok, negative = error, mapped
 * 1:1 onto WhisperError cases, Sources/WhisperKit/Utilities/WhisperError.swift:6-19); the message of the
 * last error on the calling thread is wk_last_error().  Host pointers may be pageable or pinned; pointers
 * documented as "host or device" are resolved with cudaPointerGetAttributes.
 *
 * Threading (the reference calls the same protocol objects from up to concurrentWorkerCount tasks, WhisperKit.swift:735-791):
 * a finalized wk_model is immutable and may be used from any number of host threads - the model-level entry points
 * (wk_mel, wk_encode, wk_filter_sample, wk_tensor_*) serialise internally; a wk_session (the per-task DecodingInputs of
 * TranscribeTask.swift:83 plus its own mel/encoder workspace and CUDA streams) belongs to one thread at a time, and different
 * sessions of one model run concurrently.  wk_tensor results own their device buffer until wk_tensor_free.
 * There is NO CPU fallback: every compute entry point fails with WK_ERR_MODELS_UNAVAILABLE if no sm_90 (Hopper) device is present.
 */
#ifndef WKB200_H
#define WKB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef int32_t wk_status;
enum {
    WK_OK = 0,
    WK_ERR_INVALID_ARGUMENT = -1,       /* (no Swift twin: argument validation)             */
    WK_ERR_MODELS_UNAVAILABLE = -2,     /* WhisperError.modelsUnavailable                    */
    WK_ERR_AUDIO_PROCESSING_FAILED = -3,/* WhisperError.audioProcessingFailed                */
    WK_ERR_PREPARE_DECODER_INPUTS = -4, /* WhisperError.prepareDecoderInputsFailed           */
    WK_ERR_DECODING_LOGITS_FAILED = -5, /* WhisperError.decodingLogitsFailed                 */
    WK_ERR_DECODING_FAILED = -6,        /* WhisperError.decodingFailed                       */
    WK_ERR_TRANSCRIPTION_FAILED = -7,   /* WhisperError.transcriptionFailed                  */
    WK_ERR_CUDA = -8,                   /* CUDA runtime/driver failure (message has detail)  */
    WK_ERR_LOAD_AUDIO_FAILED = -9       /* WhisperError.loadAudioFailed                      */
};

typedef struct wk_model wk_model;
typedef struct wk_session wk_session;
typedef struct wk_tensor wk_tensor;

enum { WK_DTYPE_F32 = 0, WK_DTYPE_F16 = 1, WK_DTYPE_BF16 = 2, WK_DTYPE_I32 = 3,
       WK_DTYPE_FP8_E4M3 = 4 /* storage policies only: the cross-attention K/V cache (E4M3 codes + one f32 scale per 64-value row) and the
                                encoder's QKV / FC1 / FC2 GEMM operands (wk_model_set_encoder_dtype) */ };

/* Model dimensions.  The reference reads these off the CoreML model descriptions at run time
 * (TextDecoder.swift:313-331, AudioEncoder.swift:24-38, FeatureExtractor.swift:24-38). */
typedef struct wk_model_config {
    int32_t n_mels;      /* 80 or 128 */
    int32_t d_model;     /* embedSize */
    int32_t n_heads;     /* head dim must be 64 */
    int32_t enc_layers;
    int32_t dec_layers;
    int32_t vocab;       /* logitsSize */
    int32_t n_audio_ctx; /* 1500 */
    int32_t n_text_ctx;  /* 448 (positional table); kv_max_len is 224 = Constants.maxTokenContext */
    int32_t dtype;       /* WK_DTYPE_BF16 (default) or WK_DTYPE_F16: storage/MMA-input type; accumulation is f32 */
    int32_t max_batch;   /* windows processed per encoder/decoder pass (workspace sizing) */
} wk_model_config;

typedef struct wk_model_info {
    int32_t n_mels, n_audio_ctx, d_model, n_heads, enc_layers, dec_layers, vocab;
    int32_t kv_embed_dim;   /* kvCacheEmbedDim = dec_layers * d_model */
    int32_t kv_max_len;     /* kvCacheMaxSequenceLength = 224 */
    int32_t window_samples; /* 480000 */
    int32_t has_alignment_heads;
    int32_t is_multilingual; /* logitsSize != 51864 (ModelUtilities.swift:124-126) */
    int32_t dtype, max_batch;
    int32_t cross_kv_dtype;  /* storage of the cross-attention K/V cache: dtype, or WK_DTYPE_FP8_E4M3 */
} wk_model_info;

/* SpecialTokens (Models.swift:1111-1149) - supplied by the host tokenizer. */
typedef struct wk_special_tokens {
    int32_t end_token, english_token, no_speech_token, no_timestamps_token, special_token_begin,
        start_of_previous_token, start_of_transcript_token, time_token_begin, transcribe_token, translate_token,
        whitespace_token;
} wk_special_tokens;

/* DecodingOptions mirror (Configurations.swift:155-247), fields the hot path reads.
 * "has_*" = Swift optional is non-nil. */
typedef struct wk_decode_opts {
    int32_t task_translate;       /* task == .translate */
    int32_t language_token;       /* id of "<|xx|>" (tokenizer lookup done by the host); <0 -> english_token */
    float temperature;            /* 0 = greedy argmax; >0 = top-k multinomial (TokenSampler.swift:57-73) */
    int32_t sample_length;        /* default 224 */
    int32_t top_k;                /* default 5 */
    int32_t use_prefill_prompt;   /* default 1 */
    int32_t without_timestamps;   /* default 0 */
    int32_t suppress_blank;       /* default 0 */
    const int32_t* suppress_tokens; int32_t n_suppress_tokens;
    const int32_t* prompt_tokens;   int32_t n_prompt_tokens;   /* n < 0 -> nil */
    const int32_t* prefix_tokens;   int32_t n_prefix_tokens;   /* n < 0 -> nil */
    int32_t has_compression_ratio_threshold; float compression_ratio_threshold; /* 2.4 */
    int32_t has_logprob_threshold;           float logprob_threshold;           /* -1.0 */
    int32_t has_first_token_logprob_threshold; float first_token_logprob_threshold; /* -1.5 */
    int32_t has_no_speech_threshold;         float no_speech_threshold;         /* 0.6 */
    uint64_t seed;                /* Philox seed for temperature > 0 (the reference uses Float.random) */
    /* decodeWithFallback ladder (TranscribeTask.swift:316-411), applied by wk_transcribe_windows / wk_transcribe_streams only:
     * a window whose DecodingFallback.needsFallback is set is decoded again (same encoder output) at
     * Float16(temperature) + Float16(i) * Float16(increment), i = 1..count. */
    int32_t temperature_fallback_count;        /* default 5; 0 = no retries */
    float temperature_increment_on_fallback;   /* default 0.2 */
    int32_t word_timestamps;      /* wordTimestamps: the decode loop also fills the alignmentWeights tensor (wk_session_alignment_weights) */
    /* Beam search (SURVEY 8f row 2).  The reference's BeamSearchTokenSampler is an unimplemented stub (TokenSampler.swift:254-290) and its
     * DecodingOptions has no beam field, so these two are an extension: beam_size > 1 decodes every window with that many beams
     * (openai/whisper BeamSearchDecoder semantics inside the decodeText loop, specified by oracle/beam_ref.py; self-oracle parity only),
     * maxCandidates = Int(Float(beam_size) * beam_patience) as the stub fixes (:266).  One setting per call.  With wk_batch_opts.best_of
     * = 0 a beam call skips the temperature ladder; best_of >= 1 runs the ladder with beam search on its temperature-0 rung.  Word
     * timestamps do not combine with beam_size > 1 (wk_align_tokens aligns beam results). */
    int32_t beam_size;            /* <= 1: greedy / temperature sampling (default) */
    float beam_patience;          /* default 1 */
    /* DecodingOptions.detectLanguage (Configurations.swift:165,222; TranscribeTask.swift:340-365): on a multilingual model with
     * language_token < 0, every window detects its language inside the decode loop - TextDecoder.detectLanguage's forward ([SOT] at
     * position 0) is the loop's own step 0 when the prompt starts with SOT, else one leading step that is not counted in `steps`.
     * LanguageLogitsFilter over language_tokens + the rung's sampler (argmax at temperature 0, top-k draw with its own Philox counter
     * above); each temperature-ladder rung detects again.  With use_prefill_prompt, a language token right after the prompt's first SOT
     * (the <|xx|> prefillDecoderInputs writes, TextDecoder.swift:176-186) is replaced by the detected one; otherwise the language is only
     * reported (wk_session_languages, wk_transcription_language).  0 = off: a zeroed tail decodes as before. */
    int32_t detect_language;
    const int32_t* language_tokens;   /* tokenizer.allLanguageTokens: 1..4096 ids < vocab, one list for every detecting window of a call */
    int32_t n_language_tokens;
    /* DecodingResult.noSpeechProb (the reference leaves it 0, TextDecoder.swift:802; semantics of openai/whisper decoding.py): the f32
     * softmax over all vocab raw logits - no logits filter, no temperature - of the decode step whose input is the prompt's first
     * <|startoftranscript|>, taken at no_speech_token.  Computed inside the batched decode loop at no extra step; read it with
     * wk_session_no_speech_probs.  It replaces the 0 of the DecodingFallback silence rule (Models.swift:357-381) and, in
     * wk_transcribe_streams, of findSeekPointAndSegments' skip rule and wk_segment.no_speech_prob.  A window whose loop ended before its
     * SOT step has no value (0 is used).  A prompt without <|startoftranscript|> fails its window.  0 = off: a zeroed tail decodes as before. */
    int32_t compute_no_speech_prob;
} wk_decode_opts;

/* Per-window DecodingResult (Models.swift:383-439) in flat arrays; tokens = SOT..EOT slice. */
typedef struct wk_decode_result {
    int32_t n_tokens;                 /* filteredTokens.count */
    int32_t tokens[226];
    float token_logprobs[226];
    float avg_logprob;
    float compression_ratio;
    float temperature;
    int32_t needs_fallback;           /* DecodingFallback.needsFallback (0 if fallback == nil) */
    int32_t fallback_reason;          /* 0 nil, 1 firstTokenLogProbThreshold, 2 silence, 3 compressionRatio, 4 logProb */
    int32_t first_token_logprob_too_low;
    int32_t n_current_tokens;         /* currentTokens.count when the loop ended (before finalize) */
    int32_t steps;                    /* decoder forward passes run for this window */
} wk_decode_result;

const char* wk_last_error(void);
const char* wk_version(void);
/* 1 if a compute-capability 10.x device is visible. */
int32_t wk_device_available(void);

/* ---- model ---- */
void wk_default_config(const char* variant /* tiny[.en] base[.en] small[.en] medium[.en] large large-v2 large-v3 large-v3-turbo distil-large-v3 */,
                       wk_model_config* out);
/* ModelUtilities.detectVariant + tokenizerNameForVariant + isModelMultilingual (ModelUtilities.swift:124-205): static strings out. */
wk_status wk_detect_variant(int32_t logits_dim, int32_t encoder_dim, const char** variant, const char** tokenizer_repo, int32_t* is_multilingual);
wk_status wk_model_create(const wk_model_config* cfg, int32_t device, wk_model** out);
/* HuggingFace parameter names ("model.encoder.layers.0.self_attn.q_proj.weight", ...); data host or device. */
wk_status wk_model_set_tensor(wk_model* m, const char* name, const void* data, int32_t dtype, const int64_t* shape, int32_t ndim);
wk_status wk_model_finalize(wk_model* m);
/* HuggingFace checkpoint directory (config.json + *.safetensors, F32/F16/BF16); replaces loadModels (WhisperKit.swift:358-442). */
wk_status wk_model_load(const char* weights_dir, int32_t device, int32_t max_batch, int32_t dtype, wk_model** out);
/* Seeded synthetic weights generated on the device (benchmarks: no checkpoints are available offline). */
wk_status wk_model_init_random(wk_model* m, uint64_t seed, float std);
wk_status wk_model_info_get(const wk_model* m, wk_model_info* out);
/* Storage of the decoder's cross-attention K/V cache (default: the model's dtype).  WK_DTYPE_FP8_E4M3 stores each
 * (window, layer, K|V, head, position) row of 64 values as 64 E4M3 codes plus one f32 scale s = amax(|row|) / 448,
 * code = cvt.rn.satfinite.e4m3(x / s) (s = 0 and zero codes for an all-zero row): 0.53x the bytes the decode loop streams per step
 * and a cache about half the size; K and V keep 3 mantissa bits (4 fewer than bf16, 7 fewer than f16) under a per-row scale.  Accepts WK_DTYPE_FP8_E4M3 or the model's own dtype;
 * works after wk_model_create or wk_model_load and must be called before the model's first wk_session_create (WK_ERR_INVALID_ARGUMENT
 * after that). */
wk_status wk_model_set_cross_kv_dtype(wk_model* m, int32_t dtype);
/* The FP8 row quantizer above on the host (the code the GPU projection epilogue runs): x [rows][64] f32 -> codes [rows][64], scales [rows]. */
wk_status wk_cross_kv_quantize_rows(const float* x, int64_t rows, uint8_t* codes, float* scales);
/* Precision of the encoder's QKV, FC1 and FC2 GEMMs (default: the model's dtype).  WK_DTYPE_FP8_E4M3 runs them on the FP8 tensor cores
 * (wgmma e4m3 x e4m3, f32 accumulation): activations as E4M3 codes with one f32 scale s = amax / 448 per (row, 128-column block) -
 * the LayerNorm outputs, and FC1's GELU output quantized in its epilogue from f32 - and weights as E4M3 copies with one scale per
 * output channel, quantized on the device from the 16-bit weights now and again whenever wk_model_set_tensor / wk_model_init_random
 * changes one of them (about 0.63 GB more for large-v3).  Each k-block's products are promoted into the f32 accumulator with their row
 * scale; the weight scale is applied once in the epilogue.  The conv stem, attention, the out-projection, LayerNorm statistics, the f32
 * residual stream, the final LayerNorm and the 16-bit encoder output are unchanged, so the decoder and the cross-K/V policy see a 16-bit
 * encoder output as before.  Every scale comes from its own row: a window's result does not depend on its batch.  Applies to every
 * encoder call of the model (wk_encode, sessions, the window scheduler, long-form, streams, alignment).  Accepts WK_DTYPE_FP8_E4M3 or
 * the model's own dtype; WK_ERR_INVALID_ARGUMENT once a session exists or wk_encode has run. */
wk_status wk_model_set_encoder_dtype(wk_model* m, int32_t dtype);
/* The encoder precision policy: WK_DTYPE_FP8_E4M3 or the model's dtype. */
wk_status wk_model_encoder_dtype(const wk_model* m, int32_t* dtype);
/* The FP8 quantizer on the host (the code the GPU LayerNorm, FC1 epilogue and weight quantizer run): x [rows][cols] f32 in groups of
 * `block` columns (cols a multiple of block) -> codes [rows][cols], scales [rows][cols / block].  block = 128 is the activation rule,
 * block = cols the weight rule (one scale per row). */
wk_status wk_fp8_quantize_blocks(const float* x, int64_t rows, int64_t cols, int64_t block, uint8_t* codes, float* scales);
/* ---- draft decoder for speculative greedy decoding (wk_transcribe_windows_draft) ----
 * A second, smaller Whisper decoder that reads the model's encoder output (distil-large-v3 for large-v3: its encoder is large-v3's,
 * copied and frozen).  It only proposes tokens; the model's own decoder checks them, so the output never depends on the draft.  A draft
 * has its own embedding, positional table, layers, final LayerNorm and cross-attention K/V projections, and the model's d_model, heads,
 * vocabulary and n_audio_ctx.  Every call below fails with WK_ERR_INVALID_ARGUMENT once a session of the model exists.
 * wk_model_load_draft: an HF Whisper checkpoint directory (config.json + *.safetensors); only the model.decoder.* tensors (and
 * proj_out.weight) are read, encoder tensors are ignored; a config whose d_model, heads, vocab_size or max_source_positions differ from
 * the model's is refused.  wk_model_create_draft allocates a zeroed draft of dec_layers layers (replacing any earlier one), which
 * wk_model_set_draft_tensor (HF decoder names, as wk_model_set_tensor) and wk_model_init_draft_random (seeded, as wk_model_init_random)
 * fill.  wk_model_draft_layers: the draft's decoder layers, 0 without one. */
wk_status wk_model_load_draft(wk_model* m, const char* weights_dir);
wk_status wk_model_create_draft(wk_model* m, int32_t dec_layers);
wk_status wk_model_set_draft_tensor(wk_model* m, const char* name, const void* data, int32_t dtype, const int64_t* shape, int32_t ndim);
wk_status wk_model_init_draft_random(wk_model* m, uint64_t seed, float std);
wk_status wk_model_draft_layers(const wk_model* m, int32_t* n);
void wk_model_free(wk_model* m);

/* ---- tensors (opaque device buffers passed mel -> encoder -> decoder without touching the host) ---- */
wk_status wk_tensor_shape(const wk_tensor* t, int64_t* shape4, int32_t* ndim, int32_t* dtype);
/* Copies to the host in the REFERENCE layout as f32: mel -> [B, nMels, 3000]; encoder output -> [B, d, 1500]. */
wk_status wk_tensor_to_host(const wk_tensor* t, float* dst, int64_t dst_elems);
/* Same, into a host MLMultiArray with explicit element strides (IOSurface-backed arrays pad their rows: every host access in the
 * reference goes through `strides`, TextDecoder.swift:222-227, MLMultiArrayExtensions.swift:75-82): dst[b*stride_b + c*stride_c + t*stride_t]. */
wk_status wk_tensor_to_host_strided(const wk_tensor* t, float* dst, int64_t stride_b, int64_t stride_c, int64_t stride_t, int64_t dst_elems);
/* Releases the tensor and (stream-ordered, after its last reader) its device buffer. */
void wk_tensor_free(wk_tensor* t);

/* ---- FeatureExtracting ---- */
/* pcm: n_windows rows of `stride` floats (host or device); samples_per_window[i] <= 480000 valid samples
 * (NULL = all 480000); the rest of the window is zero-padded (padOrTrimAudio, AudioProcessor.swift:151-174). */
wk_status wk_mel(wk_model* m, const float* pcm, int64_t n_windows, int64_t stride, const int32_t* samples_per_window, wk_tensor** mel_out);

/* ---- AudioProcessing: audio at any sample rate and channel layout -> 16 kHz mono f32 ----
 *   wk_audio_info         AVAudioFile's fileFormat / length       Sources/WhisperKit/Core/Audio/AudioProcessor.swift:251-253
 *   wk_audio_load         AudioProcessor.loadAudio(fromPath:) /   AudioProcessor.swift:229-305
 *                         loadAudioAsFloatArray(fromPath:)        AudioProcessor.swift:307-350
 *   wk_audio_convert      convertToMono + resampleAudio(fromFile:) AudioProcessor.swift:381-450,526-625
 *                         on interleaved frames in memory
 *   wk_audio_filter_taps  the resampler's filter design (host)
 * Files: WAV (RIFF/WAVE) with PCM u8 / s16 / s24 / s32 or IEEE float 32, plain or WAVE_FORMAT_EXTENSIBLE, and native FLAC (RFC 9639,
 * 1-8 channels, 4-32 bits per sample, optionally behind an ID3v2 tag, with a known total length).  A FLAC file loads exactly like a WAV
 * file of the same integers: bits per sample <= 16 as s16, 17-24 as s24, 25-32 as s32, each sample left-justified in its container;
 * wk_audio_info reports that container, STREAMINFO's rate, channels and total length, and the first audio frame as data_offset.  FLAC
 * frames are found, checked (CRC-8, CRC-16, contiguous sample numbers) and decoded on the device; the MD5 is not checked.  Anything else
 * (lossy formats, Ogg, big-endian RIFX, 64-bit float, a FLAC file with a bad frame) fails with WK_ERR_LOAD_AUDIO_FAILED and a message
 * naming the format or the reason and byte offset.  Samples become f32 as
 * AVAudioFile converts them: s16 x / 32768, s24 x / 8388608, s32 float(x) / 2147483648, u8 (x - 128) / 128.
 * Mono mix: convertToMono exactly, applied per read chunk of max_read_frame_size frames as the reference reads them (sumChannels
 * rescales each chunk by max|selected channel| / max(max|sum|, 0.0001)).  Resampling: scipy.signal.resample_poly(x, 16000 / g, rate / g)
 * with its default Kaiser (beta 5) window and zero padding, one continuous filter over the selected range (the reference converts each
 * read chunk separately); the length is ceil(n * 16000 / rate).  16 kHz input is copied.  Sample rates: integer Hz in [1000, 384000],
 * else WK_ERR_INVALID_ARGUMENT.  The GPU work runs on the session's stream (sessions on different threads convert concurrently), through
 * the session's pinned staging and a fixed-size device workspace; session may be NULL (a stream and workspace for the call alone). */
enum { WK_AUDIO_U8 = 0, WK_AUDIO_S16 = 1, WK_AUDIO_S24 = 2, WK_AUDIO_S32 = 3, WK_AUDIO_F32 = 4 };
enum { WK_CHANNELS_SUM = 0 /* ChannelMode.sumChannels */, WK_CHANNELS_SPECIFIC = 1 /* ChannelMode.specificChannel */ };
typedef struct wk_audio_format {
    int32_t sample_rate, channels;
    int32_t sample_format;     /* WK_AUDIO_* */
    int32_t block_align;       /* bytes per interleaved frame */
    int64_t frames;            /* frames present in the data chunk */
    int64_t data_offset;       /* byte offset of the first frame in the file */
} wk_audio_format;
typedef struct wk_audio_load_opts {   /* all zero = sumChannels(nil), the whole file, default read size, loadAudio */
    int32_t channel_mode;      /* WK_CHANNELS_SUM or WK_CHANNELS_SPECIFIC */
    int32_t channel;           /* specificChannel(channel); out of range = channel 0 */
    const int32_t* channel_indices; int32_t n_channel_indices;   /* sumChannels(indices); NULL or 0 = all channels */
    int32_t has_end_time;      /* 0 = endTime nil (to the end of the file); else end_time is used */
    double start_time;         /* seconds, finite and >= 0 */
    double end_time;           /* seconds (has_end_time != 0); values at or past the end, +inf included, read to the end */
    int64_t max_read_frame_size;   /* frames per read chunk; <= 0 = Constants.defaultAudioReadFrameSize (1323000) */
    double piece_seconds;      /* loadAudioAsFloatArray's pieces (600); <= 0 = loadAudio (one piece) */
    int64_t segment_samples;   /* 16 kHz samples per device segment; <= 0 = at most about 32 MiB of staged input and 4 Mi outputs per
                                  segment.  Never more than the call's output; never changes the result */
} wk_audio_load_opts;
/* Header of a WAV file (host only, no GPU). */
wk_status wk_audio_info(const char* path, wk_audio_format* out);
/* Load `path` as 16 kHz mono f32 into out (host or device, capacity cap samples); *n_out = the length.  out == NULL returns the length only. */
wk_status wk_audio_load(wk_session* s, const char* path, const wk_audio_load_opts* opts, float* out, int64_t cap, int64_t* n_out);
/* The same for n_frames interleaved frames of `channels` samples in sample_format (host or device; device frames aligned to their sample
 * size) at sample_rate: the result equals wk_audio_load of a WAV file holding these frames. */
wk_status wk_audio_convert(wk_session* s, const void* frames, int32_t sample_format, int64_t n_frames, int32_t channels, int32_t sample_rate,
                           const wk_audio_load_opts* opts, float* out, int64_t cap, int64_t* n_out);
/* The resampler's filter for sample_rate (host only): up / down = 16000 / rate reduced, and the 2 * 10 * max(up, down) + 1 taps
 * firwin(., 1 / max(up, down), window=('kaiser', 5.0)) * up in double (n = 0 when up == down == 1).  taps may be NULL (sizes only). */
wk_status wk_audio_filter_taps(int32_t sample_rate, double* taps, int64_t cap, int32_t* up, int32_t* down, int32_t* n);

/* ---- AudioEncoding ---- */
wk_status wk_encode(wk_model* m, const wk_tensor* mel, wk_tensor** enc_out);

/* ---- TextDecoding ---- */
wk_status wk_session_create(wk_model* m, int32_t max_batch, wk_session** out);
void wk_session_free(wk_session* s);
/* Bind encoder output for `batch` windows: computes the per-layer cross-attention K/V cache. */
wk_status wk_session_set_encoder_output(wk_session* s, const wk_tensor* enc);
/* Zero caches/masks (prepareDecoderInputs / DecodingInputs.reset). */
wk_status wk_session_reset(wk_session* s);
/* prefillDecoderInputs: builds initialPrompt into out (capacity cap); returns length in *n. */
wk_status wk_build_prompt(const wk_model* m, const wk_special_tokens* st, const wk_decode_opts* opts, int32_t use_options, int32_t* out, int32_t cap, int32_t* n);
/* predictLogits for every bound window: input_ids[B], cache_length[B] (host) -> logits [B, vocab] f32 (host, may be NULL). */
wk_status wk_decode_step(wk_session* s, const int32_t* input_ids, const int32_t* cache_length, float* logits_out);
/* TextDecoding.detectLanguage (TextDecoder.swift:420-539): one step on [SOT] + LanguageLogitsFilter + sampler, per bound window. */
wk_status wk_detect_language(wk_session* s, const wk_special_tokens* st, const int32_t* language_tokens, int32_t n_language_tokens,
                             float temperature, int32_t* token_out, float* logprob_out);
/* Filters + sampler alone (parity entry): logits [B, vocab] f32 host; tokens [B, ld_tokens], n_tokens[B] = currentTokens;
 * sample_begin_ts = TimestampRulesFilter.sampleBegin (<0: filter absent), sample_begin_blank = SuppressBlankFilter.sampleBegin
 * (<0: absent); language_tokens != NULL adds LanguageLogitsFilter(sampleBegin = language_sample_begin).
 * Writes token_out[B], logprob_out[B] and (optional) the masked logits back into filtered_out [B, vocab]. */
wk_status wk_filter_sample(wk_model* m, const wk_special_tokens* st, const wk_decode_opts* opts, int32_t is_multilingual,
                           const float* logits, int32_t batch, int32_t vocab, const int32_t* tokens, int32_t ld_tokens,
                           const int32_t* n_tokens, int32_t sample_begin_ts, int32_t sample_begin_blank,
                           const int32_t* language_tokens, int32_t n_language_tokens, int32_t language_sample_begin,
                           int32_t* token_out, float* logprob_out, float* filtered_out);
/* decodeText for every bound window with one shared prompt (device-resident loop: no per-token host round trip).
 * results: array of `batch` wk_decode_result. */
wk_status wk_decode_text(wk_session* s, const wk_special_tokens* st, const wk_decode_opts* opts,
                         const int32_t* prompt, int32_t n_prompt, wk_decode_result* results);
/* Scheduler counters of the session's last batched call: [0] decode steps launched, [1] sum over those steps of the windows that were
 * live when their burst started (an upper bound of the rows that actually streamed K/V), [2] windows admitted to a slot, [3] ladder
 * re-admissions. */
wk_status wk_session_stats(const wk_session* s, int64_t* out4);
/* Speculative decoding counters of the session's last batched call (wk_transcribe_windows_draft, wk_decode_text_draft): [0] rounds in which a window verified
 * proposals, [1] tokens the draft proposed in them, [2] proposals accepted.  All 0 after a call without a draft. */
wk_status wk_session_draft_stats(const wk_session* s, int64_t* out3);
/* Language detected for windows [first, first + n) of the session's last batched call (DecodingResult.language as a token id):
 * tokens[i] = the <|xx|> id from the rung whose result was returned, logprobs[i] = its log-prob (log-softmax over language_tokens at
 * temperature 0); -1 and 0 for a window that did not detect.  Either output may be NULL. */
wk_status wk_session_languages(const wk_session* s, int32_t first, int32_t n, int32_t* tokens, float* logprobs);
/* No-speech probability of windows [first, first + n) of the session's last batched call (wk_transcribe_windows(_ex),
 * wk_decode_text(_ex); opts->compute_no_speech_prob), from the rung whose result was returned; NaN where it was not computed. */
wk_status wk_session_no_speech_probs(const wk_session* s, int32_t first, int32_t n, float* out);
/* Device logits of the last step, copied to host (debug / parity). */
wk_status wk_session_last_logits(wk_session* s, float* logits_out);

/* TranscriptionCallback (Models.swift TranscriptionProgress; TextDecoder.swift:724-762): called from the thread that runs the decode
 * every `progress_every` decoder steps with each live window's current tokens.  Returning 0 is the reference's `callback -> false`:
 * that window stops early (EarlyStopActor) and its result is built from the tokens it has. */
typedef int32_t (*wk_progress_fn)(void* user, int32_t window, const int32_t* tokens, int32_t n_tokens, float avg_logprob);

/* Per-item arguments of the batched entry points (transcribeWithOptions' decodeOptionsArray, WhisperKit.swift:716-735). */
typedef struct wk_batch_opts {
    const wk_decode_opts* opts;         /* n_opts == 1: shared by every window; else one per window */
    int32_t n_opts;
    const int32_t* const* prompts;      /* per-window initial prompts (prefillDecoderInputs output); NULL = one shared `prompt` */
    const int32_t* prompt_lens;
    const int32_t* prompt; int32_t n_prompt;   /* shared prompt when prompts == NULL; NULL too = built per window with wk_build_prompt */
    wk_progress_fn progress; void* progress_user;
    int32_t progress_every;             /* decoder steps between callbacks / completion polls; <= 0 = 16 */
    wk_status* status;                  /* per-window Result<> (WhisperKit.swift:775-790): WK_OK or that window's error; may be NULL */
    int32_t encoder_chunk;              /* windows per mel+encoder pass; <= 0 = the model's max_batch */
    /* Best-of-N sampling inside the temperature ladder (openai/whisper best_of with decode_with_fallback's per-rung rule; the reference's
     * DecodingOptions has no bestOf, so this is an extension like wk_decode_opts.beam_size).  One value per call: it sizes the rows every
     * window holds.  0 = off (the zeroed struct; the field sits in what was tail padding): every call decodes as before, and a beam call
     * skips the ladder.  1..8: on every rung of the ladder (which now runs for beam calls too), temperature 0 decodes with beam_size beams
     * if beam_size > 1, else one row; temperature > 0 draws best_of independent samples if best_of > 1 (row j of the group: Philox
     * subsequence = its decode row), else one row.  The kept sample maximises the sum of its token log-probs / max(sampled tokens, 1),
     * ties to the lowest row, and then goes through DecodingFallback as usual.  Each window takes G = max(beam_size, best_of) decode rows
     * for the whole call, so a session holds max_batch / G windows in flight; a rung that uses fewer rows (the greedy rung of
     * beam_size 1, best_of 5 uses one of five) leaves the others idle.  G must fit the session's rows.  Word timestamps work with
     * beam_size <= 1: the kept sample's alignment rows are returned. */
    int32_t best_of;
} wk_batch_opts;

/* ---- whole hot path: host PCM in, token IDs out (TranscribeTask.run body, batched) ----
 * Windows are independent units.  The session's max_batch decode slots run as one device-resident loop; a window that ends (EOT,
 * sampleLength, first-token threshold, early stop) retires from every kernel of the step at once and its slot is handed to the next
 * encoded window, while the mel + encoder pass of the following chunk runs on a second stream (tensor-bound encoder under the
 * HBM-bound decode).  The temperature ladder re-admits a window that asks for a fallback into its own slot (cross K/V kept). */
wk_status wk_transcribe_windows(wk_model* m, wk_session* s, const float* pcm_host /* host (pageable/pinned) or device */, int64_t n_windows, int64_t stride,
                                const int32_t* samples_per_window, const wk_special_tokens* st, const wk_decode_opts* opts,
                                const int32_t* prompt, int32_t n_prompt, wk_decode_result* results);
/* decodeText on the bound windows with per-window options / prompts / status and the progress callback (no temperature ladder, like
 * TextDecoding.decodeText itself). */
wk_status wk_decode_text_ex(wk_session* s, const wk_special_tokens* st, const wk_batch_opts* bo, wk_decode_result* results);
/* Same with per-window options / prompts / status and a progress callback.  Returns WK_OK when the call itself ran; per-window
 * failures are reported through bo->status (and fail the call only when status is NULL). */
wk_status wk_transcribe_windows_ex(wk_model* m, wk_session* s, const float* pcm_host, int64_t n_windows, int64_t stride,
                                   const int32_t* samples_per_window, const wk_special_tokens* st, const wk_batch_opts* bo,
                                   wk_decode_result* results);
/* Speculative greedy decoding with the model's draft decoder: wk_transcribe_windows_ex / wk_decode_text_ex with draft_tokens = k
 * (0 = the plain entries).  The setting is an argument, not a wk_batch_opts field, so that struct keeps its size and layout for callers
 * built against it.  Each window takes G = k + 1 decode rows, so a session holds max_batch / G windows in flight.  On a
 * temperature-0 rung, once a window is past its prompt, every step of the loop becomes a round: the draft proposes k tokens, the model's
 * decoder checks all k + 1 positions in one step, and the longest prefix on which they agree is committed together with the model's own
 * next token.  The draft only changes how many decoder steps run, never which tokens come out: compared with the plain entry on a session
 * with as many decode slots, the result of every window decoded at temperature 0 is byte-identical, and so is every window's result
 * when the call has no more windows than slots.  A draw at temperature > 0 (a hotter ladder rung, a first rung above 0, language
 * detection on such a rung) uses the Philox subsequence of the window's slot; with more windows than slots, the slot a window is admitted
 * to depends on when earlier windows retire, which the draft changes, so such a window draws a different, equally valid sample.
 * Prompts and rungs at temperature > 0 advance one token per round.
 * One exception: a progress callback that stops a window takes effect at a round boundary, so such a window may carry up to k more
 * tokens; progress_every counts rounds.  Refused (WK_ERR_INVALID_ARGUMENT): a model without a draft decoder, k outside [1, 7], G above
 * the session's rows, beam_size > 1, best_of >= 1 and word timestamps. */
wk_status wk_transcribe_windows_draft(wk_model* m, wk_session* s, const float* pcm_host, int64_t n_windows, int64_t stride,
                                      const int32_t* samples_per_window, const wk_special_tokens* st, const wk_batch_opts* bo,
                                      int32_t draft_tokens, wk_decode_result* results);
wk_status wk_decode_text_draft(wk_session* s, const wk_special_tokens* st, const wk_batch_opts* bo, int32_t draft_tokens,
                               wk_decode_result* results);

/* ---- contextual biasing (DecodingOptions.biasPhrases): boost caller-given token phrases inside the fused decode loop ----
 * A set is P phrases (1..256) of 1..16 text token ids each (ids below special_token_begin), 1024 ids in all, and one boost λ >= 0.
 * Every decode row keeps a KMP match length m_p per phrase, 0 at its first sampled position (forced prompt tokens and detection steps
 * leave it alone; every window and every ladder rung starts over).  With G = max_p m_p and g(v) = max_p δ_p(m_p, v) (the match length
 * token v leads to, a completion counting as the phrase's length), token v gets b(v) = λ·(g(v) - G) on top of the filtered logits:
 * a partial match earns λ per token, breaking it takes that back, and completing a phrase keeps it.  Suppressed tokens stay
 * suppressed.  The choice (argmax, the top-k draw, beam ranking, the finished list and the best-of pick) follows the biased scores;
 * every reported value (token log-probs, avgLogProb, the fallback thresholds, compressionRatio, noSpeechProb, word timings) stays the
 * model's own.  λ = 0 decodes byte-identically to no set. */
typedef struct wk_bias wk_bias;
/* host only: validates the phrases (tokens: the phrases back to back, phrase_lens: their lengths) and builds the match tables */
wk_status wk_bias_create(const int32_t* tokens, const int32_t* phrase_lens, int32_t n_phrases, float boost, int32_t special_token_begin,
                         wk_bias** out);
void wk_bias_free(wk_bias* b);
/* Attaches sets to the session's following calls (copied: the sets may be freed afterwards); n_sets = 0 detaches.  n_sets = 1: every
 * window; else one per window (wk_transcribe_windows*, wk_decode_text*) or per stream (wk_transcribe_streams*), a call of another size
 * failing with WK_ERR_INVALID_ARGUMENT.  A NULL entry leaves its window unbiased; a set passed twice is stored once.  While a set is
 * attached the draft entry points and wk_streamer_round return WK_ERR_INVALID_ARGUMENT. */
wk_status wk_session_set_bias(wk_session* s, const wk_bias* const* sets, int64_t n_sets);

/* ---- top log-probs (DecodingOptions.topLogProbs): the k most likely tokens at every sampled position ----
 * k in [0, 20] applies to the session's following calls; 0 (the default) turns it off.  At every position the loop sampled and
 * appended, the sampler ranks the candidates its choice was made from: the filtered row over the range the draw uses (only the
 * timestamp tokens when the timestamp rule wins), larger value first, ties to the lower id.  Each carries the log-prob its token would
 * have been reported with: the filtered log-softmax at temperature 0, the log of the tempered probability before the top-k cut at
 * temperature > 0, and with a bias set the model's unbiased values and ranking.  At temperature 0 without bias, entry 0 is the
 * sampled token and its log-prob.  Forced prompt positions and the closing EOT (whose token log-prob is the 0 that finalize appends)
 * get none.  Calls with beam_size > 1, draft_tokens, the stream stop rule and wk_streamer_create return WK_ERR_INVALID_ARGUMENT while
 * k > 0, as does k outside [0, 20]. */
wk_status wk_session_set_top_logprobs(wk_session* s, int32_t k);
/* The pairs of one window of the session's last batched call (wk_transcribe_windows*, wk_decode_text*) for its result tokens [0, n):
 * tokens / logprobs [n][k] with k the setting the call ran with, best first, padded with -1 / -inf (positions without candidates,
 * fewer finite candidates than k, positions >= the result's n_tokens).  Nothing is written when the call ran with k = 0. */
wk_status wk_session_top_logprobs(const wk_session* s, int32_t window, int32_t n, int32_t* tokens, float* logprobs);

/* ---- multi-GPU edges (SURVEY section 8e): one process per GPU, windows sharded, weights replicated; NCCL only moves PCM out and
 * results back (grouped ncclSend / ncclRecv over NVLink).  NCCL is resolved at run time from the process; wk_comm_unique_id fails with
 * WK_ERR_MODELS_UNAVAILABLE if it is not there.  The 128-byte id from rank 0 reaches the other ranks by whatever the host uses for
 * rendezvous (torch.distributed in bench.py, MPI, a file). */
typedef struct wk_comm wk_comm;
void wk_comm_shard_bounds(int64_t n_windows, int32_t world, int32_t rank, int64_t* lo, int64_t* hi);   /* contiguous, order preserving */
wk_status wk_comm_unique_id(uint8_t* out128);
wk_status wk_comm_create(const uint8_t* id128, int32_t rank, int32_t world, int32_t device, wk_comm** out);
void wk_comm_free(wk_comm* c);
/* root holds all_pcm [n_windows][stride] (host or device); every rank receives its shard into shard_dev (device). */
wk_status wk_comm_scatter_windows(wk_comm* c, const float* all_pcm, int64_t n_windows, int64_t stride, int32_t root, float* shard_dev, int64_t* n_local);
/* every rank hands in the results of its shard; root receives all n_windows in window order. */
wk_status wk_comm_gather_results(wk_comm* c, const wk_decode_result* local, int64_t n_local, int64_t n_windows, int32_t root, wk_decode_result* all);
/* scatter -> wk_transcribe_windows_ex on the shard -> gather; bo must carry shared options (n_opts == 1, no per-window arrays). */
wk_status wk_transcribe_windows_sharded(wk_comm* c, wk_model* m, wk_session* s, const float* all_pcm, int64_t n_windows, int64_t stride, int32_t root,
                                        const wk_special_tokens* st, const wk_batch_opts* bo, wk_decode_result* results);
/* host wall-clock milliseconds of the last sharded call on this rank: [0] scatter [1] transcribe [2] gather [3] total */
wk_status wk_comm_last_stage_ms(const wk_comm* c, float* ms4);

/* ---- long-form windowing (SURVEY section 8f rows 1 and 3): host logic, callable without a GPU ---- */
typedef struct wk_tokenizer_hooks wk_tokenizer_hooks;   /* defined with the word-timestamp API below */
typedef struct wk_word wk_word;
typedef struct wk_segment {             /* TranscriptionSegment (Models.swift), token-level fields */
    int32_t stream, id;
    int64_t seek;                       /* window start sample inside the stream */
    float start, end;                   /* seconds from the start of the stream */
    int64_t token_offset; int32_t n_tokens; /* slice of the flat token / logprob arrays */
    float temperature, avg_logprob, compression_ratio, no_speech_prob;
} wk_segment;
/* SegmentSeeking.findSeekPointAndSegments (Sources/WhisperKit/Core/Text/SegmentSeeker.swift:41-189).
 * *n_segs = -1 means the Swift function returned nil segments (window skipped as silent). token_offset is relative to `tokens`. */
wk_status wk_find_seek_point_and_segments(const int32_t* tokens, const float* token_logprobs, int32_t n_tokens, float no_speech_prob,
                                          float avg_logprob, float compression_ratio, float temperature, const wk_decode_opts* opts,
                                          int32_t all_segments_count, int64_t current_seek, int64_t segment_size, int32_t sample_rate,
                                          int32_t time_token, int64_t* new_seek, wk_segment* segs, int32_t cap, int32_t* n_segs);
/* DecodingOptions.prepareSeekClips (Sources/WhisperKit/Utilities/Extensions+Internal.swift:111-130); clips = [start0,end0,start1,...] */
wk_status wk_prepare_seek_clips(const float* clip_timestamps, int32_t n, int64_t content_frames, int64_t* clips, int32_t cap, int32_t* n_clips);
/* EnergyVAD.voiceActivity (EnergyVAD.swift:41-56, AudioProcessor.swift:674-702): RMS per frame > threshold */
wk_status wk_vad_voice_activity(const float* wav, int64_t n, int32_t frame_len, int32_t frame_overlap, float threshold, uint8_t* out,
                                int64_t cap, int64_t* n_frames);
/* VoiceActivityDetector.findLongestSilence (VoiceActivityDetector.swift:95-125); start = end = -1 when there is none */
wk_status wk_vad_find_longest_silence(const uint8_t* vad, int64_t n, int64_t* start, int64_t* end);
/* VoiceActivityDetector.calculateActiveChunks (:52-80); chunks = [start0,end0,...] */
wk_status wk_vad_active_chunks(const float* wav, int64_t n, int32_t frame_len, int32_t frame_overlap, float threshold, int64_t* chunks,
                               int32_t cap, int32_t* n_chunks);
/* VADAudioChunker.chunkAll (Sources/WhisperKit/Core/Audio/AudioChunker.swift:53-107); chunks = [seekOffsetIndex0,end0,...] */
wk_status wk_vad_chunk_all(const float* wav, int64_t n, int64_t max_chunk_len, const float* clip_timestamps, int32_t n_clip_timestamps,
                           int64_t window_padding, int32_t frame_len, int32_t frame_overlap, float threshold, int64_t* chunks, int32_t cap,
                           int32_t* n_chunks);
/* TranscribeTask.run's seek loop (TranscribeTask.swift:98-279) for MANY audio streams at once: every round the next <= 30 s
 * window of each unfinished stream is batched through the GPU path, then each stream's seek advances by its own decoded
 * timestamps.  chunking_vad != 0 first splits every stream with VADAudioChunker (WhisperKit.swift:878-911) so chunks become
 * independent units.  With opts->word_timestamps (and `hooks`, the host tokenizer) every window also runs addWordTimestamps
 * (TranscribeTask.swift:197-239): segment bounds follow the word timings, zero-length segments are dropped and the last word end
 * can pull the seek forward.  hooks may be NULL otherwise. */
typedef struct wk_transcription wk_transcription;
wk_status wk_transcribe_streams(wk_model* m, wk_session* s, const float* const* audio, const int64_t* n_samples, int32_t n_streams,
                                const wk_special_tokens* st, const wk_decode_opts* opts, const int32_t* prompt, int32_t n_prompt,
                                const float* clip_timestamps, int32_t n_clip_timestamps, float window_clip_time, int64_t max_window_seek,
                                int32_t chunking_vad, const wk_tokenizer_hooks* hooks, wk_transcription** out);
/* The same with wk_batch_opts.best_of for every window of the call (0 = wk_transcribe_streams). */
wk_status wk_transcribe_streams_ex(wk_model* m, wk_session* s, const float* const* audio, const int64_t* n_samples, int32_t n_streams,
                                   const wk_special_tokens* st, const wk_decode_opts* opts, const int32_t* prompt, int32_t n_prompt,
                                   const float* clip_timestamps, int32_t n_clip_timestamps, float window_clip_time, int64_t max_window_seek,
                                   int32_t chunking_vad, const wk_tokenizer_hooks* hooks, int32_t best_of, wk_transcription** out);
/* The same with speculative decoding (wk_transcribe_windows_draft) for every window of the call (0 = wk_transcribe_streams_ex). */
wk_status wk_transcribe_streams_draft(wk_model* m, wk_session* s, const float* const* audio, const int64_t* n_samples, int32_t n_streams,
                                      const wk_special_tokens* st, const wk_decode_opts* opts, const int32_t* prompt, int32_t n_prompt,
                                      const float* clip_timestamps, int32_t n_clip_timestamps, float window_clip_time, int64_t max_window_seek,
                                      int32_t chunking_vad, const wk_tokenizer_hooks* hooks, int32_t best_of, int32_t draft_tokens,
                                      wk_transcription** out);
int32_t wk_transcription_segment_count(const wk_transcription* t);
int32_t wk_transcription_window_count(const wk_transcription* t);
int64_t wk_transcription_token_count(const wk_transcription* t);
wk_status wk_transcription_segments(const wk_transcription* t, wk_segment* segs, int32_t cap);
wk_status wk_transcription_tokens(const wk_transcription* t, int32_t* tokens, float* logprobs, int64_t cap);
/* wk_session_top_logprobs for every entry of wk_transcription_tokens: [token_count][k] pairs, k the session's topLogProbs setting when
 * the call ran (cap: pairs the arrays hold, at least token_count * k); nothing when k was 0.  Refused with beam_size > 1 or draft_tokens. */
wk_status wk_transcription_top_logprobs(const wk_transcription* t, int32_t* tokens, float* logprobs, int64_t cap);
int32_t wk_transcription_word_count(const wk_transcription* t);
wk_status wk_transcription_word(const wk_transcription* t, int32_t i, wk_word* out);   /* .segment indexes wk_transcription_segments */
/* TranscriptionResult.language of one stream (TranscribeTask.swift:71,292,352): the language of the stream's last window (in stream time)
 * that detected one (opts->detect_language), else token -1 and log-prob 0. */
wk_status wk_transcription_language(const wk_transcription* t, int32_t stream, int32_t* token, float* logprob);
void wk_transcription_free(wk_transcription* t);

/* ---- live transcription of many streams (AudioStreamTranscriber, Sources/WhisperKit/Core/Audio/AudioStreamTranscriber.swift) ----
 * The caller pushes 16 kHz mono f32 audio per stream.  A round takes every stream whose new audio since its lastBufferSize passes
 * transcribeCurrentBuffer's gates (:126-158: more than 1 s, and AudioProcessor.isVoiceDetected when use_vad) and runs all of them in ONE
 * batched pass of the seek loop (TranscribeTask.run with clipTimestamps = [lastConfirmedSegmentEndSeconds], :195-206), with
 * shouldStopEarly (:208-227) applied deterministically inside the window scheduler: a window ends at its first appended token whose
 * history meets the rule, is finalized there and walks the temperature fallback ladder as usual.  Each stream then applies the
 * segment confirmation of :164-192.  A stream holds its audio from the current clip start on (its unconfirmed plus untranscribed
 * audio; all of it while nothing confirms, as in the reference). */
typedef struct wk_streamer wk_streamer;
typedef struct wk_stream_config {
    int32_t required_segments_for_confirmation;   /* requiredSegmentsForConfirmation (default 2) */
    float silence_threshold;                      /* silenceThreshold (default 0.3) */
    int32_t compression_check_window;             /* compressionCheckWindow (default 60, >= 1) */
    int32_t use_vad;                              /* useVAD (default 1) */
} wk_stream_config;
typedef struct wk_stream_state {                  /* AudioStreamTranscriber.State, the fields a server reads */
    int64_t last_buffer_size;                     /* samples the last transcription of this stream covered */
    float last_confirmed_segment_end_seconds;
    int32_t n_confirmed_segments, n_unconfirmed_segments;
    int32_t transcribed;                          /* the last round transcribed this stream */
    int64_t pushed_samples;                       /* samples pushed so far */
    int64_t held_samples;                         /* samples held: absolute [held_from, pushed_samples) */
    int64_t held_from;
    int64_t duplicate_confirmations;              /* rounds of this stream whose candidates were already confirmed (:178) */
} wk_stream_state;
/* One streamer per option set: opts (copied; beam_size > 1 is refused), the decoder prompt (prefillDecoderInputs), cfg.  hooks (copied;
 * the functions and user pointer must outlive the streamer) are required with opts->word_timestamps.  Rounds run on session s, which
 * must not be used by anything else while a round runs. */
wk_status wk_streamer_create(wk_model* m, wk_session* s, const wk_special_tokens* st, const wk_decode_opts* opts, const int32_t* prompt,
                             int32_t n_prompt, const wk_stream_config* cfg, const wk_tokenizer_hooks* hooks, wk_streamer** out);
wk_status wk_streamer_add_stream(wk_streamer* t, int32_t* id);
wk_status wk_streamer_remove_stream(wk_streamer* t, int32_t id);
/* AudioProcessor.processBuffer (AudioProcessor.swift:907-917): appends samples; one relative energy per complete 1600-sample block
 * counted from the start of the stream, whatever the push sizes.  Safe against a running round and against other pushes; a round holds
 * the lock a push takes only to read its streams' sizes and energies, and copies their audio after releasing it. */
wk_status wk_streamer_push(wk_streamer* t, int32_t id, const float* pcm, int64_t n);
/* One round over all streams; ids[0..*n) = the streams it transcribed (cap >= number of streams is always enough).  No ready stream:
 * no GPU work.  A failing round returns its error and changes no stream's state. */
wk_status wk_streamer_round(wk_streamer* t, int32_t* ids, int32_t cap, int32_t* n);
wk_status wk_streamer_state(wk_streamer* t, int32_t id, wk_stream_state* out);
/* confirmedSegments then unconfirmedSegments of one stream, read with the wk_transcription_* accessors (words included; stream 0 for
 * wk_transcription_language).  Free with wk_transcription_free. */
wk_status wk_streamer_result(wk_streamer* t, int32_t id, wk_transcription** out);
void wk_streamer_free(wk_streamer* t);
/* AudioProcessor's public helpers as the streams use them: relative energies of the complete 1600-sample blocks of pcm
 * (calculateRelativeEnergy against the lowest RMS of the previous <= 20 blocks, AudioProcessor.swift:724-741,907-917; the first block
 * has no reference and is 0), and isVoiceDetected (:636-655). */
wk_status wk_stream_relative_energy(const float* pcm, int64_t n, float* out, int64_t cap, int64_t* n_blocks);
wk_status wk_stream_voice_detected(const float* energies, int64_t n, float next_buffer_seconds, float silence_threshold, int32_t* out);

/* ---- word timestamps (SURVEY section 8f row 1) ----
 * Device side: with wk_decode_opts.word_timestamps set, every decode step also writes the mean cross-attention softmax row of the
 * model's alignment heads into row tokenIndex + 1 of a [224][1500] Float16 tensor per window - the decoder model's
 * `alignment_heads_weights` output spliced by TextDecoder.updateAlignmentWeights (TextDecoder.swift:272-296,310,414,709-717).
 * Host side (C++, callable without a GPU): SegmentSeeker's DTW / alignment / punctuation / duration logic
 * (SegmentSeeker.swift:195-659).  The tokenizer stays with the host and is reached through wk_tokenizer_hooks. */
/* (layer, head) pairs, e.g. openai-whisper's per-checkpoint alignment heads; n_pairs = 0 restores the default
 * (all heads of the last half of the decoder layers). */
wk_status wk_model_set_alignment_heads(wk_model* m, const int32_t* layer_head_pairs, int32_t n_pairs);
/* DecodingResult.cache.alignmentWeights of one window of the last wk_decode_text, first `rows` rows, as f32 [rows][n_audio_ctx]. */
wk_status wk_session_alignment_weights(wk_session* s, int32_t window, int32_t rows, float* out);
/* The same rows as stored, Float16 (FloatType): an asynchronous device-to-host copy on the session stream into out (pinned memory for it
 * to be truly asynchronous); sync != 0 waits for it and for every copy queued before it. */
wk_status wk_session_alignment_weights_f16(wk_session* s, int32_t window, int32_t rows, uint16_t* out, int32_t sync);

/* ---- forced alignment of given token sequences (openai-whisper timing.py find_alignment) ----
 * One teacher-forced decoder pass over every position of every sequence: word timings for any transcript (edited text, subtitles, another
 * system's output, beam-search results) and the model's per-token log-probs of it.  Sequence w is tokens[offsets[w] .. offsets[w + 1]): the
 * full decoder input as the decode loop consumes it - prompt, text, EOT (DecodingResult.tokens can be passed back unchanged).  It must hold
 * 1..224 ids below the vocabulary size; a sequence that does not fails its own window (status[w]; status may be NULL, then the first
 * failure fails the call), the other windows still run.  Outputs stay in the session until its next call:
 *   wk_session_alignment_weights(_f16)  rows 0..n of window w: row t + 1 = the alignment heads' mean cross-attention row at input
 *                                        position t (Float16), row 0 = 0 - the decode loop's layout, ready for wk_find_alignment /
 *                                        wk_add_word_timestamps
 *   wk_session_aligned_logprobs          n values: [t] = log softmax(logits[t - 1][:end_token])[tokens[t]] for t >= 1 (raw logits, no
 *                                        filters, temperature 1), NaN at t = 0 and where tokens[t] >= end_token
 * Results do not depend on the other windows of the call. */
/* against the encoder output bound with wk_session_set_encoder_output (n_windows <= bound windows; window w = bound window w) */
wk_status wk_align_tokens(wk_session* s, const wk_special_tokens* st, const int32_t* tokens, const int32_t* offsets, int64_t n_windows,
                          int32_t* status);
/* from PCM, as wk_transcribe_windows takes it (mel, encoder and cross K/V per chunk of the session's slots) */
wk_status wk_align_windows(wk_model* m, wk_session* s, const float* pcm_host, int64_t n_windows, int64_t stride, const int32_t* samples_per_window,
                           const wk_special_tokens* st, const int32_t* tokens, const int32_t* offsets, int32_t* status);
wk_status wk_session_aligned_logprobs(const wk_session* s, int32_t window, int32_t n, float* out);

struct wk_word {                   /* WordTiming (Models.swift:617-633) */
    const char* word;              /* UTF-8, NUL-terminated */
    const int32_t* tokens; int32_t n_tokens;
    float start, end, probability;
    int32_t segment;               /* set by the segment update: index of the segment that owns the word, else -1 */
};
typedef struct wk_words wk_words;  /* owning word list returned by the functions below */
int32_t wk_words_count(const wk_words* w);
wk_status wk_words_get(const wk_words* w, int32_t i, wk_word* out);   /* pointers stay valid until wk_words_free */
void wk_words_free(wk_words* w);

struct wk_tokenizer_hooks {
    /* WhisperTokenizer.splitToWordTokens (Models.swift:1291-1306): write the words as consecutive NUL-terminated UTF-8 strings into
     * `text` and each word's token count into `counts`; return the number of words, or < 0 on error / overflow. */
    int32_t (*split_to_word_tokens)(void* user, const int32_t* tokens, int32_t n_tokens, char* text, int32_t text_cap, int32_t* counts, int32_t counts_cap);
    /* WhisperTokenizer.decode(tokens:): NUL-terminated UTF-8 into `text`; return bytes written (without NUL) or < 0. May be NULL. */
    int32_t (*decode)(void* user, const int32_t* tokens, int32_t n_tokens, char* text, int32_t text_cap);
    void* user;
};

/* SegmentSeeker.dynamicTimeWarping (SegmentSeeker.swift:195-276); matrix row-major [rows][ld], dtype WK_DTYPE_F32 or WK_DTYPE_F16.
 * The path has at most rows + cols entries. */
wk_status wk_dtw(const void* matrix, int32_t dtype, int32_t rows, int32_t cols, int64_t ld, int32_t* text_indices, int32_t* time_indices,
                 int32_t cap, int32_t* n_path);
/* findAlignment (:340-408); `words` carry word + tokens (the host's splitToWordTokens), timings are ignored. */
wk_status wk_find_alignment(const wk_word* words, int32_t n_words, const void* matrix, int32_t dtype, int32_t rows, int32_t cols, int64_t ld,
                            const float* token_logprobs, int32_t n_logprobs, wk_words** out);
/* mergePunctuations (:278-338); NULL prepended/appended = Constants.default{Prepend,Append}Punctuations (Models.swift:1459-1460). */
wk_status wk_merge_punctuations(const wk_word* alignment, int32_t n, const char* prepended, const char* appended, wk_words** out);
/* calculateWordDurationConstraints (:498-508) and truncateLongWordsAtSentenceBoundaries (:510-526). */
wk_status wk_word_duration_constraints(const wk_word* alignment, int32_t n, float* constrained_median, float* max_duration);
wk_status wk_truncate_long_words(const wk_word* alignment, int32_t n, float max_duration, wk_words** out);
/* updateSegmentsWithWordTimings (:528-659): segs[i].start/end are updated in place; segment tokens are
 * tokens[segs[i].token_offset .. + n_tokens); out = every word with .segment set. */
wk_status wk_update_segments_with_word_timings(wk_segment* segs, int32_t n_segs, const int32_t* tokens, const wk_word* merged, int32_t n_merged,
                                               int64_t seek, float last_speech_timestamp, float constrained_median, float max_duration,
                                               int32_t special_token_begin, const wk_tokenizer_hooks* hooks, wk_words** out);
/* addWordTimestamps (:410-496), the whole per-window word-timing pass; alignment = [rows][ld] with row i = window token i. */
wk_status wk_add_word_timestamps(wk_segment* segs, int32_t n_segs, const int32_t* tokens, const float* token_logprobs,
                                 const void* alignment, int32_t dtype, int32_t rows, int32_t cols, int64_t ld,
                                 const wk_tokenizer_hooks* hooks, int64_t seek, float last_speech_timestamp, int32_t special_token_begin,
                                 const char* prepended, const char* appended, wk_words** out);

/* ---- tokenizer, decode side (SURVEY section 8f row 4): ids -> text without a Swift host ----
 * Byte-level BPE decode as swift-transformers does it (Tokenizer.swift:510-530, Decoder.swift:126-170): added tokens verbatim, the rest
 * through the GPT-2 byte alphabet into lossy UTF-8, then cleanUp; WhisperTokenizerWrapper's special-token lookups and word splitting
 * (Models.swift:1201-1306).  wk_tokenizer_encode is text -> ids WITHOUT the post-processor (no <|startoftranscript|> ... template): the
 * reference filters special tokens out of encoded prompts anyway (TranscribeCLIUtils / promptTokens). */
typedef struct wk_tokenizer wk_tokenizer;
/* path: a checkpoint directory (tokenizer.json, else vocab.json + added_tokens.json), or one of those files. */
wk_status wk_tokenizer_load(const char* path, wk_tokenizer** out);
/* From memory: flags bit 0 = added token (emitted verbatim), bit 1 = special (dropped by skip_special_tokens). */
wk_status wk_tokenizer_create(const char* const* tokens, const int32_t* ids, const uint8_t* flags, int32_t n, int32_t clean_up_tokenization_spaces,
                              wk_tokenizer** out);
void wk_tokenizer_free(wk_tokenizer* t);
int32_t wk_tokenizer_vocab_size(const wk_tokenizer* t);
int32_t wk_tokenizer_token_to_id(const wk_tokenizer* t, const char* token);   /* convertTokenToId; -1 = nil */
/* decode(tokens:skipSpecialTokens:): NUL-terminated UTF-8 into text; returns bytes written (without NUL), or -(bytes needed) if cap is short. */
int32_t wk_tokenizer_decode(const wk_tokenizer* t, const int32_t* tokens, int32_t n, int32_t skip_special_tokens, char* text, int32_t cap);
/* encode(text:) minus the post-processor: added tokens verbatim, then the GPT-2 pre-tokenizer pattern, byte alphabet and BPE merges
 * (merges come from tokenizer.json / merges.txt, or wk_tokenizer_set_merges).  Returns the id count, or -(ids needed) if cap is short. */
int32_t wk_tokenizer_encode(const wk_tokenizer* t, const char* text_utf8, int32_t* ids, int32_t cap);
wk_status wk_tokenizer_set_merges(wk_tokenizer* t, const char* const* left, const char* const* right, int32_t n);
/* SpecialTokens as WhisperTokenizerWrapper.init derives them, with its defaults for absent tokens. */
wk_status wk_tokenizer_special_tokens(const wk_tokenizer* t, wk_special_tokens* out);
/* splitToWordTokens in the wk_tokenizer_hooks layout (words as consecutive NUL-terminated strings, one token count per word; a NUL
 * byte inside a decoded word is dropped). */
int32_t wk_tokenizer_split_to_word_tokens(const wk_tokenizer* t, const int32_t* tokens, int32_t n, char* text, int32_t text_cap, int32_t* counts,
                                          int32_t counts_cap);
/* Fills `hooks` with this tokenizer's split / decode so wk_transcribe_streams and wk_add_word_timestamps run without host callbacks. */
wk_status wk_tokenizer_hooks_init(wk_tokenizer* t, wk_tokenizer_hooks* hooks);

/* ---- result writers (SURVEY section 8f row 4; Sources/WhisperKit/Utilities/ResultWriter.swift) ----
 * Cues are flat: one per word where the segment has word timings, else one per segment (the order WriteSRT / WriteVTT iterate).
 * Each function writes NUL-terminated UTF-8 into out and returns the byte count (without NUL), or -(bytes needed) if cap is short. */
int32_t wk_format_time(float seconds, int32_t always_include_hours, const char* decimal_marker, char* out, int32_t cap);   /* ResultWriting.formatTime, :14-26 */
int32_t wk_write_srt(const float* starts, const float* ends, const char* const* texts, int32_t n, char* out, int32_t cap);   /* WriteSRT, :70-101 */
int32_t wk_write_vtt(const float* starts, const float* ends, const char* const* texts, int32_t n, char* out, int32_t cap);   /* WriteVTT, :103-134 */

/* ---- instrumentation ---- */
/* Number of kernels launched by this library on the calling process since the last reset. */
int64_t wk_kernel_launch_count(int32_t reset);
/* Bytes of device and pinned host memory the library holds through its buffer owner (all models, sessions and workspaces of the
 * process; not wk_tensor data, which is stream-ordered).  Test instrumentation. */
wk_status wk_debug_live_bytes(int64_t* device_bytes, int64_t* pinned_bytes);
/* Last-run stage timings in ms, TranscriptionTimings buckets (Models.swift:730-776):
 * [0] logmels [1] encoding [2] crossKV [3] decodingLoop [4] h2d [5] d2h */
wk_status wk_last_timings(wk_model* m, float* ms6);
/* Stream all work is enqueued on (cudaStream_t as void*), for CUDA-event timing by the host harness. */
void* wk_model_stream(wk_model* m);

/* ---- kernel-level test/bench hooks (used by tests/ and bench.py; device pointers) ---- */
/* C[M,N] = A[M,K] * W[N,K]^T (+bias) with the wgmma GEMM; out_dtype WK_DTYPE_BF16/F16/F32. */
wk_status wk_test_gemm(wk_model* m, const void* a, const void* w, const float* bias, void* out, int32_t M, int32_t N, int32_t K,
                       int32_t in_dtype, int32_t out_dtype, int32_t gelu);
/* out[M,N] (f32, in place) += A[M,K] * W[N,K]^T + bias: the residual-update epilogue of the encoder's out-proj / FC2. */
wk_status wk_test_gemm_residual(wk_model* m, const void* a, const void* w, const float* bias, float* out, int32_t M, int32_t N, int32_t K, int32_t in_dtype);
/* The FP8 encoder GEMM (wk_model_set_encoder_dtype) alone: a [M][K] E4M3 codes with block scales a_scale [K / 128][round_up(M, 128)]
 * (one per row and 128-column block), w [N][K] E4M3 with one scale per row w_scale [N]; N, K multiples of 128.  kind 0 (QKV):
 * out [M][N] dtype = (sum_kb (a w^T)[kb] * a_scale[kb][row]) * w_scale[col] + bias; kind 1 (FC1): the same value through exact GELU,
 * quantized per (row, 128-column block) into out [M][N] E4M3 and out_scale [N / 128][round_up(M, 128)]; kind 2 (FC2): out [M][N] f32
 * += the value. */
wk_status wk_test_gemm_fp8(wk_model* m, int32_t kind, const uint8_t* a, const float* a_scale, const uint8_t* w, const float* w_scale,
                           const float* bias, void* out, float* out_scale, int32_t M, int32_t N, int32_t K, int32_t dtype);
/* Same product through the decoder's swap-AB split-K path: out f32 [rows_x, N]. */
wk_status wk_test_gemm_splitk(wk_model* m, const void* w, const void* x, float* out, int32_t N, int32_t rows_x, int32_t K, int32_t in_dtype, int32_t splits);
/* Encoder attention on packed qkv [B*T, 3*d] -> out [B*T, d]. */
wk_status wk_test_attention(wk_model* m, const void* qkv, void* out, int32_t B, int32_t T, int32_t n_heads, int32_t dtype);
/* Decoder cross-attention kernel alone: q [B][H*64] f32, K/V [B][H][T][64] 16-bit -> out [B][H*64] 16-bit; done (device, may be NULL)
 * marks rows to skip. */
wk_status wk_test_cross_attention(wk_model* m, const float* q, const void* kcross, const void* vcross, void* out, int32_t B, int32_t H,
                                  int32_t T, int32_t dtype, const int32_t* done);
/* The beam-search form of the same kernel: groups of kv_div adjacent rows share one K/V block, K/V [B / kv_div][H][T][64]. */
wk_status wk_test_cross_attention_shared(wk_model* m, const float* q, const void* kcross, const void* vcross, void* out, int32_t B, int32_t H,
                                         int32_t T, int32_t dtype, const int32_t* done, int32_t kv_div);
/* FP8-cache form of both: K/V codes [B / kv_div][H][T][64] (E4M3) with row scales [B / kv_div][H][T] f32; dtype is the type of out;
 * kv_div = 1 runs the single-query kernel, 2..8 the beam kernel.  align_out (device, may be NULL): every head also writes its normalised
 * softmax row to align_out [H][B][T] (the word-timestamp export; runs the single-query kernel whatever kv_div is). */
wk_status wk_test_cross_attention_fp8(wk_model* m, const float* q, const uint8_t* kcodes, const uint8_t* vcodes, const float* kscale,
                                      const float* vscale, void* out, int32_t B, int32_t H, int32_t T, int32_t dtype, const int32_t* done,
                                      int32_t kv_div, float* align_out);
/* Packed bf16 cross K/V cache (the default cache of a bf16 model).  wk_test_cross_kv_project: the cross-K/V projection GEMM alone,
 * x [windows * T][d] times w [d][d] (+ bias [d], may be NULL) of one K or V, d = H * 64, bf16.  packed == 0: the 16-bit cache blocks
 * out [windows][H][T][64]; packed != 0: the packed blocks (T x 128 bytes each) in out and the row headers [windows][H][round_up(T, 16)]
 * in hdr. */
wk_status wk_test_cross_kv_project(wk_model* m, const void* x, const void* w, const float* bias, int32_t windows, int32_t T, int32_t H,
                                   int32_t packed, void* out, uint8_t* hdr);
/* wk_test_cross_attention_fp8 on the packed cache (blocks and headers as wk_test_cross_kv_project writes them); out is bf16. */
wk_status wk_test_cross_attention_packed(wk_model* m, const float* q, const void* kc, const void* vc, const uint8_t* khdr, const uint8_t* vhdr,
                                         void* out, int32_t B, int32_t H, int32_t T, const int32_t* done, int32_t kv_div, float* align_out);
/* The word-timestamp pass's cross-attention alone (bf16): q [nw * 224][H * 64] against the cache blocks of slots 0 .. nw - 1 (16-bit, or
 * packed when khdr / vhdr are not NULL), seq_len [nw] device -> out [nw * 224][H * 64]; then the export of the heads in `mask` into
 * acc [nw * 224][T] f32. */
wk_status wk_test_align_cross_attention(wk_model* m, const void* q, const void* kc, const void* vc, const uint8_t* khdr, const uint8_t* vhdr,
                                        const int32_t* seq_len, int32_t nw, int32_t H, int32_t T, uint32_t mask, void* out, float* acc);
/* Decoder self-attention kernel alone: qkv [B][3*H*64] f32 of the new token, caches [B][H][224][64] 16-bit (positions < pos[b] valid;
 * row pos[b] is appended), pos [B] device -> out [B][H*64] 16-bit. */
wk_status wk_test_self_attention(wk_model* m, const float* qkv, void* kcache, void* vcache, const int32_t* pos, void* out, int32_t B,
                                 int32_t H, int32_t dtype, const int32_t* done);
/* The decoder's swap-AB split-K GEMM alone, configured as the decode step configures it: W [N,K], x [rows_x,K] 16-bit (rows_x = the padded
 * batch Bp, a multiple of 16 <= 256) -> raw partials [splits][partial_cols][N] f32, written into the caller's buffer and nowhere else.
 * partial_cols = rows_x is the layer GEMM's form, partial_cols = B < rows_x (splits 1) the logits GEMM's. */
wk_status wk_test_gemm_partial(wk_model* m, const void* w, const void* x, float* partial_out, int32_t N, int32_t rows_x, int32_t partial_cols,
                               int32_t K, int32_t dtype, int32_t splits);
/* The split-K consumers on partials [splits][Bp][n] f32 (rows >= B are never read): kind 0 reduce + bias (may be NULL) + residual x [B][n]
 * f32 (in place) + LayerNorm -> out16 [B][n]; kind 1 reduce + bias + exact GELU -> out16 [B][n]. */
wk_status wk_test_decoder_reduce(wk_model* m, int32_t kind, const float* partial, int32_t splits, int32_t Bp, const float* bias, const float* gamma,
                                 const float* beta, float* x, void* out16, int32_t B, int32_t n, int32_t dtype);
/* Decoder self-attention on q|k|v split-K partials [splits][Bp][3*H*64] with biases bq / bv [H*64]; caches [B][H][224][64]; anc [B][224]
 * (may be NULL) names the cache row holding position t of row b (beam search).  The new K/V row goes to row b's own cache. */
wk_status wk_test_self_attention_splitk(wk_model* m, const float* partial, int32_t splits, int32_t Bp, const float* bq, const float* bv, void* kcache,
                                        void* vcache, const int32_t* pos, const int32_t* done, const int32_t* anc, void* out, int32_t B, int32_t H,
                                        int32_t dtype);
/* The K/V append a draft verification step runs before the self-attention: every row b with done[b] == 0 (done may be NULL) gets the
 * reduced, rounded k / v of its partials at position pos[b] of its own cache row, as wk_test_self_attention_splitk would write it. */
wk_status wk_test_kv_append(wk_model* m, const float* partial, int32_t splits, int32_t Bp, const float* bv, void* kcache, void* vcache,
                            const int32_t* pos, const int32_t* done, int32_t B, int32_t H, int32_t dtype);
/* Decoder cross-attention on q split-K partials [splits][Bp][H*64] with bias bq; K/V [B / kv_div][H][T][64] 16-bit, or E4M3 codes with row
 * scales [B / kv_div][H][T] when kscale / vscale are non-NULL; kv_div = 1 runs the single-query kernel, 2..8 the beam kernel. */
wk_status wk_test_cross_attention_splitk(wk_model* m, const float* partial, int32_t splits, int32_t Bp, const float* bq, const void* kcross,
                                         const void* vcross, const float* kscale, const float* vscale, void* out, int32_t B, int32_t H, int32_t T,
                                         int32_t dtype, const int32_t* done, int32_t kv_div);

/* Average device time (ms) of one launch of a named hot kernel on the live buffers, plus its algorithmic work
 * (bytes for HBM-bound kernels, FLOPs for tensor-bound ones): 0 decoder cross-attention, 1 encoder FC1 GEMM,
 * 2 log-mel, 3 encoder attention, 4 decoder QKV swap-AB GEMM, 5 encoder QKV GEMM.  Used by bench.py's roofline.
 * Kernel 0 of a session with an FP8 cross K/V cache runs the FP8 kernel and counts its bytes (codes + row scales). */
wk_status wk_bench_kernel(wk_model* m, wk_session* s, int32_t which, int32_t batch, int32_t iters, float* ms_out, double* work_out);

/* Debug readback of an internal device buffer converted to f32 (stage-by-stage parity debugging; see session.cu).  An FP8 cross K/V
 * cache (which = 15) is returned dequantized: code * row scale. */
wk_status wk_debug_read(wk_model* m, wk_session* s, int32_t which, int64_t offset_elems, float* dst, int64_t n);

#ifdef __cplusplus
}
#endif
#endif /* WKB200_H */
