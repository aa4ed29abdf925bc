// Audio loading: WAV (RIFF/WAVE) parse on the host, then on the GPU the reference's channel mix (AudioProcessor.convertToMono,
// Sources/WhisperKit/Core/Audio/AudioProcessor.swift:526-625) and a polyphase FIR resampler to 16 kHz mono, fused into one kernel that
// reads the frames in their stored format.  The host side reproduces loadAudio / loadAudioAsFloatArray's frame ranges (:229-350) and
// resampleAudio(fromFile:)'s read chunks (:381-450), because the reference normalises the mono mix's peak per read chunk.
//
// Resampler spec: scipy.signal.resample_poly(x, up, down) with its default Kaiser (beta 5) window and zero padding; up / down = 16000 / rate
// reduced.  The reference's AVAudioConverter has no portable definition; two deliberate differences from it:
//   1. one continuous filter runs over the whole selected range (the reference restarts its converter per read chunk and leaves seams);
//   2. the length is ceil(n * up / down); the reference sums per-chunk lengths, which differs by at most one sample on a partial last chunk.
//
// Memory is bounded: the selected range is processed in segments of output samples (plus the filter's input halo) through pinned host
// staging and a fixed-size device workspace.  Every output is computed from absolute indices in a fixed tap order, so the segment size never
// changes a bit of the result.
#include <math.h>
#include <stdio.h>
#include <string.h>
#include <sys/stat.h>

#include <algorithm>
#include <numeric>
#include <vector>

#include "audio.h"
#include "common.cuh"
#include "engine.h"

namespace wk {

constexpr int kOutRate = 16000;
constexpr int kMaxMixChannels = 64;     // channels of a file, and entries of a sumChannels index list
constexpr int kFirThreads = 256;
constexpr int kPeakFrames = 8192;       // frames per CTA of the peak pass
constexpr int64_t kDefaultReadFrames = 1323000;   // Constants.defaultAudioReadFrameSize
constexpr size_t kSegmentBytes = 32u << 20;        // default segment size: at most this many raw input bytes staged per segment ...
constexpr int64_t kSegmentOutputs = 1 << 22;       // ... and at most this many f32 outputs (16 MiB) written per segment
constexpr int kTabSmemFloats = 16384;   // coefficient tables up to 64 KB live in shared memory, larger ones are read through L1 / L2

// ------------------------------------------------------------------------------------------------ device side
struct MixParams {
    int fmt, bytes, channels;   // stored sample format (WK_AUDIO_*), bytes per sample, interleaved channels
    int sum;                    // 1: sumChannels with its per-chunk peak normalisation; 0: copy channel `ch`
    int ch, n_idx;
    int idx[kMaxMixChannels];   // sumChannels: the valid indices in list order, duplicates kept
};

struct FirParams {
    int up, down, p, r, taps, ld;   // ld: row stride of the [up][ld] coefficient table (taps rounded up to odd: no bank conflicts)
    int copy;                       // up == down == 1: the mono signal itself
    int tile;                       // outputs per CTA
    int tab_in_smem, stage_cap;
    int64_t n_in;
    const float* tab;
};

__device__ __forceinline__ float decode_sample(const uint8_t* p, int fmt) {
    switch (fmt) {
        case WK_AUDIO_U8: return (float)((int)p[0] - 128) / 128.f;
        case WK_AUDIO_S16: return (float)*reinterpret_cast<const int16_t*>(p) / 32768.f;
        case WK_AUDIO_S24: {
            const int v = (int)((uint32_t)p[0] << 8 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 24) >> 8;
            return (float)v / 8388608.f;
        }
        case WK_AUDIO_S32: return __int2float_rn(*reinterpret_cast<const int32_t*>(p)) / 2147483648.f;
        default: return *reinterpret_cast<const float*>(p);
    }
}

// largest c with starts[c] <= i (starts[0] = 0 <= i < starts[n])
__device__ __forceinline__ int find_chunk(const int64_t* starts, int n, int64_t i) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (starts[mid] <= i) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__device__ __forceinline__ float chunk_scale(const unsigned* peaks, int c) {
    // convertToMono: scale = maxOriginalPeak / max(monoPeak, 0.0001), in f32
    return __uint_as_float(peaks[2 * c]) / fmaxf(__uint_as_float(peaks[2 * c + 1]), 0.0001f);
}

// Mono value of frame i (relative to `raw`), before the chunk scale: the channel copy, or the f32 sum in list order starting from 0
__device__ __forceinline__ float mix_frame(const uint8_t* raw, const MixParams& mx, int64_t i) {
    const uint8_t* f = raw + i * (int64_t)(mx.channels * mx.bytes);
    if (!mx.sum) return decode_sample(f + mx.ch * mx.bytes, mx.fmt);
    float acc = 0.f;
    for (int k = 0; k < mx.n_idx; ++k) acc += decode_sample(f + mx.idx[k] * mx.bytes, mx.fmt);
    return acc;
}

// Peak pass (sumChannels over a multi-channel input): per read chunk, max |x| over the selected channels and max |mono sum|, kept as
// f32 bit patterns (non-negative floats order like their bits, so atomicMax on the patterns is an exact max).  Frames [f0, f0 + nf) of the
// selected range; raw holds frames from raw_first on.
__global__ void __launch_bounds__(256)
audio_peak_kernel(const uint8_t* __restrict__ raw, int64_t raw_first, MixParams mx, int64_t f0, int64_t nf,
                  const int64_t* __restrict__ starts, int n_chunks, unsigned* __restrict__ peaks) {
    const int64_t a = f0 + (int64_t)blockIdx.x * kPeakFrames;
    const int64_t b = min(a + kPeakFrames, f0 + nf);
    const int c_first = find_chunk(starts, n_chunks, a), c_last = find_chunk(starts, n_chunks, b - 1);
    const int bytes = mx.bytes, fb = mx.channels * bytes;
    float po = 0.f, pm = 0.f;
    int c = c_first;
    for (int64_t i = a + threadIdx.x; i < b; i += blockDim.x) {
        if (c_first != c_last) {   // this CTA straddles a chunk edge: flush on every change of chunk
            const int ci = find_chunk(starts, n_chunks, i);
            if (ci != c) {
                atomicMax(&peaks[2 * c], __float_as_uint(po));
                atomicMax(&peaks[2 * c + 1], __float_as_uint(pm));
                po = pm = 0.f;
                c = ci;
            }
        }
        const uint8_t* f = raw + (i - raw_first) * fb;
        float acc = 0.f;
        for (int k = 0; k < mx.n_idx; ++k) {
            const float x = decode_sample(f + mx.idx[k] * bytes, mx.fmt);
            po = fmaxf(po, fabsf(x));
            acc += x;
        }
        pm = fmaxf(pm, fabsf(acc));
    }
    if (c_first != c_last) {
        atomicMax(&peaks[2 * c], __float_as_uint(po));
        atomicMax(&peaks[2 * c + 1], __float_as_uint(pm));
        return;
    }
    __shared__ float red[2][8];
    po = warp_max(po);
    pm = warp_max(pm);
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = po; red[1][threadIdx.x >> 5] = pm; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w) { po = fmaxf(po, red[0][w]); pm = fmaxf(pm, red[1][w]); }
        atomicMax(&peaks[2 * c_first], __float_as_uint(po));
        atomicMax(&peaks[2 * c_first + 1], __float_as_uint(pm));
    }
}

// Fused decode + mix + polyphase FIR.  CTA = `tile` consecutive outputs [m0, m1) of the segment [o0, o_end).  Output m reads input frames
// i = i_max(m) - k, k = 0 .. taps - 1, with i_max(m) = floor(((m + r) * down - p) / up) and coefficient h[phi + k * up], phi = the remainder;
// frames outside [0, n_in) are zero.  The CTA decodes the frames it needs to mono once into shared memory (format -> f32, ordered channel
// sum, x its chunk's scale: the separate mono signal bit for bit), then every thread accumulates its outputs with FMAs in tap order k.
__global__ void __launch_bounds__(kFirThreads)
audio_fir_kernel(const uint8_t* __restrict__ raw, int64_t raw_first, MixParams mx, FirParams fp, const int64_t* __restrict__ starts,
                 int n_chunks, const unsigned* __restrict__ peaks, int64_t o0, int64_t o_end, float* __restrict__ out) {
    extern __shared__ __align__(16) float smem[];
    const int64_t m0 = o0 + (int64_t)blockIdx.x * fp.tile;
    const int64_t m1 = min(m0 + fp.tile, o_end);
    const uint8_t* rb = raw - raw_first * (int64_t)(mx.channels * mx.bytes);   // rb indexes frames of the selected range
    if (fp.copy) {
        for (int64_t m = m0 + threadIdx.x; m < m1; m += blockDim.x) {
            float v = mix_frame(rb, mx, m);
            if (mx.sum) v *= chunk_scale(peaks, find_chunk(starts, n_chunks, m));
            out[m - o0] = v;
        }
        return;
    }
    const int up = fp.up, down = fp.down, taps = fp.taps;
    const int64_t lo = ((m0 + fp.r) * down - fp.p) / up - taps + 1;
    const int64_t hi = ((m1 - 1 + fp.r) * down - fp.p) / up;   // inclusive
    float* stage = smem;
    const float* tab = fp.tab;
    if (fp.tab_in_smem) {
        float* t = smem + fp.stage_cap;
        const int n = up * fp.ld;
        for (int j = threadIdx.x; j < n; j += blockDim.x) t[j] = fp.tab[j];
        tab = t;
    }
    const int64_t a = max(lo, (int64_t)0), b = min(hi + 1, fp.n_in);
    int c_a = 0, c_b = 0;
    if (mx.sum && a < b) { c_a = find_chunk(starts, n_chunks, a); c_b = find_chunk(starts, n_chunks, b - 1); }
    const float s_a = (mx.sum && a < b) ? chunk_scale(peaks, c_a) : 1.f;
    for (int64_t i = lo + threadIdx.x; i <= hi; i += blockDim.x) {
        float v = 0.f;
        if (i >= 0 && i < fp.n_in) {
            v = mix_frame(rb, mx, i);
            if (mx.sum) v *= (c_a == c_b) ? s_a : chunk_scale(peaks, find_chunk(starts, n_chunks, i));
        }
        stage[i - lo] = v;
    }
    __syncthreads();
    for (int64_t m = m0 + threadIdx.x; m < m1; m += blockDim.x) {
        const int64_t t = (m + fp.r) * down - fp.p;
        const int64_t im = t / up;
        const int phi = (int)(t - im * up);
        const float* x = stage + (im - lo);
        const float* h = tab + (size_t)phi * fp.ld;
        float acc = 0.f;
        for (int k = 0; k < taps; ++k) acc = fmaf(x[-k], h[k], acc);
        out[m - o0] = acc;
    }
}

// ------------------------------------------------------------------------------------------------ host: WAV header
static const char* fmt_name(int f) {
    static const char* n[] = {"u8", "s16", "s24", "s32", "f32"};
    return f >= 0 && f < 5 ? n[f] : "?";
}
static int fmt_bytes(int f) { return f == WK_AUDIO_U8 ? 1 : f == WK_AUDIO_S16 ? 2 : f == WK_AUDIO_S24 ? 3 : 4; }

static uint32_t le32(const uint8_t* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }
static uint16_t le16(const uint8_t* p) { return (uint16_t)(p[0] | p[1] << 8); }

static const char* tag_name(int tag) {
    switch (tag) {
        case 0x0002: return "MS ADPCM";
        case 0x0006: return "A-law";
        case 0x0007: return "mu-law";
        case 0x0011: return "IMA ADPCM";
        case 0x0031: return "GSM 6.10";
        case 0x0050: return "MPEG";
        case 0x0055: return "MPEG layer 3";
        default: return "compressed";
    }
}

wk_status fail_load(const char* path, const char* what) {
    set_error("loadAudioFailed: %s: %s", path, what);
    return WK_ERR_LOAD_AUDIO_FAILED;
}

// RIFF/WAVE: PCM u8 / s16 / s24 / s32, IEEE float 32, EXTENSIBLE wrapping either.  Unknown chunks are skipped (odd sizes carry a pad
// byte); a data chunk shorter than its header says holds the frames that are present.
static wk_status parse_wav(FILE* f, const char* path, wk_audio_format* out) {
    struct stat sb;
    if (fstat(fileno(f), &sb) != 0) return fail_load(path, "cannot stat the file");
    const int64_t fsize = (int64_t)sb.st_size;
    uint8_t hdr[12];
    if (fread(hdr, 1, 12, f) != 12) return fail_load(path, "not a WAV file (shorter than a RIFF header)");
    if (!memcmp(hdr, "RIFX", 4)) return fail_load(path, "big-endian RIFX WAV is not supported");
    if (memcmp(hdr, "RIFF", 4) || memcmp(hdr + 8, "WAVE", 4)) return fail_load(path, "neither a RIFF/WAVE nor a FLAC file (WAV and FLAC are supported)");
    bool have_fmt = false, have_data = false;
    int tag = 0, channels = 0, bits = 0, block = 0;
    uint32_t rate = 0;
    int64_t data_off = 0, data_size = 0;
    int64_t pos = 12;
    while (pos + 8 <= fsize && !(have_fmt && have_data)) {
        uint8_t ch[8];
        if (fseeko(f, pos, SEEK_SET) != 0 || fread(ch, 1, 8, f) != 8) break;
        const int64_t size = le32(ch + 4);
        if (!memcmp(ch, "fmt ", 4)) {
            uint8_t b[40] = {0};
            const size_t want = (size_t)std::min<int64_t>(size, 40);
            if (size < 16 || fread(b, 1, want, f) != want) return fail_load(path, "truncated fmt chunk");
            tag = le16(b); channels = le16(b + 2); rate = le32(b + 4); block = le16(b + 12); bits = le16(b + 14);
            if (tag == 0xFFFE) {   // WAVE_FORMAT_EXTENSIBLE: the sub-format GUID starts with the format tag
                if (size < 40) return fail_load(path, "truncated WAVE_FORMAT_EXTENSIBLE fmt chunk");
                tag = le16(b + 24);
            }
            have_fmt = true;
        } else if (!memcmp(ch, "data", 4)) {
            data_off = pos + 8;
            data_size = std::min<int64_t>(size, fsize - data_off);
            have_data = true;
        }
        pos += 8 + size + (size & 1);
    }
    if (!have_fmt) return fail_load(path, "no fmt chunk");
    if (!have_data) return fail_load(path, "no data chunk");
    int fmt = -1;
    char msg[160];
    if (tag == 1) {
        fmt = bits == 8 ? WK_AUDIO_U8 : bits == 16 ? WK_AUDIO_S16 : bits == 24 ? WK_AUDIO_S24 : bits == 32 ? WK_AUDIO_S32 : -1;
        if (fmt < 0) { snprintf(msg, sizeof msg, "%d-bit integer PCM is not supported (8, 16, 24, 32)", bits); return fail_load(path, msg); }
    } else if (tag == 3) {
        if (bits != 32) { snprintf(msg, sizeof msg, "%d-bit float is not supported (32-bit only)", bits); return fail_load(path, msg); }
        fmt = WK_AUDIO_F32;
    } else {
        snprintf(msg, sizeof msg, "WAV format tag 0x%04x (%s) is not supported (PCM and IEEE float only)", tag, tag_name(tag));
        return fail_load(path, msg);
    }
    if (channels < 1 || channels > kMaxMixChannels) { snprintf(msg, sizeof msg, "%d channels (1..%d supported)", channels, kMaxMixChannels); return fail_load(path, msg); }
    if (block != channels * fmt_bytes(fmt)) { snprintf(msg, sizeof msg, "block align %d does not match %d channels of %s", block, channels, fmt_name(fmt)); return fail_load(path, msg); }
    out->sample_rate = (int32_t)std::min<uint32_t>(rate, 0x7fffffff);
    out->channels = channels;
    out->sample_format = fmt;
    out->block_align = block;
    out->frames = data_size / block;
    out->data_offset = data_off;
    return WK_OK;
}

// FLAC by its "fLaC" marker, optionally behind an ID3v2 tag; Ogg is refused by name; anything else goes to the WAV parser
static wk_status parse_audio(FILE* f, const char* path, wk_audio_format* out, FlacStream* fs, bool* is_flac) {
    uint8_t h[10] = {0};
    const size_t n = fread(h, 1, 10, f);
    *is_flac = false;
    int64_t start = 0;
    if (n == 10 && !memcmp(h, "ID3", 3)) {
        start = (int64_t)flac::id3v2_size(h);
        if (fseeko(f, start, SEEK_SET) != 0 || fread(h, 1, 4, f) != 4 || memcmp(h, "fLaC", 4))
            return fail_load(path, "an ID3v2 tag not followed by FLAC audio");
    }
    if (n >= 4 && !memcmp(h, "OggS", 4)) return fail_load(path, "Ogg files (Ogg-encapsulated FLAC included) are not supported");
    if (n >= 4 && !memcmp(h, "fLaC", 4)) {
        *is_flac = true;
        return flac_parse(f, path, start, out, fs);
    }
    if (fseeko(f, 0, SEEK_SET) != 0) return fail_load(path, "cannot seek in the file");
    return parse_wav(f, path, out);
}

// ------------------------------------------------------------------------------------------------ host: filter design
// scipy.special.i0 for the Kaiser window's arguments (0 <= x <= 5): the power series sum ((x/2)^k / k!)^2 has only positive terms
static double bessel_i0(double x) {
    const double q = 0.25 * x * x;
    double term = 1.0, sum = 1.0;
    for (int k = 1; k < 200; ++k) {
        term *= q / ((double)k * k);
        sum += term;
        if (term < 1e-18 * sum) break;
    }
    return sum;
}

static bool rate_ok(int64_t rate) { return rate >= 1000 && rate <= 384000; }

// up / down = 16000 / rate reduced
static void resample_ratio(int rate, int* up, int* down) {
    const int g = std::gcd(kOutRate, rate);
    *up = kOutRate / g;
    *down = rate / g;
}

// scipy.signal.resample_poly's filter: firwin(2 * half + 1, 1 / max(up, down), window=('kaiser', 5.0)) * up, half = 10 * max(up, down).
// Empty for 16 kHz (up == down == 1, an exact copy).
static void design_filter(int rate, int* up, int* down, std::vector<double>* h) {
    resample_ratio(rate, up, down);
    h->clear();
    if (*up == 1 && *down == 1) return;
    const int mr = std::max(*up, *down);
    const int64_t half = 10LL * mr, n = 2 * half + 1;
    const double cutoff = 1.0 / mr, alpha = 0.5 * (double)(n - 1), beta = 5.0, i0b = bessel_i0(beta);
    h->resize(n);
    double sum = 0.0, comp = 0.0;   // Neumaier-compensated sum of the taps (firwin's scale to unit DC gain)
    for (int64_t i = 0; i < n; ++i) {
        const double m = (double)i - alpha;
        const double x = M_PI * (cutoff * m);
        const double sinc = x == 0.0 ? 1.0 : sin(x) / x;
        const double r = (m) / alpha;
        const double w = bessel_i0(beta * sqrt(1.0 - r * r)) / i0b;
        const double v = cutoff * sinc * w;
        (*h)[i] = v;
        const double t = sum + v;
        comp += fabs(sum) >= fabs(v) ? (sum - t) + v : (v - t) + sum;
        sum = t;
    }
    sum += comp;
    for (auto& v : *h) v = v / sum * (double)*up;
}

// ------------------------------------------------------------------------------------------------ host: frame plan
struct Plan {
    int64_t first = 0, n = 0;          // selected frames [first, first + n) of the input
    std::vector<int64_t> starts;       // read chunks relative to `first`: chunk c = [starts[c], starts[c + 1]); starts.back() == n
};

// loadAudio (piece_seconds <= 0: one piece) or loadAudioAsFloatArray (pieces of piece_seconds): the frame ranges the reference reads,
// computed in double as AudioProcessor.swift:253-262 and :318-347 do, each split into reads of max_read frames (:408-447)
// min(Int64(x * sr), length) as the reference computes a frame position, clamped below at 0: the clamps only replace values for which
// the reference reads nothing (negative) or everything (at or past the end, +inf included), and keep the conversion defined
static int64_t frame_at(double x, double sr, int64_t length) {
    const double f = x * sr;
    if (!(f > 0.0)) return 0;
    if (f >= (double)length) return length;
    return (int64_t)f;
}

static wk_status make_plan(int64_t length, int rate, const wk_audio_load_opts* o, Plan* plan) {
    const double sr = (double)rate;
    const double start = o ? o->start_time : 0.0;
    const bool has_end = o && o->has_end_time;
    const int64_t max_read = (o && o->max_read_frame_size > 0) ? o->max_read_frame_size : kDefaultReadFrames;
    if (!(start >= 0.0) || !std::isfinite(start)) { set_error("audio: startTime %g must be finite and >= 0", start); return WK_ERR_INVALID_ARGUMENT; }
    if (has_end && std::isnan(o->end_time)) { set_error("audio: endTime is NaN"); return WK_ERR_INVALID_ARGUMENT; }
    if (o && (std::isnan(o->piece_seconds) || (o->piece_seconds > 0.0 && o->piece_seconds < 1.0))) {
        set_error("audio: piece_seconds %g must be <= 0 (one piece) or >= 1", o->piece_seconds);
        return WK_ERR_INVALID_ARGUMENT;
    }
    std::vector<std::pair<int64_t, int64_t>> pieces;
    if (!o || o->piece_seconds <= 0.0) {
        pieces.push_back({frame_at(start, sr, length), has_end ? frame_at(o->end_time, sr, length) : length});
    } else {
        const double duration = (double)length / sr;
        const double end = std::min(has_end ? o->end_time : duration, duration);
        for (double t = start; t < end;) {
            const double ce = std::min(t + o->piece_seconds, end);
            pieces.push_back({frame_at(t, sr, length), frame_at(ce, sr, length)});
            t = ce;
        }
    }
    // consecutive pieces are contiguous: piece k ends at the frame piece k + 1 starts from
    plan->starts.clear();
    plan->first = pieces.empty() ? 0 : std::min(pieces[0].first, length);
    int64_t cur = plan->first;
    for (auto& pc : pieces) {
        if (pc.second <= pc.first) continue;   // an empty range reads nothing
        for (int64_t p = pc.first; p < pc.second; p = cur) {
            plan->starts.push_back(p - plan->first);
            cur = std::min(p + max_read, pc.second);
        }
    }
    plan->n = cur - plan->first;
    plan->starts.push_back(plan->n);
    return WK_OK;
}

// convertToMono's channel selection (AudioProcessor.swift:567-622)
static wk_status make_mix(int fmt, int channels, const wk_audio_load_opts* o, MixParams* mx) {
    memset(mx, 0, sizeof(*mx));
    mx->fmt = fmt; mx->bytes = fmt_bytes(fmt); mx->channels = channels;
    if (channels <= 1) return WK_OK;   // already mono: unchanged
    const int mode = o ? o->channel_mode : WK_CHANNELS_SUM;
    if (mode == WK_CHANNELS_SPECIFIC) {
        mx->ch = (o->channel >= 0 && o->channel < channels) ? o->channel : 0;
        return WK_OK;
    }
    if (mode != WK_CHANNELS_SUM) { set_error("audio: channel_mode %d is neither sum (0) nor specific (1)", mode); return WK_ERR_INVALID_ARGUMENT; }
    std::vector<int> idx;
    if (o && o->channel_indices && o->n_channel_indices > 0) {
        for (int k = 0; k < o->n_channel_indices; ++k)
            if (o->channel_indices[k] >= 0 && o->channel_indices[k] < channels) idx.push_back(o->channel_indices[k]);
        if (idx.empty()) return WK_OK;   // no valid index: channel 0, not normalised
    } else {
        for (int c = 0; c < channels; ++c) idx.push_back(c);
    }
    if ((int)idx.size() > kMaxMixChannels) { set_error("audio: %zu channel indices (limit %d)", idx.size(), kMaxMixChannels); return WK_ERR_INVALID_ARGUMENT; }
    mx->sum = 1;
    mx->n_idx = (int)idx.size();
    for (size_t k = 0; k < idx.size(); ++k) mx->idx[k] = idx[k];
    return WK_OK;
}

// ------------------------------------------------------------------------------------------------ host: workspace and driver
void audio_ws_free(AudioWs* w) { delete w; }

// Where the stored frames come from: a WAV file (data chunk at data_offset), host memory, or device memory (read in place).
struct Source {
    FILE* file = nullptr; int64_t data_offset = 0;
    const uint8_t* host = nullptr;
    const uint8_t* dev = nullptr;
    int64_t first = 0;      // selected range start, in frames of the stored data
    int frame_bytes = 0;
    const char* path = "";
    const FlacStream* flac = nullptr;   // a FLAC file: frames are decoded on the device, in the container format of frame_bytes
};

static wk_status fill(const Source& src, int64_t a, int64_t b, uint8_t* dst) {
    const size_t bytes = (size_t)(b - a) * src.frame_bytes;
    const int64_t off = (src.first + a) * src.frame_bytes;
    if (src.host) { memcpy(dst, src.host + off, bytes); return WK_OK; }
    if (fseeko(src.file, src.data_offset + off, SEEK_SET) != 0 || fread(dst, 1, bytes, src.file) != bytes)
        return fail_load(src.path, "read error in the data chunk");
    return WK_OK;
}

struct Staging {
    AudioWs* w;
    const Source* src;
    int k = 0;
    // frames [a, b) of the selected range -> device; returns the device pointer and the frame it starts at
    wk_status stage(int64_t a, int64_t b, const uint8_t** raw, int64_t* raw_first) {
        if (src->dev) { *raw = src->dev + src->first * (int64_t)src->frame_bytes; *raw_first = 0; return WK_OK; }
        *raw = w->d_raw; *raw_first = a;
        if (b <= a) return WK_OK;
        if (src->flac) return flac_stage(w, *src->flac, src->first + a, src->first + b, k++ & 1);
        const int i = k++ & 1;
        WK_CUDA_CHECK(cudaEventSynchronize(w->ev_in[i]));   // the copy that last read this pinned buffer is done
        WK_CHECK(fill(*src, a, b, w->h_in[i]));
        WK_CUDA_CHECK(cudaMemcpyAsync(w->d_raw, w->h_in[i], (size_t)(b - a) * src->frame_bytes, cudaMemcpyHostToDevice, w->stream));
        WK_CUDA_CHECK(cudaEventRecord(w->ev_in[i], w->stream));
        return WK_OK;
    }
};

static bool is_device_ptr(const void* p) {
    cudaPointerAttributes at;
    const bool dev = p && cudaPointerGetAttributes(&at, p) == cudaSuccess && (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged);
    cudaGetLastError();
    return dev;
}

static int64_t out_len(int64_t n, int up, int down) { return (n * up + down - 1) / down; }

// Mix + resample the plan's frames of `src` into out (host or device) on the workspace's stream.  segment_samples: outputs per segment
// (0 = sized so that a segment stages at most about kSegmentBytes of input and writes at most kSegmentOutputs samples).  The segment never
// exceeds the call's output, so a short file allocates little; the workspace keeps the largest buffers a call needed, which these two
// limits bound.
static wk_status run_convert(AudioWs* w, const Source& src, int rate, const MixParams& mx, const Plan& plan, float* out, int64_t segment_samples) {
    int up, down;
    resample_ratio(rate, &up, &down);
    const int64_t n_in = plan.n, n_out = out_len(n_in, up, down);
    if (n_out == 0) return WK_OK;
    const bool copy = (up == 1 && down == 1);
    const int64_t half = 10LL * std::max(up, down);
    FirParams fp;
    memset(&fp, 0, sizeof(fp));
    fp.up = up; fp.down = down; fp.copy = copy; fp.n_in = n_in;
    if (!copy) {
        fp.p = (int)(down - half % down);
        fp.r = (int)((half + fp.p) / down);
        fp.taps = (int)((2 * half + 1 + up - 1) / up);
        fp.ld = fp.taps | 1;
        if (w->tab_rate != rate) {   // design and upload the table only when the workspace holds another rate's
            std::vector<double> h;
            design_filter(rate, &up, &down, &h);
            std::vector<float> tab((size_t)up * fp.ld, 0.f);
            for (int phi = 0; phi < up; ++phi)
                for (int k = 0; k < fp.taps; ++k) {
                    const int64_t j = phi + (int64_t)k * up;
                    if (j < (int64_t)h.size()) tab[(size_t)phi * fp.ld + k] = (float)h[j];
                }
            WK_CHECK(w->mem.grow(&w->d_tab, tab.size()));
            WK_CUDA_CHECK(cudaMemcpyAsync(w->d_tab, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice, w->stream));
            WK_CUDA_CHECK(cudaStreamSynchronize(w->stream));   // `tab` is pageable and goes out of scope
            w->tab_rate = rate;
        }
        fp.tab = w->d_tab;
        fp.tile = 4 * kFirThreads;
        if ((int64_t)(fp.tile - 1) * down / up + fp.taps + 2 > 4096) fp.tile = kFirThreads;
        fp.stage_cap = (int)(((int64_t)(fp.tile - 1) * down / up + fp.taps + 2 + 3) & ~3LL);
        fp.tab_in_smem = (int64_t)up * fp.ld <= kTabSmemFloats;
    } else {
        fp.tile = 4 * kFirThreads;
    }
    const int fb = src.frame_bytes;
    // segment size in outputs: a multiple of the tile, within the input and output limits, no larger than the output rounded up to a tile
    int64_t seg = segment_samples > 0 ? segment_samples
                                      : std::min<int64_t>(kSegmentOutputs, (int64_t)((double)kSegmentBytes / ((double)fb * down / up)));
    seg = std::max<int64_t>(fp.tile, seg / fp.tile * fp.tile);
    seg = std::min<int64_t>(seg, (n_out + fp.tile - 1) / fp.tile * fp.tile);
    // input frames one segment stages: the FIR segment's frames plus the filter halo; the peak pass uses segments of the same size
    const int64_t seg_in_frames = (seg - 1) * down / up + fp.taps + 2;
    const int n_chunks = (int)plan.starts.size() - 1;
    WK_CUDA_CHECK(cudaSetDevice(w->device));
    if (!src.dev) {
        WK_CHECK(w->mem.grow(&w->d_raw, (size_t)seg_in_frames * fb));
        for (uint8_t*& h : w->h_in) WK_CHECK(w->mem.grow_pinned(&h, (size_t)seg_in_frames * fb));
    }
    const bool out_dev = is_device_ptr(out);
    if (!out_dev) {
        WK_CHECK(w->mem.grow(&w->d_out, (size_t)seg));
        for (float*& h : w->h_out) WK_CHECK(w->mem.grow_pinned(&h, (size_t)seg));
    }
    for (int i = 0; i < 2; ++i) {
        if (!w->ev_in[i]) WK_CUDA_CHECK(cudaEventCreateWithFlags(&w->ev_in[i], cudaEventDisableTiming));
        if (!w->ev_out[i]) WK_CUDA_CHECK(cudaEventCreateWithFlags(&w->ev_out[i], cudaEventDisableTiming));
    }
    WK_CHECK(w->mem.grow(&w->d_starts, plan.starts.size()));
    WK_CHECK(w->mem.grow(&w->d_peaks, (size_t)std::max(n_chunks, 1) * 2));   // two peaks per chunk
    WK_CUDA_CHECK(cudaMemcpyAsync(w->d_starts, plan.starts.data(), plan.starts.size() * 8, cudaMemcpyHostToDevice, w->stream));
    WK_CUDA_CHECK(cudaMemsetAsync(w->d_peaks, 0, (size_t)std::max(n_chunks, 1) * 8, w->stream));
    WK_CUDA_CHECK(cudaStreamSynchronize(w->stream));   // plan.starts is pageable

    Staging st{w, &src};
    // pass 1: the per-chunk peaks of a normalised channel sum
    if (mx.sum) {
        const int64_t seg_frames = src.dev ? n_in : seg_in_frames;
        for (int64_t a = 0; a < n_in; a += seg_frames) {
            const int64_t b = std::min(n_in, a + seg_frames);
            const uint8_t* raw; int64_t raw_first;
            WK_CHECK(st.stage(a, b, &raw, &raw_first));
            const int64_t blocks = (b - a + kPeakFrames - 1) / kPeakFrames;
            audio_peak_kernel<<<(unsigned)blocks, 256, 0, w->stream>>>(raw, raw_first, mx, a, b - a, w->d_starts, n_chunks, w->d_peaks);
            count_launch();
        }
    }
    // pass 2: decode + mix + FIR, segment by segment
    const size_t smem = copy ? 0 : (size_t)(fp.stage_cap + (fp.tab_in_smem ? up * fp.ld : 0)) * 4;
    if (smem > 48 * 1024) WK_CUDA_CHECK(cudaFuncSetAttribute(audio_fir_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int64_t pend_o0 = -1, pend_n = 0; int pend_buf = 0;
    auto drain = [&]() -> wk_status {   // copy the previous segment's host output out of pinned staging
        if (pend_o0 < 0) return WK_OK;
        WK_CUDA_CHECK(cudaEventSynchronize(w->ev_out[pend_buf]));
        memcpy(out + pend_o0, w->h_out[pend_buf], (size_t)pend_n * 4);
        pend_o0 = -1;
        return WK_OK;
    };
    int k = 0;
    for (int64_t o0 = 0; o0 < n_out; o0 += seg, ++k) {
        const int64_t o1 = std::min(n_out, o0 + seg);
        int64_t a, b;
        if (copy) { a = o0; b = o1; }
        else {
            a = std::max<int64_t>(0, ((o0 + fp.r) * down - fp.p) / up - fp.taps + 1);
            b = std::min<int64_t>(n_in, ((o1 - 1 + fp.r) * down - fp.p) / up + 1);
        }
        const uint8_t* raw; int64_t raw_first;
        WK_CHECK(st.stage(a, std::max(a, b), &raw, &raw_first));
        float* dst = out_dev ? out + o0 : w->d_out;
        const int64_t blocks = (o1 - o0 + fp.tile - 1) / fp.tile;
        audio_fir_kernel<<<(unsigned)blocks, kFirThreads, smem, w->stream>>>(raw, raw_first, mx, fp, w->d_starts, n_chunks, w->d_peaks, o0, o1, dst);
        count_launch();
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) { set_error("audio kernel launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
        if (!out_dev) {
            const int i = k & 1;
            WK_CHECK(drain());
            WK_CUDA_CHECK(cudaMemcpyAsync(w->h_out[i], w->d_out, (size_t)(o1 - o0) * 4, cudaMemcpyDeviceToHost, w->stream));
            WK_CUDA_CHECK(cudaEventRecord(w->ev_out[i], w->stream));
            pend_o0 = o0; pend_n = o1 - o0; pend_buf = i;
        }
    }
    WK_CHECK(drain());
    WK_CUDA_CHECK(cudaStreamSynchronize(w->stream));
    return WK_OK;
}

// The session's workspace (created on first use), or one for this call alone on the current device when s is NULL
struct WsHandle {
    AudioWs* w = nullptr;
    bool temp = false;
    ~WsHandle() { if (temp) delete w; }
    wk_status open(wk_session* s) {
        if (!wk_device_available()) { set_error("audio: no sm_90 (Hopper) device"); return WK_ERR_MODELS_UNAVAILABLE; }
        if (s) {
            AudioWs** slot = session_audio_ws(s);
            if (!*slot) {
                *slot = new AudioWs();
                (*slot)->device = session_device(s);
                (*slot)->stream = session_stream(s);
            }
            w = *slot;
            WK_CUDA_CHECK(cudaSetDevice(w->device));
            return WK_OK;
        }
        w = new AudioWs();
        temp = true;
        WK_CUDA_CHECK(cudaGetDevice(&w->device));
        WK_CUDA_CHECK(cudaStreamCreateWithFlags(&w->stream, cudaStreamNonBlocking));
        w->own_stream = true;
        return WK_OK;
    }
};

static wk_status finish_len(int64_t n_out, float* out, int64_t cap, int64_t* n_out_p) {
    if (n_out_p) *n_out_p = n_out;
    if (out && cap < n_out) { set_error("audio: output capacity %lld < %lld samples", (long long)cap, (long long)n_out); return WK_ERR_INVALID_ARGUMENT; }
    return WK_OK;
}

}  // namespace wk

using namespace wk;

wk_status wk_audio_info(const char* path, wk_audio_format* out) {
    if (!path || !out) { set_error("wk_audio_info: null argument"); return WK_ERR_INVALID_ARGUMENT; }
    FILE* f = fopen(path, "rb");
    if (!f) return fail_load(path, "resource path does not exist or cannot be opened");
    FlacStream fs;
    bool is_flac;
    const wk_status st = parse_audio(f, path, out, &fs, &is_flac);
    fclose(f);
    return st;
}

wk_status wk_audio_filter_taps(int32_t sample_rate, double* taps, int64_t cap, int32_t* up, int32_t* down, int32_t* n) {
    if (!rate_ok(sample_rate)) { set_error("audio: sample rate %d Hz outside [1000, 384000]", sample_rate); return WK_ERR_INVALID_ARGUMENT; }
    int u, d;
    std::vector<double> h;
    design_filter(sample_rate, &u, &d, &h);
    if (up) *up = u;
    if (down) *down = d;
    if (n) *n = (int32_t)h.size();
    if (taps) {
        if (cap < (int64_t)h.size()) { set_error("wk_audio_filter_taps: capacity %lld < %zu taps", (long long)cap, h.size()); return WK_ERR_INVALID_ARGUMENT; }
        memcpy(taps, h.data(), h.size() * sizeof(double));
    }
    return WK_OK;
}

wk_status wk_audio_load(wk_session* s, const char* path, const wk_audio_load_opts* opts, float* out, int64_t cap, int64_t* n_out) {
    if (!path) { set_error("wk_audio_load: null path"); return WK_ERR_INVALID_ARGUMENT; }
    FILE* f = fopen(path, "rb");
    if (!f) return fail_load(path, "resource path does not exist or cannot be opened");
    struct Closer { FILE* f; ~Closer() { fclose(f); } } closer{f};
    wk_audio_format fmt;
    FlacStream fs;
    bool is_flac;
    WK_CHECK(parse_audio(f, path, &fmt, &fs, &is_flac));
    if (!rate_ok(fmt.sample_rate)) { set_error("audio: %s: sample rate %d Hz outside [1000, 384000]", path, fmt.sample_rate); return WK_ERR_INVALID_ARGUMENT; }
    Plan plan;
    WK_CHECK(make_plan(fmt.frames, fmt.sample_rate, opts, &plan));
    MixParams mx;
    WK_CHECK(make_mix(fmt.sample_format, fmt.channels, opts, &mx));
    int up, down;
    resample_ratio(fmt.sample_rate, &up, &down);
    WK_CHECK(finish_len(out_len(plan.n, up, down), out, cap, n_out));
    if (!out) return WK_OK;
    WsHandle h;
    WK_CHECK(h.open(s));
    Source src;
    src.file = f; src.data_offset = fmt.data_offset; src.first = plan.first; src.frame_bytes = fmt.block_align; src.path = path;
    if (!is_flac) return run_convert(h.w, src, fmt.sample_rate, mx, plan, out, opts ? opts->segment_samples : 0);
    WK_CHECK(flac_index(h.w, &fs));
    src.flac = &fs;
    WK_CHECK(run_convert(h.w, src, fmt.sample_rate, mx, plan, out, opts ? opts->segment_samples : 0));
    return flac_check(h.w, fs);
}

wk_status wk_audio_convert(wk_session* s, const void* frames, int32_t sample_format, int64_t n_frames, int32_t channels, int32_t sample_rate,
                           const wk_audio_load_opts* opts, float* out, int64_t cap, int64_t* n_out) {
    if (sample_format < WK_AUDIO_U8 || sample_format > WK_AUDIO_F32 || channels < 1 || channels > kMaxMixChannels || n_frames < 0 ||
        (!frames && n_frames > 0)) {
        set_error("wk_audio_convert: bad arguments (format %d, %d channels, %lld frames)", sample_format, channels, (long long)n_frames);
        return WK_ERR_INVALID_ARGUMENT;
    }
    if (!rate_ok(sample_rate)) { set_error("audio: sample rate %d Hz outside [1000, 384000]", sample_rate); return WK_ERR_INVALID_ARGUMENT; }
    Plan plan;
    WK_CHECK(make_plan(n_frames, sample_rate, opts, &plan));
    MixParams mx;
    WK_CHECK(make_mix(sample_format, channels, opts, &mx));
    int up, down;
    resample_ratio(sample_rate, &up, &down);
    WK_CHECK(finish_len(out_len(plan.n, up, down), out, cap, n_out));
    if (!out) return WK_OK;
    WsHandle h;
    WK_CHECK(h.open(s));
    Source src;
    src.first = plan.first; src.frame_bytes = channels * fmt_bytes(sample_format);
    if (is_device_ptr(frames)) {
        if ((reinterpret_cast<uintptr_t>(frames) % (sample_format == WK_AUDIO_S24 ? 1 : fmt_bytes(sample_format))) != 0) {
            set_error("wk_audio_convert: device frames must be aligned to their sample size");
            return WK_ERR_INVALID_ARGUMENT;
        }
        src.dev = static_cast<const uint8_t*>(frames);
    } else {
        src.host = static_cast<const uint8_t*>(frames);
    }
    return run_convert(h.w, src, sample_rate, mx, plan, out, opts ? opts->segment_samples : 0);
}
