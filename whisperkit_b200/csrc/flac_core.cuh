// FLAC (RFC 9639) as __host__ __device__ functions: the bit reader, CRC-8 / CRC-16, STREAMINFO, the frame header and the subframe
// decode.  flac.cu runs them in its discovery and decode kernels; tests/hostcheck/flac_hostcheck.cpp runs the same code on the CPU.
//
// Every read goes through Bits, which is bounded by the byte span it was given and never reads past it, whatever the input: a read past
// the end sets `over` and returns zeros.  Each function returns one of the Err codes below; none of them can write outside the sample
// buffer the caller sized for the block (block_size samples per channel).
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define FL_HD __host__ __device__ __forceinline__
#else
#define FL_HD inline
#endif

namespace wk {
namespace flac {

enum Err {
    OK = 0,
    E_TRUNCATED,          // the frame's bytes end before its contents do
    E_SYNC,               // no frame sync code
    E_RESERVED,           // a reserved bit is set
    E_BLOCK_SIZE_CODE,    // block-size code 0 (reserved)
    E_RATE_CODE,          // sample-rate code 15
    E_CHANNEL_CODE,       // channel codes 11-15 (reserved)
    E_BPS_CODE,           // sample-size code 3 (reserved)
    E_NUMBER,             // a malformed coded frame / sample number
    E_HEADER_CRC,         // CRC-8 mismatch
    E_STREAM_MISMATCH,    // channels, sample size, rate or block size contradict STREAMINFO
    E_SUBFRAME_TYPE,      // a reserved subframe type or a set padding bit
    E_WASTED,             // wasted bits not below the subframe's sample size
    E_PRECISION,          // LPC precision code 15
    E_SHIFT,              // negative LPC shift
    E_RESIDUAL_CODING,    // residual coding methods 2 and 3 (reserved)
    E_PARTITION,          // a partition smaller than the predictor order, or a block not divisible into the partitions
    E_FRAME_CRC,          // CRC-16 mismatch
};

FL_HD const char* err_name(int e) {
    switch (e) {
        case OK: return "ok";
        case E_TRUNCATED: return "frame truncated";
        case E_SYNC: return "no frame sync code";
        case E_RESERVED: return "reserved bit set";
        case E_BLOCK_SIZE_CODE: return "reserved block-size code 0";
        case E_RATE_CODE: return "invalid sample-rate code 15";
        case E_CHANNEL_CODE: return "reserved channel code";
        case E_BPS_CODE: return "reserved sample-size code 3";
        case E_NUMBER: return "malformed coded frame number";
        case E_HEADER_CRC: return "frame header CRC-8 mismatch";
        case E_STREAM_MISMATCH: return "frame header contradicts STREAMINFO";
        case E_SUBFRAME_TYPE: return "reserved subframe type";
        case E_WASTED: return "wasted bits not below the sample size";
        case E_PRECISION: return "reserved LPC precision code 15";
        case E_SHIFT: return "negative LPC shift";
        case E_RESIDUAL_CODING: return "reserved residual coding method";
        case E_PARTITION: return "residual partition smaller than the predictor order";
        case E_FRAME_CRC: return "frame CRC-16 mismatch";
        default: return "?";
    }
}

constexpr int kMaxHeaderBytes = 16;   // sync 2 + codes 2 + coded number 7 + block size 2 + rate 2 + CRC-8 1
constexpr int kMaxChannels = 8;
constexpr int kMaxLpcOrder = 32;

FL_HD int clz32(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return __clz((int)x);
#else
    return x ? __builtin_clz(x) : 32;
#endif
}

// ------------------------------------------------------------------------------------------------ CRCs (MSB first, initial value 0)
FL_HD uint8_t crc8_byte(uint8_t crc, uint8_t b) {   // polynomial x^8 + x^2 + x + 1
    uint32_t c = crc ^ b;
    for (int i = 0; i < 8; ++i) c = (c & 0x80) ? ((c << 1) ^ 0x07) : (c << 1);
    return (uint8_t)c;
}
FL_HD uint8_t crc8(const uint8_t* p, int n) {
    uint8_t c = 0;
    for (int i = 0; i < n; ++i) c = crc8_byte(c, p[i]);
    return c;
}
// crc16 of the single byte i (the table entry of a byte-at-a-time CRC-16): polynomial x^16 + x^15 + x^2 + 1
FL_HD uint16_t crc16_entry(uint32_t i) {
    uint32_t c = i << 8;
    for (int k = 0; k < 8; ++k) c = (c & 0x8000) ? ((c << 1) ^ 0x8005) : (c << 1);
    return (uint16_t)c;
}
FL_HD uint16_t crc16_byte(uint16_t crc, uint8_t b) { return (uint16_t)((crc << 8) ^ crc16_entry((uint32_t)(crc >> 8) ^ b)); }

// ------------------------------------------------------------------------------------------------ bit reader
struct Bits {
    const uint8_t* p;
    uint64_t pos, end;   // in bits
    bool over;
};
FL_HD Bits bits_init(const uint8_t* p, uint64_t n_bytes) { Bits b; b.p = p; b.pos = 0; b.end = n_bytes * 8; b.over = false; return b; }

// n <= 57 bits, MSB first; past the end: `over` and 0
FL_HD uint64_t get(Bits& b, int n) {
    if (n == 0) return 0;
    if (b.pos + (uint64_t)n > b.end) { b.over = true; b.pos = b.end; return 0; }
    const uint64_t byte = b.pos >> 3;
    const int off = (int)(b.pos & 7);
    const int need = (off + n + 7) >> 3;
    uint64_t v = 0;
    for (int i = 0; i < need; ++i) v = (v << 8) | b.p[byte + i];
    v >>= need * 8 - off - n;
    b.pos += (uint64_t)n;
    return v & ((n == 64) ? ~0ull : ((1ull << n) - 1));
}
FL_HD int64_t sget(Bits& b, int n) {   // two's complement, n <= 57
    if (n == 0) return 0;
    const uint64_t v = get(b, n);
    return (int64_t)(v << (64 - n)) >> (64 - n);
}
// zeros before the next 1 bit, which is consumed; `over` at the end of the span
FL_HD uint32_t unary(Bits& b) {
    uint32_t q = 0;
    while (b.pos < b.end) {
        const int off = (int)(b.pos & 7);
        const uint32_t byte = (uint32_t)(uint8_t)(b.p[b.pos >> 3] << off);
        const int avail = 8 - off;
        if (byte) {
            const int z = clz32(byte) - 24;
            if (z < avail) {
                b.pos += (uint64_t)z + 1;
                return q + (uint32_t)z;
            }
        }
        q += (uint32_t)avail;
        b.pos += (uint64_t)avail;
    }
    b.over = true;
    return q;
}
FL_HD void align_byte(Bits& b) { b.pos = (b.pos + 7) & ~7ull; if (b.pos > b.end) { b.pos = b.end; b.over = true; } }

// ------------------------------------------------------------------------------------------------ STREAMINFO and the frame header
struct StreamInfo {
    int min_block, max_block;
    uint32_t min_frame, max_frame;
    int rate, channels, bps;
    uint64_t total;   // samples per channel (inter-channel samples)
    uint8_t md5[16];
};

// The 34-byte STREAMINFO body; 0 or E_STREAM_MISMATCH (a malformed field)
FL_HD int parse_streaminfo(const uint8_t* p, StreamInfo* si) {
    Bits b = bits_init(p, 34);
    si->min_block = (int)get(b, 16);
    si->max_block = (int)get(b, 16);
    si->min_frame = (uint32_t)get(b, 24);
    si->max_frame = (uint32_t)get(b, 24);
    si->rate = (int)get(b, 20);
    si->channels = (int)get(b, 3) + 1;
    si->bps = (int)get(b, 5) + 1;
    si->total = get(b, 36);
    for (int i = 0; i < 16; ++i) si->md5[i] = p[18 + i];
    if (si->min_block < 16 || si->max_block < si->min_block || si->bps < 4 || si->rate == 0) return E_STREAM_MISMATCH;
    if (si->min_frame && si->max_frame && si->max_frame < si->min_frame) return E_STREAM_MISMATCH;
    return OK;
}

struct FrameHeader {
    int block;       // samples per channel
    int rate;        // Hz, 0 = STREAMINFO's
    int assign;      // channel code: 0-7 independent (code + 1 channels), 8 left/side, 9 side/right, 10 mid/side
    int channels;
    int bps;
    int variable;    // blocking strategy bit
    uint64_t number; // frame number (fixed blocking) or first sample (variable blocking)
    int length;      // header bytes, CRC-8 included
};

// Parses the header at p (n bytes available) and checks its CRC-8 and its agreement with STREAMINFO
FL_HD int parse_header(const uint8_t* p, int n, const StreamInfo& si, FrameHeader* h) {
    if (n < 6) return E_TRUNCATED;
    if (p[0] != 0xFF || (p[1] & 0xFE) != 0xF8) return E_SYNC;
    h->variable = p[1] & 1;
    const int bs_code = p[2] >> 4, rate_code = p[2] & 15, ch_code = p[3] >> 4, bps_code = (p[3] >> 1) & 7;
    if (p[3] & 1) return E_RESERVED;
    if (bs_code == 0) return E_BLOCK_SIZE_CODE;
    if (rate_code == 15) return E_RATE_CODE;
    if (ch_code > 10) return E_CHANNEL_CODE;
    if (bps_code == 3) return E_BPS_CODE;
    // the coded number: UTF-8 style, up to 31 bits (6 bytes) for a frame number, 36 bits (7 bytes) for a sample number
    int i = 4;
    const uint32_t c0 = p[i++];
    int extra;
    uint64_t v;
    if (!(c0 & 0x80)) { extra = 0; v = c0; }
    else if ((c0 & 0xE0) == 0xC0) { extra = 1; v = c0 & 0x1F; }
    else if ((c0 & 0xF0) == 0xE0) { extra = 2; v = c0 & 0x0F; }
    else if ((c0 & 0xF8) == 0xF0) { extra = 3; v = c0 & 0x07; }
    else if ((c0 & 0xFC) == 0xF8) { extra = 4; v = c0 & 0x03; }
    else if ((c0 & 0xFE) == 0xFC) { extra = 5; v = c0 & 0x01; }
    else if (c0 == 0xFE && h->variable) { extra = 6; v = 0; }
    else return E_NUMBER;
    if (i + extra > n) return E_TRUNCATED;
    for (int k = 0; k < extra; ++k) {
        const uint32_t c = p[i++];
        if ((c & 0xC0) != 0x80) return E_NUMBER;
        v = (v << 6) | (c & 0x3F);
    }
    h->number = v;
    // block size
    int block;
    if (bs_code == 1) block = 192;
    else if (bs_code <= 5) block = 576 << (bs_code - 2);
    else if (bs_code == 6) { if (i + 1 > n) return E_TRUNCATED; block = p[i] + 1; i += 1; }
    else if (bs_code == 7) { if (i + 2 > n) return E_TRUNCATED; block = (p[i] << 8 | p[i + 1]) + 1; i += 2; }
    else block = 256 << (bs_code - 8);
    // sample rate
    int rate = 0;
    switch (rate_code) {
        case 0: rate = 0; break;
        case 1: rate = 88200; break;
        case 2: rate = 176400; break;
        case 3: rate = 192000; break;
        case 4: rate = 8000; break;
        case 5: rate = 16000; break;
        case 6: rate = 22050; break;
        case 7: rate = 24000; break;
        case 8: rate = 32000; break;
        case 9: rate = 44100; break;
        case 10: rate = 48000; break;
        case 11: rate = 96000; break;
        case 12: if (i + 1 > n) return E_TRUNCATED; rate = p[i] * 1000; i += 1; break;
        case 13: if (i + 2 > n) return E_TRUNCATED; rate = p[i] << 8 | p[i + 1]; i += 2; break;
        default: if (i + 2 > n) return E_TRUNCATED; rate = (p[i] << 8 | p[i + 1]) * 10; i += 2; break;
    }
    if (i + 1 > n) return E_TRUNCATED;
    if (crc8(p, i) != p[i]) return E_HEADER_CRC;
    h->length = i + 1;
    h->block = block;
    h->rate = rate;
    h->assign = ch_code;
    h->channels = ch_code < 8 ? ch_code + 1 : 2;
    h->bps = bps_code == 0 ? si.bps : bps_code == 1 ? 8 : bps_code == 2 ? 12 : bps_code == 7 ? 32 : 16 + 4 * (bps_code - 4);
    if (h->channels != si.channels || h->bps != si.bps || (rate && rate != si.rate) || block > si.max_block) return E_STREAM_MISMATCH;
    if (!h->variable && v > 0x7FFFFFFFull) return E_NUMBER;
    return OK;
}

// Extra bit of a channel's subframe: the side channel of a stereo decorrelation
FL_HD int subframe_bps(const FrameHeader& h, int ch) {
    return h.bps + ((h.assign == 8 && ch == 1) || (h.assign == 9 && ch == 0) || (h.assign == 10 && ch == 1) ? 1 : 0);
}

// ------------------------------------------------------------------------------------------------ subframes
// Residual of a predictor of `order` into out[order .. block): Rice (4-bit parameter) or Rice2 (5-bit), partitions, escapes
template <typename T>
FL_HD int decode_residual(Bits& b, int block, int order, T* out) {
    const int method = (int)get(b, 2);
    if (method > 1) return E_RESIDUAL_CODING;
    const int pbits = method ? 5 : 4, esc = method ? 31 : 15;
    const int po = (int)get(b, 4);
    const int parts = 1 << po;
    if ((block >> po) << po != block || (block >> po) < order) return E_PARTITION;
    const int psize = block >> po;
    int i = order;
    for (int pi = 0; pi < parts; ++pi) {
        const int end = (pi + 1) * psize;
        const int k = (int)get(b, pbits);
        if (b.over) return E_TRUNCATED;
        if (k == esc) {
            const int nb = (int)get(b, 5);
            for (; i < end; ++i) out[i] = (T)sget(b, nb);
        } else {
            for (; i < end; ++i) {
                const uint64_t q = unary(b);
                const uint64_t u = (q << k) | get(b, k);
                out[i] = (T)((int64_t)(u >> 1) ^ -(int64_t)(u & 1));
                if (b.over) return E_TRUNCATED;
            }
        }
        if (b.over) return E_TRUNCATED;
    }
    return OK;
}

// The recurrences wrap modulo 2^bits(A) instead of overflowing: a well-formed stream never wraps, a malformed one decodes to garbage that
// its CRC or the caller rejects, without undefined behaviour on the way.
template <typename A> struct Wrap;
template <> struct Wrap<int32_t> { typedef uint32_t U; };
template <> struct Wrap<int64_t> { typedef uint64_t U; };

// Fixed predictor of order 0-4 over the residual in out[order ..]: accumulator type A (int32 when bps + 4 bits fit)
template <typename T, typename A>
FL_HD void fixed_predict(T* out, int block, int order) {
    typedef typename Wrap<A>::U U;
    switch (order) {
        case 1: for (int i = 1; i < block; ++i) out[i] = (T)(A)((U)out[i] + (U)out[i - 1]); break;
        case 2: for (int i = 2; i < block; ++i) out[i] = (T)(A)((U)out[i] + 2 * (U)out[i - 1] - (U)out[i - 2]); break;
        case 3: for (int i = 3; i < block; ++i) out[i] = (T)(A)((U)out[i] + 3 * (U)out[i - 1] - 3 * (U)out[i - 2] + (U)out[i - 3]); break;
        case 4: for (int i = 4; i < block; ++i) out[i] = (T)(A)((U)out[i] + 4 * (U)out[i - 1] - 6 * (U)out[i - 2] + 4 * (U)out[i - 3] - (U)out[i - 4]); break;
        default: break;
    }
}

// LPC prediction: out[i] += (sum_j c[j] * out[i - 1 - j]) >> shift, in accumulator type A
template <typename T, typename A>
FL_HD void lpc_predict(T* out, int block, int order, const int32_t* c, int shift) {
    typedef typename Wrap<A>::U U;
    for (int i = order; i < block; ++i) {
        U s = 0;
        for (int j = 0; j < order; ++j) s += (U)(A)c[j] * (U)(A)out[i - 1 - j];
        out[i] = (T)(A)((U)(A)out[i] + (U)((A)s >> shift));
    }
}

FL_HD int ceil_log2(int x) { int r = 0; while ((1 << r) < x) ++r; return r; }

// What a subframe's prediction needs once its residual is parsed
struct Sub {
    int kind;      // 0 samples as parsed (CONSTANT, VERBATIM, FIXED order 0), 1 FIXED, 2 LPC
    int order, shift, wasted, wide;   // wide: the recurrence needs 64-bit arithmetic
    int32_t c[kMaxLpcOrder];
};

// Entropy half of one subframe of `block` samples at sample size sbps (4-33) into out[0 .. block): the samples of CONSTANT and VERBATIM,
// the warm-up samples and the residual of FIXED and LPC.  T: int32_t when sbps <= 32, int64_t for 33.
template <typename T>
FL_HD int parse_subframe(Bits& b, int block, int sbps, T* out, Sub* s) {
    s->kind = 0; s->order = 0; s->shift = 0; s->wasted = 0; s->wide = 0;
    if (get(b, 1)) return E_SUBFRAME_TYPE;
    const int type = (int)get(b, 6);
    if (get(b, 1)) {
        s->wasted = (int)unary(b) + 1;
        if (b.over) return E_TRUNCATED;
        if (s->wasted >= sbps) return E_WASTED;
        sbps -= s->wasted;
    }
    if (b.over) return E_TRUNCATED;
    if (type == 0) {   // CONSTANT
        const T v = (T)sget(b, sbps);
        for (int i = 0; i < block; ++i) out[i] = v;
    } else if (type == 1) {   // VERBATIM
        for (int i = 0; i < block; ++i) out[i] = (T)sget(b, sbps);
    } else if ((type >= 8 && type <= 12) || type >= 32) {   // FIXED order 0-4, LPC order 1-32
        const bool lpc = type >= 32;
        const int order = lpc ? type - 31 : type - 8;
        if (order > block) return E_PARTITION;
        for (int i = 0; i < order; ++i) out[i] = (T)sget(b, sbps);
        s->order = order;
        if (lpc) {
            const int pc = (int)get(b, 4);
            if (pc == 15) return E_PRECISION;
            const int prec = pc + 1;
            s->shift = (int)sget(b, 5);
            if (s->shift < 0) return E_SHIFT;
            for (int j = 0; j < order; ++j) s->c[j] = (int32_t)sget(b, prec);
            s->kind = 2;
            s->wide = sbps + prec + ceil_log2(order) > 32 || sizeof(T) > 4;
        } else {
            s->kind = order ? 1 : 0;
            s->wide = sbps + 4 > 32 || sizeof(T) > 4;   // |coefficients| sum to at most 16 (order 4)
        }
        if (b.over) return E_TRUNCATED;
        const int e = decode_residual(b, block, order, out);
        if (e) return e;
    } else {
        return E_SUBFRAME_TYPE;
    }
    return b.over ? E_TRUNCATED : OK;
}

// Prediction half: the recurrence over the parsed residual, then the wasted bits
template <typename T>
FL_HD void predict_subframe(const Sub& s, int block, T* out) {
    if (s.kind == 1) {
        if (s.wide) fixed_predict<T, int64_t>(out, block, s.order);
        else fixed_predict<T, int32_t>(out, block, s.order);
    } else if (s.kind == 2) {
        if (s.wide) lpc_predict<T, int64_t>(out, block, s.order, s.c, s.shift);
        else lpc_predict<T, int32_t>(out, block, s.order, s.c, s.shift);
    }
    if (s.wasted)
        for (int i = 0; i < block; ++i) out[i] = (T)(int64_t)((uint64_t)(int64_t)out[i] << s.wasted);
}

template <typename T>
FL_HD int decode_subframe(Bits& b, int block, int sbps, T* out) {
    Sub s;
    const int e = parse_subframe(b, block, sbps, out, &s);
    if (!e) predict_subframe(s, block, out);
    return e;
}

// Channel c's sample i after decorrelation, from the decoded subframes a = channel 0 and s = channel 1 (stereo codes 8-10)
FL_HD int64_t decorrelate(int assign, int c, int64_t a, int64_t s) {
    switch (assign) {
        case 8: return c == 0 ? a : (int64_t)((uint64_t)a - (uint64_t)s);   // left, side
        case 9: return c == 0 ? (int64_t)((uint64_t)a + (uint64_t)s) : s;   // side, right
        case 10: {                                     // mid, side
            const uint64_t m = ((uint64_t)a << 1) | (uint64_t)(s & 1);
            return c == 0 ? (int64_t)(m + (uint64_t)s) >> 1 : (int64_t)(m - (uint64_t)s) >> 1;
        }
        default: return c == 0 ? a : s;
    }
}

// Size of an ID3v2 tag from its 10-byte header (0 if there is none)
FL_HD uint64_t id3v2_size(const uint8_t* h) {
    if (h[0] != 'I' || h[1] != 'D' || h[2] != '3') return 0;
    const uint64_t s = (uint64_t)(h[6] & 0x7F) << 21 | (uint64_t)(h[7] & 0x7F) << 14 | (uint64_t)(h[8] & 0x7F) << 7 | (h[9] & 0x7F);
    return 10 + s + ((h[5] & 0x10) ? 10 : 0);
}

// Upper bound of one frame's bytes: the header, a VERBATIM subframe at 33 bits per sample for every channel (wasted-bit unary included),
// padding and the CRC-16.  STREAMINFO's max_frame, when present, is the encoder's own bound; this one holds for any well-formed frame
// whose residual codes no worse than verbatim at the subframe's sample size plus one bit.
FL_HD uint64_t frame_bound(const StreamInfo& si) {
    const uint64_t per_ch = 1 + 5 + ((uint64_t)si.max_block * 34 + 7) / 8 + 64;
    return (uint64_t)kMaxHeaderBytes + (uint64_t)si.channels * per_ch + 2;
}

}  // namespace flac
}  // namespace wk
