// CPU build of whisperkit_b200/csrc/flac_core.cuh (test infrastructure): a serial FLAC decoder over the same __host__ __device__ functions
// the GPU kernels run: frame header, subframe parse and prediction, decorrelation, CRC-16.  Frames are walked one after another, each
// starting where the previous one's CRC-16 ends, so the discovery the GPU does by sync-code scan is not needed here.
//
// Built as a shared library for ctypes (the round-trip tests and the host baseline of tools/bench_flac.py) and, with
// -DFLAC_HOSTCHECK_MAIN and -fsanitize=address,undefined, as an executable that decodes the malformed corpus.
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../whisperkit_b200/csrc/flac_core.cuh"

using namespace wk::flac;

enum HostErr { H_NOT_FLAC = 100, H_METADATA = 101, H_UNKNOWN_LENGTH = 102, H_GAP = 103, H_BLOCKING = 104, H_CAPACITY = 105 };

// fmt: [rate, channels, bps, variable blocking]; out: total * channels int32, interleaved, the samples as coded (not left-justified).
// Returns 0 or an error code (Err or HostErr); *err_off is the byte offset it refers to.
extern "C" int wk_flac_host_decode(const uint8_t* data, int64_t n, int32_t* fmt, int64_t* total, int32_t* out, int64_t cap, int64_t* err_off) {
    *err_off = 0;
    int64_t pos = 0;
    if (n >= 10) pos = (int64_t)id3v2_size(data);
    if (pos + 4 > n || memcmp(data + pos, "fLaC", 4)) { *err_off = pos; return H_NOT_FLAC; }
    pos += 4;
    StreamInfo si{};
    bool first = true, last = false;
    while (!last) {
        if (pos + 4 > n) { *err_off = pos; return H_METADATA; }
        last = data[pos] & 0x80;
        const int type = data[pos] & 0x7F;
        const int64_t len = (int64_t)data[pos + 1] << 16 | data[pos + 2] << 8 | data[pos + 3];
        if (first && (type != 0 || len != 34)) { *err_off = pos; return H_METADATA; }
        if (!first && (type == 0 || type == 127)) { *err_off = pos; return H_METADATA; }
        if (pos + 4 + len > n) { *err_off = pos; return H_METADATA; }
        if (first && parse_streaminfo(data + pos + 4, &si)) { *err_off = pos; return H_METADATA; }
        first = false;
        pos += 4 + len;
    }
    if (si.total == 0) { *err_off = pos; return H_UNKNOWN_LENGTH; }
    fmt[0] = si.rate; fmt[1] = si.channels; fmt[2] = si.bps; fmt[3] = 0;
    *total = (int64_t)si.total;
    if (!out) return 0;
    if (cap < (int64_t)si.total * si.channels) return H_CAPACITY;
    std::vector<int64_t> buf[kMaxChannels];
    uint64_t sample = 0;
    int variable = -1, nominal = 0;
    while (sample < si.total) {
        *err_off = pos;
        FrameHeader h;
        const int avail = (int)(n - pos < kMaxHeaderBytes ? n - pos : kMaxHeaderBytes);
        int e = parse_header(data + pos, avail, si, &h);
        if (e) return e;
        if (variable < 0) { variable = h.variable; nominal = h.block; fmt[3] = variable; }
        if (h.variable != variable) return H_BLOCKING;
        const uint64_t start = variable ? h.number : h.number * (uint64_t)nominal;
        if (start != sample || sample + (uint64_t)h.block > si.total) return H_GAP;
        Bits b = bits_init(data + pos, (uint64_t)(n - pos));
        b.pos = (uint64_t)h.length * 8;
        for (int c = 0; c < h.channels; ++c) {
            buf[c].resize(h.block);
            e = decode_subframe(b, h.block, subframe_bps(h, c), buf[c].data());
            if (e) return e;
        }
        align_byte(b);
        const int64_t end = pos + (int64_t)(b.pos >> 3);
        if (b.over || end + 2 > n) return E_TRUNCATED;
        uint16_t crc = 0;
        for (int64_t i = pos; i < end + 2; ++i) crc = crc16_byte(crc, data[i]);
        if (crc) return E_FRAME_CRC;
        for (int i = 0; i < h.block; ++i)
            for (int c = 0; c < h.channels; ++c) {
                const int64_t v = h.assign >= 8 ? decorrelate(h.assign, c, buf[0][i], buf[1][i]) : buf[c][i];
                out[(int64_t)(sample + i) * h.channels + c] = (int32_t)v;
            }
        sample += (uint64_t)h.block;
        pos = end + 2;
    }
    return 0;
}

#ifdef FLAC_HOSTCHECK_MAIN
// Decodes each file named on the command line; prints "<status> <offset> <path>" per file and writes the samples of a decoded file to
// <path>.s32 (int32, little-endian, interleaved)
int main(int argc, char** argv) {
    for (int a = 1; a < argc; ++a) {
        FILE* f = fopen(argv[a], "rb");
        if (!f) { printf("-1 0 %s\n", argv[a]); continue; }
        std::vector<uint8_t> data;
        uint8_t tmp[65536];
        size_t got;
        while ((got = fread(tmp, 1, sizeof tmp, f)) > 0) data.insert(data.end(), tmp, tmp + got);
        fclose(f);
        int32_t fmt[4];
        int64_t total = 0, off = 0;
        int st = wk_flac_host_decode(data.data(), (int64_t)data.size(), fmt, &total, nullptr, 0, &off);
        std::vector<int32_t> out;
        if (!st) {
            out.resize((size_t)total * fmt[1]);
            st = wk_flac_host_decode(data.data(), (int64_t)data.size(), fmt, &total, out.data(), (int64_t)out.size(), &off);
        }
        printf("%d %lld %s\n", st, (long long)off, argv[a]);
        if (!st) {
            const std::string p = std::string(argv[a]) + ".s32";
            FILE* g = fopen(p.c_str(), "wb");
            if (g) { fwrite(out.data(), 4, out.size(), g); fclose(g); }
        }
    }
    return 0;
}
#endif
