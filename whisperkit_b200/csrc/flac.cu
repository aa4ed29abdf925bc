// FLAC (RFC 9639) decoding on the GPU for the audio loader.  The format itself is in flac_core.cuh; this file holds the kernels and the
// host driver.
//
//   1. Host: ID3v2 skip, "fLaC", metadata blocks skipped by their lengths, STREAMINFO, the first frame header (blocking strategy).
//   2. Discovery: the audio bytes stream through the pinned staging in chunks that overlap by the longest possible frame.
//      flac_scan_kernel finds byte-aligned sync codes and keeps the headers whose CRC-8 passes and whose fields agree with STREAMINFO
//      and the stream's blocking strategy, compacted in byte order (per-CTA counts, an exclusive scan, then ordered writes: no order
//      from atomics reaches the result).  flac_chain_kernel runs one thread per candidate: it feeds the frame's bytes through CRC-16 and
//      stops at the first later candidate that continues the sample count with a zero CRC remainder, or at the end of the audio.
//   3. Chain: the host walks the candidates from the first frame by their `next` links.  The result is the frame table (byte offset and
//      first sample per frame) covering [0, total) without gaps; any break fails the load, naming the byte offset.
//   4. Decode: for a segment of the loader, the frames covering its samples are uploaded and flac_decode_kernel (one CTA per frame)
//      parses the subframes (one thread: the subframes follow each other in the bit stream), predicts each channel on its own warp,
//      then all threads decorrelate and write the samples inside the segment to d_raw, interleaved and left-justified in the WAV
//      container of the same width.  Everything after that is the WAV path.
#include <string.h>
#include <sys/stat.h>

#include <algorithm>

#include "audio.h"
#include "common.cuh"

namespace wk {

using namespace flac;

constexpr int kScanThreads = 256;
constexpr int kScanBytes = 4096;            // positions per CTA of the scan
constexpr int64_t kChunkBytes = 16 << 20;   // discovery chunk, before the overlap
constexpr int kChainThreads = 128;

struct FlacCand {
    int64_t off;     // file offset of the header
    int64_t first;   // first sample
    int32_t block;
    int32_t why;     // chain result: 0 next found, 1 CRC-16 mismatch, 2 sample gap or overlap, 3 no following frame
    int64_t next;    // file offset of the next frame (or of the end of the audio)
};

struct ScanCtx {
    StreamInfo si;
    int variable, nominal;
    int64_t total;
};

// The header at p (n bytes available) as a candidate of this stream: 0 or the first sample and block size
__device__ __forceinline__ bool scan_at(const uint8_t* p, int64_t n, const ScanCtx& c, int64_t* first, int* block) {
    if (n < 2 || p[0] != 0xFF || (p[1] & 0xFE) != 0xF8) return false;
    FrameHeader h;
    if (parse_header(p, (int)(n < kMaxHeaderBytes ? n : (int64_t)kMaxHeaderBytes), c.si, &h) != OK || h.variable != c.variable) return false;
    const int64_t s = c.variable ? (int64_t)h.number : (int64_t)h.number * c.nominal;
    if (s < 0 || s + h.block > c.total) return false;
    if (!c.variable && h.block != c.nominal && s + h.block != c.total) return false;   // only the last frame of fixed blocking is short
    *first = s;
    *block = h.block;
    return true;
}

// kWrite = false: counts[cta] = candidates among this CTA's positions.  kWrite = true: writes them in byte order from offsets[cta] on.
template <bool kWrite>
__global__ void __launch_bounds__(kScanThreads)
flac_scan_kernel(const uint8_t* __restrict__ buf, int64_t n_buf, int64_t n_scan, int64_t buf_off, ScanCtx ctx, unsigned* __restrict__ counts,
                 FlacCand* __restrict__ out, unsigned cap) {
    const int64_t base = (int64_t)blockIdx.x * kScanBytes;
    __shared__ unsigned warp_n[kScanThreads / 32];
    __shared__ unsigned run;
    if (threadIdx.x == 0) run = kWrite ? counts[blockIdx.x] : 0u;   // write pass: counts holds the exclusive offsets
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int it = 0; it < kScanBytes / kScanThreads; ++it) {
        const int64_t p = base + (int64_t)it * kScanThreads + threadIdx.x;
        int64_t first = 0;
        int block = 0;
        const bool hit = p < n_scan && scan_at(buf + p, n_buf - p, ctx, &first, &block);
        const unsigned bal = __ballot_sync(0xffffffffu, hit);
        if (lane == 0) warp_n[warp] = __popc(bal);
        __syncthreads();
        unsigned before = run;
        for (int w2 = 0; w2 < warp; ++w2) before += warp_n[w2];
        if (kWrite && hit) {
            const unsigned idx = before + __popc(bal & ((1u << lane) - 1));
            if (idx < cap) {
                FlacCand c;
                c.off = buf_off + p; c.first = first; c.block = block; c.why = 3; c.next = -1;
                out[idx] = c;
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) for (int w2 = 0; w2 < kScanThreads / 32; ++w2) run += warp_n[w2];
        __syncthreads();
    }
    if (!kWrite && threadIdx.x == 0) counts[blockIdx.x] = run;
}

// counts[0 .. n) -> exclusive offsets in place, counts[n] = the total (one thread: a few thousand additions in a fixed order)
__global__ void flac_scan_offsets_kernel(unsigned* counts, int n) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    unsigned s = 0;
    for (int i = 0; i < n; ++i) { const unsigned c = counts[i]; counts[i] = s; s += c; }
    counts[n] = s;
}

// One thread per owned candidate: CRC-16 over its bytes, up to the first later candidate that continues its samples with a zero
// remainder, or up to the end of the audio for the frame that ends the stream
__global__ void __launch_bounds__(kChainThreads)
flac_chain_kernel(const uint8_t* __restrict__ buf, int64_t buf_off, int64_t buf_end, FlacCand* __restrict__ cand, const unsigned* __restrict__ n_cand,
                  int64_t own_end, int64_t audio_end, int64_t total, int64_t bound) {
    __shared__ uint16_t tab[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) tab[i] = crc16_entry(i);
    __syncthreads();
    const unsigned n = *n_cand;
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || cand[i].off >= own_end) return;
    FlacCand c = cand[i];
    const int64_t expect = c.first + c.block;
    const int64_t limit = min(buf_end, c.off + bound);
    unsigned j = i + 1;
    uint16_t crc = 0;
    int why = 3;
    for (int64_t pos = c.off;; ++pos) {
        if (pos > c.off) {
            while (j < n && cand[j].off < pos) ++j;
            if (j < n && cand[j].off == pos) {
                if (cand[j].first == expect) {
                    if (crc == 0) { why = 0; c.next = pos; break; }
                    why = 1;
                } else if (crc == 0 && why == 3) {
                    why = 2;
                }
            }
            if (pos == audio_end) {
                if (expect == total && crc == 0) { why = 0; c.next = pos; break; }
                if (expect == total) why = 1;
            }
        }
        if (pos >= limit) break;
        crc = (uint16_t)((crc << 8) ^ tab[(crc >> 8) ^ buf[pos - buf_off]]);
    }
    cand[i].why = why;
    cand[i].next = c.next;
}

// One CTA per frame of [f0, f0 + gridDim.x): decoded subframes in scratch (channel-major per frame), then the samples in [s0, s1) to raw
template <typename T>
__global__ void __launch_bounds__(256)
flac_decode_kernel(const uint8_t* __restrict__ bytes, int64_t bytes_off, const int64_t* __restrict__ f_off, const int64_t* __restrict__ f_first,
                   int f0, StreamInfo si, T* __restrict__ scratch, int64_t s0, int64_t s1, uint8_t* __restrict__ raw, int cbytes, int shift,
                   unsigned long long* __restrict__ err) {
    const int f = f0 + blockIdx.x;
    const int64_t first = f_first[f], block64 = f_first[f + 1] - first;
    const int ch = si.channels;
    T* x = scratch + (first - f_first[f0]) * ch;
    __shared__ Sub subs[kMaxChannels];
    __shared__ FrameHeader hdr;
    __shared__ int bad;
    if (threadIdx.x == 0) {
        const uint8_t* p = bytes + (f_off[f] - bytes_off);
        const int64_t n = f_off[f + 1] - f_off[f];
        int e = parse_header(p, (int)(n < kMaxHeaderBytes ? n : (int64_t)kMaxHeaderBytes), si, &hdr);
        if (!e && hdr.block != block64) e = E_STREAM_MISMATCH;
        Bits b = bits_init(p, (uint64_t)n);
        b.pos = (uint64_t)hdr.length * 8;
        for (int c = 0; c < ch && !e; ++c) e = parse_subframe(b, hdr.block, subframe_bps(hdr, c), x + (int64_t)c * block64, &subs[c]);
        bad = e;
        if (e) atomicMin(err, (unsigned long long)f << 8 | (unsigned)e);
    }
    __syncthreads();
    if (bad) return;
    const int block = (int)block64;
    if ((threadIdx.x & 31) == 0 && (int)(threadIdx.x >> 5) < ch) {
        const int c = threadIdx.x >> 5;
        predict_subframe(subs[c], block, x + (int64_t)c * block);
    }
    __syncthreads();
    const int64_t a = max(first, s0), b = min(first + block64, s1);
    const int assign = hdr.assign;
    for (int64_t k = (a - first) * ch + threadIdx.x; k < (b - first) * ch; k += blockDim.x) {
        const int64_t i = k / ch;
        const int c = (int)(k - i * ch);
        int64_t v = x[(int64_t)c * block + i];
        if (assign >= 8) v = decorrelate(assign, c, x[i], x[(int64_t)block + i]);
        const uint32_t u = (uint32_t)((uint64_t)v << shift);
        uint8_t* d = raw + ((first + i - s0) * ch + c) * cbytes;
        if (cbytes == 2) *reinterpret_cast<uint16_t*>(d) = (uint16_t)u;
        else if (cbytes == 4) *reinterpret_cast<uint32_t*>(d) = u;
        else { d[0] = (uint8_t)u; d[1] = (uint8_t)(u >> 8); d[2] = (uint8_t)(u >> 16); }
    }
}

// ------------------------------------------------------------------------------------------------ host
static wk_status fail_at(const char* path, int64_t off, const char* what) {
    char msg[200];
    snprintf(msg, sizeof msg, "FLAC: %s at byte %lld", what, (long long)off);
    return fail_load(path, msg);
}

static int container_bytes(int bps) { return bps <= 16 ? 2 : bps <= 24 ? 3 : 4; }

wk_status flac_parse(FILE* f, const char* path, int64_t start, wk_audio_format* out, FlacStream* fs) {
    struct stat sb;
    if (fstat(fileno(f), &sb) != 0) return fail_load(path, "cannot stat the file");
    const int64_t fsize = (int64_t)sb.st_size;
    int64_t pos = start + 4;   // past "fLaC"
    bool first = true, last = false;
    while (!last) {
        uint8_t h[4];
        if (pos + 4 > fsize || fseeko(f, pos, SEEK_SET) != 0 || fread(h, 1, 4, f) != 4) return fail_at(path, pos, "metadata truncated");
        last = h[0] & 0x80;
        const int type = h[0] & 0x7F;
        const int64_t len = (int64_t)h[1] << 16 | h[2] << 8 | h[3];
        if (pos + 4 + len > fsize) return fail_at(path, pos, "metadata block runs past the end of the file");
        if (first) {
            if (type != 0 || len != 34) return fail_at(path, pos, "missing STREAMINFO (the first metadata block)");
            uint8_t b[34];
            if (fread(b, 1, 34, f) != 34) return fail_at(path, pos, "STREAMINFO truncated");
            if (parse_streaminfo(b, &fs->si) != OK) return fail_at(path, pos, "malformed STREAMINFO");
        } else if (type == 0) {
            return fail_at(path, pos, "a second STREAMINFO");
        } else if (type == 127) {
            return fail_at(path, pos, "invalid metadata block type 127");
        }
        first = false;
        pos += 4 + len;
    }
    const StreamInfo& si = fs->si;
    if (si.total == 0) return fail_at(path, start + 8, "STREAMINFO total sample count 0 (unknown length) is not supported");
    fs->file = f;
    fs->path = path;
    fs->audio_off = pos;
    fs->audio_end = fsize;
    if (fsize - pos >= 128) {   // an ID3v1 tag after the audio
        uint8_t t[3];
        if (fseeko(f, fsize - 128, SEEK_SET) == 0 && fread(t, 1, 3, f) == 3 && !memcmp(t, "TAG", 3)) fs->audio_end = fsize - 128;
    }
    uint8_t hb[kMaxHeaderBytes] = {0};
    const int n = (int)std::min<int64_t>(kMaxHeaderBytes, fs->audio_end - pos);
    FrameHeader h;
    if (n <= 0 || fseeko(f, pos, SEEK_SET) != 0 || fread(hb, 1, n, f) != (size_t)n) return fail_at(path, pos, "no audio frames");
    const int e = parse_header(hb, n, si, &h);
    if (e) return fail_at(path, pos, err_name(e));
    fs->variable = h.variable;
    fs->nominal = h.block;
    const int cb = container_bytes(si.bps);
    out->sample_rate = si.rate;
    out->channels = si.channels;
    out->sample_format = cb == 2 ? WK_AUDIO_S16 : cb == 3 ? WK_AUDIO_S24 : WK_AUDIO_S32;
    out->block_align = si.channels * cb;
    out->frames = (int64_t)si.total;
    out->data_offset = pos;
    return WK_OK;
}

static int64_t chain_bound(const StreamInfo& si) { return (int64_t)std::max<uint64_t>(si.max_frame, frame_bound(si)); }

wk_status flac_index(AudioWs* w, FlacStream* fs) {
    const StreamInfo& si = fs->si;
    const int64_t bound = chain_bound(si);
    const int64_t overlap = bound + kMaxHeaderBytes;
    ScanCtx ctx;
    ctx.si = si; ctx.variable = fs->variable; ctx.nominal = fs->nominal; ctx.total = (int64_t)si.total;
    const int64_t buf_cap = kChunkBytes + overlap;
    for (uint8_t*& h : w->h_in) WK_CHECK(w->mem.grow_pinned(&h, (size_t)buf_cap));
    WK_CHECK(w->mem.grow(&w->d_bytes, (size_t)buf_cap, w->stream));
    const int max_ctas = (int)((buf_cap + kScanBytes - 1) / kScanBytes);
    WK_CHECK(w->mem.grow(&w->d_counts, (size_t)max_ctas + 1, w->stream));
    for (int i = 0; i < 2; ++i)
        if (!w->ev_in[i]) WK_CUDA_CHECK(cudaEventCreateWithFlags(&w->ev_in[i], cudaEventDisableTiming));
    std::vector<FlacCand> all, part;
    auto read_chunk = [&](int64_t c0, int i, int64_t* len) -> wk_status {
        *len = std::min(fs->audio_end, c0 + buf_cap) - c0;
        WK_CUDA_CHECK(cudaEventSynchronize(w->ev_in[i]));
        if (fseeko(fs->file, c0, SEEK_SET) != 0 || fread(w->h_in[i], 1, (size_t)*len, fs->file) != (size_t)*len)
            return fail_at(fs->path, c0, "read error");
        return WK_OK;
    };
    int64_t len = 0;
    int k = 0;
    WK_CHECK(read_chunk(fs->audio_off, 0, &len));
    for (int64_t c0 = fs->audio_off; c0 < fs->audio_end; c0 += kChunkBytes, ++k) {
        const int i = k & 1;
        const int64_t n_buf = len;
        const int64_t own_end = std::min(fs->audio_end, c0 + kChunkBytes);
        const int64_t n_scan = std::min(n_buf, own_end - c0 + bound);
        const int ctas = (int)((n_scan + kScanBytes - 1) / kScanBytes);
        WK_CUDA_CHECK(cudaMemcpyAsync(w->d_bytes, w->h_in[i], (size_t)n_buf, cudaMemcpyHostToDevice, w->stream));
        WK_CUDA_CHECK(cudaEventRecord(w->ev_in[i], w->stream));
        flac_scan_kernel<false><<<ctas, kScanThreads, 0, w->stream>>>(w->d_bytes, n_buf, n_scan, c0, ctx, w->d_counts, nullptr, 0);
        count_launch();
        flac_scan_offsets_kernel<<<1, 32, 0, w->stream>>>(w->d_counts, ctas);
        count_launch();
        unsigned n_cand = 0;
        WK_CUDA_CHECK(cudaMemcpyAsync(&n_cand, w->d_counts + ctas, 4, cudaMemcpyDeviceToHost, w->stream));
        WK_CUDA_CHECK(cudaStreamSynchronize(w->stream));
        if (n_cand > (unsigned)(n_scan / 2 + 1)) return fail_at(fs->path, c0, "frame scan overflow");
        if (n_cand) {
            WK_CHECK(w->mem.grow(&w->d_cand, n_cand, w->stream));
            flac_scan_kernel<true><<<ctas, kScanThreads, 0, w->stream>>>(w->d_bytes, n_buf, n_scan, c0, ctx, w->d_counts, w->d_cand, n_cand);
            count_launch();
            flac_chain_kernel<<<(n_cand + kChainThreads - 1) / kChainThreads, kChainThreads, 0, w->stream>>>(
                w->d_bytes, c0, c0 + n_buf, w->d_cand, w->d_counts + ctas, own_end, fs->audio_end, (int64_t)si.total, bound);
            count_launch();
            const cudaError_t e = cudaGetLastError();
            if (e != cudaSuccess) { set_error("FLAC kernel launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
            part.resize(n_cand);
            WK_CUDA_CHECK(cudaMemcpyAsync(part.data(), w->d_cand, (size_t)n_cand * sizeof(FlacCand), cudaMemcpyDeviceToHost, w->stream));
        }
        if (own_end < fs->audio_end) WK_CHECK(read_chunk(own_end, (k + 1) & 1, &len));   // the next chunk's read overlaps this chunk's kernels
        WK_CUDA_CHECK(cudaStreamSynchronize(w->stream));
        for (unsigned c = 0; c < n_cand; ++c)
            if (part[c].off < own_end) all.push_back(part[c]);
    }
    // the chain from the first frame
    fs->off.clear();
    fs->first.clear();
    int64_t pos = fs->audio_off, sample = 0;
    size_t at = 0;
    while (sample < (int64_t)si.total) {
        while (at < all.size() && all[at].off < pos) ++at;
        if (at == all.size() || all[at].off != pos) return fail_at(fs->path, pos, "no valid frame header where the previous frame ends");
        const FlacCand& c = all[at];
        if (c.first != sample) return fail_at(fs->path, pos, "frame sample numbers leave a gap or overlap");
        if (c.why == 1) return fail_at(fs->path, pos, "frame CRC-16 mismatch");
        if (c.why == 2) return fail_at(fs->path, pos, "the next frame's sample number leaves a gap or overlap");
        if (c.why != 0) return fail_at(fs->path, pos, "no valid frame follows (truncated or corrupt)");
        fs->off.push_back(c.off);
        fs->first.push_back(c.first);
        sample = c.first + c.block;
        pos = c.next;
    }
    fs->off.push_back(pos);
    fs->first.push_back(sample);
    const size_t nf = fs->off.size();
    WK_CHECK(w->mem.grow(&w->d_frames, 2 * nf, w->stream));
    WK_CUDA_CHECK(cudaMemcpyAsync(w->d_frames, fs->off.data(), nf * 8, cudaMemcpyHostToDevice, w->stream));
    WK_CUDA_CHECK(cudaMemcpyAsync(w->d_frames + nf, fs->first.data(), nf * 8, cudaMemcpyHostToDevice, w->stream));
    WK_CHECK(w->mem.grow(&w->d_err, 1, w->stream));
    WK_CUDA_CHECK(cudaMemsetAsync(w->d_err, 0xFF, 8, w->stream));
    WK_CUDA_CHECK(cudaStreamSynchronize(w->stream));   // the frame table is pageable
    return WK_OK;
}

wk_status flac_stage(AudioWs* w, const FlacStream& fs, int64_t s0, int64_t s1, int buf) {
    const int nf = (int)fs.off.size() - 1;
    const int f0 = (int)(std::upper_bound(fs.first.begin(), fs.first.begin() + nf, s0) - fs.first.begin()) - 1;
    const int f1 = (int)(std::lower_bound(fs.first.begin(), fs.first.begin() + nf, s1) - fs.first.begin());   // frames [f0, f1)
    const int64_t b0 = fs.off[f0], nbytes = fs.off[f1] - b0;
    const int ch = fs.si.channels, cb = container_bytes(fs.si.bps);
    const bool wide = fs.si.bps == 32;   // the side channel of 32-bit stereo has 33 bits
    const size_t scratch = (size_t)(fs.first[f1] - fs.first[f0]) * ch * (wide ? 8 : 4);
    WK_CUDA_CHECK(cudaEventSynchronize(w->ev_in[buf]));   // the copy that last read this pinned buffer is done
    WK_CHECK(w->mem.grow_pinned(&w->h_in[buf], (size_t)nbytes));
    WK_CHECK(w->mem.grow(&w->d_bytes, (size_t)nbytes, w->stream));
    WK_CHECK(w->mem.grow(reinterpret_cast<uint8_t**>(&w->d_scratch), scratch, w->stream));
    if (fseeko(fs.file, b0, SEEK_SET) != 0 || fread(w->h_in[buf], 1, (size_t)nbytes, fs.file) != (size_t)nbytes)
        return fail_at(fs.path, b0, "read error");
    WK_CUDA_CHECK(cudaMemcpyAsync(w->d_bytes, w->h_in[buf], (size_t)nbytes, cudaMemcpyHostToDevice, w->stream));
    WK_CUDA_CHECK(cudaEventRecord(w->ev_in[buf], w->stream));
    const size_t nft = fs.off.size();
    const int shift = cb * 8 - fs.si.bps;
    const unsigned threads = 32u * (unsigned)ch;
    if (wide)
        flac_decode_kernel<int64_t><<<f1 - f0, threads, 0, w->stream>>>(w->d_bytes, b0, w->d_frames, w->d_frames + nft, f0, fs.si,
                                                                        (int64_t*)w->d_scratch, s0, s1, w->d_raw, cb, shift, w->d_err);
    else
        flac_decode_kernel<int32_t><<<f1 - f0, threads, 0, w->stream>>>(w->d_bytes, b0, w->d_frames, w->d_frames + nft, f0, fs.si,
                                                                        (int32_t*)w->d_scratch, s0, s1, w->d_raw, cb, shift, w->d_err);
    count_launch();
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("FLAC decode launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

wk_status flac_check(AudioWs* w, const FlacStream& fs) {
    unsigned long long e = 0;
    WK_CUDA_CHECK(cudaMemcpyAsync(&e, w->d_err, 8, cudaMemcpyDeviceToHost, w->stream));
    WK_CUDA_CHECK(cudaStreamSynchronize(w->stream));
    if (e == ~0ull) return WK_OK;
    const size_t f = (size_t)(e >> 8);
    return fail_at(fs.path, f < fs.off.size() ? fs.off[f] : 0, err_name((int)(e & 0xFF)));
}

}  // namespace wk
