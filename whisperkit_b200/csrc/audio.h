// The audio loader's per-session workspace and the FLAC source it can read from (audio.cu, flac.cu).
#pragma once
#include <stdio.h>

#include <vector>

#include "flac_core.cuh"
#include "kernels.h"

namespace wk {

struct FlacCand;

struct AudioWs {
    Buffers mem;
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    uint8_t* h_in[2] = {nullptr, nullptr};    // pinned input staging (double-buffered: the host fills one while
    float* h_out[2] = {nullptr, nullptr};     // the other is copied); pinned output staging for host outputs
    cudaEvent_t ev_in[2] = {nullptr, nullptr}, ev_out[2] = {nullptr, nullptr};
    uint8_t* d_raw = nullptr;
    float* d_out = nullptr;
    float* d_tab = nullptr; int tab_rate = 0;
    int64_t* d_starts = nullptr;
    unsigned* d_peaks = nullptr;
    // FLAC: compressed bytes of a discovery chunk or of the frames a segment covers, the scan's candidates, the frame table, the decoded
    // subframes of a segment (int32, or int64 at 32 bits per sample) and the first decode error
    uint8_t* d_bytes = nullptr;
    FlacCand* d_cand = nullptr;
    unsigned* d_counts = nullptr;
    int64_t* d_frames = nullptr;
    void* d_scratch = nullptr;
    unsigned long long* d_err = nullptr;
    ~AudioWs() {
        cudaSetDevice(device);
        if (stream) cudaStreamSynchronize(stream);
        for (int i = 0; i < 2; ++i) {
            if (ev_in[i]) cudaEventDestroy(ev_in[i]);
            if (ev_out[i]) cudaEventDestroy(ev_out[i]);
        }
        if (own_stream && stream) cudaStreamDestroy(stream);
    }
};

wk_status fail_load(const char* path, const char* what);

// A FLAC file: STREAMINFO, where the audio frames lie, and (after flac_index) the frame table
struct FlacStream {
    FILE* file = nullptr;
    const char* path = "";
    flac::StreamInfo si{};
    int64_t audio_off = 0, audio_end = 0;   // byte span of the frames
    int variable = 0, nominal = 0;          // blocking strategy and the block size of a fixed-blocking stream
    std::vector<int64_t> off, first;        // per frame, plus one entry for the end: byte offset and first sample
};

// The header: ID3v2 skip, "fLaC", metadata blocks, STREAMINFO; the first frame header for the blocking strategy (host only)
wk_status flac_parse(FILE* f, const char* path, int64_t start, wk_audio_format* out, FlacStream* fs);
// Frame discovery on the device and the chain check: fills fs->off / fs->first and uploads them
wk_status flac_index(AudioWs* w, FlacStream* fs);
// Decodes the samples [s0, s1) of the stream into w->d_raw, left-justified in the container format, through pinned buffer `buf`
wk_status flac_stage(AudioWs* w, const FlacStream& fs, int64_t s0, int64_t s1, int buf);
// The first error a decode kernel of this call met, as a load failure naming the frame's byte offset
wk_status flac_check(AudioWs* w, const FlacStream& fs);

}  // namespace wk
