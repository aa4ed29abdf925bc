// Edge collectives of the data-parallel hot path behind the C ABI (SURVEY.md section 8e): rank `root` scatters 30 s PCM windows to the
// ranks of one node and gathers the per-window DecodingResults back - grouped ncclSend / ncclRecv over NVLink / NVSwitch, nothing else.
// Windows are independent units (the reference fans them out as tasks, WhisperKit.swift:741-809), so there is no collective inside the
// model.  NCCL is resolved at run time from the process (the copy PyTorch already loaded, else libnccl.so.2): libwkb200 itself does not
// link against it, and a single-GPU host never needs it.
#include <dlfcn.h>
#include <nccl.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "common.cuh"
#include "engine.h"

namespace {

struct NcclApi {
    ncclResult_t (*GetUniqueId)(ncclUniqueId*);
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int);
    ncclResult_t (*CommDestroy)(ncclComm_t);
    ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t);
    ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t);
    ncclResult_t (*GroupStart)();
    ncclResult_t (*GroupEnd)();
    const char* (*GetErrorString)(ncclResult_t);
    bool ok = false;
};

NcclApi* nccl() {
    static NcclApi api;
    static bool tried = false;
    if (tried) return api.ok ? &api : nullptr;
    tried = true;
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);   // the copy already in the process (PyTorch's)
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return nullptr;
#define WK_SYM(field, name) *(void**)(&api.field) = dlsym(h, name); if (!api.field) return nullptr;
    WK_SYM(GetUniqueId, "ncclGetUniqueId") WK_SYM(CommInitRank, "ncclCommInitRank") WK_SYM(CommDestroy, "ncclCommDestroy")
    WK_SYM(Send, "ncclSend") WK_SYM(Recv, "ncclRecv") WK_SYM(GroupStart, "ncclGroupStart") WK_SYM(GroupEnd, "ncclGroupEnd")
    WK_SYM(GetErrorString, "ncclGetErrorString")
#undef WK_SYM
    api.ok = true;
    return &api;
}

#define WK_NCCL_CHECK(expr)                                                                      \
    do {                                                                                         \
        ncclResult_t _r = (expr);                                                                \
        if (_r != ncclSuccess) {                                                                 \
            wk::set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #expr, nccl()->GetErrorString(_r)); \
            return WK_ERR_CUDA;                                                                  \
        }                                                                                        \
    } while (0)

}  // namespace

struct wk_comm {
    ncclComm_t comm = nullptr;
    int rank = 0, world = 1, device = 0;
    cudaStream_t stream = nullptr, copy_stream = nullptr;
    wk::Buffers mem;
    float* stage[2] = {nullptr, nullptr};   // root: shards of the other ranks on their way from the host
    cudaEvent_t staged[2], sent[2];
    wk_decode_result* res_dev = nullptr;
    float stage_ms[4] = {0, 0, 0, 0};   // last sharded call on this rank: scatter, transcribe, gather, total (host wall clock)
};

extern "C" {

// the static contiguous split of SURVEY 8(e): order preserving, the first (n % world) ranks take one extra window
void wk_comm_shard_bounds(int64_t n_windows, int32_t world, int32_t rank, int64_t* lo, int64_t* hi) {
    const int64_t base = n_windows / world, rem = n_windows % world;
    *lo = rank * base + std::min<int64_t>(rank, rem);
    *hi = *lo + base + (rank < rem ? 1 : 0);
}

wk_status wk_comm_unique_id(uint8_t* out128) {
    if (!out128) return WK_ERR_INVALID_ARGUMENT;
    NcclApi* n = nccl();
    if (!n) { wk::set_error("NCCL is not available in this process (libnccl.so.2 not found)"); return WK_ERR_MODELS_UNAVAILABLE; }
    ncclUniqueId id;
    WK_NCCL_CHECK(n->GetUniqueId(&id));
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
    memcpy(out128, &id, 128);
    return WK_OK;
}

wk_status wk_comm_create(const uint8_t* id128, int32_t rank, int32_t world, int32_t device, wk_comm** out) {
    if (!id128 || !out || world < 1 || rank < 0 || rank >= world) { wk::set_error("wk_comm_create: bad arguments"); return WK_ERR_INVALID_ARGUMENT; }
    NcclApi* n = nccl();
    if (!n) { wk::set_error("NCCL is not available in this process (libnccl.so.2 not found)"); return WK_ERR_MODELS_UNAVAILABLE; }
    WK_CUDA_CHECK(cudaSetDevice(device));
    wk_comm* c = new wk_comm();
    c->rank = rank; c->world = world; c->device = device;
    ncclUniqueId id;
    memcpy(&id, id128, 128);
    WK_NCCL_CHECK(n->CommInitRank(&c->comm, world, id, rank));
    WK_CUDA_CHECK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    WK_CUDA_CHECK(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
    for (int i = 0; i < 2; ++i) {
        WK_CUDA_CHECK(cudaEventCreateWithFlags(&c->staged[i], cudaEventDisableTiming));
        WK_CUDA_CHECK(cudaEventCreateWithFlags(&c->sent[i], cudaEventDisableTiming));
    }
    *out = c;
    return WK_OK;
}

void wk_comm_free(wk_comm* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    cudaStreamSynchronize(c->copy_stream);
    if (c->comm && nccl()) nccl()->CommDestroy(c->comm);
    for (int i = 0; i < 2; ++i) { cudaEventDestroy(c->staged[i]); cudaEventDestroy(c->sent[i]); }
    cudaStreamDestroy(c->stream);
    cudaStreamDestroy(c->copy_stream);
    delete c;
}

// Rank `root` holds all_pcm [n_windows][stride] (host, pinned for full speed, or device); every rank gets its contiguous shard in
// shard_dev (device, at least (hi - lo) * stride floats).  The root walks the other ranks in order: the host-to-device copy of shard r + 1
// runs on a second stream while shard r is on the wire, and its own shard is copied last.  Returns when the shard is in place.
wk_status wk_comm_scatter_windows(wk_comm* c, const float* all_pcm, int64_t n_windows, int64_t stride, int32_t root, float* shard_dev, int64_t* n_local) {
    if (!c || !shard_dev || n_windows < 0 || root < 0 || root >= c->world || (c->rank == root && !all_pcm)) { wk::set_error("wk_comm_scatter_windows: bad arguments"); return WK_ERR_INVALID_ARGUMENT; }
    NcclApi* n = nccl();
    WK_CUDA_CHECK(cudaSetDevice(c->device));
    int64_t lo, hi;
    wk_comm_shard_bounds(n_windows, c->world, c->rank, &lo, &hi);
    if (n_local) *n_local = hi - lo;
    if (c->rank != root) {
        if (hi > lo) WK_NCCL_CHECK(n->Recv(shard_dev, (size_t)(hi - lo) * stride, ncclFloat, root, c->comm, c->stream));
        WK_CUDA_CHECK(cudaStreamSynchronize(c->stream));
        return WK_OK;
    }
    cudaPointerAttributes at;
    const bool on_dev = cudaPointerGetAttributes(&at, all_pcm) == cudaSuccess && at.type == cudaMemoryTypeDevice;
    cudaGetLastError();
    int64_t max_shard = 0;
    for (int r = 0; r < c->world; ++r) { int64_t a, b; wk_comm_shard_bounds(n_windows, c->world, r, &a, &b); if (r != root) max_shard = std::max(max_shard, b - a); }
    if (!on_dev)
        for (float*& p : c->stage) WK_CHECK(c->mem.grow(&p, (size_t)max_shard * stride));
    int k = 0;
    for (int r = 0; r < c->world; ++r) {
        if (r == root) continue;
        int64_t a, b;
        wk_comm_shard_bounds(n_windows, c->world, r, &a, &b);
        if (b <= a) continue;
        const float* src = all_pcm + a * stride;
        if (!on_dev) {
            const int buf = k & 1;
            WK_CUDA_CHECK(cudaStreamWaitEvent(c->copy_stream, c->sent[buf], 0));   // the send that last used this buffer is done
            WK_CUDA_CHECK(cudaMemcpyAsync(c->stage[buf], src, (size_t)(b - a) * stride * 4, cudaMemcpyHostToDevice, c->copy_stream));
            WK_CUDA_CHECK(cudaEventRecord(c->staged[buf], c->copy_stream));
            WK_CUDA_CHECK(cudaStreamWaitEvent(c->stream, c->staged[buf], 0));
            src = c->stage[buf];
            WK_NCCL_CHECK(n->Send(src, (size_t)(b - a) * stride, ncclFloat, r, c->comm, c->stream));
            WK_CUDA_CHECK(cudaEventRecord(c->sent[buf], c->stream));
            ++k;
        } else {
            WK_NCCL_CHECK(n->Send(src, (size_t)(b - a) * stride, ncclFloat, r, c->comm, c->stream));
        }
    }
    if (hi > lo) WK_CUDA_CHECK(cudaMemcpyAsync(shard_dev, all_pcm + lo * stride, (size_t)(hi - lo) * stride * 4, cudaMemcpyDefault, c->copy_stream));
    WK_CUDA_CHECK(cudaStreamSynchronize(c->copy_stream));   // own shard in place; the sends drain on their own stream
    return WK_OK;
}

// Every rank hands in its n_local results; rank `root` receives all n_windows of them in window order.
wk_status wk_comm_gather_results(wk_comm* c, const wk_decode_result* local, int64_t n_local, int64_t n_windows, int32_t root, wk_decode_result* all) {
    if (!c || (n_local > 0 && !local) || root < 0 || root >= c->world || (c->rank == root && !all)) { wk::set_error("wk_comm_gather_results: bad arguments"); return WK_ERR_INVALID_ARGUMENT; }
    NcclApi* n = nccl();
    WK_CUDA_CHECK(cudaSetDevice(c->device));
    const size_t need = (size_t)(c->rank == root ? n_windows : n_local);
    WK_CHECK(c->mem.grow(&c->res_dev, need, c->stream));
    int64_t lo, hi;
    wk_comm_shard_bounds(n_windows, c->world, c->rank, &lo, &hi);
    if (hi - lo != n_local) { wk::set_error("wk_comm_gather_results: rank %d holds %lld results, its shard has %lld windows", c->rank, (long long)n_local, (long long)(hi - lo)); return WK_ERR_INVALID_ARGUMENT; }
    if (c->rank != root) {
        if (n_local > 0) {
            WK_CUDA_CHECK(cudaMemcpyAsync(c->res_dev, local, (size_t)n_local * sizeof(wk_decode_result), cudaMemcpyHostToDevice, c->stream));
            WK_NCCL_CHECK(n->Send(c->res_dev, (size_t)n_local * sizeof(wk_decode_result), ncclChar, root, c->comm, c->stream));
        }
        WK_CUDA_CHECK(cudaStreamSynchronize(c->stream));
        return WK_OK;
    }
    WK_NCCL_CHECK(n->GroupStart());
    for (int r = 0; r < c->world; ++r) {
        if (r == root) continue;
        int64_t a, b;
        wk_comm_shard_bounds(n_windows, c->world, r, &a, &b);
        if (b > a) WK_NCCL_CHECK(n->Recv(c->res_dev + a, (size_t)(b - a) * sizeof(wk_decode_result), ncclChar, r, c->comm, c->stream));
    }
    WK_NCCL_CHECK(n->GroupEnd());
    WK_CUDA_CHECK(cudaMemcpyAsync(all, c->res_dev, (size_t)n_windows * sizeof(wk_decode_result), cudaMemcpyDeviceToHost, c->stream));
    WK_CUDA_CHECK(cudaStreamSynchronize(c->stream));
    if (n_local > 0) memcpy(all + lo, local, (size_t)n_local * sizeof(wk_decode_result));
    return WK_OK;
}

// The sharded batched entry: scatter -> wk_transcribe_windows_ex on the local shard -> gather.  `bo` carries options shared by every
// window (n_opts == 1) - per-window arrays would have to be sharded by the caller.  results: n_windows entries on the root, ignored elsewhere.
wk_status wk_transcribe_windows_sharded(wk_comm* c, wk_model* m, wk_session* s, const float* all_pcm, int64_t n_windows, int64_t stride, int32_t root,
                                        const wk_special_tokens* st, const wk_batch_opts* bo, wk_decode_result* results) {
    if (!c || !m || !s || !st || !bo || bo->n_opts != 1 || bo->prompts || bo->status) { wk::set_error("wk_transcribe_windows_sharded: bad arguments (shared options only)"); return WK_ERR_INVALID_ARGUMENT; }
    int64_t lo, hi;
    wk_comm_shard_bounds(n_windows, c->world, c->rank, &lo, &hi);
    const int64_t nl = hi - lo;
    WK_CUDA_CHECK(cudaSetDevice(c->device));
    wk::Buffers scratch;
    float* shard = nullptr;
    WK_CHECK(scratch.dmalloc(&shard, (size_t)std::max<int64_t>(nl, 1) * stride, false));
    auto now = []() { timespec t; clock_gettime(CLOCK_MONOTONIC, &t); return t.tv_sec * 1e3 + t.tv_nsec * 1e-6; };
    const double t0 = now();
    wk_status r = wk_comm_scatter_windows(c, all_pcm, n_windows, stride, root, shard, nullptr);
    const double t1 = now();
    std::vector<wk_decode_result> local((size_t)std::max<int64_t>(nl, 1));
    if (r == WK_OK && nl > 0) r = wk_transcribe_windows_ex(m, s, shard, nl, stride, nullptr, st, bo, local.data());
    const double t2 = now();
    if (r != WK_OK) return r;
    r = wk_comm_gather_results(c, local.data(), nl, n_windows, root, results);
    const double t3 = now();
    c->stage_ms[0] = (float)(t1 - t0); c->stage_ms[1] = (float)(t2 - t1); c->stage_ms[2] = (float)(t3 - t2); c->stage_ms[3] = (float)(t3 - t0);
    return r;
}

wk_status wk_comm_last_stage_ms(const wk_comm* c, float* ms4) {
    if (!c || !ms4) return WK_ERR_INVALID_ARGUMENT;
    memcpy(ms4, c->stage_ms, sizeof(c->stage_ms));
    return WK_OK;
}

}  // extern "C"
