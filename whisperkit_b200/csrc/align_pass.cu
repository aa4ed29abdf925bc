// Teacher-forced alignment pass: every position of every window of a chunk goes through the decoder at once (wk_align_tokens /
// wk_align_windows).  The rows are (window, position) pairs at a fixed stride of kAlignStride = 224 rows per window, so row w * 224 + t is
// position t of window w; the GEMMs are the encoder's plain wgmma GEMMs over all rows (session.cu), the kernels here are what is specific
// to the pass:
//   align_embed_kernel            x = token embedding + positional embedding (padding rows: 0)
//   align_attention_kernel        causal self-attention (K / V from the QKV output) and multi-query cross-attention (K / V from the
//                                 cross-attention cache, 16-bit or FP8), flash-style online softmax on the tensor cores
//   align_export_kernel           the alignment heads' normalised softmax rows, recomputed with each row's final max / sum and summed
//                                 over the heads in a fixed order into an f32 accumulator
//   align_rows_f16_kernel         the accumulator as the decode loop's Float16 alignmentWeights layout (row t + 1 = position t)
//   align_logprob_kernel          log softmax(logits[t][:eot])[tokens[t + 1]] (openai-whisper's text_token_probs rule)
// Results do not depend on what else is in the batch: every row is computed from its own window's rows only and every reduction has a
// fixed order.
#include <math.h>

#include <type_traits>

#include "common.cuh"
#include "kernels.h"

namespace wk {

static constexpr int kAlignStride = 224;   // rows per window (Constants.maxTokenContext)
static constexpr int kAtQ = 128;           // query rows per CTA: 8 warps x 16
static constexpr int kAtThreads = 256;
static constexpr int kAtKeys = 64;         // keys per tile
static constexpr int kAtLd = 72;           // smem row stride (elements): 144 bytes keeps ldmatrix rows on distinct banks

// =====================================================================================================
// embedding
// =====================================================================================================
template <typename T>
__global__ void __launch_bounds__(256)
align_embed_kernel(const T* __restrict__ emb, const float* __restrict__ pos_emb, const int32_t* __restrict__ row_tok, float* __restrict__ x, int d) {
    const long long r = blockIdx.x;
    const int tok = row_tok[r], t = (int)(r % kAlignStride);
    for (int i = threadIdx.x; i < d; i += blockDim.x)
        x[r * d + i] = tok >= 0 ? T16<T>::to_f(emb[(long long)tok * d + i]) + pos_emb[(long long)t * d + i] : 0.f;
}

wk_status align_embed(const void* emb, const float* pos_emb, const int32_t* row_tok, float* x, int64_t rows, int d, int dtype, cudaStream_t stream) {
    if (dtype == WK_DTYPE_F16)
        launch_k(align_embed_kernel<__half>, dim3((unsigned)rows), dim3(256), 0, stream, 0, (const __half*)emb, pos_emb, row_tok, x, d);
    else
        launch_k(align_embed_kernel<__nv_bfloat16>, dim3((unsigned)rows), dim3(256), 0, stream, 0, (const __nv_bfloat16*)emb, pos_emb, row_tok, x, d);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("align_embed launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

// =====================================================================================================
// tensor-core helpers (mma.sync m16n8k16, f32 accumulate)
// =====================================================================================================
__device__ __forceinline__ void at_ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void at_ldsm_x4_trans(uint32_t addr, uint32_t (&r)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
template <typename T> __device__ __forceinline__ void at_mma(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1);
template <> __device__ __forceinline__ void at_mma<__nv_bfloat16>(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <> __device__ __forceinline__ void at_mma<__half>(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// x, y (f32) -> 16-bit pair and the 16-bit pair of what its rounding dropped: hi + lo carries ~16 mantissa bits through two MMAs
template <typename T> __device__ __forceinline__ void at_split2(float x, float y, uint32_t& hi, uint32_t& lo) {
    hi = T16<T>::pack2(x, y);
    const float2 h = T16<T>::unpack2(hi);
    lo = T16<T>::pack2(x - h.x, y - h.y);
}

// A fragments of a warp's 16 query rows (rows row0 + g, row0 + g + 8; 64 dims = 4 k-steps) straight from global memory
template <typename T>
__device__ __forceinline__ void at_load_q(const T* __restrict__ q, long long ldq, long long row0, int g, int tq, uint32_t (&qa)[4][4]) {
    const T* r0 = q + (row0 + g) * ldq;
    const T* r1 = q + (row0 + g + 8) * ldq;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
        const int c = ks * 16 + 2 * tq;
        qa[ks][0] = *reinterpret_cast<const uint32_t*>(r0 + c);
        qa[ks][1] = *reinterpret_cast<const uint32_t*>(r1 + c);
        qa[ks][2] = *reinterpret_cast<const uint32_t*>(r0 + c + 8);
        qa[ks][3] = *reinterpret_cast<const uint32_t*>(r1 + c + 8);
    }
}

// raw scores of a warp's 16 rows against the 64 keys of a tile ([key][kAtLd] 16-bit in smem): s[nt][0..1] = row g, keys nt*8 + 2tq (+1);
// s[nt][2..3] = row g + 8
template <typename T>
__device__ __forceinline__ void at_scores(uint32_t ks_base, const uint32_t (&qa)[4][4], int lane, float (&s)[8][4]) {
    const int lm = lane >> 3, lr = lane & 7;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
        uint32_t b[2][4];
#pragma unroll
        for (int half = 0; half < 2; ++half) at_ldsm_x4(ks_base + ((nt * 8 + lr) * kAtLd + (half * 4 + lm) * 8) * 2, b[half]);
        s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) at_mma<T>(s[nt], qa[ks], b[ks >> 1][(ks & 1) * 2], b[ks >> 1][(ks & 1) * 2 + 1]);
    }
}

// cp.async of rows [key0, key0 + 64) of a [keys][ld] 16-bit (or, FP8, byte) source into a smem tile; rows >= nkeys are zero-filled
template <bool FP8>
__device__ __forceinline__ void at_issue_tile(uint8_t* dst, const uint8_t* __restrict__ src, long long ld_bytes, int key0, int nkeys, int tid) {
    constexpr int kChunks = FP8 ? 4 : 8;           // 16-byte pieces per row
    constexpr int kDstLd = FP8 ? 64 : kAtLd * 2;   // FP8 codes land unpadded, 16-bit rows padded
    for (int i = tid; i < kAtKeys * kChunks; i += kAtThreads) {
        const int r = i / kChunks, c = i % kChunks, key = key0 + r;
        const bool ok = key < nkeys;
        cp_async16(dst + r * kDstLd + c * 16, src + (long long)(ok ? key : 0) * ld_bytes + c * 16, ok);
    }
}

// FP8: widen a [64][64] code tile exactly to the 16-bit [64][kAtLd] layout
template <typename T>
__device__ __forceinline__ void at_widen(const uint8_t* codes, T* dst, int tid) {
    for (int i = tid; i < kAtKeys * 8; i += kAtThreads) {   // 8 codes per item
        const int r = i >> 3, c = i & 7;
        const uint2 u = *reinterpret_cast<const uint2*>(codes + r * 64 + c * 8);
        uint32_t h[4];
        fp8x4_to_half2(u.x, h[0], h[1]);
        fp8x4_to_half2(u.y, h[2], h[3]);
        if constexpr (!std::is_same<T, __half>::value) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float2 a = T16<__half>::unpack2(h[k]);
                h[k] = T16<T>::pack2(a.x, a.y);
            }
        }
        *reinterpret_cast<uint4*>(dst + r * kAtLd + c * 8) = make_uint4(h[0], h[1], h[2], h[3]);
    }
}

// Packed bf16 cache: cp.async of the 96-byte primary slots of rows [key0, key0 + 64) of block `blk` and of their 64 header bytes (at
// kAtKeys * 96); rows >= nkeys are zero-filled (header 0, value 0)
__device__ __forceinline__ void at_issue_tile_packed(uint8_t* dst, const uint8_t* __restrict__ blk, const uint8_t* __restrict__ hdr, int key0,
                                                     int nkeys, int tid) {
    for (int i = tid; i < kAtKeys * 6 + 4; i += kAtThreads) {
        if (i < kAtKeys * 6) {
            const int r = i / 6, c = i % 6, key = key0 + r;
            const bool ok = key < nkeys;
            cp_async16(dst + r * kPackedRowBytes + c * 16, blk + (long long)(ok ? key : 0) * kPackedRowBytes + c * 16, ok);
        } else {
            const int c = i - kAtKeys * 6;
            const bool ok = key0 + 16 * c < nkeys;   // the header vector is padded to 16 bytes
            cp_async16(dst + kAtKeys * kPackedRowBytes + c * 16, hdr + (ok ? key0 + 16 * c : 0), ok);
        }
    }
}
// Packed: rebuild the exact bf16 tile in the 16-bit [64][kAtLd] layout (a raw row's last 32 bytes from global memory)
template <typename T>
__device__ __forceinline__ void at_widen_packed(const uint8_t* tile, T* dst, const uint8_t* __restrict__ blk, int Tlen, int key0, int tid) {
    for (int i = tid; i < kAtKeys * 8; i += kAtThreads) {
        const int r = i >> 3, c = i & 7;
        const uint8_t h = tile[kAtKeys * kPackedRowBytes + r];
        const uint8_t* pr = tile + r * kPackedRowBytes;
        uint4 u;
        if (h == kPackedRaw)
            u = c < 6 ? *reinterpret_cast<const uint4*>(pr + 16 * c)
                      : __ldg(reinterpret_cast<const uint4*>(blk + (long long)Tlen * kPackedRowBytes + (long long)(key0 + r) * 32 + 16 * (c - 6)));
        else
            u = unpack_bf16x8(*reinterpret_cast<const uint2*>(pr + 8 * c), *reinterpret_cast<const uint32_t*>(pr + 64 + 4 * c), h);
        *reinterpret_cast<uint4*>(dst + r * kAtLd + c * 8) = u;
    }
}

// =====================================================================================================
// attention.  KIND 0: causal self-attention over the window's own rows of the QKV output (keys <= the query position);
// KIND 1: cross-attention against the 16-bit cache block [T][64] of the window's slot; KIND 2: the same against the FP8 cache (codes widened
// exactly to 16-bit in shared memory, the K row scale applied to the scores, the V row scale folded into p relative to the block's largest);
// KIND 3: the same against the packed bf16 cache (rows rebuilt exactly in shared memory, at_widen_packed).
// One CTA = (query tile of 128 rows, head, window); K / V stream through a double-buffered 64-key ring; each warp keeps its 16 rows' running
// max / sum / output in registers.  Query tiles that start past the window's sequence exit at once; rows past it are computed but not stored.
// stats != nullptr (cross only): each row's final (max, sum) of the head, [H][rows], for align_export_kernel.
// =====================================================================================================
template <typename T, int KIND>
__global__ void __launch_bounds__(kAtThreads)
align_attention_kernel(const T* __restrict__ q, long long ldq, const uint8_t* __restrict__ kb, const uint8_t* __restrict__ vb, long long ld_kv,
                       const float* __restrict__ kscale, const float* __restrict__ vscale, const int32_t* __restrict__ seq_len, int slot0,
                       T* __restrict__ out, int H, int Tlen, float2* __restrict__ stats, long long stat_rows, const uint8_t* __restrict__ khdr,
                       const uint8_t* __restrict__ vhdr) {
    constexpr bool FP8 = KIND == 2, PK = KIND == 3, WIDE = FP8 || PK;
    constexpr int kTileBytes = FP8 ? kAtKeys * 64 : PK ? kAtKeys * (kPackedRowBytes + 1) : kAtKeys * kAtLd * 2;
    __shared__ __align__(128) uint8_t ring[2][2][kTileBytes];           // [stage][K|V]
    __shared__ __align__(128) T wide[WIDE ? 2 : 1][WIDE ? kAtKeys * kAtLd : 8];   // FP8 / packed: the widened K and V tiles
    __shared__ float ksc_s[FP8 ? kAtKeys : 1], vsc_s[FP8 ? kAtKeys : 1], red[8];
    const int qt = blockIdx.x, h = blockIdx.y, w = blockIdx.z;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, tq = lane & 3;
    const int n = seq_len[w];
    const int q0 = qt * kAtQ;
    if (q0 >= n) return;
    const int dm = H * 64;
    const int nkeys = KIND == 0 ? min(n, q0 + kAtQ) : Tlen;
    const int ntiles = (nkeys + kAtKeys - 1) / kAtKeys;
    const long long row_base = (long long)w * kAlignStride;
    const int rw0 = q0 + warp * 16;                 // the warp's first position
    const bool active = rw0 < n;
    // K / V source of this (window, head)
    const long long blk = KIND == 0 ? 0 : (long long)(slot0 + w) * H + h;
    const uint8_t* ksrc = KIND == 0 ? kb + (row_base * ld_kv + h * 64) * 2 : kb + blk * Tlen * ld_kv;
    const uint8_t* vsrc = KIND == 0 ? vb + (row_base * ld_kv + h * 64) * 2 : vb + blk * Tlen * ld_kv;
    const long long ld_bytes = KIND == 0 ? ld_kv * 2 : ld_kv;
    const long long hoff = PK ? blk * packed_hdr_stride(Tlen) : 0;
    auto issue = [&](uint8_t* kd, uint8_t* vd, int key0) {
        if constexpr (PK) {
            at_issue_tile_packed(kd, ksrc, khdr + hoff, key0, nkeys, tid);
            at_issue_tile_packed(vd, vsrc, vhdr + hoff, key0, nkeys, tid);
        } else {
            at_issue_tile<FP8>(kd, ksrc, ld_bytes, key0, nkeys, tid);
            at_issue_tile<FP8>(vd, vsrc, ld_bytes, key0, nkeys, tid);
        }
    };
    float vmax = 1.f;
    if constexpr (FP8) {   // V scales are used relative to the block's largest, so p * vsc / vmax stays <= 1
        float vm = 0.f;
        for (int t = tid; t < Tlen; t += kAtThreads) vm = fmaxf(vm, vscale[blk * Tlen + t]);
        vm = warp_max(vm);
        if (lane == 0) red[warp] = vm;
        __syncthreads();
        vm = red[0];
        for (int i = 1; i < 8; ++i) vm = fmaxf(vm, red[i]);
        vmax = vm;
    }
    const float inv_vmax = vmax > 0.f ? 1.f / vmax : 0.f;

    uint32_t qa[4][4];
    if (active) at_load_q<T>(q + h * 64, ldq, row_base + rw0, g, tq, qa);
    float o[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) o[nt][0] = o[nt][1] = o[nt][2] = o[nt][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    const int pos0 = rw0 + g, pos1 = rw0 + g + 8;   // positions of the thread's two rows

    issue(ring[0][0], ring[0][1], 0);
    cp_async_commit();
    for (int kt = 0; kt < ntiles; ++kt) {
        const int stg = kt & 1;
        if (kt + 1 < ntiles) {
            issue(ring[stg ^ 1][0], ring[stg ^ 1][1], (kt + 1) * kAtKeys);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const T* kt16 = reinterpret_cast<const T*>(ring[stg][0]);
        const T* vt16 = reinterpret_cast<const T*>(ring[stg][1]);
        if constexpr (FP8) {
            at_widen<T>(ring[stg][0], wide[0], tid);
            at_widen<T>(ring[stg][1], wide[1], tid);
            if (tid < kAtKeys) {
                const int key = kt * kAtKeys + tid;
                ksc_s[tid] = key < Tlen ? kscale[blk * Tlen + key] : 0.f;
                vsc_s[tid] = key < Tlen ? vscale[blk * Tlen + key] * inv_vmax : 0.f;
            }
            __syncthreads();
            kt16 = wide[0];
            vt16 = wide[1];
        }
        if constexpr (PK) {
            at_widen_packed<T>(ring[stg][0], wide[0], ksrc, Tlen, kt * kAtKeys, tid);
            at_widen_packed<T>(ring[stg][1], wide[1], vsrc, Tlen, kt * kAtKeys, tid);
            __syncthreads();
            kt16 = wide[0];
            vt16 = wide[1];
        }
        // self-attention: a tile that starts past the warp's last position is masked for all of its rows
        const bool skip = KIND == 0 && kt * kAtKeys > rw0 + 15;
        if (active && !skip) {
            float s[8][4];
            at_scores<T>(smem_u32(kt16), qa, lane, s);
            float tmax0 = -INFINITY, tmax1 = -INFINITY;
#pragma unroll
            for (int nt = 0; nt < 8; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int kl = nt * 8 + 2 * tq + (e & 1), key = kt * kAtKeys + kl;
                    float v = s[nt][e] * 0.125f;
                    if constexpr (FP8) v *= ksc_s[kl];
                    const bool valid = KIND == 0 ? key <= (e < 2 ? pos0 : pos1) : key < Tlen;
                    v = valid ? v : -INFINITY;
                    s[nt][e] = v;
                    if (e < 2) tmax0 = fmaxf(tmax0, v); else tmax1 = fmaxf(tmax1, v);
                }
#pragma unroll
            for (int off = 1; off < 4; off <<= 1) {
                tmax0 = fmaxf(tmax0, __shfl_xor_sync(0xffffffffu, tmax0, off));
                tmax1 = fmaxf(tmax1, __shfl_xor_sync(0xffffffffu, tmax1, off));
            }
            const float mn0 = fmaxf(m0, tmax0), mn1 = fmaxf(m1, tmax1);
            // a row with every key so far masked keeps max -inf: exponentiate against 0 so that the masked scores give exactly 0
            const float base0 = mn0 == -INFINITY ? 0.f : mn0, base1 = mn1 == -INFINITY ? 0.f : mn1;
            const float al0 = __expf(m0 - base0), al1 = __expf(m1 - base1);
            m0 = mn0; m1 = mn1;
            l0 *= al0; l1 *= al1;
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) { o[nt][0] *= al0; o[nt][1] *= al0; o[nt][2] *= al1; o[nt][3] *= al1; }
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                s[nt][0] = __expf(s[nt][0] - base0); s[nt][1] = __expf(s[nt][1] - base0);
                s[nt][2] = __expf(s[nt][2] - base1); s[nt][3] = __expf(s[nt][3] - base1);
                l0 += s[nt][0] + s[nt][1];
                l1 += s[nt][2] + s[nt][3];
                if constexpr (FP8) {
                    const float va = vsc_s[nt * 8 + 2 * tq], vb2 = vsc_s[nt * 8 + 2 * tq + 1];
                    s[nt][0] *= va; s[nt][1] *= vb2; s[nt][2] *= va; s[nt][3] *= vb2;
                }
            }
            // O += P V: k-step j covers keys 16j .. 16j + 15 (score n-tiles 2j, 2j + 1); P enters as hi + lo 16-bit halves
            const uint32_t vbase = smem_u32(vt16);
            const int lm = lane >> 3, lr = lane & 7;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                uint32_t ph[4], pl[4];
                at_split2<T>(s[2 * j][0], s[2 * j][1], ph[0], pl[0]);
                at_split2<T>(s[2 * j][2], s[2 * j][3], ph[1], pl[1]);
                at_split2<T>(s[2 * j + 1][0], s[2 * j + 1][1], ph[2], pl[2]);
                at_split2<T>(s[2 * j + 1][2], s[2 * j + 1][3], ph[3], pl[3]);
#pragma unroll
                for (int np = 0; np < 4; ++np) {   // output dims 16np .. 16np + 15
                    uint32_t bv[4];
                    at_ldsm_x4_trans(vbase + ((j * 16 + (lm & 1) * 8 + lr) * kAtLd + np * 16 + (lm >> 1) * 8) * 2, bv);
                    at_mma<T>(o[2 * np], ph, bv[0], bv[1]);
                    at_mma<T>(o[2 * np], pl, bv[0], bv[1]);
                    at_mma<T>(o[2 * np + 1], ph, bv[2], bv[3]);
                    at_mma<T>(o[2 * np + 1], pl, bv[2], bv[3]);
                }
            }
        }
        __syncthreads();   // the stage (and the widened tiles) may be overwritten from here on
    }
    if (!active) return;
#pragma unroll
    for (int off = 1; off < 4; off <<= 1) {
        l0 += __shfl_xor_sync(0xffffffffu, l0, off);
        l1 += __shfl_xor_sync(0xffffffffu, l1, off);
    }
    const float f0 = vmax / l0, f1 = vmax / l1;
    if (pos0 < n) {
        T* dst = out + (row_base + pos0) * dm + h * 64;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) *reinterpret_cast<uint32_t*>(dst + nt * 8 + 2 * tq) = T16<T>::pack2(o[nt][0] * f0, o[nt][1] * f0);
        if (stats != nullptr && tq == 0) stats[h * stat_rows + row_base + pos0] = make_float2(m0, l0);
    }
    if (pos1 < n) {
        T* dst = out + (row_base + pos1) * dm + h * 64;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) *reinterpret_cast<uint32_t*>(dst + nt * 8 + 2 * tq) = T16<T>::pack2(o[nt][2] * f1, o[nt][3] * f1);
        if (stats != nullptr && tq == 0) stats[h * stat_rows + row_base + pos1] = make_float2(m1, l1);
    }
}

template <typename T, int KIND>
static void launch_attention(const void* q, long long ldq, const void* k, const void* v, long long ld_kv, const float* ks, const float* vs,
                             const int32_t* seq_len, int slot0, void* out, int nw, int H, int Tlen, float2* stats, long long stat_rows,
                             cudaStream_t stream, const uint8_t* kh = nullptr, const uint8_t* vh = nullptr) {
    launch_k(align_attention_kernel<T, KIND>, dim3((kAlignStride + kAtQ - 1) / kAtQ, H, nw), dim3(kAtThreads), 0, stream, 0, (const T*)q, ldq,
             (const uint8_t*)k, (const uint8_t*)v, ld_kv, ks, vs, seq_len, slot0, (T*)out, H, Tlen, stats, stat_rows, kh, vh);
}

wk_status align_self_attention(const void* qkv, const int32_t* seq_len, void* out, int nw, int H, int dtype, cudaStream_t stream) {
    const int d = H * 64;
    if (dtype == WK_DTYPE_F16)
        launch_attention<__half, 0>(qkv, 3 * d, (const __half*)qkv + d, (const __half*)qkv + 2 * d, 3 * d, nullptr, nullptr, seq_len, 0, out, nw, H,
                                    kAlignStride, nullptr, 0, stream);
    else
        launch_attention<__nv_bfloat16, 0>(qkv, 3 * d, (const __nv_bfloat16*)qkv + d, (const __nv_bfloat16*)qkv + 2 * d, 3 * d, nullptr, nullptr,
                                           seq_len, 0, out, nw, H, kAlignStride, nullptr, 0, stream);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("align_self_attention launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

wk_status align_cross_attention(const void* q, const void* kc, const void* vc, const float* kscale, const float* vscale, const int32_t* seq_len,
                                int slot0, void* out, float* stats, int64_t stat_rows, int nw, int H, int Tlen, int dtype, cudaStream_t stream,
                                const uint8_t* khdr, const uint8_t* vhdr) {
    const bool fp8 = kscale != nullptr, f16 = dtype == WK_DTYPE_F16;
    const long long ldq = (long long)H * 64;
    float2* st2 = reinterpret_cast<float2*>(stats);
    if (khdr) {
        if (f16 || fp8 || !vhdr) { set_error("align_cross_attention: the packed cache is bf16 and needs both header vectors"); return WK_ERR_INVALID_ARGUMENT; }
        launch_attention<__nv_bfloat16, 3>(q, ldq, kc, vc, 128, nullptr, nullptr, seq_len, slot0, out, nw, H, Tlen, st2, stat_rows, stream, khdr, vhdr);
    } else if (fp8) {
        if (f16) launch_attention<__half, 2>(q, ldq, kc, vc, 64, kscale, vscale, seq_len, slot0, out, nw, H, Tlen, st2, stat_rows, stream);
        else launch_attention<__nv_bfloat16, 2>(q, ldq, kc, vc, 64, kscale, vscale, seq_len, slot0, out, nw, H, Tlen, st2, stat_rows, stream);
    } else {
        if (f16) launch_attention<__half, 1>(q, ldq, kc, vc, 128, nullptr, nullptr, seq_len, slot0, out, nw, H, Tlen, st2, stat_rows, stream);
        else launch_attention<__nv_bfloat16, 1>(q, ldq, kc, vc, 128, nullptr, nullptr, seq_len, slot0, out, nw, H, Tlen, st2, stat_rows, stream);
    }
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("align_cross_attention launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

// =====================================================================================================
// alignment export.  One CTA = (64-key tile, query tile of 128 rows, window).  For every alignment head of the layer, in ascending order,
// the scores of the tile are recomputed exactly as align_attention_kernel computes them and normalised with the row's final (max, sum);
// the heads' rows are added to the accumulator in that order (first != 0: the layer is the first with alignment heads, so the sum starts
// at 0).  Each accumulator element belongs to one thread of one CTA: the mean is deterministic, in the decode loop's order (layers, then
// heads, decoder_align_mean_kernel).
// =====================================================================================================
// F: 0 the 16-bit cache, 1 FP8, 2 packed bf16
template <typename T, int F>
__global__ void __launch_bounds__(kAtThreads)
align_export_kernel(const T* __restrict__ q, const uint8_t* __restrict__ kc, const float* __restrict__ kscale, const float2* __restrict__ stats,
                    long long stat_rows, const int32_t* __restrict__ seq_len, int slot0, uint32_t mask, int first, float* __restrict__ acc, int H,
                    int Tlen, const uint8_t* __restrict__ khdr) {
    constexpr bool FP8 = F == 1, PK = F == 2;
    constexpr int kTileBytes = FP8 ? kAtKeys * 64 : PK ? kAtKeys * (kPackedRowBytes + 1) : kAtKeys * kAtLd * 2;
    __shared__ __align__(128) uint8_t tile[kTileBytes];
    __shared__ __align__(128) T wide[FP8 || PK ? kAtKeys * kAtLd : 8];
    __shared__ float ksc_s[FP8 ? kAtKeys : 1];
    const int kt = blockIdx.x, qt = blockIdx.y, w = blockIdx.z;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, tq = lane & 3;
    const int n = seq_len[w];
    const int q0 = qt * kAtQ;
    if (q0 >= n) return;
    const long long row_base = (long long)w * kAlignStride;
    const int rw0 = q0 + warp * 16;
    const bool active = rw0 < n;
    const int pos0 = rw0 + g, pos1 = rw0 + g + 8;
    const long long ld_bytes = FP8 ? 64 : 128;   // packed: blocks of T x 128 bytes too
    float a[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int key = kt * kAtKeys + nt * 8 + 2 * tq + (e & 1), pos = e < 2 ? pos0 : pos1;
            a[nt][e] = (!first && active && pos < n && key < Tlen) ? acc[(row_base + pos) * Tlen + key] : 0.f;
        }
    for (uint32_t hm = mask; hm != 0; hm &= hm - 1) {
        const int h = __ffs(hm) - 1;
        const long long blk = (long long)(slot0 + w) * H + h;
        if constexpr (PK) at_issue_tile_packed(tile, kc + blk * Tlen * ld_bytes, khdr + blk * packed_hdr_stride(Tlen), kt * kAtKeys, Tlen, tid);
        else at_issue_tile<FP8>(tile, kc + blk * Tlen * ld_bytes, ld_bytes, kt * kAtKeys, Tlen, tid);
        cp_async_commit();
        cp_async_wait<0>();
        __syncthreads();
        const T* k16 = reinterpret_cast<const T*>(tile);
        if constexpr (FP8) {
            at_widen<T>(tile, wide, tid);
            if (tid < kAtKeys) {
                const int key = kt * kAtKeys + tid;
                ksc_s[tid] = key < Tlen ? kscale[blk * Tlen + key] : 0.f;
            }
            __syncthreads();
            k16 = wide;
        }
        if constexpr (PK) {
            at_widen_packed<T>(tile, wide, kc + blk * Tlen * ld_bytes, Tlen, kt * kAtKeys, tid);
            __syncthreads();
            k16 = wide;
        }
        if (active) {
            uint32_t qa[4][4];
            at_load_q<T>(q + h * 64, (long long)H * 64, row_base + rw0, g, tq, qa);
            float s[8][4];
            at_scores<T>(smem_u32(k16), qa, lane, s);
            const float2 st0 = pos0 < n ? stats[h * stat_rows + row_base + pos0] : make_float2(0.f, 1.f);
            const float2 st1 = pos1 < n ? stats[h * stat_rows + row_base + pos1] : make_float2(0.f, 1.f);
            const float inv0 = 1.f / st0.y, inv1 = 1.f / st1.y;
#pragma unroll
            for (int nt = 0; nt < 8; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    float v = s[nt][e] * 0.125f;
                    if constexpr (FP8) v *= ksc_s[nt * 8 + 2 * tq + (e & 1)];
                    a[nt][e] += __expf(v - (e < 2 ? st0.x : st1.x)) * (e < 2 ? inv0 : inv1);
                }
        }
        __syncthreads();   // the tile is reloaded for the next head
    }
    if (!active) return;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int key = kt * kAtKeys + nt * 8 + 2 * tq + (e & 1), pos = e < 2 ? pos0 : pos1;
            if (pos < n && key < Tlen) acc[(row_base + pos) * Tlen + key] = a[nt][e];
        }
}

wk_status align_export(const void* q, const void* kc, const float* kscale, const float* stats, int64_t stat_rows, const int32_t* seq_len, int slot0,
                       uint32_t mask, int first, float* acc, int nw, int H, int Tlen, int dtype, cudaStream_t stream, const uint8_t* khdr) {
    const dim3 grid((Tlen + kAtKeys - 1) / kAtKeys, (kAlignStride + kAtQ - 1) / kAtQ, nw);
    const float2* st2 = reinterpret_cast<const float2*>(stats);
    const bool fp8 = kscale != nullptr, f16 = dtype == WK_DTYPE_F16;
#define WK_EXPORT(TT, F) launch_k(align_export_kernel<TT, F>, grid, dim3(kAtThreads), 0, stream, 0, (const TT*)q, (const uint8_t*)kc, kscale, st2, \
                                  (long long)stat_rows, seq_len, slot0, mask, first, acc, H, Tlen, khdr)
    if (khdr) {
        if (f16 || fp8) { set_error("align_export: the packed cache is bf16"); return WK_ERR_INVALID_ARGUMENT; }
        WK_EXPORT(__nv_bfloat16, 2);
    } else if (fp8) { if (f16) WK_EXPORT(__half, 1); else WK_EXPORT(__nv_bfloat16, 1); }
    else { if (f16) WK_EXPORT(__half, 0); else WK_EXPORT(__nv_bfloat16, 0); }
#undef WK_EXPORT
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("align_export launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

// out[w][r][t] (Float16, store_rows rows per window): row 0 and rows past the sequence 0, row r = acc[position r - 1] / n_slots
__global__ void align_rows_f16_kernel(const float* __restrict__ acc, const int32_t* __restrict__ seq_len, float n_slots, __half* __restrict__ out,
                                      int Tlen, int store_rows) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y, w = blockIdx.z;
    if (t >= Tlen) return;
    const bool on = r >= 1 && r <= seq_len[w] && n_slots > 0.f;
    const float v = on ? acc[((long long)w * kAlignStride + r - 1) * Tlen + t] / n_slots : 0.f;
    out[((long long)w * store_rows + r) * Tlen + t] = __float2half(v);
}

wk_status align_rows_f16(const float* acc, const int32_t* seq_len, int n_slots, void* out, int nw, int Tlen, int store_rows, cudaStream_t stream) {
    launch_k(align_rows_f16_kernel, dim3((Tlen + 255) / 256, store_rows, nw), dim3(256), 0, stream, 0, acc, seq_len, (float)n_slots, (__half*)out,
             Tlen, store_rows);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("align_rows_f16 launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

// =====================================================================================================
// token log-probs.  One CTA per logits row (position t of window w, rows [r0, r0 + rows) of the pass): out[w][t + 1] =
// logits[target] - max - log(sum exp(logits[:eot] - max)) with target = tokens[t + 1]; NaN when the target is a special or timestamp token
// (>= eot).  Fixed thread-to-element assignment and a fixed reduction tree: the value does not depend on the batch.
// =====================================================================================================
static constexpr int kLpThreads = 256;
__global__ void __launch_bounds__(kLpThreads)
align_logprob_kernel(const float* __restrict__ logits, long long ld, long long r0, const int32_t* __restrict__ row_tok, const int32_t* __restrict__ seq_len,
                     int eot, float* __restrict__ out) {
    __shared__ float red[kLpThreads / 32];
    const long long r = r0 + blockIdx.x;
    const int w = (int)(r / kAlignStride), t = (int)(r % kAlignStride);
    if (t + 1 >= seq_len[w]) return;
    const int target = row_tok[r + 1];
    if (target < 0 || target >= eot) {
        if (threadIdx.x == 0) out[r + 1] = __int_as_float(0x7fc00000);
        return;
    }
    const float* lg = logits + (long long)blockIdx.x * ld;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    float mx = -INFINITY;
    for (int v = tid; v < eot; v += kLpThreads) mx = fmaxf(mx, lg[v]);
    mx = warp_max(mx);
    if (lane == 0) red[warp] = mx;
    __syncthreads();
    mx = red[0];
    for (int i = 1; i < kLpThreads / 32; ++i) mx = fmaxf(mx, red[i]);
    __syncthreads();
    float sm = 0.f;
    for (int v = tid; v < eot; v += kLpThreads) sm += expf(lg[v] - mx);
    sm = warp_sum(sm);
    if (lane == 0) red[warp] = sm;
    __syncthreads();
    if (tid == 0) {
        float tot = 0.f;
        for (int i = 0; i < kLpThreads / 32; ++i) tot += red[i];
        out[r + 1] = lg[target] - mx - logf(tot);
    }
}

wk_status align_token_logprobs(const float* logits, int64_t ld, int64_t r0, int64_t rows, const int32_t* row_tok, const int32_t* seq_len, int eot,
                               float* out, cudaStream_t stream) {
    launch_k(align_logprob_kernel, dim3((unsigned)rows), dim3(kLpThreads), 0, stream, 0, logits, (long long)ld, (long long)r0, row_tok, seq_len, eot, out);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("align_token_logprobs launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

}  // namespace wk
