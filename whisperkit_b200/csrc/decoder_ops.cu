// Decoder-side kernels: everything one autoregressive step needs besides the (swap-AB, split-K) wgmma GEMMs.
//
// Reference behaviour restated on the device (so the host sees only final token IDs):
//   decodeText loop state machine            Sources/WhisperKit/Core/TextDecoder.swift:566-686
//   updateKVCache (host splice, eliminated)  Sources/WhisperKit/Core/TextDecoder.swift:218-270
//   LogitsFiltering x4                       Sources/WhisperKit/Core/Text/LogitsFilter.swift:12-276
//   GreedyTokenSampler.update                Sources/WhisperKit/Core/Text/TokenSampler.swift:42-83,215-240
#include <curand_kernel.h>
#include <math.h>

#include <stdlib.h>

#include "common.cuh"
#include <algorithm>
#include "kernels.h"

namespace wk {

static constexpr int kMaxCtx = 224;  // Constants.maxTokenContext (Models.swift:1334)

__device__ __forceinline__ float block_sum(float v, float* scratch) {
    v = warp_sum(v);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
    __syncthreads();
    if (lane == 0) scratch[warp] = v;
    __syncthreads();
    float r = (lane < nw) ? scratch[lane] : 0.f;
    r = warp_sum(r);
    return r;
}
__device__ __forceinline__ float block_max(float v, float* scratch) {
    v = warp_max(v);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
    __syncthreads();
    if (lane == 0) scratch[warp] = v;
    __syncthreads();
    float r = (lane < nw) ? scratch[lane] : -INFINITY;
    r = warp_max(r);
    return r;
}

// =====================================================================================================
// decode state
// =====================================================================================================
__global__ void decode_slots_init_kernel(DecodeState st, RowParams* __restrict__ rp_dev, const int32_t* __restrict__ slot_ids,
                                         const int32_t* __restrict__ prompts, const RowParams* __restrict__ rp_new, BeamState bs) {
    const int i = blockIdx.x, b = slot_ids[i];
    const RowParams R = rp_new[i];
    const int n_prompt = R.prompt_len;
    for (int t = threadIdx.x; t < kMaxCtx; t += blockDim.x) {
        st.tokens[b * kMaxCtx + t] = t < n_prompt ? prompts[i * kMaxCtx + t] : 0;
        st.logprobs[b * kMaxCtx + t] = 0.f;
        // the call has beam rows, so the self-attention reads every row through the cache ancestry: a row that never reorders (single or
        // sample rung) must read its own cache rows.  beam_update_kernel rewrites the entries of beam rows before they are read
        if (bs.use_anc) bs.anc[b * kMaxCtx + t] = b;
    }
    if (st.bias_pool)   // every phrase match starts over with the window and with each ladder rung
        for (int t = threadIdx.x; t < kMaxBiasPhrases; t += blockDim.x) st.bias_m[b * kMaxBiasPhrases + t] = 0;
    if (threadIdx.x == 0) {
        if (st.bias_pool) st.bias_acc[b] = 0;
        rp_dev[b] = R;
        st.n_tokens[b] = n_prompt;
        st.next_token[b] = n_prompt > 0 ? prompts[i * kMaxCtx + n_prompt - 1] : 0;
        st.done[b] = 0;
        st.first_low[b] = 0;
        st.steps[b] = 0;
        st.input_ids[b] = 0;
        st.error[b] = 0;
        st.lang_token[b] = -1;
        st.lang_logprob[b] = 0.f;
        st.lang_state[b] = R.detect == 2 ? kLangLead : 0;
        st.no_speech[b] = __int_as_float(0x7fc00000);   // NaN: not computed (yet)
        if (bs.beam > 1) {
            bs.sum_lp[b] = 0.f;
            if (b % bs.group == 0) bs.n_fin[b / bs.group] = 0;
        }
    }
}

wk_status decode_slots_init(DecodeState st, RowParams* rp_dev, const int32_t* slot_ids, const int32_t* prompts, const RowParams* rp_new,
                            int n, cudaStream_t stream, BeamState beam) {
    if (n < 1) return WK_OK;
    decode_slots_init_kernel<<<n, 64, 0, stream>>>(st, rp_dev, slot_ids, prompts, rp_new, beam);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("decode_slots_init launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

// =====================================================================================================
// token + position embedding, prompt forcing (TextDecoder.swift:581-594), first LayerNorm
// =====================================================================================================
template <typename T>
__global__ void __launch_bounds__(256)
decoder_embed_ln_kernel(const T* __restrict__ emb, const float* __restrict__ pos_emb, const float* __restrict__ gamma,
                        const float* __restrict__ beta, DecodeState st, int vocab, int ts_begin, float* __restrict__ x,
                        T* __restrict__ xn, int d, const int32_t* __restrict__ explicit_pos) {
    __shared__ float scratch[32];
    const int b = blockIdx.x, tid = threadIdx.x;
    pdl_launch_dependents();
    pdl_wait();
    int tok, pos;
    if (explicit_pos) {
        tok = st.input_ids[b];
        pos = explicit_pos[b];
    } else {
        if (st.done[b]) return;          // the window has ended: its row of the step is dead (x / xn keep their last values)
        const int step = st.steps[b];
        const int prompt_len = st.rp[b].prompt_len;
        pos = step;
        tok = st.next_token[b];
        bool overwrite = false;
        const int lang_state = st.lang_state[b];
        if (lang_state == kLangLead) {
            tok = st.rp[b].lead_token;   // leading language-detection step: [SOT] at position 0 (steps[b] is still 0)
        } else if (step < prompt_len) {
            const int cur = st.tokens[b * kMaxCtx + step];
            const bool is_ts = cur >= ts_begin, pred_ts = tok >= ts_begin;
            if (!(step == prompt_len - 1 && is_ts && pred_ts)) tok = cur;
            else overwrite = true;  // model-predicted first timestamp replaces the forced <|0.00|>
        }
        __syncthreads();
        if (tid == 0) {
            if (overwrite) st.tokens[b * kMaxCtx + step] = tok;
            st.input_ids[b] = tok;
            if (lang_state == kLangLeadRan) st.lang_state[b] = 0;   // the previous step was the leading detection step: this is step 0
        }
    }
    tok = min(max(tok, 0), vocab - 1);   // never index the embedding table out of bounds
    float v[8];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int i = tid + k * 256;
        v[k] = 0.f;
        if (i < d) {
            v[k] = T16<T>::to_f(emb[(long long)tok * d + i]) + pos_emb[(long long)pos * d + i];
            x[(long long)b * d + i] = v[k];
            s += v[k];
        }
    }
    const float mean = block_sum(s, scratch) / d;
    float q = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int i = tid + k * 256;
        if (i < d) { const float a = v[k] - mean; q += a * a; }
    }
    const float rstd = rsqrtf(block_sum(q, scratch) / d + 1e-5f);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int i = tid + k * 256;
        if (i < d) xn[(long long)b * d + i] = T16<T>::from_f((v[k] - mean) * rstd * gamma[i] + beta[i]);
    }
}

wk_status decoder_embed_ln(const void* emb16, const float* pos, const float* gamma, const float* beta, DecodeState st, int vocab,
                           int ts_begin, float* x, void* xn, int B, int d, int dtype, const int32_t* explicit_pos, cudaStream_t stream) {
    if (d > 2048) { set_error("decoder_embed_ln: d_model %d > 2048", d); return WK_ERR_INVALID_ARGUMENT; }
    if (dtype == WK_DTYPE_F16)
        launch_k(decoder_embed_ln_kernel<__half>, dim3(B), dim3(256), 0, stream, 1, (const __half*)emb16, pos, gamma, beta, st, vocab, ts_begin, x, (__half*)xn, d, explicit_pos);
    else
        launch_k(decoder_embed_ln_kernel<__nv_bfloat16>, dim3(B), dim3(256), 0, stream, 1, (const __nv_bfloat16*)emb16, pos, gamma, beta, st, vocab, ts_begin, x, (__nv_bfloat16*)xn, d, explicit_pos);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("decoder_embed_ln launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

// =====================================================================================================
// split-K reduce + bias + residual + LayerNorm      (partials [S][Bp][d] f32, written by the swap-AB GEMM)
// =====================================================================================================
static constexpr int kReduceThreads = 320;   // one float4 per thread at d = 1280
static constexpr int kMaxSplits = 20;

// All split-K partial loads of a thread are issued back to back (fully unrolled, predicated) so the kernel pays one
// L2 round trip instead of `splits` serial ones; the sum runs in a fixed order (deterministic).
template <typename T>
__global__ void __launch_bounds__(kReduceThreads)
decoder_reduce_resid_ln_kernel(const float* __restrict__ partial, int splits, int Bp, const float* __restrict__ bias,
                               const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ x,
                               T* __restrict__ xn, int d) {
    __shared__ float scratch[32];
    const int b = blockIdx.x, tid = threadIdx.x;
    const int d4 = d >> 2;
    pdl_launch_dependents();
    pdl_wait();
    float4 v[2];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const int i4 = tid + k * kReduceThreads;
        v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i4 < d4) {
            float4 p[kMaxSplits];
#pragma unroll
            for (int sp = 0; sp < kMaxSplits; ++sp)
                if (sp < splits) p[sp] = __ldcg(reinterpret_cast<const float4*>(partial + ((long long)sp * Bp + b) * d) + i4);
            float4 a = reinterpret_cast<const float4*>(x + (long long)b * d)[i4];
            if (bias) {
                const float4 bb = __ldg(reinterpret_cast<const float4*>(bias) + i4);
                a.x += bb.x; a.y += bb.y; a.z += bb.z; a.w += bb.w;
            }
#pragma unroll
            for (int sp = 0; sp < kMaxSplits; ++sp)
                if (sp < splits) { a.x += p[sp].x; a.y += p[sp].y; a.z += p[sp].z; a.w += p[sp].w; }
            v[k] = a;
            reinterpret_cast<float4*>(x + (long long)b * d)[i4] = a;
            s += a.x + a.y + a.z + a.w;
        }
    }
    const float mean = block_sum(s, scratch) / d;
    float q = 0.f;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const int i4 = tid + k * kReduceThreads;
        if (i4 < d4) {
            const float a0 = v[k].x - mean, a1 = v[k].y - mean, a2 = v[k].z - mean, a3 = v[k].w - mean;
            q += a0 * a0 + a1 * a1 + a2 * a2 + a3 * a3;
        }
    }
    const float rstd = rsqrtf(block_sum(q, scratch) / d + 1e-5f);
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const int i4 = tid + k * kReduceThreads;
        if (i4 < d4) {
            const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + i4), bb = __ldg(reinterpret_cast<const float4*>(beta) + i4);
            uint2 pk;
            pk.x = T16<T>::pack2((v[k].x - mean) * rstd * g.x + bb.x, (v[k].y - mean) * rstd * g.y + bb.y);
            pk.y = T16<T>::pack2((v[k].z - mean) * rstd * g.z + bb.z, (v[k].w - mean) * rstd * g.w + bb.w);
            reinterpret_cast<uint2*>(xn + (long long)b * d)[i4] = pk;
        }
    }
}

wk_status decoder_reduce_resid_ln(const float* partial, int splits, int Bp, const float* bias, const float* gamma,
                                  const float* beta, float* x, void* xn, int B, int d, int dtype, cudaStream_t stream) {
    if (splits > kMaxSplits || d > 8 * kReduceThreads || (d & 3)) {
        set_error("decoder_reduce_resid_ln: unsupported splits %d / d %d", splits, d);
        return WK_ERR_INVALID_ARGUMENT;
    }
    if (dtype == WK_DTYPE_F16)
        launch_k(decoder_reduce_resid_ln_kernel<__half>, dim3(B), dim3(kReduceThreads), 0, stream, 32, partial, splits, Bp, bias, gamma, beta, x, (__half*)xn, d);
    else
        launch_k(decoder_reduce_resid_ln_kernel<__nv_bfloat16>, dim3(B), dim3(kReduceThreads), 0, stream, 32, partial, splits, Bp, bias, gamma, beta, x, (__nv_bfloat16*)xn, d);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("decoder_reduce_resid_ln launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

template <typename T>
__global__ void __launch_bounds__(256)
decoder_reduce_bias_gelu_kernel(const float* __restrict__ partial, int splits, int Bp, const float* __restrict__ bias,
                                T* __restrict__ out, int B, int n) {
    pdl_launch_dependents();
    pdl_wait();
    const long long idx = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (idx >= (long long)B * n) return;
    const int b = (int)(idx / n), i = (int)(idx - (long long)b * n);
    float4 a = *reinterpret_cast<const float4*>(bias + i);
    float4 p[8];
#pragma unroll
    for (int sp = 0; sp < 8; ++sp)
        if (sp < splits) p[sp] = __ldcg(reinterpret_cast<const float4*>(partial + ((long long)sp * Bp + b) * n + i));
#pragma unroll
    for (int sp = 0; sp < 8; ++sp)
        if (sp < splits) { a.x += p[sp].x; a.y += p[sp].y; a.z += p[sp].z; a.w += p[sp].w; }
    for (int sp = 8; sp < splits; ++sp) {
        const float4 pp = __ldcg(reinterpret_cast<const float4*>(partial + ((long long)sp * Bp + b) * n + i));
        a.x += pp.x; a.y += pp.y; a.z += pp.z; a.w += pp.w;
    }
    uint2 pk;
    pk.x = T16<T>::pack2(gelu_erf(a.x), gelu_erf(a.y));
    pk.y = T16<T>::pack2(gelu_erf(a.z), gelu_erf(a.w));
    *reinterpret_cast<uint2*>(out + (long long)b * n + i) = pk;
}

wk_status decoder_reduce_bias_gelu(const float* partial, int splits, int Bp, const float* bias, void* out, int B, int n,
                                   int dtype, cudaStream_t stream) {
    const long long threads = (long long)B * n / 4;
    const unsigned grid = (unsigned)((threads + 255) / 256);
    if (dtype == WK_DTYPE_F16)
        launch_k(decoder_reduce_bias_gelu_kernel<__half>, dim3(grid), dim3(256), 0, stream, 32, partial, splits, Bp, bias, (__half*)out, B, n);
    else
        launch_k(decoder_reduce_bias_gelu_kernel<__nv_bfloat16>, dim3(grid), dim3(256), 0, stream, 32, partial, splits, Bp, bias, (__nv_bfloat16*)out, B, n);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("decoder_reduce_bias_gelu launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

// =====================================================================================================
// self attention for one new token: one CTA (4 warps) per (b, h).  Warp 0 reduces the q/k/v split-K partials and appends K/V in place
// in the device cache (replaces the host-side updateKVCache splice); the cached positions are then split over the 4 warps - 8 lanes
// per 128-byte row, 4 rows per warp instruction, several instructions in flight - so that B*H*4 warps keep enough loads in the air
// for what is a latency-bound gather (<= 223 rows of K and of V per head).  cache layout [B][H][max_len][64]
// =====================================================================================================
template <typename T, bool kAnc>
__global__ void __launch_bounds__(128)
decoder_self_attention_kernel(const float* __restrict__ partial, int splits, int Bp, const float* __restrict__ bq,
                              const float* __restrict__ bv, T* __restrict__ kcache, T* __restrict__ vcache,
                              const int32_t* __restrict__ pos_ptr, const int32_t* __restrict__ done,
                              T* __restrict__ out, int B, int H, int max_len, const int32_t* __restrict__ anc) {
    __shared__ float sq[64], skc[64], svc[64];
    __shared__ float sp[kMaxCtx];
    __shared__ float red[4][64];
    __shared__ float sstat[8];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int bh = blockIdx.x, b = bh / H, h = bh % H;
    pdl_launch_dependents();
    pdl_wait();
    if (done != nullptr && done[b]) return;   // ended window: no cache traffic
    const int dm = H * 64;
    const int pos = pos_ptr[b];
    // cache row of position t: this sequence's own row, or (beam search) the row of the ancestor beam that produced position t
    const int32_t* arow = kAnc ? anc + (long long)b * max_len : nullptr;
    const long long own = (long long)bh * max_len;
    auto row_of = [&](int t) -> long long { return kAnc ? ((long long)arow[t] * H + h) * max_len + t : own + t; };
    if (warp == 0) {
        const int e = 2 * lane;
        float2 q = make_float2(bq[h * 64 + e], bq[h * 64 + e + 1]);
        float2 k = make_float2(0.f, 0.f);
        float2 v = make_float2(bv[h * 64 + e], bv[h * 64 + e + 1]);
        for (int s = 0; s < splits; ++s) {
            const float* pr = partial + ((long long)s * Bp + b) * (3LL * dm) + h * 64 + e;
            const float2 pq = *reinterpret_cast<const float2*>(pr);
            const float2 pk = *reinterpret_cast<const float2*>(pr + dm);
            const float2 pv = *reinterpret_cast<const float2*>(pr + 2 * dm);
            q.x += pq.x; q.y += pq.y; k.x += pk.x; k.y += pk.y; v.x += pv.x; v.y += pv.y;
        }
        // append to the cache (16-bit rounding is part of the precision policy); the new row always goes to the sequence's own cache row
        const uint32_t k16 = T16<T>::pack2(k.x, k.y), v16 = T16<T>::pack2(v.x, v.y);
        *reinterpret_cast<uint32_t*>(kcache + (own + pos) * 64 + e) = k16;
        *reinterpret_cast<uint32_t*>(vcache + (own + pos) * 64 + e) = v16;
        const float2 kr = T16<T>::unpack2(k16), vr = T16<T>::unpack2(v16);
        sq[e] = q.x; sq[e + 1] = q.y;
        skc[e] = kr.x; skc[e + 1] = kr.y;
        svc[e] = vr.x; svc[e + 1] = vr.y;
        const float self = warp_sum(q.x * kr.x + q.y * kr.y);   // the current position's score comes from registers
        if (lane == 0) sp[pos] = self * 0.125f;
    }
    __syncthreads();
    const int sub = lane & 7, rsel = lane >> 3;   // 16-byte piece of the 128-byte row / row within a group of 4
    float qv[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) qv[j] = sq[sub * 8 + j];
    // ---- scores over the cached positions: warp w takes rows 16 i + 4 w + rsel
    const T* kb = kcache + sub * 8;
#pragma unroll 4
    for (int t0 = warp * 4; t0 < pos; t0 += 16) {
        const int t = t0 + rsel;
        float acc = 0.f;
        if (t < pos) {
            const uint4 u = *reinterpret_cast<const uint4*>(kb + row_of(t) * 64);
            const float2 a0 = T16<T>::unpack2(u.x), a1 = T16<T>::unpack2(u.y), a2 = T16<T>::unpack2(u.z), a3 = T16<T>::unpack2(u.w);
            acc = qv[0] * a0.x + qv[1] * a0.y + qv[2] * a1.x + qv[3] * a1.y + qv[4] * a2.x + qv[5] * a2.y + qv[6] * a3.x + qv[7] * a3.y;
        }
        acc += __shfl_xor_sync(0xffffffffu, acc, 1);
        acc += __shfl_xor_sync(0xffffffffu, acc, 2);
        acc += __shfl_xor_sync(0xffffffffu, acc, 4);
        if (sub == 0 && t < pos) sp[t] = acc * 0.125f;
    }
    __syncthreads();
    // ---- softmax over positions 0..pos
    float mx = -INFINITY;
    for (int t = tid; t <= pos; t += 128) mx = fmaxf(mx, sp[t]);
    mx = warp_max(mx);
    if (lane == 0) sstat[warp] = mx;
    __syncthreads();
    mx = fmaxf(fmaxf(sstat[0], sstat[1]), fmaxf(sstat[2], sstat[3]));
    float sm = 0.f;
    for (int t = tid; t <= pos; t += 128) {
        const float pr = __expf(sp[t] - mx);
        sp[t] = pr;
        sm += pr;
    }
    sm = warp_sum(sm);
    if (lane == 0) sstat[4 + warp] = sm;
    __syncthreads();
    const float inv = 1.f / (sstat[4] + sstat[5] + sstat[6] + sstat[7]);
    // ---- output: sum_t p[t] V[t]
    float o8[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o8[j] = 0.f;
    const T* vb = vcache + sub * 8;
#pragma unroll 4
    for (int t0 = warp * 4; t0 < pos; t0 += 16) {
        const int t = t0 + rsel;
        if (t < pos) {
            const float pr = sp[t];
            const uint4 u = *reinterpret_cast<const uint4*>(vb + row_of(t) * 64);
            const float2 a0 = T16<T>::unpack2(u.x), a1 = T16<T>::unpack2(u.y), a2 = T16<T>::unpack2(u.z), a3 = T16<T>::unpack2(u.w);
            o8[0] += pr * a0.x; o8[1] += pr * a0.y; o8[2] += pr * a1.x; o8[3] += pr * a1.y;
            o8[4] += pr * a2.x; o8[5] += pr * a2.y; o8[6] += pr * a3.x; o8[7] += pr * a3.y;
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        o8[j] += __shfl_xor_sync(0xffffffffu, o8[j], 8);
        o8[j] += __shfl_xor_sync(0xffffffffu, o8[j], 16);
    }
    if (rsel == 0) {
#pragma unroll
        for (int j = 0; j < 8; ++j) red[warp][sub * 8 + j] = o8[j];
    }
    __syncthreads();
    if (tid < 64) {
        // the current position comes from shared memory (its cache row was written by this CTA just above)
        const float o = red[0][tid] + red[1][tid] + red[2][tid] + red[3][tid] + sp[pos] * svc[tid];
        out[(long long)b * dm + h * 64 + tid] = T16<T>::from_f(o * inv);
    }
}

wk_status decoder_self_attention(const float* partial, int splits, int Bp, const float* bq, const float* bv, void* kcache,
                                 void* vcache, const int32_t* pos, const int32_t* done, void* out, int B, int H,
                                 int max_len, int dtype, cudaStream_t stream, const int32_t* anc) {
    if (max_len > kMaxCtx) { set_error("decoder_self_attention: max_len %d > %d", max_len, kMaxCtx); return WK_ERR_INVALID_ARGUMENT; }
    const unsigned grid = (unsigned)(B * H);
    if (dtype == WK_DTYPE_F16) {
        if (anc) launch_k(decoder_self_attention_kernel<__half, true>, dim3(grid), dim3(128), 0, stream, 2, partial, splits, Bp, bq, bv, (__half*)kcache, (__half*)vcache, pos, done, (__half*)out, B, H, max_len, anc);
        else launch_k(decoder_self_attention_kernel<__half, false>, dim3(grid), dim3(128), 0, stream, 2, partial, splits, Bp, bq, bv, (__half*)kcache, (__half*)vcache, pos, done, (__half*)out, B, H, max_len, anc);
    } else {
        if (anc) launch_k(decoder_self_attention_kernel<__nv_bfloat16, true>, dim3(grid), dim3(128), 0, stream, 2, partial, splits, Bp, bq, bv, (__nv_bfloat16*)kcache, (__nv_bfloat16*)vcache, pos, done, (__nv_bfloat16*)out, B, H, max_len, anc);
        else launch_k(decoder_self_attention_kernel<__nv_bfloat16, false>, dim3(grid), dim3(128), 0, stream, 2, partial, splits, Bp, bq, bv, (__nv_bfloat16*)kcache, (__nv_bfloat16*)vcache, pos, done, (__nv_bfloat16*)out, B, H, max_len, anc);
    }
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("decoder_self_attention launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

// The K/V append of decoder_self_attention_kernel's warp 0 alone (same sums in the same order, same rounding): one warp per (b, h)
template <typename T>
__global__ void __launch_bounds__(32)
decoder_kv_append_kernel(const float* __restrict__ partial, int splits, int Bp, const float* __restrict__ bv, T* __restrict__ kcache,
                         T* __restrict__ vcache, const int32_t* __restrict__ pos_ptr, const int32_t* __restrict__ done, int H, int max_len) {
    const int lane = threadIdx.x, bh = blockIdx.x, b = bh / H, h = bh % H;
    pdl_launch_dependents();
    pdl_wait();
    if (done != nullptr && done[b]) return;
    const int dm = H * 64, e = 2 * lane;
    const long long own = (long long)bh * max_len + pos_ptr[b];
    float2 k = make_float2(0.f, 0.f);
    float2 v = make_float2(bv[h * 64 + e], bv[h * 64 + e + 1]);
    for (int s = 0; s < splits; ++s) {
        const float* pr = partial + ((long long)s * Bp + b) * (3LL * dm) + h * 64 + e;
        const float2 pk = *reinterpret_cast<const float2*>(pr + dm);
        const float2 pv = *reinterpret_cast<const float2*>(pr + 2 * dm);
        k.x += pk.x; k.y += pk.y; v.x += pv.x; v.y += pv.y;
    }
    *reinterpret_cast<uint32_t*>(kcache + own * 64 + e) = T16<T>::pack2(k.x, k.y);
    *reinterpret_cast<uint32_t*>(vcache + own * 64 + e) = T16<T>::pack2(v.x, v.y);
}

wk_status decoder_kv_append(const float* partial, int splits, int Bp, const float* bv, void* kcache, void* vcache, const int32_t* pos,
                            const int32_t* done, int B, int H, int max_len, int dtype, cudaStream_t stream) {
    if (max_len > kMaxCtx) { set_error("decoder_kv_append: max_len %d > %d", max_len, kMaxCtx); return WK_ERR_INVALID_ARGUMENT; }
    if (dtype == WK_DTYPE_F16)
        launch_k(decoder_kv_append_kernel<__half>, dim3(B * H), dim3(32), 0, stream, 2, partial, splits, Bp, bv, (__half*)kcache, (__half*)vcache, pos, done, H, max_len);
    else
        launch_k(decoder_kv_append_kernel<__nv_bfloat16>, dim3(B * H), dim3(32), 0, stream, 2, partial, splits, Bp, bv, (__nv_bfloat16*)kcache,
                 (__nv_bfloat16*)vcache, pos, done, H, max_len);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("decoder_kv_append launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

// =====================================================================================================
// cross attention for one query per (b, h) over T encoder positions.  HBM-streaming kernel: each CTA pulls its
// contiguous K block then V block through a ring of 16000-byte bulk-copy stages (cp.async.bulk + mbarrier), a dedicated producer warp
// keeps the ring full while 4 consumer warps compute.  K/V layout [B][H][T][64] (written head-major by the cross-KV GEMM epilogue).
//   16-bit cache: 128-byte rows, 125 rows per stage, 2 stages (5 CTAs per SM); a lane takes 8 values (16 bytes) of a row.
//   packed bf16 cache (common.cuh): the producer bulk-loads the block's K and V header vectors, then per stage the 12000 bytes of primary
//   slots and, on the same barrier, one 32-byte copy of each raw row's secondary slot into the stage's side area; a lane rebuilds the exact
//   uint4 the 16-bit row holds (cross_piece), so the dot products, the row-to-lane mapping and the reduction order are the 16-bit ones.
//   FP8 cache (FP8 = true): 64-byte rows of E4M3 codes with one f32 scale per row ([B][H][T], see fp8_row_scale), 250 rows per stage,
//   2 stages (4 CTAs per SM); the producer first bulk-loads the block's two scale vectors, a lane widens 16
//   codes exactly to f32, the K scale multiplies each key's dot product before the softmax and the V scale is folded into p for the P.V
//   phase - the alignment export stays the normalised softmax row.
// =====================================================================================================
enum CrossFmt { kCrossRaw16 = 0, kCrossFp8 = 1, kCrossPacked = 2 };
template <int F> struct CrossCfg {
    static constexpr bool FP8 = F == kCrossFp8;
    static constexpr int kRowBytes = FP8 ? 64 : 128;
    static constexpr int kRows = FP8 ? 250 : 125;             // rows per stage: kRows * kRowBytes = 16000 B (multiple of 16)
    // bytes a stage occupies in the ring: packed, the 12000-byte primary slots, then one 32-byte secondary slot per row (filled for raw rows)
    static constexpr int kStageBytes = kRows * kRowBytes;
    static constexpr int kLoadBytes = F == kCrossPacked ? kRows * kPackedRowBytes : kStageBytes;   // bytes of a stage's bulk copy
    // 2 stages: 38.6 KB of shared memory per 16-bit CTA (5 per SM), 50.3 KB per FP8 CTA (4 per SM).  More, smaller CTAs per SM keep
    // more K/V streams in flight and shorten the last wave: a deeper ring (4 stages, 3 CTAs per SM) moved the same bytes more slowly
    static constexpr int kStages = 2;
    static constexpr int kLanesPerRow = kRowBytes / 16;       // a lane reads 16 bytes of a row
    static constexpr int kRowsPerWarp = 32 / kLanesPerRow;    // rows per warp instruction
    static constexpr int kDims = 64 / kLanesPerRow;           // values per lane
};
static constexpr int kCrossRows = CrossCfg<kCrossRaw16>::kRows;
static constexpr int kCrossThreads = 160;           // 4 consumer warps + 1 producer warp

__device__ __forceinline__ void fp8x16_to_f32(const uint4 u, float (&x)[16]) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        uint32_t lo, hi;
        fp8x4_to_half2(w[k], lo, hi);
        const float2 a = T16<__half>::unpack2(lo), b = T16<__half>::unpack2(hi);
        x[4 * k] = a.x; x[4 * k + 1] = a.y; x[4 * k + 2] = b.x; x[4 * k + 3] = b.y;
    }
}
// q . (this lane's 16 bytes of a K row)
template <typename T, int F>
__device__ __forceinline__ float cross_row_dot(const uint4 u, const float (&qv)[CrossCfg<F>::kDims]) {
    if constexpr (CrossCfg<F>::FP8) {
        float x[16];
        fp8x16_to_f32(u, x);
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < 16; ++j) acc = fmaf(qv[j], x[j], acc);
        return acc;
    } else {
        const float2 a0 = T16<T>::unpack2(u.x), a1 = T16<T>::unpack2(u.y), a2 = T16<T>::unpack2(u.z), a3 = T16<T>::unpack2(u.w);
        return qv[0] * a0.x + qv[1] * a0.y + qv[2] * a1.x + qv[3] * a1.y + qv[4] * a2.x + qv[5] * a2.y + qv[6] * a3.x + qv[7] * a3.y;
    }
}
// acc += p * (this lane's 16 bytes of a V row)
template <typename T, int F>
__device__ __forceinline__ void cross_row_axpy(const uint4 u, float p, float (&acc)[CrossCfg<F>::kDims]) {
    if constexpr (CrossCfg<F>::FP8) {
        float x[16];
        fp8x16_to_f32(u, x);
#pragma unroll
        for (int j = 0; j < 16; ++j) acc[j] = fmaf(p, x[j], acc[j]);
    } else {
        const float2 a0 = T16<T>::unpack2(u.x), a1 = T16<T>::unpack2(u.y), a2 = T16<T>::unpack2(u.z), a3 = T16<T>::unpack2(u.w);
        acc[0] += p * a0.x; acc[1] += p * a0.y; acc[2] += p * a1.x; acc[3] += p * a1.y;
        acc[4] += p * a2.x; acc[5] += p * a2.y; acc[6] += p * a3.x; acc[7] += p * a3.y;
    }
}

// this lane's 16 bytes (8 16-bit values, or 16 FP8 codes) of row r of a stage; packed: rebuilt from the row's slots (header byte h)
template <int F>
__device__ __forceinline__ uint4 cross_piece(const uint8_t* tile, int r, int sub, uint8_t h) {
    using C = CrossCfg<F>;
    if constexpr (F == kCrossPacked) {
        const uint8_t* row = tile + r * kPackedRowBytes;
        if (h == kPackedRaw) return *reinterpret_cast<const uint4*>(sub < 6 ? row + 16 * sub : tile + C::kLoadBytes + r * 32 + 16 * (sub - 6));
        return unpack_bf16x8(*reinterpret_cast<const uint2*>(row + 8 * sub), *reinterpret_cast<const uint32_t*>(row + 64 + 4 * sub), h);
    } else {
        return *reinterpret_cast<const uint4*>(tile + r * C::kRowBytes + sub * 16);
    }
}

template <typename T, int F>
__global__ void __launch_bounds__(kCrossThreads)
decoder_cross_attention_kernel(const float* __restrict__ partial, int splits, int Bp, const float* __restrict__ bq,
                               const uint8_t* __restrict__ kcross, const uint8_t* __restrict__ vcross, const float* __restrict__ kscale,
                               const float* __restrict__ vscale, T* __restrict__ out, int B, int H, int Tlen, const int32_t* __restrict__ done,
                               float* __restrict__ align_scratch, uint32_t align_mask, int kv_div, const uint8_t* __restrict__ khdr,
                               const uint8_t* __restrict__ vhdr) {
    using C = CrossCfg<F>;
    constexpr bool FP8 = C::FP8, PACKED = F == kCrossPacked;
    extern __shared__ __align__(128) uint8_t smem[];
    const int Tp = (Tlen + 3) & ~3;
    uint8_t* ring = smem;                                                   // C::kStages * 16000
    float* scores = reinterpret_cast<float*>(smem + C::kStages * C::kStageBytes);   // [Tlen]
    float* ksc = scores + Tp;                                               // FP8: [Tlen] K row scales
    float* vsc = ksc + Tp;                                                  // FP8: [Tlen] V row scales
    const int hs = packed_hdr_stride(Tlen);
    uint8_t* hdr = reinterpret_cast<uint8_t*>(scores + Tp);                 // packed: [2][hs] K then V row headers
    float* sq = FP8 ? vsc + Tp : PACKED ? reinterpret_cast<float*>(hdr + 2 * hs) : scores + Tp;   // [64]
    float* red = sq + 64;                                                   // [4][64] + scratch
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(red + 4 * 64 + 32);
    uint64_t* empty_bar = full_bar + C::kStages;
    uint64_t* scale_bar = empty_bar + C::kStages;                           // FP8: the row scales, packed: the row headers

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // grid order: (window, head, beam) - the kv_div rows that share one K/V block are adjacent, so their streams meet in L2
    const int beam_j = blockIdx.x % kv_div, wh = blockIdx.x / kv_div;
    const int win = wh / H, h = wh % H, b = win * kv_div + beam_j;
    const int kvh = win * H + h;             // K/V block index: [window][head]
    const int dm = H * 64;
    const int chunks = Tlen / C::kRows;  // per K and per V
    pdl_launch_dependents();
    // ended window: skip its K/V stream.  done[] was written by the sampler of the previous step, many kernels upstream, so it
    // may be read before griddepcontrol.wait; the load is issued here and consumed after the barrier set-up so that its latency hides
    // under it (the CTA lives ~8 us: a dependent L2 round trip at its start would cost several per cent of the kernel)
    const int ended = done != nullptr ? done[b] : 0;
    if (tid == 0) {
        for (int i = 0; i < C::kStages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 4); }
        if constexpr (FP8 || PACKED) mbar_init(scale_bar, 1);
        fence_barrier_init();
    }
    __syncthreads();
    if (ended) { pdl_wait(); return; }   // (the wait still runs: this grid must not complete before its upstream does)

    if (warp == 4) {
        // ---------------- producer ----------------
        // no griddepcontrol.wait here: the cross K/V cache is written once before the decode loop starts, so when this kernel is
        // launched as a programmatic dependent the first K chunks are already in flight while the upstream GEMM drains
        if constexpr (PACKED) {
            // packed: the two header vectors, then per stage the primary slots and a 32-byte copy of the secondary slot of each raw row
            // into the stage's side area, all on the stage's barrier.  The primary copy is issued before the headers are read, so only
            // the first stage's raw copies wait for the header load
            const uint8_t* kb = kcross + (long long)kvh * Tlen * 128;
            const uint8_t* vb = vcross + (long long)kvh * Tlen * 128;
            if (lane == 0) {
                mbar_expect_tx(scale_bar, 2u * hs);
                bulk_load_1d(hdr, khdr + (long long)kvh * hs, hs, scale_bar);
                bulk_load_1d(hdr + hs, vhdr + (long long)kvh * hs, hs, scale_bar);
            }
            for (int c = 0; c < 2 * chunks; ++c) {
                const int stage = c % C::kStages;
                const uint32_t ph = (c / C::kStages) & 1;
                const int cc = c < chunks ? c : c - chunks;
                const uint8_t* blk = c < chunks ? kb : vb;
                uint8_t* dst = ring + stage * C::kStageBytes;
                mbar_wait(&empty_bar[stage], ph ^ 1);
                if (lane == 0) {
                    mbar_expect_tx_only(&full_bar[stage], C::kLoadBytes);
                    bulk_load_1d(dst, blk + (long long)cc * C::kLoadBytes, C::kLoadBytes, &full_bar[stage]);
                }
                mbar_wait(scale_bar, 0);
                const uint8_t* h = hdr + (c < chunks ? 0 : hs) + cc * C::kRows;
                int raw = 0;
                for (int r = lane; r < C::kRows; r += 32)
                    if (h[r] == kPackedRaw) {
                        bulk_load_1d(dst + C::kLoadBytes + r * 32, blk + (long long)Tlen * kPackedRowBytes + (long long)(cc * C::kRows + r) * 32, 32,
                                     &full_bar[stage]);
                        ++raw;
                    }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) raw += __shfl_xor_sync(0xffffffffu, raw, o);
                if (lane == 0) mbar_expect_tx(&full_bar[stage], 32u * raw);   // the stage's one arrival
            }
            return;
        }
        if (lane == 0) {
            if constexpr (FP8) {
                mbar_expect_tx(scale_bar, 2u * Tlen * 4);
                bulk_load_1d(ksc, kscale + (long long)kvh * Tlen, Tlen * 4, scale_bar);
                bulk_load_1d(vsc, vscale + (long long)kvh * Tlen, Tlen * 4, scale_bar);
            }
            const uint8_t* kb = kcross + (long long)kvh * Tlen * C::kRowBytes;
            const uint8_t* vb = vcross + (long long)kvh * Tlen * C::kRowBytes;
            for (int c = 0; c < 2 * chunks; ++c) {
                const int stage = c % C::kStages;
                const uint32_t ph = (c / C::kStages) & 1;
                mbar_wait(&empty_bar[stage], ph ^ 1);
                mbar_expect_tx(&full_bar[stage], C::kStageBytes);
                const uint8_t* src = c < chunks ? kb + (long long)c * C::kStageBytes : vb + (long long)(c - chunks) * C::kStageBytes;
                bulk_load_1d(ring + stage * C::kStageBytes, src, C::kStageBytes, &full_bar[stage]);
            }
        }
        return;
    }
    // ---------------- consumers (128 threads) ----------------
    pdl_wait();                      // the q partials come from the upstream GEMM
    if (tid < 64) {
        float q = bq[h * 64 + tid];
        for (int s = 0; s < splits; ++s) q += partial[((long long)s * Bp + b) * dm + h * 64 + tid];
        sq[tid] = q * 0.125f;
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    const int sub = lane % C::kLanesPerRow;   // 16-byte piece of the row: dims sub*kDims .. sub*kDims + kDims - 1
    const int rsel = lane / C::kLanesPerRow;  // row within the warp's group of kRowsPerWarp
    float qv[C::kDims];
#pragma unroll
    for (int j = 0; j < C::kDims; ++j) qv[j] = sq[sub * C::kDims + j];
    if constexpr (FP8 || PACKED) mbar_wait(scale_bar, 0);

    // K phase: scores[t] = q . K[t]  (FP8: ksc[t] * (q . code[t]))
    for (int c = 0; c < chunks; ++c) {
        const int stage = c % C::kStages;
        const uint32_t ph = (c / C::kStages) & 1;
        mbar_wait(&full_bar[stage], ph);
        const uint8_t* tile = ring + stage * C::kStageBytes;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int r = warp * C::kRowsPerWarp + rsel + 4 * C::kRowsPerWarp * i;
            float acc = 0.f;
            if (r < C::kRows) acc = cross_row_dot<T, F>(cross_piece<F>(tile, r, sub, PACKED ? hdr[c * C::kRows + r] : 0), qv);
#pragma unroll
            for (int o = 1; o < C::kLanesPerRow; o <<= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
            if (sub == 0 && r < C::kRows) scores[c * C::kRows + r] = FP8 ? acc * ksc[c * C::kRows + r] : acc;
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    // softmax over Tlen scores (consumers only)
    float mx = -INFINITY;
    for (int t = tid; t < Tlen; t += 128) mx = fmaxf(mx, scores[t]);
    mx = warp_max(mx);
    if (lane == 0) red[warp] = mx;
    asm volatile("bar.sync 1, 128;" ::: "memory");
    mx = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
    float sm = 0.f;
    for (int t = tid; t < Tlen; t += 128) {
        const float p = __expf(scores[t] - mx);
        scores[t] = p;
        sm += p;
    }
    sm = warp_sum(sm);
    asm volatile("bar.sync 1, 128;" ::: "memory");   // everyone has read red[] (max) before it is reused
    if (lane == 0) red[warp] = sm;
    asm volatile("bar.sync 1, 128;" ::: "memory");
    const float inv = 1.f / (red[0] + red[1] + red[2] + red[3]);
    if (align_scratch != nullptr && ((align_mask >> h) & 1u)) {
        // alignment head: export the normalised softmax row (word timestamps); slot = rank of h among the layer's alignment heads
        const int slot = __popc(align_mask & ((1u << h) - 1u));
        float* dst = align_scratch + ((long long)slot * B + b) * Tlen;
        for (int t = tid; t < Tlen; t += 128) dst[t] = scores[t] * inv;
    }

    // V phase: out[d] = sum_t p[t] V[t][d]  (FP8: p[t] vsc[t] code[t][d])
    float acc[C::kDims];
#pragma unroll
    for (int j = 0; j < C::kDims; ++j) acc[j] = 0.f;
    for (int c = chunks; c < 2 * chunks; ++c) {
        const int stage = c % C::kStages;
        const uint32_t ph = (c / C::kStages) & 1;
        mbar_wait(&full_bar[stage], ph);
        const uint8_t* tile = ring + stage * C::kStageBytes;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int r = warp * C::kRowsPerWarp + rsel + 4 * C::kRowsPerWarp * i;
            if (r < C::kRows) {
                const int t = (c - chunks) * C::kRows + r;
                const float p = FP8 ? scores[t] * vsc[t] : scores[t];
                cross_row_axpy<T, F>(cross_piece<F>(tile, r, sub, PACKED ? hdr[hs + t] : 0), p, acc);
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);
    }
#pragma unroll
    for (int j = 0; j < C::kDims; ++j) {
#pragma unroll
        for (int o = C::kLanesPerRow; o < 32; o <<= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");   // red[] (sum) consumed by everyone
    if (rsel == 0) {
#pragma unroll
        for (int j = 0; j < C::kDims; ++j) red[warp * 64 + sub * C::kDims + j] = acc[j];
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    if (tid < 64) {
        const float o = (red[tid] + red[64 + tid] + red[128 + tid] + red[192 + tid]) * inv;
        out[(long long)b * dm + h * 64 + tid] = T16<T>::from_f(o);
    }
}

template <int F> static size_t cross_smem_bytes(int T) {
    using C = CrossCfg<F>;
    return (size_t)C::kStages * C::kStageBytes + (size_t)((T + 3) & ~3) * 4 * (C::FP8 ? 3 : 1) + (F == kCrossPacked ? 2 * packed_hdr_stride(T) : 0) +
           64 * 4 + (4 * 64 + 32) * 4 + (2 * C::kStages + (F != kCrossRaw16 ? 1 : 0)) * 8 + 64;
}

template <typename T, int F>
static wk_status launch_cross(const float* partial, int splits, int Bp, const float* bq, const void* kcross, const void* vcross, const float* kscale,
                              const float* vscale, void* out, int B, int H, int Tlen, cudaStream_t stream, const int32_t* done, float* align_scratch,
                              uint32_t align_mask, int kv_div, const uint8_t* khdr, const uint8_t* vhdr) {
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(decoder_cross_attention_kernel<T, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
        if (e != cudaSuccess) { set_error("cudaFuncSetAttribute(cross): %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
        attr_set = true;
    }
    launch_k(decoder_cross_attention_kernel<T, F>, dim3(B * H), dim3(kCrossThreads), cross_smem_bytes<F>(Tlen), stream, 4, partial, splits, Bp, bq,
             (const uint8_t*)kcross, (const uint8_t*)vcross, kscale, vscale, (T*)out, B, H, Tlen, done, align_scratch, align_mask, kv_div, khdr, vhdr);
    return WK_OK;
}

__global__ void cross_kv_unpack_kernel(const uint8_t* __restrict__ packed, const uint8_t* __restrict__ hdr, uint4* __restrict__ out, int64_t groups, int T) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;   // group of 8 values
    if (i >= groups) return;
    const int64_t row = i >> 3, blk = row / T;
    const int t = (int)(row - blk * T);
    out[i] = packed_group(packed + blk * T * 128, T, t, (int)(i & 7), hdr[blk * packed_hdr_stride(T) + t]);
}

wk_status cross_kv_unpack(const void* packed, const uint8_t* hdr, void* out, int64_t blocks, int T, cudaStream_t stream) {
    const int64_t groups = blocks * T * 8;
    if (groups == 0) return WK_OK;
    cross_kv_unpack_kernel<<<(unsigned)((groups + 255) / 256), 256, 0, stream>>>((const uint8_t*)packed, hdr, (uint4*)out, groups, T);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("cross_kv_unpack launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

// The beam-search form (NQ rows share one K/V block) lives in cross_attention_mq.cu: both products on the tensor cores.

__global__ void decoder_align_mean_kernel(const float* __restrict__ scratch, int n_slots, const int32_t* __restrict__ steps,
                                          const int32_t* __restrict__ done, const int32_t* __restrict__ lang_state, __half* __restrict__ out,
                                          int B, int Tlen, int max_rows) {
    const int b = blockIdx.y, t = blockIdx.x * blockDim.x + threadIdx.x;
    // launched after the sampler advanced the row's step: steps[b] = tokenIndex + 1 = the row of this step's slice; a window whose
    // segment just completed (or completed earlier) gets no row - the reference breaks out of its loop before updateAlignmentWeights
    // (TextDecoder.swift:668-674,709-717); nor does the leading language-detection step, which is not a step of decodeText
    const int row = steps[b];
    if (t >= Tlen || row >= max_rows || done[b] || (lang_state != nullptr && lang_state[b] == kLangLeadRan)) return;
    float a = 0.f;
    for (int s = 0; s < n_slots; ++s) a += scratch[((long long)s * B + b) * Tlen + t];   // fixed order: deterministic
    out[((long long)b * max_rows + row) * Tlen + t] = __float2half(a / (float)n_slots);
}

wk_status decoder_align_mean(const float* scratch, int n_slots, const int32_t* steps, const int32_t* done, const int32_t* lang_state,
                             void* out_f16, int B, int T, int max_rows, cudaStream_t stream) {
    launch_k(decoder_align_mean_kernel, dim3((T + 255) / 256, B), dim3(256), 0, stream, 0, scratch, n_slots, steps, done, lang_state, (__half*)out_f16, B, T, max_rows);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("decoder_align_mean launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

wk_status decoder_cross_attention(const float* partial, int splits, int Bp, const float* bq, const void* kcross,
                                  const void* vcross, void* out, int B, int H, int T, int dtype, cudaStream_t stream,
                                  const int32_t* done, float* align_scratch, uint32_t align_mask, int kv_div, const float* kscale,
                                  const float* vscale, bool single_query, const uint8_t* khdr, const uint8_t* vhdr) {
    const bool fp8 = kscale != nullptr;
    if (kv_div < 1 || B % kv_div != 0) { set_error("decoder_cross_attention: %d rows do not split into groups of %d", B, kv_div); return WK_ERR_INVALID_ARGUMENT; }
    if (!fp8 && T % kCrossRows != 0) { set_error("decoder_cross_attention: n_audio_ctx %d not a multiple of %d", T, kCrossRows); return WK_ERR_INVALID_ARGUMENT; }
    if (kv_div > 1 && kv_div <= 8 && align_scratch == nullptr && !single_query)   // beam search: one CTA per (window, head) serves all beams from one K/V pass
        return decoder_cross_attention_mq(partial, splits, Bp, bq, kcross, vcross, out, B, H, T, dtype, stream, done, kv_div, kscale, vscale, khdr, vhdr);
    // FP8: the scale vectors are bulk-copied, so T * 4 bytes per (window, head) must keep 16-byte alignment
    if (fp8 && (T % CrossCfg<kCrossFp8>::kRows != 0 || T % 4 != 0)) { set_error("decoder_cross_attention (fp8): n_audio_ctx %d not a multiple of 500", T); return WK_ERR_INVALID_ARGUMENT; }
    const bool f16 = dtype == WK_DTYPE_F16;
    if (khdr && (fp8 || f16 || !vhdr)) { set_error("decoder_cross_attention: the packed cache is bf16 and needs both header vectors"); return WK_ERR_INVALID_ARGUMENT; }
#define WK_CROSS(TT, FF) launch_cross<TT, FF>(partial, splits, Bp, bq, kcross, vcross, kscale, vscale, out, B, H, T, stream, done, align_scratch, align_mask, kv_div, khdr, vhdr)
    wk_status st = khdr ? WK_CROSS(__nv_bfloat16, kCrossPacked)
                 : fp8 ? (f16 ? WK_CROSS(__half, kCrossFp8) : WK_CROSS(__nv_bfloat16, kCrossFp8))
                       : (f16 ? WK_CROSS(__half, kCrossRaw16) : WK_CROSS(__nv_bfloat16, kCrossRaw16));
#undef WK_CROSS
    if (st != WK_OK) return st;
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("decoder_cross_attention launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

// =====================================================================================================
// K7: fused logits filters + greedy sampler + decode-loop state update.  One CTA per sequence; the logits row
// (V f32, 207 KB for V = 51866) is staged once in shared memory, masks are applied while it streams in, and the
// max / log-sum-exp / argmax reductions of TimestampRulesFilter and GreedyTokenSampler run out of smem.
// =====================================================================================================
static constexpr int kSamplerThreads = 1024;

struct ArgMax { float v; int i; };
__device__ __forceinline__ ArgMax argmax_better(ArgMax a, ArgMax b) {
    // larger value wins; ties -> lower index (first maximal index, like argmax)
    if (b.v > a.v || (b.v == a.v && b.i < a.i)) return b;
    return a;
}

// block-wide argmax (first maximal index) over srow[lo, V); srow is only read; the result is identical in every thread
__device__ __forceinline__ ArgMax block_argmax_row(const float* srow, int lo, int V, ArgMax* sarg) {
    const int tid = threadIdx.x;
    ArgMax best = {-INFINITY, 0x7fffffff};
    for (int i = lo + tid; i < V; i += kSamplerThreads) {
        const float x = srow[i];
        if (x > best.v) { best.v = x; best.i = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        ArgMax other;
        other.v = __shfl_xor_sync(0xffffffffu, best.v, o);
        other.i = __shfl_xor_sync(0xffffffffu, best.i, o);
        best = argmax_better(best, other);
    }
    __syncthreads();
    if ((tid & 31) == 0) sarg[tid >> 5] = best;
    __syncthreads();
    best = sarg[tid & 31];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        ArgMax other;
        other.v = __shfl_xor_sync(0xffffffffu, best.v, o);
        other.i = __shfl_xor_sync(0xffffffffu, best.i, o);
        best = argmax_better(best, other);
    }
    return best;
}

// the softmax at temperature 1 / inv_t over srow[lo, V) whose scaled max is zmax: its normaliser, and the probability of a value x
__device__ __forceinline__ float tempered_sum(const float* srow, int lo, int V, float inv_t, float zmax, float* scratch) {
    float z = 0.f;
    for (int i = lo + threadIdx.x; i < V; i += kSamplerThreads) {
        const float x = srow[i];
        if (x != -INFINITY) z += __expf(x * inv_t - zmax);
    }
    return block_sum(z, scratch);
}
__device__ __forceinline__ float tempered_prob(float x, float inv_t, float zmax, float z) { return __expf(x * inv_t - zmax) / z; }

// GreedyTokenSampler.update on a filtered row staged in smem, restricted to [lo, V) whose max is `m` and log-sum-exp `lse`:
// temperature 0 = argmax; > 0 = logits / T, softmax over the whole (filtered) range, top-k, multinomial draw inside the top-k mass,
// logprob = log softmax prob of the draw (TokenSampler.swift:57-73 / :140-180).  The reference draws with Float.random
// (non-deterministic); here the draw is Philox(seed, subsequence, offset).  Returns the token in .i (out of [0, V) if the row has no
// finite logit) and its log-prob in .v; srow is modified at T > 0.  z_out (T > 0, may be nullptr): the tempered normaliser
__device__ __forceinline__ ArgMax sample_row(float* srow, int lo, int V, float m, float lse, float temperature, int top_k, uint64_t seed,
                                             unsigned long long subsequence, unsigned long long offset, float* scratch, ArgMax* sarg,
                                             float* z_out = nullptr) {
    const int tid = threadIdx.x;
    ArgMax best;
    if (temperature == 0.f) {
        best = block_argmax_row(srow, lo, V, sarg);
        best.v = best.v - lse;
        return best;
    }
    const float inv_t = 1.f / temperature;
    const float zmax = m * inv_t;
    const float z = tempered_sum(srow, lo, V, inv_t, zmax, scratch);
    if (z_out) *z_out = z;
    __shared__ float topv[32];
    __shared__ int topi[32];
    const int k = top_k < 1 ? 1 : (top_k > 32 ? 32 : top_k);
    int kk = 0;
    for (; kk < k; ++kk) {
        const ArgMax a = block_argmax_row(srow, lo, V, sarg);
        if (a.v == -INFINITY) break;
        if (tid == 0) { topv[kk] = tempered_prob(a.v, inv_t, zmax, z); topi[kk] = a.i; srow[a.i] = -INFINITY; }
        __syncthreads();
    }
    __syncthreads();
    float mass = 0.f;
    for (int j = 0; j < kk; ++j) mass += topv[j];
    curandStatePhilox4_32_10_t rng;
    curand_init(seed, subsequence, offset, &rng);
    const float u = 1.f - curand_uniform(&rng);   // [0, 1)
    const float rnd = u * mass;
    float acc = 0.f;
    int chosen = kk > 0 ? kk - 1 : 0;
    for (int j = 0; j < kk; ++j) {
        acc += topv[j];
        if (rnd < acc) { chosen = j; break; }
    }
    best.i = kk > 0 ? topi[chosen] : 0x7fffffff;
    best.v = kk > 0 ? logf(topv[chosen]) : -INFINITY;
    return best;
}

// Philox subsequences of the in-loop language detection draws: row b uses kDetectSubsequence + b, apart from the loop's own draws
// (subsequence b), so that detecting moves no token draw of the decode
static constexpr unsigned long long kDetectSubsequence = 1ull << 32;

// ---- DecodingOptions.biasPhrases (tests/bias_ref.py is the specification).  A row keeps one KMP match length m_p per phrase; a token v
// earns b(v) = λ·(g(v) - G) with G = max_p m_p and g(v) = max_p δ_p(m_p, v).  Only the tokens on some phrase's failure chain from m_p
// have g > 0: at most Σ L_p = 1024 of them, one per thread of the sampler's CTA.
struct BiasSet {
    const int32_t* desc; const int32_t* tok; const int32_t* fail; int n;
    __device__ BiasSet(const int32_t* pool, const RowParams& R)
        : desc(pool + R.bias_off), tok(pool + R.bias_off + R.bias_n), fail(pool + R.bias_off + R.bias_n + R.bias_len), n(R.bias_n) {}
};

// δ_p(k, v), a completion counting as L_p; *stored: the state the row keeps (f_p(L_p) after a completion)
__device__ __forceinline__ int bias_step(const BiasSet& B, int p, int k, int v, int* stored) {
    const int d = B.desc[p], start = d & 0xffff, len = d >> 16;
    const int32_t* w = B.tok + start;
    const int32_t* f = B.fail + start;
    while (k > 0 && w[k] != v) k = f[k - 1];
    k = w[k] == v ? k + 1 : 0;
    *stored = k == len ? f[len - 1] : k;
    return k;
}

// adds b(v) to srow[lo, V) in place (−inf stays −inf); returns G.  cand: kMaxBiasTotal packed (token | g << 20) entries of shared memory
__device__ int bias_apply(float* srow, int lo, int V, const BiasSet& B, const uint8_t* m, float boost, float* scratch, int* cand, int* ncand) {
    const int tid = threadIdx.x;
    const int mp = tid < B.n ? m[tid] : 0;
    if (tid == 0) *ncand = 0;
    const int G = (int)block_max((float)mp, scratch);   // (its barriers also publish *ncand = 0)
    if (tid < B.n) {   // the failure chain mp, f(mp), ..., 0: token w[k] continues the match to k + 1 (the first such k is δ, the largest)
        const int d = B.desc[tid], start = d & 0xffff;
        const int32_t* w = B.tok + start;
        const int32_t* f = B.fail + start;
        for (int k = mp;; k = f[k - 1]) {
            cand[atomicAdd(ncand, 1)] = w[k] | (k + 1) << 20;
            if (k == 0) break;
        }
    }
    __syncthreads();
    const int nc = *ncand;
    int tok = -1;
    float val = 0.f;
    if (tid < nc) {   // one owner per token (its first entry) applies the maximum over the phrases
        const int c = cand[tid];
        tok = c & 0xfffff;
        int g = c >> 20;
        for (int j = 0; j < nc && tok >= 0; ++j) {
            const int o = cand[j];
            if ((o & 0xfffff) != tok) continue;
            if (j < tid) tok = -1;
            else g = max(g, o >> 20);
        }
        if (tok < lo || tok >= V) tok = -1;
        if (tok >= 0) val = srow[tok] + boost * (float)(g - G);
    }
    const float base = boost * (float)(0 - G);   // b of every token outside the chains
    if (base != 0.f) {
        __syncthreads();
        for (int i = lo + tid; i < V; i += kSamplerThreads) srow[i] += base;
        __syncthreads();
    }
    if (tok >= 0) srow[tok] = val;
    __syncthreads();
    return G;
}

// the row's states after token v; returns g(v) (block-uniform)
__device__ int bias_advance(const BiasSet& B, uint8_t* m, int v, float* scratch) {
    const int tid = threadIdx.x;
    int g = 0;
    if (tid < B.n) {
        int stored;
        g = bias_step(B, tid, m[tid], v, &stored);
        m[tid] = (uint8_t)stored;
    }
    return (int)block_max((float)g, scratch);
}

// ---- DecodingOptions.topLogProbs (tests/top_logprobs_ref.py is the specification): the k best candidates of the filtered row, ordered
// like block_argmax_row (larger value first, ties to the lower index), in one pass over the row.  Each warp keeps a register top-k of
// its threads' strided slices, entry j in lane j, and warp 0 then merges the 32 warp lists with the same insertion.  (A list per
// thread would need 2k registers of the 64 that a 1024-thread CTA allows.)
__device__ __forceinline__ bool top_better(float av, int ai, float bv, int bi) { return av > bv || (av == bv && ai < bi); }

// offers every lane's (x, i) to the warp's list (lv, li) of k entries; only finite values enter.  Called by whole warps
__device__ __forceinline__ void warp_top_offer(float x, int i, int k, float& lv, int& li) {
    const int lane = threadIdx.x & 31;
    const float tv = __shfl_sync(0xffffffffu, lv, k - 1);
    const int ti = __shfl_sync(0xffffffffu, li, k - 1);
    unsigned cand = __ballot_sync(0xffffffffu, x > -INFINITY && top_better(x, i, tv, ti));
    while (cand) {
        const int src = __ffs(cand) - 1;
        cand &= cand - 1;
        const float cv = __shfl_sync(0xffffffffu, x, src);
        const int ci = __shfl_sync(0xffffffffu, i, src);
        // the entries better than the candidate keep their lanes, the others move down one lane and the last falls off
        const int pos = __popc(__ballot_sync(0xffffffffu, lane < k && top_better(lv, li, cv, ci)));
        const float uv = __shfl_up_sync(0xffffffffu, lv, 1);
        const int ui = __shfl_up_sync(0xffffffffu, li, 1);
        if (pos < k) {
            if (lane == pos) { lv = cv; li = ci; }
            else if (lane > pos) { lv = uv; li = ui; }
        }
    }
}

// the k best entries of srow[lo, V) (only read) into tv / ti [0, k), padded with (-inf, INT_MAX); tv / ti: 32 * k entries of shared
// memory.  Thread j < k (lane j of warp 0) writes entry j
__device__ void block_top_row(const float* srow, int lo, int V, int k, float* tv, int* ti) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float lv = -INFINITY;
    int li = 0x7fffffff;
    for (int i0 = lo + (tid & ~31); i0 < V; i0 += kSamplerThreads) {   // thread tid sees srow[lo + tid + j * kSamplerThreads]
        const int i = i0 + lane;
        warp_top_offer(i < V ? srow[i] : -INFINITY, i, k, lv, li);
    }
    if (lane < k) { tv[warp * k + lane] = lv; ti[warp * k + lane] = li; }
    __syncthreads();
    if (warp != 0) return;
    lv = -INFINITY;
    li = 0x7fffffff;
    const int n = (kSamplerThreads / 32) * k;
    for (int c = 0; c < n; c += 32) warp_top_offer(c + lane < n ? tv[c + lane] : -INFINITY, c + lane < n ? ti[c + lane] : 0, k, lv, li);
    __syncwarp();
    if (lane < k) { tv[lane] = lv; ti[lane] = li; }
}

// kTop: the variant with the DecodingOptions.topLogProbs pass (SamplerParams.top_n > 0); the other one is the sampler without it
template <bool kTop>
__global__ void __launch_bounds__(kSamplerThreads)
sampler_kernel(const float* __restrict__ logits, long long ld_logits, SamplerParams p, DecodeState st,
               const int32_t* __restrict__ tokens_in, int ld_tokens, const int32_t* __restrict__ n_tokens_in,
               int32_t* __restrict__ token_out, float* __restrict__ logprob_out, float* __restrict__ filtered_out) {
    extern __shared__ __align__(16) float srow[];  // [V]; kTop: then the candidate lists [32 * 20] values, [32 * 20] ids, the position
    __shared__ float scratch[32];
    __shared__ int sflag[8];     // 0: ts filter active, 1: lo0, 2: hi0 (interval A), 3: lo1, 4: hi1 (interval B), 5: blank active
    __shared__ ArgMax sarg[32];
    __shared__ int s_cand[kMaxBiasTotal];   // biasPhrases: the row's (token, g) candidates, then the appended token (s_adv)
    __shared__ int s_ncand, s_adv;
    const int b = blockIdx.x, tid = threadIdx.x;
    const int V = p.vocab;
    const bool loop_mode = p.loop_mode != 0;
    pdl_launch_dependents();
    pdl_wait();
    if (loop_mode && st.done[b]) return;   // ended window: its logits row is not even read
    // per-row options: the decode loop reads them from the row's RowParams, the stateless entry from the call
    RowParams R;
    if (loop_mode) {
        R = st.rp[b];
    } else {
        R.prompt_len = -1; R.sample_begin_ts = p.sample_begin_ts; R.sample_begin_blank = p.sample_begin_blank; R.max_steps = 0;
        R.temperature = p.temperature; R.top_k = p.top_k; R.has_first_thr = 0; R.first_thr = 0.f; R.seed = p.seed;
        R.suppress_off = 0; R.n_suppress = p.n_suppress;
        R.detect = 0; R.lang_pos = -1; R.n_lang = 0; R.lead_token = 0; R.no_speech_pos = -1; R.mode = kRowSingle;
    }
    const int32_t* toks = loop_mode ? st.tokens + b * kMaxCtx : tokens_in + (long long)b * ld_tokens;
    const wk_special_tokens& S = p.st;

    if (loop_mode && R.detect) {
        // DecodingOptions.detectLanguage: this step's logits are those of TextDecoder.detectLanguage (TextDecoder.swift:420-539) - [SOT] at
        // position 0 - either because the row's step 0 is that forward or because this is the row's leading detection step.
        // LanguageLogitsFilter alone on the raw row, then the rung's sampler; the <|xx|> slot of the prompt takes the detected language
        // before a later step forces it (prefillDecoderInputs with the detected language, TranscribeTask.swift:354-357)
        const bool lead = st.lang_state[b] == kLangLead;
        if (lead || (R.detect == 1 && st.steps[b] == 0)) {
            const float* row = logits + (long long)b * ld_logits;
            for (int i = tid; i < V; i += kSamplerThreads) srow[i] = -INFINITY;
            __syncthreads();
            for (int j = tid; j < R.n_lang; j += kSamplerThreads) {
                const int t = p.detect_tokens[j];
                if (t >= 0 && t < V) srow[t] = row[t];
            }
            __syncthreads();
            float mx = -INFINITY;
            for (int i = tid; i < V; i += kSamplerThreads) mx = fmaxf(mx, srow[i]);
            mx = block_max(mx, scratch);
            float sm = 0.f;
            for (int i = tid; i < V; i += kSamplerThreads) {
                const float x = srow[i];
                if (x != -INFINITY) sm += __expf(x - mx);
            }
            sm = block_sum(sm, scratch);
            // every row of a group draws with the group's first row's subsequence: the group's rows are copies of one window, so its
            // best-of candidates (and beams) share one detected language
            const int g0 = p.beam.group > 1 ? b - b % p.beam.group : b;
            const ArgMax d = sample_row(srow, 0, V, mx, mx + logf(sm), R.temperature, R.top_k, R.seed,
                                        kDetectSubsequence + (unsigned long long)(g0 / max(1, p.rng_div)), 0ull,
                                        scratch, sarg);
            if (tid == 0) {
                const bool ok = d.i >= 0 && d.i < V;
                st.lang_token[b] = ok ? d.i : -1;
                st.lang_logprob[b] = ok ? d.v : 0.f;
                if (ok && R.lang_pos >= 0) st.tokens[b * kMaxCtx + R.lang_pos] = d.i;
                if (lead) st.lang_state[b] = kLangLeadRan;
            }
            __syncthreads();
            // the leading step ends here: no sample, no bookkeeping - the row starts its step 0 next
            if (lead) return;
        }
    }
    if (loop_mode && R.no_speech_pos == st.steps[b] && st.lang_state[b] != kLangLead) {
        // DecodingResult.noSpeechProb (openai/whisper decoding.py): the softmax of the RAW logits of the step whose input is the prompt's
        // SOT - before any logits filter, at no temperature - taken at <|nospeech|>.  Fixed-order block reductions: deterministic.
        // expf, not __expf: the value is compared against a threshold and reported.
        const float* row = logits + (long long)b * ld_logits;
        float mx = -INFINITY;
        for (int i = tid; i < V; i += kSamplerThreads) mx = fmaxf(mx, row[i]);
        mx = block_max(mx, scratch);
        float sm = 0.f;
        for (int i = tid; i < V; i += kSamplerThreads) sm += expf(row[i] - mx);
        sm = block_sum(sm, scratch);
        if (tid == 0) {
            const int ns = S.no_speech_token;
            st.no_speech[b] = (ns >= 0 && ns < V) ? expf(row[ns] - mx) / sm : __int_as_float(0x7fc00000);
        }
    }
    const int n_tok = loop_mode ? st.n_tokens[b] : n_tokens_in[b];

    if (tid == 0) {
        // ---- TimestampRulesFilter rule state (LogitsFilter.swift:72-109)
        int active = 0, loA = 0, hiA = 0, loB = 0, hiB = 0;
        if (R.sample_begin_ts >= 0) {
            int sb = -1;
            if (p.is_multilingual) {
                const int lim = n_tok < 3 ? n_tok : 3;
                for (int i = 0; i < lim; ++i)
                    if (toks[i] == S.transcribe_token || toks[i] == S.translate_token) { sb = max(i + 1, R.sample_begin_ts); break; }
            } else {
                sb = R.sample_begin_ts;
            }
            if (sb >= 0 && sb <= n_tok) {
                active = 1;
                if (n_tok > sb) {
                    const int ns = n_tok - sb;
                    const bool last_ts = ns >= 1 && toks[n_tok - 1] >= S.time_token_begin;
                    const bool pen_ts = ns < 2 || toks[n_tok - 2] >= S.time_token_begin;
                    if (last_ts) {
                        if (pen_ts) { loA = S.time_token_begin; hiA = V; }   // has to be non-timestamp
                        else { loA = 0; hiA = S.end_token; }                 // cannot be normal text
                    }
                    int last_time = -1;
                    for (int i = n_tok - 1; i >= sb; --i)
                        if (toks[i] >= S.time_token_begin) { last_time = toks[i]; break; }
                    if (last_time >= 0) {
                        const int ts_last = (last_ts && !pen_ts) ? last_time : last_time + 1;
                        loB = S.time_token_begin; hiB = ts_last;
                    }
                }
            }
        }
        sflag[0] = active; sflag[1] = loA; sflag[2] = hiA; sflag[3] = loB; sflag[4] = hiB;
        sflag[5] = (R.sample_begin_blank >= 0 && n_tok == R.sample_begin_blank) ? 1 : 0;   // SuppressBlankFilter
        sflag[6] = (p.language_tokens != nullptr && n_tok >= p.language_sample_begin) ? 1 : 0;  // LanguageLogitsFilter
    }
    __syncthreads();
    const int ts_active = sflag[0], loA = sflag[1], hiA = sflag[2], loB = sflag[3], hiB = sflag[4];
    const int blank_active = sflag[5], lang_active = sflag[6];
    const float* row = logits + (long long)b * ld_logits;

    // ---- stream the row into smem with the interval / single-token masks applied
    for (int i = tid; i < V; i += kSamplerThreads) {
        float x = lang_active ? -INFINITY : row[i];
        if (blank_active && (i == S.whitespace_token || i == S.end_token)) x = -INFINITY;
        if (ts_active) {
            if (i == S.no_timestamps_token) x = -INFINITY;
            if ((i >= loA && i < hiA) || (i >= loB && i < hiB)) x = -INFINITY;
        }
        srow[i] = x;
    }
    __syncthreads();
    if (lang_active) {
        for (int j = tid; j < p.n_language_tokens; j += kSamplerThreads) {
            const int t = p.language_tokens[j];
            if (t >= 0 && t < V) srow[t] = row[t];
        }
        __syncthreads();
        // re-apply the filters that run after a (custom-positioned) language filter
        for (int j = tid; j < p.n_language_tokens; j += kSamplerThreads) {
            const int i = p.language_tokens[j];
            if (i < 0 || i >= V) continue;
            if (blank_active && (i == S.whitespace_token || i == S.end_token)) srow[i] = -INFINITY;
            if (ts_active && (i == S.no_timestamps_token || (i >= loA && i < hiA) || (i >= loB && i < hiB))) srow[i] = -INFINITY;
        }
        __syncthreads();
    }
    for (int j = tid; j < R.n_suppress; j += kSamplerThreads) {   // SuppressTokensFilter
        const int t = p.suppress[R.suppress_off + j];
        if (t >= 0 && t < V) srow[t] = -INFINITY;
    }
    __syncthreads();

    // ---- reductions: max over text / timestamp partitions
    const int tsb = (ts_active && S.time_token_begin > 0 && S.time_token_begin < V) ? S.time_token_begin : V;
    float mtext = -INFINITY, mts = -INFINITY;
    for (int i = tid; i < V; i += kSamplerThreads) {
        const float x = srow[i];
        if (i < tsb) mtext = fmaxf(mtext, x); else mts = fmaxf(mts, x);
    }
    mtext = block_max(mtext, scratch);
    mts = block_max(mts, scratch);
    const float mall = fmaxf(mtext, mts);
    float sall = 0.f, sts = 0.f;
    for (int i = tid; i < V; i += kSamplerThreads) {
        const float x = srow[i];
        if (x == -INFINITY) continue;
        sall += __expf(x - mall);
        if (i >= tsb) sts += __expf(x - mts);
    }
    sall = block_sum(sall, scratch);
    sts = block_sum(sts, scratch);
    float lse = mall + logf(sall);
    // "sum of probability over timestamps is above any other token" (LogitsFilter.swift:124-127,144-242)
    bool ts_wins = false;
    if (tsb < V && mts > -INFINITY) {
        const float lse_ts = mts + logf(sts);
        const float ts_logprob = lse_ts - lse;
        const float max_text_logprob = mtext - lse;
        ts_wins = ts_logprob > max_text_logprob;
        if (ts_wins) lse = lse_ts;
    }
    const int lo = ts_wins ? tsb : 0;
    if (ts_wins && filtered_out) {
        for (int i = tid; i < tsb; i += kSamplerThreads) srow[i] = -INFINITY;
        __syncthreads();
    }
    if (filtered_out) {
        for (int i = tid; i < V; i += kSamplerThreads) filtered_out[(long long)b * V + i] = srow[i];
        __syncthreads();
    }
    // DecodingOptions.biasPhrases: from the row's first sampled position on (prompt forcing and detection steps are left alone), the
    // phrase bonus joins the filtered row after every filter.  The choice sees it; the reported log-probs stay the model's: a chosen
    // token's filtered value is its raw logit, so they come from `row`, against the unbiased normaliser
    const bool biased = loop_mode && st.bias_pool != nullptr && R.bias_n > 0 && st.steps[b] >= R.prompt_len - 1;
    // DecodingOptions.topLogProbs: a position the row may record ranks its candidates here, on the filtered row before the bonus or the
    // draw change it.  The values are raw logits until they are written, against the normaliser of the position's reported log-prob
    float* top_v = srow + V;
    int* top_i = (int*)(top_v + 32 * kMaxTopLogprobs);
    int* top_pos = top_i + 32 * kMaxTopLogprobs;
    bool top = false;
    if constexpr (kTop) {
        top = loop_mode && R.mode != kRowBeam && st.steps[b] >= R.prompt_len - 1;
        if (top) block_top_row(srow, lo, V, p.top_n, top_v, top_i);
    }
    float m_draw = ts_wins ? mts : mall;
    float z_unbiased = 0.f;
    int bias_G = 0;
    if (biased) {
        if (R.mode != kRowBeam && R.temperature != 0.f) z_unbiased = tempered_sum(srow, lo, V, 1.f / R.temperature, m_draw * (1.f / R.temperature), scratch);
        const BiasSet B(st.bias_pool, R);
        bias_G = bias_apply(srow, lo, V, B, st.bias_m + b * kMaxBiasPhrases, R.bias_boost, scratch, s_cand, &s_ncand);
        float mx = -INFINITY;
        for (int i = lo + tid; i < V; i += kSamplerThreads) mx = fmaxf(mx, srow[i]);
        mx = block_max(mx, scratch);
        if (R.temperature != 0.f) m_draw = mx;
    }
    if (loop_mode && R.mode == kRowBeam) {
        // beam search: rank the row's (beam + 1) best tokens of the filtered log-softmax, best first (whisper BeamSearchDecoder.update step 1);
        // the per-window merge and every state update happen in beam_update_kernel
        const int k = p.beam.beam + 1;
        for (int kk = 0; kk < k; ++kk) {
            const ArgMax a = block_argmax_row(srow, lo, V, sarg);
            const bool ok = a.v != -INFINITY && a.i >= 0 && a.i < V;   // (a NaN row yields the initial index: no candidate)
            if (tid == 0) {
                p.beam.cand_tok[b * (kMaxBeam + 1) + kk] = ok ? a.i : -1;
                p.beam.cand_lp[b * (kMaxBeam + 1) + kk] = ok ? (biased ? row[a.i] : a.v) - lse : -INFINITY;
                p.beam.cand_sc[b * (kMaxBeam + 1) + kk] = ok ? a.v - lse : -INFINITY;
                if (ok) srow[a.i] = -INFINITY;
            }
            __syncthreads();
        }
        return;
    }
    // the row's draw: Philox(seed, row, step) at temperature > 0 (row: the slot in a draft call, whose windows sample on row 0 only)
    float z_draw = 0.f;
    const ArgMax best = sample_row(srow, lo, V, m_draw, lse, R.temperature, R.top_k, R.seed, (unsigned long long)(b / max(1, p.rng_div)),
                                   (unsigned long long)(loop_mode ? st.steps[b] : n_tok), scratch, sarg, kTop && top ? &z_draw : nullptr);
    float lp_sampled = best.v;
    if (biased && best.i >= 0 && best.i < V)
        lp_sampled = R.temperature == 0.f ? row[best.i] - lse
                                          : logf(tempered_prob(row[best.i], 1.f / R.temperature, (ts_wins ? mts : mall) * (1.f / R.temperature), z_unbiased));
    if (tid == 0) s_adv = -1;
    if (tid == 0) {
        if constexpr (kTop) *top_pos = -1;
        int tok = best.i;
        float lp = lp_sampled;
        // a row with no finite logit (every token masked, or a NaN from upstream) has no argmax: end the window there and flag it instead
        // of feeding an out-of-range id to the next embedding lookup (the host reports WhisperError.decodingLogitsFailed for the window)
        const bool bad = tok < 0 || tok >= V;
        if (bad) { tok = S.end_token; lp = -INFINITY; }
        if (token_out) token_out[b] = bad ? -1 : tok;
        if (logprob_out) logprob_out[b] = lp;
        if (loop_mode) {
            // decodeText bookkeeping (TextDecoder.swift:654-686)
            const int step = st.steps[b];
            const bool first_low = (step == 0) && R.has_first_thr && (lp < R.first_thr);
            const bool completed = (tok == S.end_token) || (n_tok >= p.max_ctx - 1) || first_low;
            st.next_token[b] = tok;
            st.steps[b] = step + 1;
            if (bad) st.error[b] = 1;
            if (completed) {
                st.done[b] = 1;
                st.first_low[b] = first_low ? 1 : 0;
            } else {
                if (!(step < R.prompt_len - 1)) {   // !isPrefill
                    st.tokens[b * kMaxCtx + n_tok] = tok;
                    st.logprobs[b * kMaxCtx + n_tok] = lp;
                    st.n_tokens[b] = n_tok + 1;
                    if (biased) s_adv = tok;
                    if constexpr (kTop) *top_pos = n_tok;
                }
                if (step + 1 >= R.max_steps) st.done[b] = 1;   // loop bound min(sampleLength, 223) reached (TextDecoder.swift:566)
            }
        }
    }
    if constexpr (kTop) {   // the candidates of an appended token at its position, with the normaliser of its log-prob (unbiased)
        if (top) {
            __syncthreads();
            const int pos = *top_pos;
            if (pos >= 0 && tid < p.top_n) {
                const float v = top_v[tid];
                const bool ok = v > -INFINITY;
                const float lp = R.temperature == 0.f ? v - lse
                                                      : logf(tempered_prob(v, 1.f / R.temperature, (ts_wins ? mts : mall) * (1.f / R.temperature),
                                                                           biased ? z_unbiased : z_draw));
                const long long at = ((long long)b * kMaxCtx + pos) * p.top_n + tid;
                p.top_tok[at] = ok ? top_i[tid] : -1;
                p.top_lp[at] = ok ? lp : -INFINITY;
            }
        }
    }
    if (biased) {   // the appended token moves the row's matches on; the bonus it earned is banked for the best-of ranking
        __syncthreads();
        if (s_adv >= 0) {
            const int g = bias_advance(BiasSet(st.bias_pool, R), st.bias_m + b * kMaxBiasPhrases, s_adv, scratch);
            if (tid == 0) st.bias_acc[b] += g - bias_G;
        }
    }
}

// =====================================================================================================
// Beam search step (oracle/beam_ref.py is the specification).  One CTA per window; rows r0 .. r0 + beam - 1 are its beams.
// =====================================================================================================
static constexpr int kBeamThreads = 128;

__global__ void __launch_bounds__(kBeamThreads)
beam_update_kernel(DecodeState st, BeamState bs, wk_special_tokens S, int max_ctx) {
    __shared__ int32_t s_tok[kMaxBeam][kMaxCtx];
    __shared__ float s_lp[kMaxBeam][kMaxCtx];
    __shared__ int32_t s_anc[kMaxBeam][kMaxCtx];
    __shared__ float c_score[kMaxBeam * (kMaxBeam + 1)], c_lp[kMaxBeam * (kMaxBeam + 1)];
    __shared__ int c_src[kMaxBeam * (kMaxBeam + 1)], c_tok[kMaxBeam * (kMaxBeam + 1)], c_ord[kMaxBeam * (kMaxBeam + 1)];
    __shared__ int n_src[kMaxBeam], n_tokv[kMaxBeam];
    __shared__ float n_lp[kMaxBeam], n_score[kMaxBeam];
    __shared__ int f_src[kMaxCand]; __shared__ float f_score[kMaxCand];
    __shared__ int sh[4];   // 0: mode (0 prefill/plain advance, 1 ranked, 2 ended without ranking)  1: new finished count  2: window done  3: finished before
    const int g = blockIdx.x, tid = threadIdx.x, beam = bs.beam, r0 = g * bs.group;   // a beam group uses the first `beam` of its rows
    pdl_launch_dependents();
    pdl_wait();
    if (st.done[r0]) return;
    if (st.lang_state[r0] == kLangLeadRan) return;   // the leading language-detection step ranked nothing: no beam bookkeeping
    const RowParams R = st.rp[r0];
    if (R.mode != kRowBeam) return;                  // a single / best-of rung: the sampler did the rows' bookkeeping
    const int step = st.steps[r0], n_tok = st.n_tokens[r0], P = R.prompt_len;
    const int C1 = kMaxBeam + 1;
    if (tid == 0) {
        const int gtok = bs.cand_tok[r0 * C1];
        const float glp = bs.cand_lp[r0 * C1];
        const bool bad = gtok < 0;
        const bool first_low = (step == 0) && R.has_first_thr && (glp < R.first_thr);
        int mode = 0, done = 0;
        int nf_before = bs.n_fin[g];
        int nf_new = 0;
        if (bad) { done = 1; mode = 2; }
        else if (step < P - 1) {                       // prefill: every beam is the same forced copy; greedy bookkeeping
            if (gtok == S.end_token || first_low) done = 1;
        } else if (n_tok >= max_ctx - 1 || first_low) {
            done = 1; mode = 2;
        } else {
            mode = 1;
            const int considered = (step == P - 1) ? 1 : beam;   // identical beams count once
            int nc = 0;
            for (int j = 0; j < considered; ++j)
                for (int k = 0; k <= beam; ++k) {
                    const int t = bs.cand_tok[(r0 + j) * C1 + k];
                    if (t < 0) continue;
                    const float v = bs.cand_lp[(r0 + j) * C1 + k];
                    c_score[nc] = bs.sum_lp[r0 + j] + bs.cand_sc[(r0 + j) * C1 + k]; c_lp[nc] = v; c_src[nc] = j; c_tok[nc] = t; c_ord[nc] = nc; ++nc;
                }
            for (int i = 1; i < nc; ++i) {             // stable insertion sort, best score first
                const int o = c_ord[i];
                int k = i - 1;
                while (k >= 0 && c_score[c_ord[k]] < c_score[o]) { c_ord[k + 1] = c_ord[k]; --k; }
                c_ord[k + 1] = o;
            }
            int saved = 0;
            for (int i = 0; i < nc && saved < beam; ++i) {
                const int o = c_ord[i];
                if (c_tok[o] == S.end_token) {
                    if (nf_before + nf_new < bs.max_candidates) { f_src[nf_new] = c_src[o]; f_score[nf_new] = c_score[o]; ++nf_new; }
                } else {
                    n_src[saved] = c_src[o]; n_tokv[saved] = c_tok[o]; n_lp[saved] = c_lp[o]; n_score[saved] = c_score[o]; ++saved;
                }
            }
            for (; saved < beam; ++saved) {            // (cannot happen with beam + 1 candidates per beam; keeps the state well formed)
                n_src[saved] = n_src[saved > 0 ? saved - 1 : 0]; n_tokv[saved] = n_tokv[saved > 0 ? saved - 1 : 0]; n_lp[saved] = 0.f; n_score[saved] = -INFINITY;
            }
            if (nf_before + nf_new >= bs.max_candidates) done = 1;
        }
        if (!done && step + 1 >= R.max_steps) done = 1;   // loop bound (TextDecoder.swift:566)
        sh[0] = mode; sh[1] = nf_new; sh[2] = done; sh[3] = nf_before;
        for (int j = 0; j < beam; ++j) {
            const int r = r0 + j;
            st.steps[r] = step + 1;
            if (bad) st.error[r] = 1;
            if (mode != 1) st.next_token[r] = bad ? S.end_token : gtok;
            if (done) { st.done[r] = 1; st.first_low[r] = first_low ? 1 : 0; }
            bs.anc[r * kMaxCtx + step] = r;             // position `step` of this row's cache was written by the row itself
        }
    }
    __syncthreads();
    if (sh[0] != 1) return;
    // ---- ranked step: histories and ancestry move to the surviving beams
    for (int i = tid; i < beam * kMaxCtx; i += kBeamThreads) {
        const int j = i / kMaxCtx, t = i % kMaxCtx;
        s_tok[j][t] = st.tokens[(r0 + j) * kMaxCtx + t];
        s_lp[j][t] = st.logprobs[(r0 + j) * kMaxCtx + t];
        s_anc[j][t] = bs.anc[(r0 + j) * kMaxCtx + t];
    }
    __syncthreads();
    for (int f = 0; f < sh[1]; ++f) {                   // newly finished: prefix of the source beam + EOT (log-prob 0, like sampler.finalize)
        const int slot = g * kMaxCand + sh[3] + f, src = f_src[f];
        for (int t = tid; t < n_tok; t += kBeamThreads) {
            bs.fin_tokens[slot * kMaxCtx + t] = s_tok[src][t];
            bs.fin_lps[slot * kMaxCtx + t] = s_lp[src][t];
        }
        if (tid == 0) {
            bs.fin_tokens[slot * kMaxCtx + n_tok] = S.end_token;
            bs.fin_lps[slot * kMaxCtx + n_tok] = 0.f;
            bs.fin_len[slot] = n_tok + 1;
            bs.fin_score[slot] = f_score[f];
        }
    }
    if (tid == 0) bs.n_fin[g] = sh[3] + sh[1];
    for (int i = tid; i < beam * kMaxCtx; i += kBeamThreads) {
        const int j = i / kMaxCtx, t = i % kMaxCtx, r = r0 + j, src = n_src[j];
        if (t < n_tok) { st.tokens[r * kMaxCtx + t] = s_tok[src][t]; st.logprobs[r * kMaxCtx + t] = s_lp[src][t]; }
        else if (t == n_tok) { st.tokens[r * kMaxCtx + t] = n_tokv[j]; st.logprobs[r * kMaxCtx + t] = n_lp[j]; }
        if (t <= step) bs.anc[r * kMaxCtx + t] = (t == step) ? r0 + src : s_anc[src][t];
    }
    if (tid < beam) {
        const int r = r0 + tid;
        st.n_tokens[r] = n_tok + 1;
        st.next_token[r] = n_tokv[tid];
        bs.sum_lp[r] = n_score[tid];
    }
    if (st.bias_pool && R.bias_n > 0) {   // biasPhrases: each surviving beam takes its source beam's matches, moved on by its new token
        __shared__ uint8_t s_m[kMaxBeam][kMaxBiasPhrases];
        const BiasSet B(st.bias_pool, R);
        for (int i = tid; i < beam * B.n; i += kBeamThreads) s_m[i / B.n][i % B.n] = st.bias_m[(r0 + i / B.n) * kMaxBiasPhrases + i % B.n];
        __syncthreads();
        for (int i = tid; i < beam * B.n; i += kBeamThreads) {
            const int j = i / B.n, ph = i % B.n;
            int stored;
            bias_step(B, ph, s_m[n_src[j]][ph], n_tokv[j], &stored);
            st.bias_m[(r0 + j) * kMaxBiasPhrases + ph] = (uint8_t)stored;
        }
    }
}

wk_status beam_update(DecodeState st, BeamState beam, wk_special_tokens sp, int max_ctx, int groups, cudaStream_t stream) {
    if (beam.beam < 2 || beam.beam > kMaxBeam || beam.max_candidates < 1 || beam.max_candidates > kMaxCand || beam.group < beam.beam ||
        beam.group > kMaxBeam) {
        set_error("beam_update: beam %d / candidates %d / group %d outside [2, %d] / [1, %d] / [beam, %d]", beam.beam, beam.max_candidates,
                  beam.group, kMaxBeam, kMaxCand, kMaxBeam);
        return WK_ERR_INVALID_ARGUMENT;
    }
    launch_k(beam_update_kernel, dim3(groups), dim3(kBeamThreads), 0, stream, 8, st, beam, sp, max_ctx);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("beam_update launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

// =====================================================================================================
// Speculative greedy decoding: the draft rounds' bookkeeping kernels (session.cu enqueue_round).  Row r0 = q * group is the window's
// committed row; its state after the main step is exactly the sequential decode's, and verify row j (input: proposal j - 1 at position
// p0 + j, history: row 0's plus proposals 0..j-1) is the sequential step p0 + j whenever proposals 0..j-1 match what the model sampled.
// =====================================================================================================
__global__ void draft_round_begin_kernel(DecodeState st, DecodeState ds, RowParams* __restrict__ drp, DraftRound R) {
    const int q = blockIdx.x, r0 = q * R.group;
    const bool live = !st.done[r0];
    const int p0 = st.steps[r0], n = st.n_tokens[r0];
    const RowParams rp = st.rp[r0];
    for (int t = threadIdx.x; t < kMaxCtx; t += blockDim.x) ds.tokens[q * kMaxCtx + t] = st.tokens[r0 * kMaxCtx + t];
    if (threadIdx.x != 0) return;
    // past the prompt (tokens[p0] is the committed input of position p0), greedy, not in a leading language-detection step
    R.verify[q] = live && p0 >= rp.prompt_len && rp.temperature == 0.f && rp.mode == kRowSingle && st.lang_state[r0] == 0;
    R.p0[q] = live ? p0 : -1;
    R.nprop[q] = 0;
    R.cur[q] = -1;
    if (live) R.fed[q] = min(R.fed[q], p0);   // positions past the committed ones held rejected proposals (or a previous window's)
    ds.done[q] = 1;
    ds.n_tokens[q] = n;
    // the draft's filters are the window's; it always feeds its input token (no prompt forcing, no detection) and proposes greedily
    RowParams d = rp;
    d.prompt_len = 0; d.temperature = 0.f; d.has_first_thr = 0; d.detect = 0; d.lang_pos = -1; d.n_lang = 0; d.no_speech_pos = -1;
    d.mode = kRowSingle;
    drp[q] = d;
}

wk_status draft_round_begin(DecodeState st, DecodeState ds, RowParams* drp, DraftRound R, cudaStream_t stream) {
    launch_k(draft_round_begin_kernel, dim3(R.slots), dim3(64), 0, stream, 0, st, ds, drp, R);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("draft_round_begin launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

__device__ __forceinline__ void draft_collect(DecodeState ds, DraftRound R, int q) {
    const int c = R.cur[q];
    if (c < 0) return;
    R.prop[q * 8 + c] = ds.next_token[q];   // the draft sampler's token (EOT when its row had no finite logit)
    R.nprop[q] = c + 1;
    R.cur[q] = -1;
}

__global__ void draft_feed_kernel(DecodeState st, DecodeState ds, DraftRound R, int collect_only) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= R.slots) return;
    draft_collect(ds, R, q);
    if (collect_only) return;
    const bool ended = ds.done[q];              // the previous draft step ended the draft's sequence (EOT, length limit)
    ds.done[q] = 1;
    const int p0 = R.p0[q], f = R.fed[q], r0 = q * R.group;
    if (p0 < 0) return;
    int tok, n;
    if (f < p0) {                               // catch up on a committed token (its sample is not a proposal)
        tok = st.tokens[r0 * kMaxCtx + f];
        n = st.n_tokens[r0];
    } else {
        const int i = f - p0;                   // proposal i: input = the committed token at p0, then the draft's own proposals
        if (!R.verify[q] || i >= R.k || f >= st.rp[r0].max_steps || i != R.nprop[q] || (i > 0 && ended)) return;
        tok = i == 0 ? st.tokens[r0 * kMaxCtx + p0] : R.prop[q * 8 + i - 1];
        n = p0 + 1 + i;
        R.cur[q] = i;
    }
    ds.n_tokens[q] = n;
    ds.next_token[q] = tok;
    ds.steps[q] = f;
    ds.done[q] = 0;
    R.fed[q] = f + 1;
}

wk_status draft_feed(DecodeState st, DecodeState ds, DraftRound R, int collect_only, cudaStream_t stream) {
    launch_k(draft_feed_kernel, dim3((R.slots + 127) / 128), dim3(128), 0, stream, 0, st, ds, R, collect_only);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("draft_feed launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

__global__ void draft_verify_setup_kernel(DecodeState st, RowParams* __restrict__ rp, int32_t* __restrict__ anc, DraftRound R) {
    const int q = blockIdx.x, r0 = q * R.group, tid = threadIdx.x;
    __shared__ int s_nv;
    if (tid == 0) {
        const int p0 = R.p0[q];
        int nv = 0;
        if (p0 >= 0 && R.verify[q]) {
            // row j runs step p0 + j, which the sequential loop reaches only below max_steps (<= 223: positions stay inside the cache)
            nv = min(min(R.nprop[q], R.group - 1), st.rp[r0].max_steps - 1 - p0);
            nv = max(nv, 0);
        }
        R.rows[q] = nv;
        s_nv = nv;
    }
    __syncthreads();
    const int nv = s_nv;
    if (nv == 0) return;
    const int p0 = R.p0[q];
    const int32_t* prop = R.prop + q * 8;
    for (int i = tid; i < nv * kMaxCtx; i += blockDim.x) {
        const int j = 1 + i / kMaxCtx, t = i % kMaxCtx, r = r0 + j;
        if (t <= p0) st.tokens[r * kMaxCtx + t] = st.tokens[r0 * kMaxCtx + t];
        else if (t <= p0 + j) st.tokens[r * kMaxCtx + t] = prop[t - p0 - 1];
        if (t < p0) anc[r * kMaxCtx + t] = anc[r0 * kMaxCtx + t];
        else if (t < p0 + j) anc[r * kMaxCtx + t] = r0 + (t - p0);   // position p0 + i of this step is row i's
    }
    if (tid < nv) {
        const int j = tid + 1, r = r0 + j;
        rp[r] = st.rp[r0];
        st.next_token[r] = prop[j - 1];
        st.steps[r] = p0 + j;
        st.n_tokens[r] = p0 + 1 + j;
        st.done[r] = 0;
        st.error[r] = 0;
        st.first_low[r] = 0;
        st.lang_state[r] = 0;
    }
}

wk_status draft_verify_setup(DecodeState st, RowParams* rp, int32_t* anc, DraftRound R, cudaStream_t stream) {
    launch_k(draft_verify_setup_kernel, dim3(R.slots), dim3(256), 0, stream, 0, st, rp, anc, R);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("draft_verify_setup launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

__global__ void draft_accept_kernel(DecodeState st, int32_t* __restrict__ anc, DraftRound R) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= R.slots) return;
    const int r0 = q * R.group, rows = R.rows[q], p0 = R.p0[q];
    const int compared = rows > 0 ? min(R.nprop[q], rows + 1) : 0;   // proposal i is checked against the sample of row i
    int a = 0;
    for (int i = 0; i < compared; ++i) {
        // row 0 holds the state after step p0 + i: its sample must be proposal i, which row i + 1 took as its input
        if (st.next_token[r0] != R.prop[q * 8 + i]) break;
        ++a;
        if (st.done[r0] || i + 1 > rows) break;   // the window ended at this token, or step p0 + i + 1 had no row
        const int j = i + 1, r = r0 + j, at = p0 + 1 + j, n = st.n_tokens[r];
        if (n > at) {   // row j appended its sample to the history
            st.tokens[r0 * kMaxCtx + at] = st.tokens[r * kMaxCtx + at];
            st.logprobs[r0 * kMaxCtx + at] = st.logprobs[r * kMaxCtx + at];
        }
        st.n_tokens[r0] = n;
        st.steps[r0] = st.steps[r];
        st.next_token[r0] = st.next_token[r];
        st.done[r0] = st.done[r];
        st.first_low[r0] = st.first_low[r];
        st.error[r0] = st.error[r];
        anc[r0 * kMaxCtx + p0 + j] = r;
    }
    for (int j = 1; j < R.group; ++j) st.done[r0 + j] = 1;
    if (compared > 0) {
        atomicAdd(&R.counters[0], 1ull);
        atomicAdd(&R.counters[1], (unsigned long long)compared);
        atomicAdd(&R.counters[2], (unsigned long long)a);
    }
}

wk_status draft_accept(DecodeState st, int32_t* anc, DraftRound R, cudaStream_t stream) {
    launch_k(draft_accept_kernel, dim3((R.slots + 127) / 128), dim3(128), 0, stream, 0, st, anc, R);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("draft_accept launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

wk_status sampler_filter_sample(const float* logits, int64_t ld_logits, SamplerParams p, DecodeState st, const int32_t* tokens,
                                int ld_tokens, const int32_t* n_tokens, int32_t* token_out, float* logprob_out,
                                float* filtered_out, int B, cudaStream_t stream) {
    const bool top = p.top_n > 0;
    if (top && (p.top_n > kMaxTopLogprobs || !p.loop_mode || !p.top_tok || !p.top_lp)) {
        set_error("sampler: top_n %d needs the decode loop, its buffers and top_n <= %d", p.top_n, kMaxTopLogprobs);
        return WK_ERR_INVALID_ARGUMENT;
    }
    const size_t smem = (size_t)p.vocab * sizeof(float) + (top ? (2 * 32 * kMaxTopLogprobs + 1) * sizeof(float) : 0);
    if (smem > 220 * 1024) { set_error("sampler: vocab %d too large for the shared-memory row", p.vocab); return WK_ERR_INVALID_ARGUMENT; }
    static bool attr_set[2] = {false, false};
    auto kernel = top ? sampler_kernel<true> : sampler_kernel<false>;
    if (!attr_set[top]) {
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
        if (e != cudaSuccess) { set_error("cudaFuncSetAttribute(sampler): %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
        attr_set[top] = true;
    }
    launch_k(kernel, dim3(B), dim3(kSamplerThreads), smem, stream, 8, logits, (long long)ld_logits, p, st, tokens, ld_tokens,
             n_tokens, token_out, logprob_out, filtered_out);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("sampler launch: %s", cudaGetErrorString(e)); return WK_ERR_CUDA; }
    return WK_OK;
}

}  // namespace wk
