// The decoder plumbing the two Tacotron models share: the attention step (TacoAttention), the loop state at the start of
// the workspace and its reset, and the frame layout changes around the postnet.
// Reference: TTS/tts/layers/tacotron/attentions.py:9-37, 127-320, 323-438 (LocationLayer, OriginalAttention,
//            MonotonicDynamicConvolutionAttention).
#include <math.h>

#include "engines.cuh"

namespace b200tts {

namespace {

constexpr int A = 128;   // attention_dim of both models
constexpr int LOC_F = 32, LOC_K = 31, DCA_F = 8, DCA_K = 21, PRIOR_K = 11;
constexpr int PADL = 15;   // zero margin around the staged weights: the widest conv reach (31 taps, centred)

template <class Op>
__device__ float block_reduce(float v, float* red, Op op) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    v = red[0];
    for (int i = 1; i < nw; ++i) v = op(v, red[i]);
    return v;
}

__device__ __forceinline__ float warp_sum1(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

}  // namespace

// The attention kernel's arguments, one CTA per running row over its len_b tokens
struct AttnArgs {
    const float* q = nullptr;                 // [B, Q] attention-RNN output
    const float* enc = nullptr;               // [B, Tt, E] encoder outputs
    const float* pin = nullptr;               // [B, A, Tt] inputs_layer(encoder outputs)
    float* alpha = nullptr; float* cum = nullptr;   // [B, Tt] previous / cumulative weights
    float* ctx = nullptr;                     // [B, E]
    float* align = nullptr; int max_steps = 0;      // [B, max_steps, Tt]
    const long long* lens = nullptr; const int* done = nullptr; const int* ctl = nullptr;
    int Tt = 0, type = 0, location = 0, softmax = 0;
    // original: Wq [A][Q], v [A], vb; location: Wc [F][2][K], Wd [A][F]
    // DCA: Wq [A][Q], bq [A], Wk [F*K][A], Ws [F][K], Wsl [A][F], Wdl [A][F], bdl [A], v [A], prior [11]
    const float *Wq = nullptr, *bq = nullptr, *v = nullptr, *Wc = nullptr, *Wd = nullptr;
    const float *Wk = nullptr, *Ws = nullptr, *Wsl = nullptr, *Wdl = nullptr, *bdl = nullptr, *prior = nullptr;
    float vb = 0.f;
};

namespace {

// One attention step for row b = blockIdx.x over its len_b tokens (OriginalAttention.forward with mask None /
// MonotonicDynamicConvolutionAttention.forward), then the context and the alignment row of step ctl[1].  Q / E: the
// query and encoder widths.
template <int Q, int E>
__global__ void __launch_bounds__(256) taco_attn_kernel(AttnArgs a) {
    extern __shared__ float sm[];
    const int b = blockIdx.x;
    if (a.done[b]) return;
    const int len = (int)a.lens[b], Tt = a.Tt, t = a.ctl[1];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    float* qs = sm;                      // [Q]
    float* pq = qs + Q;                  // [A]
    float* tq = pq + A;                  // [A]
    float* G = tq + A;                   // [DCA_F * DCA_K]
    float* red = G + DCA_F * DCA_K;      // [32]
    float* ap = red + 32;                // [Tt + 2 PADL] previous weights, zero margins
    float* cp = ap + Tt + 2 * PADL;      // [Tt + 2 PADL] cumulative weights
    float* e = cp + Tt + 2 * PADL;       // [Tt] energies, then weights
    // the per-token weights, staged so that lane j reads consecutive words: location dense (original) or
    // static / dynamic filter layers (DCA) transposed to [filter][A], and the conv taps
    float* wT = e + Tt;                  // [LOC_F][A]
    float* wc = wT + LOC_F * A;          // [LOC_F][2][LOC_K] (original) or [DCA_F][DCA_K] (DCA)
    for (int i = threadIdx.x; i < Q; i += blockDim.x) qs[i] = a.q[(size_t)b * Q + i];
    if (a.type == 0 && a.location) {
        for (int i = threadIdx.x; i < A * LOC_F; i += blockDim.x) wT[(i % LOC_F) * A + i / LOC_F] = a.Wd[i];
        for (int i = threadIdx.x; i < LOC_F * 2 * LOC_K; i += blockDim.x) wc[i] = a.Wc[i];
    } else if (a.type == 1) {
        for (int i = threadIdx.x; i < A * DCA_F; i += blockDim.x) {
            wT[(i % DCA_F) * A + i / DCA_F] = a.Wsl[i];
            wT[(DCA_F + i % DCA_F) * A + i / DCA_F] = a.Wdl[i];
        }
        for (int i = threadIdx.x; i < DCA_F * DCA_K; i += blockDim.x) wc[i] = a.Ws[i];
    }
    for (int i = threadIdx.x; i < Tt + 2 * PADL; i += blockDim.x) {
        const int n = i - PADL;
        const bool in = n >= 0 && n < len;
        ap[i] = in ? a.alpha[(size_t)b * Tt + n] : 0.f;
        cp[i] = in && a.cum ? a.cum[(size_t)b * Tt + n] : 0.f;
    }
    __syncthreads();
    for (int j = warp; j < A; j += nw) {   // processed query
        float s = 0.f;
        for (int k = lane; k < Q; k += 32) s = fmaf(a.Wq[(size_t)j * Q + k], qs[k], s);
        s = warp_sum1(s);
        if (lane == 0) pq[j] = a.bq ? s + a.bq[j] : s;
    }
    __syncthreads();
    if (a.type == 1) {   // G = key_layer(tanh(query_layer(q)))
        for (int j = threadIdx.x; j < A; j += blockDim.x) tq[j] = tanhf(pq[j]);
        __syncthreads();
        for (int r = warp; r < DCA_F * DCA_K; r += nw) {
            float s = 0.f;
            for (int k = lane; k < A; k += 32) s = fmaf(a.Wk[(size_t)r * A + k], tq[k], s);
            s = warp_sum1(s);
            if (lane == 0) G[r] = s;
        }
        __syncthreads();
    }
    for (int n = warp; n < len; n += nw) {   // energies: one warp per token
        const float* x = ap + PADL + n;      // x[k] = alpha[n + k]
        float acc = 0.f;
        if (a.type == 0) {
            float f = 0.f;                   // location feature LOC_F of lane
            if (a.location) {
                const float* w = wc + lane * 2 * LOC_K;
                const float* xc = cp + PADL + n;
                for (int k = 0; k < LOC_K; ++k) {
                    f = fmaf(w[k], x[k - LOC_K / 2], f);
                    f = fmaf(w[LOC_K + k], xc[k - LOC_K / 2], f);
                }
            }
#pragma unroll
            for (int m = 0; m < A / 32; ++m) {
                const int j = lane + 32 * m;
                float u = pq[j];
                if (a.location) {
                    float l = 0.f;
#pragma unroll 8
                    for (int i = 0; i < LOC_F; ++i) l = fmaf(wT[i * A + j], __shfl_sync(0xffffffffu, f, i), l);
                    u += l;
                }
                u += a.pin[((size_t)b * A + j) * Tt + n];
                acc = fmaf(a.v[j], tanhf(u), acc);
            }
            acc = warp_sum1(acc) + a.vb;
        } else {
            float f = 0.f;                   // lanes 0..7: static filter i, lanes 8..15: dynamic filter i - 8
            if (lane < 2 * DCA_F) {
                const float* w = lane < DCA_F ? wc + lane * DCA_K : G + (lane - DCA_F) * DCA_K;
                for (int k = 0; k < DCA_K; ++k) f = fmaf(w[k], x[k - DCA_K / 2], f);
            }
#pragma unroll
            for (int m = 0; m < A / 32; ++m) {
                const int j = lane + 32 * m;
                float s = 0.f, dd = 0.f;
#pragma unroll
                for (int i = 0; i < DCA_F; ++i) {
                    s = fmaf(wT[i * A + j], __shfl_sync(0xffffffffu, f, i), s);
                    dd = fmaf(wT[(DCA_F + i) * A + j], __shfl_sync(0xffffffffu, f, DCA_F + i), dd);
                }
                acc = fmaf(a.v[j], tanhf(s + (dd + a.bdl[j])), acc);
            }
            acc = warp_sum1(acc);
            float pr = 0.f;                  // causal prior: sum_k prior[k] alpha[n + k - 10]
            for (int k = 0; k < PRIOR_K; ++k) pr = fmaf(a.prior[k], x[k - (PRIOR_K - 1)], pr);
            acc += logf(fmaxf(pr, 1e-6f));
        }
        if (lane == 0) e[n] = acc;
    }
    __syncthreads();
    // normalisation over the row's tokens
    if (a.type == 1 || a.softmax) {
        float m = -INFINITY;
        for (int n = threadIdx.x; n < len; n += blockDim.x) m = fmaxf(m, e[n]);
        m = block_reduce(m, red, [](float x, float y) { return fmaxf(x, y); });
        float s = 0.f;
        for (int n = threadIdx.x; n < len; n += blockDim.x) {
            const float v = expf(e[n] - m);
            e[n] = v;
            s += v;
        }
        s = block_reduce(s, red, [](float x, float y) { return x + y; });
        for (int n = threadIdx.x; n < len; n += blockDim.x) e[n] = e[n] / s;
    } else {
        float s = 0.f;
        for (int n = threadIdx.x; n < len; n += blockDim.x) {
            const float v = 1.f / (1.f + expf(-e[n]));
            e[n] = v;
            s += v;
        }
        s = block_reduce(s, red, [](float x, float y) { return x + y; });
        for (int n = threadIdx.x; n < len; n += blockDim.x) e[n] = e[n] / s;
    }
    __syncthreads();
    for (int n = threadIdx.x; n < len; n += blockDim.x) {
        const float w = e[n];
        a.alpha[(size_t)b * Tt + n] = w;
        if (a.cum) a.cum[(size_t)b * Tt + n] = cp[PADL + n] + w;
        a.align[((size_t)b * a.max_steps + t) * Tt + n] = w;
    }
    const float* eb = a.enc + (size_t)b * Tt * E;
    for (int c = threadIdx.x; c < E; c += blockDim.x) {
        float s = 0.f;
        for (int n = 0; n < len; ++n) s = fmaf(e[n], eb[(size_t)n * E + c], s);
        a.ctx[(size_t)b * E + c] = s;
    }
}

// loop state at step 0: zero RNN states, context and go frame; alpha zero (original) or one-hot at token 0 (DCA)
__global__ void taco_reset_kernel(float* zero, size_t nzero, float* alpha, int Tt, int one_hot, int* done, int* ctl, int B) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nzero; i += (size_t)gridDim.x * blockDim.x)
        zero[i] = 0.f;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < B * Tt; i += gridDim.x * blockDim.x)
        alpha[i] = (one_hot && i % Tt == 0) ? 1.f : 0.f;
    if (blockIdx.x == 0)
        for (int b = threadIdx.x; b < B; b += blockDim.x) {
            done[b] = 0;
            ctl[2 + b] = 0;
            if (b == 0) { ctl[0] = B; ctl[1] = 0; }
        }
}

// postnet input: x[b, c, t] = dec[b, t, c] below frames[b], else 0; mask[b, t] likewise
__global__ void postnet_in_kernel(const float* dec, int Fpitch, const int* frames, float* x, float* mask, int C, int Tp) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x, c = blockIdx.y, b = blockIdx.z;
    if (t >= Tp) return;
    const bool valid = t < frames[b];
    x[((size_t)b * C + c) * Tp + t] = valid ? dec[((size_t)b * Fpitch + t) * C + c] : 0.f;
    if (c == 0) mask[(size_t)b * Tp + t] = valid ? 1.f : 0.f;
}

// out[b, t, c] = y[b, c, t] for t < F
__global__ void postnet_out_kernel(const float* y, int Tp, float* out, int F, int C) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (i >= F * C) return;
    const int t = i / C, c = i - t * C;
    out[(size_t)b * F * C + i] = y[((size_t)b * C + c) * Tp + t];
}

size_t attn_smem_bytes(int Qd, int Tt) {
    return sizeof(float) * (Qd + 2 * A + DCA_F * DCA_K + 32 + 3 * (size_t)Tt + 4 * PADL + LOC_F * A + LOC_F * 2 * LOC_K);
}

}  // namespace

// ------------------------------------------------------------------ the attention
int TacoAttention::init(int q_dim, int e_dim, int attention_type, int location_attn, int attention_softmax,
                        WeightList& wl) {
    Q = q_dim; E = e_dim; type = attention_type; location = location_attn; softmax = attention_softmax;
    B200_REQUIRE((Q == 1024 && E == 512) || (Q == 256 && E == 256), "taco_attn: no kernel for Q %d / E %d", Q, E);
    int rc;
    if (type == 0) {
        if ((rc = upload(wq, wl.take(), (size_t)A * Q))) return rc;
        if ((rc = pack_conv(inproj, wl.take(), nullptr, A, E, 1, 1, 0))) return rc;
        if ((rc = upload(v, wl.take(), A))) return rc;
        const float* v_bias = wl.take();
        B200_REQUIRE(v_bias, "taco_attn: null v.bias");
        vb = v_bias[0];
        if (location) {
            if ((rc = upload(wc, wl.take(), (size_t)LOC_F * 2 * LOC_K))) return rc;
            if ((rc = upload(wd, wl.take(), (size_t)A * LOC_F))) return rc;
        }
    } else {
        if ((rc = upload(prior, wl.take(), PRIOR_K))) return rc;
        if ((rc = upload(wq, wl.take(), (size_t)A * Q))) return rc;
        if ((rc = upload(bq, wl.take(), A))) return rc;
        if ((rc = upload(wk, wl.take(), (size_t)DCA_F * DCA_K * A))) return rc;
        if ((rc = upload(ws, wl.take(), (size_t)DCA_F * DCA_K))) return rc;
        if ((rc = upload(wsl, wl.take(), (size_t)A * DCA_F))) return rc;
        if ((rc = upload(wdl, wl.take(), (size_t)A * DCA_F))) return rc;
        if ((rc = upload(bdl, wl.take(), A))) return rc;
        if ((rc = upload(v, wl.take(), A))) return rc;
    }
    return 0;
}

int TacoAttention::keys(const float* enc, float* encT, float* pin, int B, int Tt, cudaStream_t st) const {
    if (type != 0) return 0;
    int rc;
    if ((rc = launch_transpose(enc, encT, B, Tt, E, st))) return rc;
    ConvIO io;
    io.x = dense(encT, E, Tt); io.Tin = Tt;
    io.y = dense(pin, A, Tt); io.Tout = Tt; io.B = B;
    return launch_conv(inproj, io, st);
}

int TacoAttention::prepare(int Tt, size_t* smem) const {
    const size_t n = attn_smem_bytes(Q, Tt);
    B200_REQUIRE(n <= 200 * 1024, "taco_attn: %d tokens exceed the attention kernel's shared memory", Tt);
    if (n > 48 * 1024) {
        if (Q == 1024)
            B200_CUDA_OK(cudaFuncSetAttribute(taco_attn_kernel<1024, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)n));
        else
            B200_CUDA_OK(cudaFuncSetAttribute(taco_attn_kernel<256, 256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)n));
    }
    *smem = n;
    return 0;
}

int TacoAttention::launch(const TacoLoop& p, const float* q, float* ctx, const float* enc, float* align, int S,
                          const long long* lens, int B, int Tt, size_t smem, cudaStream_t st, bool note) const {
    AttnArgs a;
    a.q = q; a.enc = enc; a.pin = p.pin; a.alpha = p.alpha; a.cum = (type == 0 && location) ? p.cum : nullptr;
    a.ctx = ctx; a.align = align; a.max_steps = S; a.lens = lens; a.done = p.done; a.ctl = p.ctl; a.Tt = Tt;
    a.type = type; a.location = location; a.softmax = softmax;
    a.Wq = wq; a.bq = bq; a.v = v; a.vb = vb; a.Wc = wc; a.Wd = wd;
    a.Wk = wk; a.Ws = ws; a.Wsl = wsl; a.Wdl = wdl; a.bdl = bdl; a.prior = prior;
    if (Q == 1024) taco_attn_kernel<1024, 512><<<B, 256, smem, st>>>(a);
    else taco_attn_kernel<256, 256><<<B, 256, smem, st>>>(a);
    if (note) dispatch_note(DISPATCH_TACO_ATTN);
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------ the loop state
void taco_loop_layout(Arena& ar, int B, int Tt, int RC, size_t nzero, TacoLoop& p) {
    p.pin = ar.f32((size_t)B * A * Tt);
    p.ctl = (int*)ar.f32(2 + B);
    p.done = (int*)ar.f32(B);
    p.alpha = ar.f32((size_t)B * Tt);
    p.cum = ar.f32((size_t)B * Tt);
    p.proj = ar.f32((size_t)B * RC);
    p.logit = ar.f32(B);
    p.zero = ar.f32(nzero);
    p.nzero = nzero;
}

int taco_loop_start(const TacoLoop& p, int B, int Tt, int S, int rC, int one_hot, float* dec_out, float* stop,
                    float* align, cudaStream_t st) {
    B200_CUDA_OK(cudaMemsetAsync(dec_out, 0, sizeof(float) * (size_t)B * S * rC, st));
    B200_CUDA_OK(cudaMemsetAsync(stop, 0, sizeof(float) * (size_t)B * S, st));
    B200_CUDA_OK(cudaMemsetAsync(align, 0, sizeof(float) * (size_t)B * S * Tt, st));
    B200_CUDA_OK(cudaMemsetAsync(p.cum, 0, sizeof(float) * (size_t)B * Tt, st));
    taco_reset_kernel<<<64, 256, 0, st>>>(p.zero, p.nzero, p.alpha, Tt, one_hot, p.done, p.ctl, B);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------ around the postnet
int launch_frames_in(const float* dec, int Fpitch, const int* frames, float* x, float* mask, int B, int C, int Tp,
                     cudaStream_t st) {
    postnet_in_kernel<<<dim3((Tp + 127) / 128, C, B), 128, 0, st>>>(dec, Fpitch, frames, x, mask, C, Tp);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

int launch_frames_out(const float* y, int Tp, float* out, int B, int F, int C, cudaStream_t st) {
    postnet_out_kernel<<<dim3((F * C + 255) / 256, B), 256, 0, st>>>(y, Tp, out, F, C);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace b200tts
