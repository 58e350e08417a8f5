// Tacotron2 inference: text -> mel spectrogram through the location-sensitive (or dynamic-convolution) attention decoder.
// Reference: TTS/tts/models/tacotron2.py:238-300 (inference), TTS/tts/layers/tacotron/tacotron2.py (Encoder, Decoder,
//            Postnet), common_layers.py:63-119 (Prenet), attentions.py:9-37, 127-320, 323-438 (LocationLayer,
//            OriginalAttention, MonotonicDynamicConvolutionAttention).
// The decoder loop is exact FP32 on the FMA pipe (the stop decision feeds back through it).  Per step: two prenet GEMVs,
// the attention LSTMCell, one attention launch per row, the decoder LSTMCell, the projection and stopnet GEMVs and the
// step epilogue -- 8 launches, captured as CUDA-graph chunks.  The two LSTMCells read ~72 MB of weights per step; with
// more than 8 rows one weight read serves 32 rows.
#include <math.h>

#include "engines.cuh"

namespace b200tts {

namespace {

constexpr int E = 512, HE = 256, Q = 1024, D = 1024, A = 128, PN = 256;
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

// The step epilogue (Decoder.inference's loop body after decode): for each running row b, the first r frames of the
// projection -> dec_out[b, t*r .. t*r + r), the next prenet input = the last of them, stop[b, t] = sigmoid(logit); done
// after step t >= 1 when that exceeds 0.5, or at t = max_steps - 1 (steps[b] = t + 1); then ctl = {running, t + 1}.
struct StepArgs {
    const float* proj = nullptr; int RC = 0; const float* logit = nullptr;
    int C = 0, r = 0, max_steps = 0;
    float* dec_out = nullptr; float* stop = nullptr; float* mem = nullptr;
    int* done = nullptr; int* ctl = nullptr; int B = 0;
};

__global__ void __launch_bounds__(256) taco_step_kernel(StepArgs a) {
    const int t = a.ctl[1], rc = a.r * a.C;
    for (int i = threadIdx.x; i < a.B * rc; i += blockDim.x) {
        const int b = i / rc, k = i - b * rc;
        if (a.done[b]) continue;
        const float v = a.proj[(size_t)b * a.RC + k];
        a.dec_out[((size_t)b * a.max_steps * a.r + (size_t)t * a.r) * a.C + k] = v;
        if (k >= rc - a.C) a.mem[(size_t)b * a.C + k - (rc - a.C)] = v;
    }
    __syncthreads();
    for (int b = threadIdx.x; b < a.B; b += blockDim.x) {
        if (a.done[b]) continue;
        const float s = 1.f / (1.f + expf(-a.logit[b]));
        a.stop[(size_t)b * a.max_steps + t] = s;
        if ((t >= 1 && s > 0.5f) || t == a.max_steps - 1) {
            a.done[b] = 1;
            a.ctl[2 + b] = t + 1;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int run = 0;
        for (int b = 0; b < a.B; ++b) run += a.done[b] ? 0 : 1;
        a.ctl[0] = run;
        a.ctl[1] = t + 1;
    }
}

// loop state at step 0: zero LSTM states, context and go frame; alpha zero (original) or one-hot at token 0 (DCA)
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

// mel[b, t, c] = y[b, c, t] for t < F
__global__ void postnet_out_kernel(const float* y, int Tp, float* mel, int F, int C) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (i >= F * C) return;
    const int t = i / C, c = i - t * C;
    mel[(size_t)b * F * C + i] = y[((size_t)b * C + c) * Tp + t];
}

struct Persist {   // the part of the workspace that lives from encode to the end of the loop
    float *pin, *mem, *pb, *q, *qc, *ctx, *dh, *dc, *alpha, *cum, *proj, *logit;
    int *ctl, *done;
};

size_t attn_smem_bytes(int Qd, int Tt) {
    return sizeof(float) * (Qd + 2 * A + DCA_F * DCA_K + 32 + 3 * (size_t)Tt + 4 * PADL + LOC_F * A + LOC_F * 2 * LOC_K);
}

}  // namespace

int taco_attn_prepare(int Qd, int Ed, int Tt, size_t* smem) {
    B200_REQUIRE((Qd == 1024 && Ed == 512) || (Qd == 256 && Ed == 256), "taco_attn: no kernel for Q %d / E %d", Qd, Ed);
    const size_t n = attn_smem_bytes(Qd, Tt);
    B200_REQUIRE(n <= 200 * 1024, "taco_attn: %d tokens exceed the attention kernel's shared memory", Tt);
    if (n > 48 * 1024) {
        if (Qd == 1024)
            B200_CUDA_OK(cudaFuncSetAttribute(taco_attn_kernel<1024, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)n));
        else
            B200_CUDA_OK(cudaFuncSetAttribute(taco_attn_kernel<256, 256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)n));
    }
    *smem = n;
    return 0;
}

int launch_taco_attn(const AttnArgs& a, int Qd, int Ed, int B, size_t smem, cudaStream_t st, bool note) {
    if (Qd == 1024 && Ed == 512) taco_attn_kernel<1024, 512><<<B, 256, smem, st>>>(a);
    else if (Qd == 256 && Ed == 256) taco_attn_kernel<256, 256><<<B, 256, smem, st>>>(a);
    else { set_error("taco_attn: no kernel for Q %d / E %d", Qd, Ed); return 1; }
    if (note) dispatch_note(DISPATCH_TACO_ATTN);
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

static bool persist_layout(const Tacotron2& e, Arena& ar, int B, int Tt, Persist& p) {
    const int C = e.c.out_channels;
    p.pin = ar.f32((size_t)B * A * Tt);
    p.ctl = (int*)ar.f32(2 + B);
    p.done = (int*)ar.f32(B);
    p.alpha = ar.f32((size_t)B * Tt);
    p.cum = ar.f32((size_t)B * Tt);
    p.proj = ar.f32((size_t)B * C * e.c.r_init);
    p.logit = ar.f32(B);
    p.pb = ar.f32((size_t)2 * B * PN);
    // zeroed at the start of the loop, one run: go frame, both query buffers, cell, context, both decoder buffers, cell
    const size_t nz = (size_t)B * (C + 2 * Q + Q + E + 2 * D + D);
    float* z = ar.f32(nz);
    if (!(p.pin && p.ctl && p.done && p.alpha && p.cum && p.proj && p.logit && p.pb && z)) return false;
    p.mem = z;
    p.q = p.mem + (size_t)B * C;
    p.qc = p.q + (size_t)2 * B * Q;
    p.ctx = p.qc + (size_t)B * Q;
    p.dh = p.ctx + (size_t)B * E;
    p.dc = p.dh + (size_t)2 * B * D;
    return true;
}

size_t Tacotron2::persist_bytes(int B, int Tt) const {
    const int C = c.out_channels;
    return arena_bytes((size_t)B * A * Tt) + arena_bytes(2 + B) + arena_bytes(B) + 2 * arena_bytes((size_t)B * Tt) +
           arena_bytes((size_t)B * C * c.r_init) + arena_bytes(B) + arena_bytes((size_t)2 * B * PN) +
           arena_bytes((size_t)B * (C + 2 * Q + Q + E + 2 * D + D));
}

size_t Tacotron2::workspace_bytes(int B, int Tt, int F) const {
    const size_t encb = persist_bytes(B, Tt) + enc.workspace_bytes(B, Tt) + arena_bytes((size_t)B * E * Tt);
    const int Tp = (F + 3) / 4 * 4, C = c.out_channels;
    const size_t postb = 2 * arena_bytes((size_t)B * C * Tp) + 2 * arena_bytes((size_t)B * 512 * Tp) +
                         arena_bytes((size_t)B * Tp);
    return std::max(encb, postb) + 1024;
}

int Tacotron2::init(const b200tts_tacotron2_config& cfg, const float* const* w, int nw) {
    c = cfg;
    const int C = c.out_channels;
    B200_REQUIRE(c.n_vocab > 0 && C > 0 && c.r_init >= 1 && (c.attention_type == 0 || c.attention_type == 1),
                 "tacotron2: unsupported config");
    const int expect = 1 + 6 * 3 + 8 + 2 * (c.prenet_bn ? 5 : 1) + 4 +
                       (c.attention_type == 1 ? 9 : 4 + (c.location_attn ? 2 : 0)) + 4 + 2 + 2 + 6 * 5;
    B200_REQUIRE(nw == expect, "tacotron2: expected %d weight tensors, got %d", expect, nw);
    int rc, i = 0, used = 0;
    if ((rc = enc.init(c.n_vocab, E, HE, 3, w, &used))) return rc;
    i += used;
    for (int l = 0; l < 2; ++l) {   // prenet (no bias); "bn": eval BatchNorm folded into the layer
        const int in = l ? PN : C;
        if (!c.prenet_bn) {
            if ((rc = upload(prenet_w[l], w[i++], (size_t)PN * in))) return rc;
            continue;
        }
        std::vector<float> wf((size_t)PN * in), bf(PN);
        for (int o = 0; o < PN; ++o) {
            const double s = (double)w[i + 1][o] / sqrt((double)w[i + 4][o] + 1e-5);
            for (int k = 0; k < in; ++k) wf[(size_t)o * in + k] = (float)(w[i][(size_t)o * in + k] * s);
            bf[o] = (float)(w[i + 2][o] - w[i + 3][o] * s);
        }
        if ((rc = upload(prenet_w[l], wf.data(), wf.size()))) return rc;
        if ((rc = upload(prenet_b[l], bf.data(), bf.size()))) return rc;
        i += 5;
    }
    auto lstm = [&](DevBuf<float>& wih, DevBuf<float>& whh, DevBuf<float>& bias, int in, int H) -> int {
        int r;
        if ((r = upload(wih, w[i], (size_t)4 * H * in))) return r;
        if ((r = upload(whh, w[i + 1], (size_t)4 * H * H))) return r;
        std::vector<float> b((size_t)4 * H);
        for (int k = 0; k < 4 * H; ++k) b[k] = w[i + 2][k] + w[i + 3][k];
        i += 4;
        return upload(bias, b.data(), b.size());
    };
    if ((rc = lstm(arnn_wih, arnn_whh, arnn_b, PN + E, Q))) return rc;
    if (c.attention_type == 0) {
        if ((rc = upload(att_wq, w[i++], (size_t)A * Q))) return rc;
        if ((rc = pack_conv(inproj, w[i++], nullptr, A, E, 1, 1, 0))) return rc;
        if ((rc = upload(att_v, w[i++], A))) return rc;
        att_vb = w[i++][0];
        if (c.location_attn) {
            if ((rc = upload(att_wc, w[i++], (size_t)LOC_F * 2 * LOC_K))) return rc;
            if ((rc = upload(att_wd, w[i++], (size_t)A * LOC_F))) return rc;
        }
    } else {
        if ((rc = upload(att_prior, w[i++], PRIOR_K))) return rc;
        if ((rc = upload(att_wq, w[i++], (size_t)A * Q))) return rc;
        if ((rc = upload(att_bq, w[i++], A))) return rc;
        if ((rc = upload(att_wk, w[i++], (size_t)DCA_F * DCA_K * A))) return rc;
        if ((rc = upload(att_ws, w[i++], (size_t)DCA_F * DCA_K))) return rc;
        if ((rc = upload(att_wsl, w[i++], (size_t)A * DCA_F))) return rc;
        if ((rc = upload(att_wdl, w[i++], (size_t)A * DCA_F))) return rc;
        if ((rc = upload(att_bdl, w[i++], A))) return rc;
        if ((rc = upload(att_v, w[i++], A))) return rc;
    }
    if ((rc = lstm(drnn_wih, drnn_whh, drnn_b, Q + E, D))) return rc;
    if ((rc = upload(proj_w, w[i], (size_t)C * c.r_init * (D + E)))) return rc;
    if ((rc = upload(proj_b, w[i + 1], (size_t)C * c.r_init))) return rc;
    if ((rc = upload(stop_w, w[i + 2], (size_t)D + C * c.r_init))) return rc;
    if ((rc = upload(stop_b, w[i + 3], 1))) return rc;
    i += 4;
    for (int l = 0; l < 5; ++l, i += 6) {   // Postnet ConvBNBlocks, BatchNorm folded
        const int ci = l ? 512 : C, co = l == 4 ? C : 512;
        std::vector<float> wf((size_t)co * ci * 5), bf(co);
        for (int o = 0; o < co; ++o) {
            const double s = (double)w[i + 2][o] / sqrt((double)w[i + 5][o] + 1e-5);
            for (size_t k = 0; k < (size_t)ci * 5; ++k) wf[(size_t)o * ci * 5 + k] = (float)(w[i][(size_t)o * ci * 5 + k] * s);
            bf[o] = (float)(((double)w[i + 1][o] - w[i + 4][o]) * s + w[i + 3][o]);
        }
        if ((rc = pack_conv(post[l], wf.data(), bf.data(), co, ci, 5, 1, 2))) return rc;
    }
    return 0;
}

int Tacotron2::encode(const long long* tokens, const long long* lengths, int B, int Tt, float* enc_out, void* ws,
                      size_t ws_bytes, cudaStream_t st) const {
    B200_REQUIRE(tokens && lengths && enc_out && ws, "tacotron2_encode: null pointer");
    B200_REQUIRE(B >= 1 && Tt >= 1, "tacotron2_encode: empty batch");
    B200_REQUIRE(ws_bytes >= workspace_bytes(B, Tt, 0), "tacotron2_encode: workspace too small");
    Arena ar(ws, ws_bytes);
    Persist p;
    B200_REQUIRE(persist_layout(*this, ar, B, Tt, p), "tacotron2_encode: arena exhausted");
    int rc;
    if ((rc = enc.encode(tokens, lengths, B, Tt, enc_out, ar, st))) return rc;
    if (c.attention_type == 0) {   // inputs_layer, step-invariant: pin [B, A, Tt]
        float* encT = ar.f32((size_t)B * E * Tt);
        B200_REQUIRE(encT, "tacotron2_encode: arena exhausted");
        if ((rc = launch_transpose(enc_out, encT, B, Tt, E, st))) return rc;
        ConvIO io;
        io.x = encT; io.x_bs = (long long)E * Tt; io.x_cs = Tt; io.Tin = Tt;
        io.y = p.pin; io.y_bs = (long long)A * Tt; io.y_cs = Tt; io.Tout = Tt; io.B = B;
        if ((rc = launch_conv(inproj, io, st))) return rc;
    }
    return 0;
}

int Tacotron2::decode_loop(const long long* lengths, const float* enc_out, int B, int Tt, int r, int max_steps,
                           const unsigned char* drop, int chunk_steps, float* dec_out, float* stop_tokens,
                           float* alignments, int* steps, void* ws, size_t ws_bytes, cudaStream_t st) const {
    B200_REQUIRE(lengths && enc_out && dec_out && stop_tokens && alignments && steps && ws,
                 "tacotron2_decode_loop: null pointer");
    B200_REQUIRE(B >= 1 && Tt >= 1 && max_steps >= 1, "tacotron2_decode_loop: B, Tt and max_steps must be >= 1");
    B200_REQUIRE(r >= 1 && r <= c.r_init, "tacotron2_decode_loop: r must be in [1, r_init = %d]", c.r_init);
    B200_REQUIRE(chunk_steps >= 2 && chunk_steps % 2 == 0, "tacotron2_decode_loop: chunk_steps must be even and >= 2");
    B200_REQUIRE(ws_bytes >= workspace_bytes(B, Tt, 0), "tacotron2_decode_loop: workspace too small");
    const int C = c.out_channels, RC = C * c.r_init;
    Arena ar(ws, ws_bytes);
    Persist p;
    B200_REQUIRE(persist_layout(*this, ar, B, Tt, p), "tacotron2_decode_loop: arena exhausted");
    B200_CUDA_OK(cudaMemsetAsync(dec_out, 0, sizeof(float) * (size_t)B * max_steps * r * C, st));
    B200_CUDA_OK(cudaMemsetAsync(stop_tokens, 0, sizeof(float) * (size_t)B * max_steps, st));
    B200_CUDA_OK(cudaMemsetAsync(alignments, 0, sizeof(float) * (size_t)B * max_steps * Tt, st));
    B200_CUDA_OK(cudaMemsetAsync(p.cum, 0, sizeof(float) * (size_t)B * Tt, st));
    int rc;
    taco_reset_kernel<<<64, 256, 0, st>>>(p.mem, (size_t)B * (C + 2 * Q + Q + E + 2 * D + D), p.alpha, Tt,
                                          c.attention_type == 1, p.done, p.ctl, B);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    const int nb = B > 8 ? 32 : 8;
    const int lstm_id = nb == 32 ? DISPATCH_LSTM_CELL32 : DISPATCH_LSTM_CELL;
    size_t attn_smem = 0;
    if ((rc = taco_attn_prepare(Q, E, Tt, &attn_smem))) return rc;
    // one step; parity = step index within the chunk (query and decoder h are double-buffered)
    auto step = [&](cudaStream_t cs, int par, bool note) -> int {
        int rc;
        const float* in = p.mem;
        for (int l = 0; l < 2; ++l) {
            LinArgs a;
            a.W = prenet_w[l]; a.bias = prenet_b[l]; a.K = l ? PN : C; a.R = PN; a.x = in; a.x_bs = a.K;
            a.y = p.pb + (size_t)l * B * PN; a.y_bs = PN; a.relu = 1;
            a.drop = c.prenet_dropout ? drop : nullptr; a.drop_layer = l; a.drop_L = 2; a.drop_F = max_steps;
            a.ctl = p.ctl; a.done = p.done; a.B = B;
            if ((rc = launch_linear(a, cs, note))) return rc;
            in = a.y;
        }
        float* q_in = p.q + (size_t)par * B * Q;
        float* q_out = p.q + (size_t)(par ^ 1) * B * Q;
        {   // attention RNN on [prenet | context], h
            LstmArgs a;
            a.seg[0] = {arnn_wih, PN + E, 0, in, PN, 0, PN};
            a.seg[1] = {arnn_wih + PN, PN + E, 0, p.ctx, E, 0, E};
            a.seg[2] = {arnn_whh, Q, 0, q_in, Q, 0, Q};
            a.nseg = 3;
            a.H = Q; a.h_out = q_out; a.h_bs = Q; a.c = p.qc; a.bias = arnn_b; a.done = p.done; a.B = B;
            if ((rc = launch_lstm(a, 1, nb, lstm_id, cs, note))) return rc;
        }
        {
            AttnArgs a;
            a.q = q_out; a.enc = enc_out; a.pin = p.pin; a.alpha = p.alpha;
            a.cum = (c.attention_type == 0 && c.location_attn) ? p.cum : nullptr;
            a.ctx = p.ctx; a.align = alignments; a.max_steps = max_steps; a.lens = lengths; a.done = p.done;
            a.ctl = p.ctl; a.Tt = Tt; a.type = c.attention_type; a.location = c.location_attn;
            a.softmax = c.attention_norm; a.Wq = att_wq; a.bq = att_bq; a.v = att_v; a.vb = att_vb; a.Wc = att_wc;
            a.Wd = att_wd; a.Wk = att_wk; a.Ws = att_ws; a.Wsl = att_wsl; a.Wdl = att_wdl; a.bdl = att_bdl;
            a.prior = att_prior;
            if ((rc = launch_taco_attn(a, Q, E, B, attn_smem, cs, note))) return rc;
        }
        float* dh_in = p.dh + (size_t)par * B * D;
        float* dh_out = p.dh + (size_t)(par ^ 1) * B * D;
        {   // decoder RNN on [query | context], h
            LstmArgs a;
            a.seg[0] = {drnn_wih, Q + E, 0, q_out, Q, 0, Q};
            a.seg[1] = {drnn_wih + Q, Q + E, 0, p.ctx, E, 0, E};
            a.seg[2] = {drnn_whh, D, 0, dh_in, D, 0, D};
            a.nseg = 3;
            a.H = D; a.h_out = dh_out; a.h_bs = D; a.c = p.dc; a.bias = drnn_b; a.done = p.done; a.B = B;
            if ((rc = launch_lstm(a, 1, nb, lstm_id, cs, note))) return rc;
        }
        {   // linear_projection([h | context]), all C * r_init rows
            LinArgs a;
            a.W = proj_w; a.bias = proj_b; a.K = D; a.R = RC; a.x = dh_out; a.x_bs = D; a.x2 = p.ctx; a.x2_bs = E;
            a.K2 = E; a.y = p.proj; a.y_bs = RC; a.done = p.done; a.B = B;
            if ((rc = launch_linear(a, cs, note))) return rc;
        }
        {   // stopnet([h | full projection])
            LinArgs a;
            a.W = stop_w; a.bias = stop_b; a.K = D; a.R = 1; a.x = dh_out; a.x_bs = D; a.x2 = p.proj; a.x2_bs = RC;
            a.K2 = RC; a.y = p.logit; a.y_bs = 1; a.done = p.done; a.B = B;
            if ((rc = launch_linear(a, cs, note))) return rc;
        }
        StepArgs s;
        s.proj = p.proj; s.RC = RC; s.logit = p.logit; s.C = C; s.r = r; s.max_steps = max_steps;
        s.dec_out = dec_out; s.stop = stop_tokens; s.mem = p.mem; s.done = p.done; s.ctl = p.ctl; s.B = B;
        taco_step_kernel<<<1, 256, 0, cs>>>(s);
        if (note) dispatch_note(DISPATCH_TACO_STEP);
        B200_CUDA_OK(cudaGetLastError());
        return 0;
    };
    std::vector<int> host;
    if ((rc = run_step_graph("tacotron2_decode_loop", chunk_steps, max_steps, 8, step, p.ctl, B, host, st))) return rc;
    for (int b = 0; b < B; ++b) steps[b] = host[2 + b];
    return 0;
}

int Tacotron2::postnet(const float* dec_out, const int* frames, int B, int F, int Fpitch, float* mel, void* ws,
                       size_t ws_bytes, cudaStream_t st) const {
    B200_REQUIRE(dec_out && frames && mel && ws, "tacotron2_postnet: null pointer");
    B200_REQUIRE(B >= 1 && F >= 1 && F <= Fpitch, "tacotron2_postnet: need B >= 1 and 1 <= F <= Fpitch");
    B200_REQUIRE(ws_bytes >= workspace_bytes(B, 1, F), "tacotron2_postnet: workspace too small");
    const int C = c.out_channels, Tp = (F + 3) / 4 * 4;
    Arena ar(ws, ws_bytes);
    float* x = ar.f32((size_t)B * C * Tp);
    float* y = ar.f32((size_t)B * C * Tp);
    float* h1 = ar.f32((size_t)B * 512 * Tp);
    float* h2 = ar.f32((size_t)B * 512 * Tp);
    float* mask = ar.f32((size_t)B * Tp);
    B200_REQUIRE(x && y && h1 && h2 && mask, "tacotron2_postnet: arena exhausted");
    {
        dim3 grid((Tp + 127) / 128, C, B);
        postnet_in_kernel<<<grid, 128, 0, st>>>(dec_out, Fpitch, frames, x, mask, C, Tp);
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
    }
    int rc;
    const float* in = x;
    // conv (BN folded) -> tanh, the last without it and plus the input.  A tanh layer's output is not masked (that
    // epilogue takes no mask); the next conv masks it as it reads it, and the last one masks its output.
    for (int l = 0; l < 5; ++l) {
        const int ci = l ? 512 : C, co = l == 4 ? C : 512;
        float* out = l == 4 ? y : (l & 1 ? h2 : h1);
        ConvIO io;
        io.x = in; io.x_bs = (long long)ci * Tp; io.x_cs = Tp; io.Tin = Tp;
        io.y = out; io.y_bs = (long long)co * Tp; io.y_cs = Tp; io.Tout = Tp; io.B = B;
        if (l) { io.xmask = mask; io.xmask_bs = Tp; }
        io.act = l == 4 ? ACT_NONE : ACT_TANH;
        if (l == 4) {
            io.res = x; io.res_bs = (long long)C * Tp; io.res_cs = Tp;
            io.ymask = mask; io.ymask_bs = Tp; io.flags = EPI_MASK_POST;
        }
        if ((rc = launch_conv(post[l], io, st))) return rc;
        in = out;
    }
    dim3 grid((F * C + 255) / 256, B);
    postnet_out_kernel<<<grid, 256, 0, st>>>(y, Tp, mel, F, C);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace b200tts
