// Tacotron (1) inference: text -> spectrogram through the GRU attention decoder.
// Reference: TTS/tts/models/tacotron.py:218-271 (inference), TTS/tts/layers/tacotron/tacotron.py (BatchNormConv1d,
//            Highway, CBHG, Encoder, PostCBHG, Decoder), common_layers.py:63-119 (Prenet), attentions.py.
// The decoder loop is exact FP32 on the FMA pipe (the stop decision feeds back through it).  Per step: two prenet GEMVs,
// the attention GRUCell, one attention launch per row, project_to_decoder_in, the two residual GRUCells, proj_to_mel,
// the stopnet and the step epilogue -- 10 launches, captured as CUDA-graph chunks.
#include <math.h>

#include "engines.cuh"

namespace b200tts {

namespace {

constexpr int EMB = 256, E = 256, Q = 256, D = 256, BANK = 128, HW = 128, NHW = 4;
constexpr int PN0 = 256, PN1 = 128;      // decoder and encoder prenet widths
constexpr int HW_TF = 16;                // frames per highway CTA
constexpr int HW_MAX_CIN = 1024;         // widest pre_highway input the highway kernel stages

__device__ __forceinline__ float sigm(float x) { return 1.f / (1.f + expf(-x)); }

// The CBHG's highway stack over a tile of HW_TF frames of row blockIdx.y, held in shared memory for all four layers:
// [pre_highway (x W_pre, no bias)], then per layer x = relu(H x + bH) sig(T x + bT) + x (1 - sig(T x + bT)).
// x [B, Cin, T] channel-major -> y [B, 128, T].  Thread o < 256 computes row o of [H | T] for the tile's frames, summing
// k in order; weights are transposed ([k][o]) so a warp reads consecutive words.
struct HighwayArgs {
    const float* x = nullptr; long long x_bs = 0; int Cin = 0, T = 0;
    const float* pre = nullptr;                // [Cin][128] or null (Cin == 128)
    const float* w = nullptr; const float* bias = nullptr;   // [NHW][128][256], [NHW][256]
    float* y = nullptr; long long y_bs = 0;
};

__global__ void __launch_bounds__(256) highway_kernel(HighwayArgs a) {
    extern __shared__ float sm[];
    float* xs = sm;                      // [128][HW_TF]
    float* hs = xs + HW * HW_TF;         // [256][HW_TF]
    float* xin = hs + 2 * HW * HW_TF;    // [Cin][HW_TF] (pre_highway only)
    const int b = blockIdx.y, t0 = blockIdx.x * HW_TF, tid = threadIdx.x;
    const float* x = a.x + (size_t)b * a.x_bs;
    float* dst = a.pre ? xin : xs;
    for (int i = tid; i < a.Cin * HW_TF; i += blockDim.x) {
        const int k = i / HW_TF, f = i - k * HW_TF, t = t0 + f;
        dst[i] = t < a.T ? x[(size_t)k * a.T + t] : 0.f;
    }
    __syncthreads();
    if (a.pre) {   // xs[j] = sum_k pre[k][j] xin[k]: thread (j, half) for 8 frames
        const int j = tid & (HW - 1), f0 = (tid >> 7) * (HW_TF / 2);
        float acc[HW_TF / 2];
#pragma unroll
        for (int f = 0; f < HW_TF / 2; ++f) acc[f] = 0.f;
        for (int k = 0; k < a.Cin; ++k) {
            const float wv = a.pre[(size_t)k * HW + j];
            const float4* xv = reinterpret_cast<const float4*>(xin + k * HW_TF + f0);
#pragma unroll
            for (int v = 0; v < HW_TF / 8; ++v) {
                const float4 q = xv[v];
                acc[4 * v + 0] = fmaf(wv, q.x, acc[4 * v + 0]);
                acc[4 * v + 1] = fmaf(wv, q.y, acc[4 * v + 1]);
                acc[4 * v + 2] = fmaf(wv, q.z, acc[4 * v + 2]);
                acc[4 * v + 3] = fmaf(wv, q.w, acc[4 * v + 3]);
            }
        }
#pragma unroll
        for (int f = 0; f < HW_TF / 2; ++f) xs[j * HW_TF + f0 + f] = acc[f];
        __syncthreads();
    }
    for (int l = 0; l < NHW; ++l) {
        const float* w = a.w + (size_t)l * HW * 2 * HW;
        float acc[HW_TF];
#pragma unroll
        for (int f = 0; f < HW_TF; ++f) acc[f] = 0.f;
        for (int k = 0; k < HW; ++k) {
            const float wv = w[(size_t)k * 2 * HW + tid];
            const float4* xv = reinterpret_cast<const float4*>(xs + k * HW_TF);
#pragma unroll
            for (int v = 0; v < HW_TF / 4; ++v) {
                const float4 q = xv[v];
                acc[4 * v + 0] = fmaf(wv, q.x, acc[4 * v + 0]);
                acc[4 * v + 1] = fmaf(wv, q.y, acc[4 * v + 1]);
                acc[4 * v + 2] = fmaf(wv, q.z, acc[4 * v + 2]);
                acc[4 * v + 3] = fmaf(wv, q.w, acc[4 * v + 3]);
            }
        }
        const float bo = a.bias[l * 2 * HW + tid];
#pragma unroll
        for (int f = 0; f < HW_TF; ++f) hs[tid * HW_TF + f] = acc[f] + bo;
        __syncthreads();
        for (int i = tid; i < HW * HW_TF; i += blockDim.x) {
            const float h = fmaxf(hs[i], 0.f), g = sigm(hs[HW * HW_TF + i]);
            xs[i] = h * g + xs[i] * (1.f - g);
        }
        __syncthreads();
    }
    float* y = a.y + (size_t)b * a.y_bs;
    for (int i = tid; i < HW * HW_TF; i += blockDim.x) {
        const int j = i / HW_TF, f = i - j * HW_TF, t = t0 + f;
        if (t < a.T) y[(size_t)j * a.T + t] = xs[i];
    }
}

// The step epilogue (Decoder.inference's loop body after decode, tacotron.py:470-482): for each running row b, the
// first r frames of the projection -> dec_out[b, t*r .. t*r + r), the memory queue update (_update_memory_input) from
// mem_in into mem_out, stop[b, t] = sigmoid(logit); with n = t + 1 steps taken, the row is done when n > len_b / 4 and
// (sigmoid > 0.6 or its attention weight at token len_b - 1 > 0.6), or when n > max_decoder_steps (steps[b] = n);
// then ctl = {running, t + 1}.
struct Step1Args {
    const float* proj = nullptr; int RC = 0; const float* logit = nullptr;
    const float* alpha = nullptr; const long long* lens = nullptr; int Tt = 0;
    int C = 0, r = 0, memory_size = 0, Cm = 0, max_decoder_steps = 0, S = 0;
    const float* mem_in = nullptr; float* mem_out = nullptr;
    float* dec_out = nullptr; float* stop = nullptr;
    int* done = nullptr; int* ctl = nullptr; int B = 0;
};

__global__ void __launch_bounds__(256) taco1_step_kernel(Step1Args a) {
    const int t = a.ctl[1], rc = a.r * a.C;
    for (int i = threadIdx.x; i < a.B * rc; i += blockDim.x) {
        const int b = i / rc, k = i - b * rc;
        if (a.done[b]) continue;
        a.dec_out[((size_t)b * a.S * a.r + (size_t)t * a.r) * a.C + k] = a.proj[(size_t)b * a.RC + k];
    }
    for (int i = threadIdx.x; i < a.B * a.Cm; i += blockDim.x) {
        const int b = i / a.Cm, k = i - b * a.Cm;
        if (a.done[b]) continue;
        const float* pj = a.proj + (size_t)b * a.RC;
        float v;
        if (a.memory_size <= 0) v = pj[a.C * (a.r - 1) + k];                      // the last frame
        else if (a.memory_size > a.r) v = k < rc ? pj[k] : a.mem_in[(size_t)b * a.Cm + k - rc];   // queue
        else v = pj[k];                                                             // the first memory_size frames
        a.mem_out[(size_t)b * a.Cm + k] = v;
    }
    __syncthreads();
    for (int b = threadIdx.x; b < a.B; b += blockDim.x) {
        if (a.done[b]) continue;
        const float s = 1.f / (1.f + expf(-a.logit[b]));
        a.stop[(size_t)b * a.S + t] = s;
        const int n = t + 1, len = (int)a.lens[b];
        const bool attn_end = a.alpha[(size_t)b * a.Tt + len - 1] > 0.6f;
        if ((4 * n > len && (s > 0.6f || attn_end)) || n > a.max_decoder_steps) {
            a.done[b] = 1;
            a.ctl[2 + b] = n;
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

// the loop state plus Tacotron's own: the prenet outputs, the decoder input, the residual GRU outputs and, zeroed,
// mem [2][B][Cm], q / dh1 / dh2 [2][B][256] and ctx [B][256]
struct Persist : TacoLoop {
    float *pb, *din, *x1, *x2;
    float *mem, *q, *ctx, *dh1, *dh2;
};

void persist_layout(const Tacotron& e, Arena& ar, int B, int Tt, Persist& p) {
    const size_t nzero = (size_t)B * (2 * e.Cm + 2 * Q + E + 4 * D);
    taco_loop_layout(ar, B, Tt, e.c.frame_channels * e.c.r_init, nzero, p);
    p.pb = ar.f32((size_t)B * (PN0 + PN1));
    p.din = ar.f32((size_t)B * D);
    p.x1 = ar.f32((size_t)B * D);
    p.x2 = ar.f32((size_t)B * D);
    p.mem = p.zero;
    p.q = p.mem + (size_t)2 * B * e.Cm;
    p.ctx = p.q + (size_t)2 * B * Q;
    p.dh1 = p.ctx + (size_t)B * E;
    p.dh2 = p.dh1 + (size_t)2 * B * D;
}

}  // namespace

// ------------------------------------------------------------------ CBHG
int Tacotron::Cbhg::init(int cin, int k_max, int p1, WeightList& wl) {
    Cin = cin; K = k_max; P1 = p1;
    B200_REQUIRE(Cin >= 1 && Cin <= HW_MAX_CIN && K >= 1, "tacotron: unsupported CBHG shape");
    int rc;
    std::vector<float> wf, bf;
    {   // the bank: conv k (taps [-(k-1)/2, k/2]) placed in the union window [-(K-1)/2, K/2] of K taps
        const int padU = (K - 1) / 2;
        std::vector<float> wb((size_t)K * BANK * Cin * K, 0.f), bb((size_t)K * BANK);
        for (int k = 1; k <= K; ++k) {
            if ((rc = fold_bn(wl, false, 1e-3, BANK, (size_t)Cin * k, wf, bf))) return rc;
            const int off = padU - (k - 1) / 2;
            for (int o = 0; o < BANK; ++o) {
                const int row = (k - 1) * BANK + o;
                bb[row] = bf[o];
                for (int ci = 0; ci < Cin; ++ci)
                    for (int j = 0; j < k; ++j)
                        wb[((size_t)row * Cin + ci) * K + off + j] = wf[((size_t)o * Cin + ci) * k + j];
            }
        }
        if ((rc = pack_conv(bank, wb.data(), bb.data(), K * BANK, Cin, K, 1, padU))) return rc;
    }
    if ((rc = fold_bn(wl, false, 1e-3, P1, (size_t)K * BANK * 3, wf, bf))) return rc;
    if ((rc = pack_conv(proj1, wf.data(), bf.data(), P1, K * BANK, 3, 1, 1))) return rc;
    if ((rc = fold_bn(wl, false, 1e-3, Cin, (size_t)P1 * 3, wf, bf))) return rc;
    if ((rc = pack_conv(proj2, wf.data(), bf.data(), Cin, P1, 3, 1, 1))) return rc;
    if (Cin != HW) {   // pre_highway [128][Cin] -> [Cin][128]
        const float* pre = wl.take();
        B200_REQUIRE(pre, "tacotron: null pre_highway weight");
        std::vector<float> pt((size_t)Cin * HW);
        for (int o = 0; o < HW; ++o)
            for (int k = 0; k < Cin; ++k) pt[(size_t)k * HW + o] = pre[(size_t)o * Cin + k];
        if ((rc = upload(pre_w, pt.data(), pt.size()))) return rc;
    }
    {   // highways: [H | T] rows transposed to [k][256]
        std::vector<float> hw((size_t)NHW * HW * 2 * HW), hb((size_t)NHW * 2 * HW);
        for (int l = 0; l < NHW; ++l) {
            const float *hw_H = wl.take(), *hb_H = wl.take(), *hw_T = wl.take(), *hb_T = wl.take();
            B200_REQUIRE(hw_H && hb_H && hw_T && hb_T, "tacotron: null highway weight or bias");
            for (int o = 0; o < 2 * HW; ++o) {
                const float* W = o < HW ? hw_H : hw_T;
                const float* bsrc = o < HW ? hb_H : hb_T;
                const int oo = o % HW;
                hb[(size_t)l * 2 * HW + o] = bsrc[oo];
                for (int k = 0; k < HW; ++k) hw[((size_t)l * HW + k) * 2 * HW + o] = W[(size_t)oo * HW + k];
            }
        }
        if ((rc = upload(hw_w, hw.data(), hw.size()))) return rc;
        if ((rc = upload(hw_b, hb.data(), hb.size()))) return rc;
    }
    {   // GRU: both directions' input projections as one 1x1 conv (rows [fwd 3H | bwd 3H]), bias b_ih + (b_hr, b_hz, 0)
        constexpr int H = GRU_H;
        std::vector<float> wi((size_t)6 * H * HW), bi((size_t)6 * H), img((size_t)2 * 3 * 32 * BIGRU_THREADS), bn(2 * H);
        for (int d = 0; d < 2; ++d) {
            const float *w_ih = wl.take(), *w_hh = wl.take(), *b_ih = wl.take(), *b_hh = wl.take();
            B200_REQUIRE(w_ih && b_ih && b_hh, "tacotron: null GRU weight or bias");
            memcpy(wi.data() + (size_t)d * 3 * H * HW, w_ih, sizeof(float) * 3 * H * HW);
            for (int r = 0; r < 3 * H; ++r) bi[(size_t)d * 3 * H + r] = b_ih[r] + (r < 2 * H ? b_hh[r] : 0.f);
            for (int j = 0; j < H; ++j) bn[d * H + j] = b_hh[2 * H + j];
            if ((rc = pack_bigru_whh(w_hh, img.data() + (size_t)d * 3 * 32 * BIGRU_THREADS))) return rc;
        }
        if ((rc = pack_conv(gru_in, wi.data(), bi.data(), 6 * H, HW, 1, 1, 0))) return rc;
        if ((rc = upload(whh, img.data(), img.size()))) return rc;
        if ((rc = upload(bhn, bn.data(), bn.size()))) return rc;
    }
    return 0;
}

Tacotron::Cbhg::Scratch Tacotron::Cbhg::carve(Arena& ar, int B, int T) const {
    Scratch s;
    s.bank = ar.f32((size_t)B * K * BANK * T);
    s.y2 = ar.f32((size_t)B * P1 * T);
    s.y3 = ar.f32((size_t)B * Cin * T);
    s.hx = ar.f32((size_t)B * HW * T);
    s.pre = ar.f32((size_t)B * 6 * GRU_H * T);
    return s;
}

int Tacotron::Cbhg::run(const float* x, const float* mask, const int* lens32, const long long* lens64, int B, int T,
                        float* out, long long out_bs, int out_ts, int out_cs, const Scratch& s, cudaStream_t st) const {
    float *bk = s.bank, *y2 = s.y2, *y3 = s.y3, *hx = s.hx, *pre = s.pre;
    int rc;
    auto conv = [&](const ConvLayer& L, const float* in, int ci, float* o, int co, int act, const float* res) {
        ConvIO io;
        io.x = dense(in, ci, T); io.Tin = T;
        io.y = dense(o, co, T); io.Tout = T; io.B = B;
        io.act = act; io.ymask = {mask, T}; io.flags = EPI_MASK_POST;
        if (res) io.res = dense(res, co, T);
        return launch_conv(L, io, st);
    };
    if ((rc = conv(bank, x, Cin, bk, K * BANK, ACT_RELU, nullptr))) return rc;
    if ((rc = conv(proj1, bk, K * BANK, y2, P1, ACT_RELU, nullptr))) return rc;
    if ((rc = conv(proj2, y2, P1, y3, Cin, ACT_NONE, x))) return rc;   // x += inputs
    {
        HighwayArgs a;
        a.x = y3; a.x_bs = (long long)Cin * T; a.Cin = Cin; a.T = T; a.pre = pre_w; a.w = hw_w; a.bias = hw_b;
        a.y = hx; a.y_bs = (long long)HW * T;
        const size_t smem = sizeof(float) * HW_TF * (3 * HW + (Cin != HW ? Cin : 0));
        static DeviceOnce once;
        if ((rc = device_once(once, nullptr, [](int) -> int {
                 B200_CUDA_OK(cudaFuncSetAttribute(highway_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                   (int)(sizeof(float) * HW_TF * (3 * HW + HW_MAX_CIN))));
                 return 0;
             })))
            return rc;
        highway_kernel<<<dim3((T + HW_TF - 1) / HW_TF, B), 256, smem, st>>>(a);
        count_launch();
        dispatch_note(DISPATCH_HIGHWAY);
        B200_CUDA_OK(cudaGetLastError());
    }
    {
        ConvIO io;
        io.x = dense(hx, HW, T); io.Tin = T;
        io.y = dense(pre, 6 * GRU_H, T); io.Tout = T; io.B = B;
        if ((rc = launch_conv(gru_in, io, st))) return rc;
    }
    BiGruArgs g;
    g.pre = pre; g.pre_bs = (long long)6 * GRU_H * T; g.pre_cs = T; g.whh = whh; g.bhn = bhn;
    g.out = out; g.out_bs = out_bs; g.out_ts = out_ts; g.out_cs = out_cs; g.lens32 = lens32; g.lens64 = lens64; g.T = T;
    return launch_bigru(g, B, st);
}

// ------------------------------------------------------------------ the model
int Tacotron::init(const b200tts_tacotron_config& cfg, const float* const* w, int nw) {
    c = cfg;
    const int C = c.frame_channels, RC = C * c.r_init;
    B200_REQUIRE(c.n_vocab > 0 && C > 0 && C <= HW_MAX_CIN && c.out_channels > 0 && c.r_init >= 1 &&
                 (c.attention_type == 0 || c.attention_type == 1), "tacotron: unsupported config");
    Cm = c.memory_size > 0 ? C * c.memory_size : C;
    WeightList wl(w, nw);
    int rc;
    if ((rc = upload(emb, wl.take(), (size_t)c.n_vocab * EMB))) return rc;
    const float *p0w = wl.take(), *p0b = wl.take(), *p1w = wl.take(), *p1b = wl.take();
    if ((rc = pack_conv(eprenet[0], p0w, p0b, PN0, EMB, 1, 1, 0))) return rc;
    if ((rc = pack_conv(eprenet[1], p1w, p1b, PN1, PN0, 1, 1, 0))) return rc;
    if ((rc = ecbhg.init(PN1, 16, 128, wl))) return rc;
    std::vector<float> wf, bf;
    for (int l = 0; l < 2; ++l) {   // decoder prenet (with bias); "bn": eval BatchNorm (eps 1e-5) folded into the layer
        const int in = l ? PN0 : Cm, out = l ? PN1 : PN0;
        if (!c.prenet_bn) {
            if ((rc = upload(prenet_w[l], wl.take(), (size_t)out * in))) return rc;
            if ((rc = upload(prenet_b[l], wl.take(), out))) return rc;
            continue;
        }
        if ((rc = fold_bn(wl, true, 1e-5, out, in, wf, bf))) return rc;
        if ((rc = upload(prenet_w[l], wf.data(), wf.size()))) return rc;
        if ((rc = upload(prenet_b[l], bf.data(), bf.size()))) return rc;
    }
    // a GRUCell: W_ih, W_hh, bias [4][H] = (b_ir + b_hr, b_iz + b_hz, b_in, b_hn)
    auto gru = [&](DevBuf<float>& wih, DevBuf<float>& whh_, DevBuf<float>& bias, int in, int H) -> int {
        int r;
        if ((r = upload(wih, wl.take(), (size_t)3 * H * in))) return r;
        if ((r = upload(whh_, wl.take(), (size_t)3 * H * H))) return r;
        const float *b_ih = wl.take(), *b_hh = wl.take();
        B200_REQUIRE(b_ih && b_hh, "tacotron: null GRUCell bias");
        std::vector<float> b((size_t)4 * H);
        for (int k = 0; k < 2 * H; ++k) b[k] = b_ih[k] + b_hh[k];
        for (int k = 0; k < H; ++k) { b[2 * H + k] = b_ih[2 * H + k]; b[3 * H + k] = b_hh[2 * H + k]; }
        return upload(bias, b.data(), b.size());
    };
    if ((rc = gru(arnn_wih, arnn_whh, arnn_b, PN1 + E, Q))) return rc;
    if ((rc = att.init(Q, E, c.attention_type, c.location_attn, c.attention_norm, wl))) return rc;
    if ((rc = upload(pdi_w, wl.take(), (size_t)D * (Q + E)))) return rc;
    if ((rc = upload(pdi_b, wl.take(), D))) return rc;
    for (int l = 0; l < 2; ++l)
        if ((rc = gru(drnn_wih[l], drnn_whh[l], drnn_b[l], D, D))) return rc;
    if ((rc = upload(proj_w, wl.take(), (size_t)RC * D))) return rc;
    if ((rc = upload(proj_b, wl.take(), RC))) return rc;
    if ((rc = upload(stop_w, wl.take(), (size_t)D + RC))) return rc;
    if ((rc = upload(stop_b, wl.take(), 1))) return rc;
    if ((rc = pcbhg.init(C, 8, 256, wl))) return rc;
    const float *lw = wl.take(), *lb = wl.take();
    if ((rc = pack_conv(last, lw, lb, c.out_channels, 2 * GRU_H, 1, 1, 0))) return rc;
    return wl.finish("tacotron");
}

// encode: the loop state (kept until the loop ends), the embedding and its mask, the prenet outputs, the transposed
// encoder outputs and the encoder CBHG's scratch
struct EncodeWs { Persist p; float *x0, *mask, *x1, *xin, *encT; Tacotron::Cbhg::Scratch cbhg; };
static EncodeWs encode_carve(const Tacotron& e, Arena& ar, int B, int Tt) {
    EncodeWs w;
    persist_layout(e, ar, B, Tt, w.p);
    w.x0 = ar.f32((size_t)B * EMB * Tt);
    w.mask = ar.f32((size_t)B * Tt);
    w.x1 = ar.f32((size_t)B * PN0 * Tt);
    w.xin = ar.f32((size_t)B * PN1 * Tt);
    w.encT = ar.f32((size_t)B * E * Tt);
    w.cbhg = e.ecbhg.carve(ar, B, Tt);
    return w;
}

// postnet, from the start of the workspace once the loop is done: its input and mask, the CBHG output and scratch
struct PostnetWs { float *x, *mask, *g, *y; Tacotron::Cbhg::Scratch cbhg; };
static PostnetWs postnet_carve(const Tacotron& e, Arena& ar, int B, int Tp) {
    PostnetWs w;
    w.x = ar.f32((size_t)B * e.c.frame_channels * Tp);
    w.mask = ar.f32((size_t)B * Tp);
    w.g = ar.f32((size_t)B * 2 * GRU_H * Tp);
    w.y = ar.f32((size_t)B * e.c.out_channels * Tp);
    w.cbhg = e.pcbhg.carve(ar, B, Tp);
    return w;
}

size_t Tacotron::workspace_bytes(int B, int Tt, int F) const {
    return std::max(arena_size([&](Arena& ar) { encode_carve(*this, ar, B, Tt); }),
                    arena_size([&](Arena& ar) { postnet_carve(*this, ar, B, (F + 3) / 4 * 4); }));
}

int Tacotron::encode(const long long* tokens, const long long* lengths, int B, int Tt, float* enc_out, void* ws,
                     size_t ws_bytes, cudaStream_t st) const {
    B200_REQUIRE(tokens && lengths && enc_out && ws, "tacotron_encode: null pointer");
    B200_REQUIRE(B >= 1 && Tt >= 1, "tacotron_encode: empty batch");
    const size_t need = workspace_bytes(B, Tt, 0);
    B200_REQUIRE(ws_bytes >= need, "tacotron_encode: workspace of %zu bytes, %zu needed", ws_bytes, need);
    Arena ar(ws, ws_bytes);
    const EncodeWs w = encode_carve(*this, ar, B, Tt);
    float *x0 = w.x0, *mask = w.mask, *x1 = w.x1, *xin = w.xin;
    int rc;
    // emb(x), zero past each row's length (the reference runs each row at its own length)
    if ((rc = launch_embed(tokens, lengths, emb, nullptr, B, Tt, EMB, EMB, x0, mask, st, false))) return rc;
    const float* in = x0;
    for (int l = 0; l < 2; ++l) {   // encoder prenet: Linear -> ReLU (eval: no dropout), masked
        const int ci = l ? PN0 : EMB, co = l ? PN1 : PN0;
        float* o = l ? xin : x1;
        ConvIO io;
        io.x = dense(in, ci, Tt); io.Tin = Tt;
        io.y = dense(o, co, Tt); io.Tout = Tt; io.B = B;
        io.act = ACT_RELU; io.ymask = {mask, Tt}; io.flags = EPI_MASK_POST;
        if ((rc = launch_conv(eprenet[l], io, st))) return rc;
        in = o;
    }
    if ((rc = ecbhg.run(xin, mask, nullptr, lengths, B, Tt, enc_out, (long long)Tt * E, E, 1, w.cbhg, st))) return rc;
    return att.keys(enc_out, w.encT, w.p.pin, B, Tt, st);
}

int Tacotron::decode_loop(const long long* lengths, const float* enc_out, int B, int Tt, int r, int max_steps,
                          const unsigned char* drop, int chunk_steps, float* dec_out, float* stop_tokens,
                          float* alignments, int* steps, void* ws, size_t ws_bytes, cudaStream_t st) const {
    B200_REQUIRE(lengths && enc_out && dec_out && stop_tokens && alignments && steps && ws,
                 "tacotron_decode_loop: null pointer");
    B200_REQUIRE(B >= 1 && Tt >= 1 && max_steps >= 1, "tacotron_decode_loop: B, Tt and max_steps must be >= 1");
    B200_REQUIRE(r >= 1 && r <= c.r_init, "tacotron_decode_loop: r must be in [1, r_init = %d]", c.r_init);
    B200_REQUIRE(chunk_steps >= 2 && chunk_steps % 2 == 0, "tacotron_decode_loop: chunk_steps must be even and >= 2");
    const size_t need = workspace_bytes(B, Tt, 0);
    B200_REQUIRE(ws_bytes >= need, "tacotron_decode_loop: workspace of %zu bytes, %zu needed", ws_bytes, need);
    const int C = c.frame_channels, RC = C * c.r_init, S = max_steps + 1;   // a row emits at most max_steps + 1 steps
    Arena ar(ws, ws_bytes);
    Persist p;
    persist_layout(*this, ar, B, Tt, p);
    int rc;
    if ((rc = taco_loop_start(p, B, Tt, S, r * C, c.attention_type == 1, dec_out, stop_tokens, alignments, st)))
        return rc;
    size_t attn_smem = 0;
    if ((rc = att.prepare(Tt, &attn_smem))) return rc;
    const int nb = B > 8 ? 32 : 8;
    // one step; parity = step index within the chunk (memory, query and both decoder h are double-buffered)
    auto step = [&](cudaStream_t cs, int par, bool note) -> int {
        int rc;
        const float* mem_in = p.mem + (size_t)par * B * Cm;
        float* mem_out = p.mem + (size_t)(par ^ 1) * B * Cm;
        float* pb0 = p.pb;
        float* pb1 = p.pb + (size_t)B * PN0;
        for (int l = 0; l < 2; ++l) {   // prenet: Linear -> ReLU -> dropout; drop is [B, S, 2, 256], layer 1 uses 128
            LinArgs a;
            a.W = prenet_w[l]; a.bias = prenet_b[l]; a.K = l ? PN0 : Cm; a.R = l ? PN1 : PN0;
            a.x = l ? pb0 : mem_in; a.x_bs = a.K; a.y = l ? pb1 : pb0; a.y_bs = a.R; a.relu = 1;
            a.drop = c.prenet_dropout ? drop : nullptr; a.drop_layer = l ? 2 : 0; a.drop_L = l ? 4 : 2; a.drop_F = S;
            a.ctl = p.ctl; a.done = p.done; a.B = B;
            if ((rc = launch_linear(a, cs, note))) return rc;
        }
        float* q_in = p.q + (size_t)par * B * Q;
        float* q_out = p.q + (size_t)(par ^ 1) * B * Q;
        {   // attention RNN on [prenet | context], h
            GruArgs a;
            a.seg[0] = {arnn_wih, PN1 + E, 0, pb1, PN1, 0, PN1};
            a.seg[1] = {arnn_wih + PN1, PN1 + E, 0, p.ctx, E, 0, E};
            a.seg[2] = {arnn_whh, Q, 0, q_in, Q, 0, Q};
            a.nseg = 3; a.nin = 2;
            a.H = Q; a.bias = arnn_b; a.h_in = q_in; a.hin_bs = Q; a.h_out = q_out; a.h_bs = Q; a.done = p.done; a.B = B;
            if ((rc = launch_gru(a, nb, cs, note))) return rc;
        }
        if ((rc = att.launch(p, q_out, p.ctx, enc_out, alignments, S, lengths, B, Tt, attn_smem, cs, note))) return rc;
        {   // project_to_decoder_in([query | context])
            LinArgs a;
            a.W = pdi_w; a.bias = pdi_b; a.K = Q; a.R = D; a.x = q_out; a.x_bs = Q; a.x2 = p.ctx; a.x2_bs = E; a.K2 = E;
            a.y = p.din; a.y_bs = D; a.done = p.done; a.B = B;
            if ((rc = launch_linear(a, cs, note))) return rc;
        }
        const float* xin = p.din;
        float* xo[2] = {p.x1, p.x2};
        float* dh[2] = {p.dh1, p.dh2};
        for (int l = 0; l < 2; ++l) {   // decoder RNN l, then the residual x = h + x
            GruArgs a;
            a.seg[0] = {drnn_wih[l], D, 0, xin, D, 0, D};
            a.seg[1] = {drnn_whh[l], D, 0, dh[l] + (size_t)par * B * D, D, 0, D};
            a.nseg = 2; a.nin = 1;
            a.H = D; a.bias = drnn_b[l]; a.h_in = a.seg[1].x; a.hin_bs = D;
            a.h_out = dh[l] + (size_t)(par ^ 1) * B * D; a.h_bs = D;
            a.res = xin; a.res_bs = D; a.x_out = xo[l]; a.xo_bs = D; a.done = p.done; a.B = B;
            if ((rc = launch_gru(a, nb, cs, note))) return rc;
            xin = xo[l];
        }
        {   // proj_to_mel, all C * r_init rows
            LinArgs a;
            a.W = proj_w; a.bias = proj_b; a.K = D; a.R = RC; a.x = p.x2; a.x_bs = D; a.y = p.proj; a.y_bs = RC;
            a.done = p.done; a.B = B;
            if ((rc = launch_linear(a, cs, note))) return rc;
        }
        {   // stopnet([decoder output | full projection])
            LinArgs a;
            a.W = stop_w; a.bias = stop_b; a.K = D; a.R = 1; a.x = p.x2; a.x_bs = D; a.x2 = p.proj; a.x2_bs = RC;
            a.K2 = RC; a.y = p.logit; a.y_bs = 1; a.done = p.done; a.B = B;
            if ((rc = launch_linear(a, cs, note))) return rc;
        }
        Step1Args s;
        s.proj = p.proj; s.RC = RC; s.logit = p.logit; s.alpha = p.alpha; s.lens = lengths; s.Tt = Tt;
        s.C = C; s.r = r; s.memory_size = c.memory_size; s.Cm = Cm; s.max_decoder_steps = max_steps; s.S = S;
        s.mem_in = mem_in; s.mem_out = mem_out; s.dec_out = dec_out; s.stop = stop_tokens;
        s.done = p.done; s.ctl = p.ctl; s.B = B;
        taco1_step_kernel<<<1, 256, 0, cs>>>(s);
        if (note) dispatch_note(DISPATCH_TACO1_STEP);
        B200_CUDA_OK(cudaGetLastError());
        return 0;
    };
    std::vector<int> host;
    if ((rc = run_step_graph("tacotron_decode_loop", chunk_steps, S, 10, step, p.ctl, B, host, st))) return rc;
    for (int b = 0; b < B; ++b) steps[b] = host[2 + b];
    return 0;
}

int Tacotron::postnet(const float* dec_out, const int* frames, int B, int F, int Fpitch, float* out, void* ws,
                      size_t ws_bytes, cudaStream_t st) const {
    B200_REQUIRE(dec_out && frames && out && ws, "tacotron_postnet: null pointer");
    B200_REQUIRE(B >= 1 && F >= 1 && F <= Fpitch, "tacotron_postnet: need B >= 1 and 1 <= F <= Fpitch");
    const size_t need = workspace_bytes(B, 1, F);
    B200_REQUIRE(ws_bytes >= need, "tacotron_postnet: workspace of %zu bytes, %zu needed", ws_bytes, need);
    const int C = c.frame_channels, O = c.out_channels, Tp = (F + 3) / 4 * 4;
    Arena ar(ws, ws_bytes);
    const PostnetWs w = postnet_carve(*this, ar, B, Tp);
    float *x = w.x, *mask = w.mask, *g = w.g, *y = w.y;
    int rc;
    if ((rc = launch_frames_in(dec_out, Fpitch, frames, x, mask, B, C, Tp, st))) return rc;
    // the biGRU writes channel-major [B, 256, Tp] for last_linear on the conv engine
    if ((rc = pcbhg.run(x, mask, frames, nullptr, B, Tp, g, (long long)2 * GRU_H * Tp, 1, Tp, w.cbhg, st))) return rc;
    {
        ConvIO io;
        io.x = dense(g, 2 * GRU_H, Tp); io.Tin = Tp;
        io.y = dense(y, O, Tp); io.Tout = Tp; io.B = B;
        io.ymask = {mask, Tp}; io.flags = EPI_MASK_POST;
        if ((rc = launch_conv(last, io, st))) return rc;
    }
    return launch_frames_out(y, Tp, out, B, F, O, st);
}

}  // namespace b200tts
