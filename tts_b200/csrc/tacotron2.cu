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

constexpr int E = 512, HE = 256, Q = 1024, D = 1024, PN = 256;

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

// the loop state plus Tacotron2's own: the prenet outputs and, zeroed, the go frame, both query buffers, the attention
// cell, the context, both decoder buffers and the decoder cell
struct Persist : TacoLoop {
    float *pb, *mem, *q, *qc, *ctx, *dh, *dc;
};

void persist_layout(const Tacotron2& e, Arena& ar, int B, int Tt, Persist& p) {
    const int C = e.c.out_channels;
    taco_loop_layout(ar, B, Tt, C * e.c.r_init, (size_t)B * (C + 2 * Q + Q + E + 2 * D + D), p);
    p.pb = ar.f32((size_t)2 * B * PN);
    p.mem = p.zero;
    p.q = p.mem + (size_t)B * C;
    p.qc = p.q + (size_t)2 * B * Q;
    p.ctx = p.qc + (size_t)B * Q;
    p.dh = p.ctx + (size_t)B * E;
    p.dc = p.dh + (size_t)2 * B * D;
}

// encode: the loop state (kept until the loop ends), the encoder's scratch and the transposed encoder outputs
struct EncodeWs { Persist p; SeqEncoder::Scratch enc; float* encT; };
EncodeWs encode_carve(const Tacotron2& e, Arena& ar, int B, int Tt) {
    EncodeWs w;
    persist_layout(e, ar, B, Tt, w.p);
    w.enc = e.enc.carve(ar, B, Tt);
    w.encT = ar.f32((size_t)B * E * Tt);
    return w;
}

// postnet, from the start of the workspace once the loop is done
struct PostnetWs { float *x, *y, *h1, *h2, *mask; };
PostnetWs postnet_carve(Arena& ar, int B, int C, int Tp) {
    PostnetWs w;
    w.x = ar.f32((size_t)B * C * Tp);
    w.y = ar.f32((size_t)B * C * Tp);
    w.h1 = ar.f32((size_t)B * 512 * Tp);
    w.h2 = ar.f32((size_t)B * 512 * Tp);
    w.mask = ar.f32((size_t)B * Tp);
    return w;
}

}  // namespace

size_t Tacotron2::workspace_bytes(int B, int Tt, int F) const {
    return std::max(arena_size([&](Arena& ar) { encode_carve(*this, ar, B, Tt); }),
                    arena_size([&](Arena& ar) { postnet_carve(ar, B, c.out_channels, (F + 3) / 4 * 4); }));
}

int Tacotron2::init(const b200tts_tacotron2_config& cfg, const float* const* w, int nw) {
    c = cfg;
    const int C = c.out_channels;
    B200_REQUIRE(c.n_vocab > 0 && C > 0 && c.r_init >= 1 && (c.attention_type == 0 || c.attention_type == 1),
                 "tacotron2: unsupported config");
    WeightList wl(w, nw);
    int rc;
    if ((rc = enc.init(c.n_vocab, E, HE, 3, wl))) return rc;
    std::vector<float> wf, bf;
    for (int l = 0; l < 2; ++l) {   // prenet (no bias); "bn": eval BatchNorm folded into the layer
        const int in = l ? PN : C;
        if (!c.prenet_bn) {
            if ((rc = upload(prenet_w[l], wl.take(), (size_t)PN * in))) return rc;
            continue;
        }
        if ((rc = fold_bn(wl, false, 1e-5, PN, in, wf, bf))) return rc;
        if ((rc = upload(prenet_w[l], wf.data(), wf.size()))) return rc;
        if ((rc = upload(prenet_b[l], bf.data(), bf.size()))) return rc;
    }
    auto lstm = [&](DevBuf<float>& wih, DevBuf<float>& whh, DevBuf<float>& bias, int in, int H) -> int {
        int r;
        if ((r = upload(wih, wl.take(), (size_t)4 * H * in))) return r;
        if ((r = upload(whh, wl.take(), (size_t)4 * H * H))) return r;
        const float *b_ih = wl.take(), *b_hh = wl.take();
        B200_REQUIRE(b_ih && b_hh, "tacotron2: null LSTMCell bias");
        std::vector<float> b((size_t)4 * H);
        for (int k = 0; k < 4 * H; ++k) b[k] = b_ih[k] + b_hh[k];
        return upload(bias, b.data(), b.size());
    };
    if ((rc = lstm(arnn_wih, arnn_whh, arnn_b, PN + E, Q))) return rc;
    if ((rc = att.init(Q, E, c.attention_type, c.location_attn, c.attention_norm, wl))) return rc;
    if ((rc = lstm(drnn_wih, drnn_whh, drnn_b, Q + E, D))) return rc;
    if ((rc = upload(proj_w, wl.take(), (size_t)C * c.r_init * (D + E)))) return rc;
    if ((rc = upload(proj_b, wl.take(), (size_t)C * c.r_init))) return rc;
    if ((rc = upload(stop_w, wl.take(), (size_t)D + C * c.r_init))) return rc;
    if ((rc = upload(stop_b, wl.take(), 1))) return rc;
    for (int l = 0; l < 5; ++l) {   // Postnet ConvBNBlocks, BatchNorm folded
        const int ci = l ? 512 : C, co = l == 4 ? C : 512;
        if ((rc = fold_bn(wl, true, 1e-5, co, (size_t)ci * 5, wf, bf))) return rc;
        if ((rc = pack_conv(post[l], wf.data(), bf.data(), co, ci, 5, 1, 2))) return rc;
    }
    return wl.finish("tacotron2");
}

int Tacotron2::encode(const long long* tokens, const long long* lengths, int B, int Tt, float* enc_out, void* ws,
                      size_t ws_bytes, cudaStream_t st) const {
    B200_REQUIRE(tokens && lengths && enc_out && ws, "tacotron2_encode: null pointer");
    B200_REQUIRE(B >= 1 && Tt >= 1, "tacotron2_encode: empty batch");
    const size_t need = workspace_bytes(B, Tt, 0);
    B200_REQUIRE(ws_bytes >= need, "tacotron2_encode: workspace of %zu bytes, %zu needed", ws_bytes, need);
    Arena ar(ws, ws_bytes);
    const EncodeWs w = encode_carve(*this, ar, B, Tt);
    int rc;
    if ((rc = enc.encode(tokens, lengths, B, Tt, enc_out, w.enc, st))) return rc;
    return att.keys(enc_out, w.encT, w.p.pin, B, Tt, st);
}

int Tacotron2::decode_loop(const long long* lengths, const float* enc_out, int B, int Tt, int r, int max_steps,
                           const unsigned char* drop, int chunk_steps, float* dec_out, float* stop_tokens,
                           float* alignments, int* steps, void* ws, size_t ws_bytes, cudaStream_t st) const {
    B200_REQUIRE(lengths && enc_out && dec_out && stop_tokens && alignments && steps && ws,
                 "tacotron2_decode_loop: null pointer");
    B200_REQUIRE(B >= 1 && Tt >= 1 && max_steps >= 1, "tacotron2_decode_loop: B, Tt and max_steps must be >= 1");
    B200_REQUIRE(r >= 1 && r <= c.r_init, "tacotron2_decode_loop: r must be in [1, r_init = %d]", c.r_init);
    B200_REQUIRE(chunk_steps >= 2 && chunk_steps % 2 == 0, "tacotron2_decode_loop: chunk_steps must be even and >= 2");
    const size_t need = workspace_bytes(B, Tt, 0);
    B200_REQUIRE(ws_bytes >= need, "tacotron2_decode_loop: workspace of %zu bytes, %zu needed", ws_bytes, need);
    const int C = c.out_channels, RC = C * c.r_init;
    Arena ar(ws, ws_bytes);
    Persist p;
    persist_layout(*this, ar, B, Tt, p);
    int rc;
    if ((rc = taco_loop_start(p, B, Tt, max_steps, r * C, c.attention_type == 1, dec_out, stop_tokens, alignments, st)))
        return rc;
    const int nb = B > 8 ? 32 : 8;
    const int lstm_id = nb == 32 ? DISPATCH_LSTM_CELL32 : DISPATCH_LSTM_CELL;
    size_t attn_smem = 0;
    if ((rc = att.prepare(Tt, &attn_smem))) return rc;
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
        if ((rc = att.launch(p, q_out, p.ctx, enc_out, alignments, max_steps, lengths, B, Tt, attn_smem, cs, note)))
            return rc;
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
    const size_t need = workspace_bytes(B, 1, F);
    B200_REQUIRE(ws_bytes >= need, "tacotron2_postnet: workspace of %zu bytes, %zu needed", ws_bytes, need);
    const int C = c.out_channels, Tp = (F + 3) / 4 * 4;
    Arena ar(ws, ws_bytes);
    const PostnetWs w = postnet_carve(ar, B, C, Tp);
    float *x = w.x, *y = w.y, *h1 = w.h1, *h2 = w.h2, *mask = w.mask;
    int rc;
    if ((rc = launch_frames_in(dec_out, Fpitch, frames, x, mask, B, C, Tp, st))) return rc;
    const float* in = x;
    // conv (BN folded) -> tanh, the last without it and plus the input.  A tanh layer's output is not masked (that
    // epilogue takes no mask); the next conv masks it as it reads it, and the last one masks its output.
    for (int l = 0; l < 5; ++l) {
        const int ci = l ? 512 : C, co = l == 4 ? C : 512;
        float* out = l == 4 ? y : (l & 1 ? h2 : h1);
        ConvIO io;
        io.x = dense(in, ci, Tp); io.Tin = Tp;
        io.y = dense(out, co, Tp); io.Tout = Tp; io.B = B;
        if (l) io.xmask = {mask, Tp};
        io.act = l == 4 ? ACT_NONE : ACT_TANH;
        if (l == 4) {
            io.res = dense(x, C, Tp);
            io.ymask = {mask, Tp}; io.flags = EPI_MASK_POST;
        }
        if ((rc = launch_conv(post[l], io, st))) return rc;
        in = out;
    }
    return launch_frames_out(y, Tp, mel, B, F, C, st);
}

}  // namespace b200tts
