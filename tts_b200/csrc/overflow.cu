// Overflow / Neural-HMM inference: text -> mel spectrogram through an autoregressive neural HMM.
// Reference: TTS/tts/models/overflow.py:207-246 (inference), neuralhmm_tts.py (inference, no decoder),
//            TTS/tts/layers/overflow/common_layers.py:12-92 (Encoder), :95-219 (ParameterModel, Outputnet),
//            neural_hmm.py:338-464 (inference, sample), :519-528 (EmissionModel.sample), decoder.py:56-78 (Decoder),
//            TTS/tts/layers/tacotron/common_layers.py:63-120 (Prenet), tacotron2.py:11-44 (ConvBNBlock).
// Everything before the Glow decoder is exact FP32 on the FMA pipe: the state transitions are thresholds on a running
// product that feed back through the loop, so they must not depend on tensor-core rounding.  The loop is GEMV work over
// at most a few dozen rows; its weights (about 6.5 M floats at the defaults) fit in L2.
#include <math.h>

#include "engines.cuh"

namespace b200tts {

namespace {

// The frame epilogue (neural_hmm.py:424-457), one block: for each running row b
//   mean = o[0:C], std = max(softplus(o[C:2C]), floor), x = temp > 0 ? mean + (std * temp) * noise[b, f] : mean
//   hmm_out[b, f] = x; prenet window <- (window[1:], x)
//   quantile *= sigmoid(-o[2C]); quantile < threshold: state += 1, quantile = 1; states_travelled[b, f + 1] = state
//   done when state == len_b * spp or f == max_frames - 1 (frames[b] = f + 1)
// then ctl = {rows still running, f + 1}.
struct StepArgs {
    const float* o = nullptr; int C = 0, ar = 0;
    const float* noise = nullptr; float temp = 0.f, floor_ = 0.f, thr = 0.f; int max_frames = 0;
    float* hmm_out = nullptr; float* pin = nullptr; int* st_tr = nullptr;
    int* state = nullptr; float* quant = nullptr; int* done = nullptr; int* ctl = nullptr;
    const long long* lens = nullptr; int spp = 1; int B = 0;
};

__global__ void __launch_bounds__(256) hmm_step_kernel(StepArgs a) {
    const int f = a.ctl[1], C = a.C, O = 2 * C + 1;
    for (int i = threadIdx.x; i < a.B * C; i += blockDim.x) {
        const int b = i / C, c = i - b * C;
        if (a.done[b]) continue;
        const float* o = a.o + (size_t)b * O;
        const float mean = o[c], sr = o[C + c];
        const float sp = sr > 20.f ? sr : log1pf(expf(sr));
        const float sd = fmaxf(sp, a.floor_);
        float x = mean;
        if (a.temp > 0.f) x = __fadd_rn(mean, __fmul_rn(__fmul_rn(sd, a.temp), a.noise[((size_t)b * a.max_frames + f) * C + c]));
        a.hmm_out[((size_t)b * a.max_frames + f) * C + c] = x;
        float* p = a.pin + (size_t)b * a.ar * C + c;
        for (int k = 0; k + 1 < a.ar; ++k) p[k * C] = p[(k + 1) * C];
        p[(a.ar - 1) * C] = x;
    }
    __syncthreads();
    for (int b = threadIdx.x; b < a.B; b += blockDim.x) {
        if (a.done[b]) continue;
        const float stay = 1.f / (1.f + expf(a.o[(size_t)b * O + 2 * C]));   // sigmoid(-v)
        float q = __fmul_rn(a.quant[b], stay);
        int s = a.state[b];
        if (q < a.thr) { s += 1; q = 1.f; }
        a.quant[b] = q;
        a.state[b] = s;
        a.st_tr[(size_t)b * (a.max_frames + 1) + f + 1] = s;
        if (s == (int)a.lens[b] * a.spp || f == a.max_frames - 1) {
            a.done[b] = 1;
            a.ctl[2 + b] = f + 1;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int run = 0;
        for (int b = 0; b < a.B; ++b) run += a.done[b] ? 0 : 1;
        a.ctl[0] = run;
        a.ctl[1] = f + 1;
    }
}

// loop state at frame 0: h = c = 0, the go-token window, state 0, quantile 1, states_travelled = {0, -1, ...}
__global__ void hmm_reset_kernel(float* hm, float* cm, int M, float* pin, const float* go, int ar, int C, int* state,
                                 float* quant, int* done, int* ctl, int* st_tr, int max_frames, int B) {
    const int b = blockIdx.x;
    for (int i = threadIdx.x; i < M; i += blockDim.x) hm[(size_t)b * M + i] = cm[(size_t)b * M + i] = 0.f;
    for (int i = threadIdx.x; i < ar * C; i += blockDim.x) pin[(size_t)b * ar * C + i] = go[i / C];
    for (int i = threadIdx.x; i <= max_frames; i += blockDim.x) st_tr[(size_t)b * (max_frames + 1) + i] = i ? -1 : 0;
    if (threadIdx.x == 0) {
        state[b] = 0; quant[b] = 1.f; done[b] = 0; ctl[2 + b] = 0;
        if (b == 0) { ctl[0] = B; ctl[1] = 0; }
    }
}

// Decoder.preprocess + the Glow squeeze (overflow/decoder.py:73-78, glow_tts/decoder.py:8-28) of the time-major HMM
// output: zs[b, k*C + c, q] = x[b, q*nsq + k, c] for q < frames[b] / nsq, else 0; msk[b, q] likewise
__global__ void squeeze_hmm_kernel(const float* x, int Fpitch, const int* frames, float* zs, float* msk, int C, int nsq,
                                   int Tq) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x, ck = blockIdx.y, b = blockIdx.z;
    if (q >= Tq) return;
    const int k = ck / C, c = ck - k * C;
    const bool valid = q < frames[b] / nsq;
    zs[((size_t)b * C * nsq + ck) * Tq + q] = valid ? x[((size_t)b * Fpitch + (size_t)q * nsq + k) * C + c] : 0.f;
    if (ck == 0) msk[(size_t)b * Tq + q] = valid ? 1.f : 0.f;
}

// inverse_normalize (overflow.py:129-130): y[b, t, c] = x * std[c] + mean[c], x channel-major (x_ts = 1, x_cs = pitch)
// or time-major (x_ts = C, x_cs = 1)
__global__ void denorm_kernel(const float* x, long long x_bs, int x_ts, int x_cs, const float* mean, const float* sd,
                              float* y, int T, int C) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (i >= T * C) return;
    const int t = i / C, c = i - t * C;
    y[(size_t)b * T * C + i] = __fadd_rn(__fmul_rn(x[b * x_bs + (size_t)t * x_ts + (size_t)c * x_cs], sd[c]), mean[c]);
}

struct Persist {   // the part of the workspace that lives from encode to sample
    float *zc, *quant, *hm, *cm, *pin, *pb, *hid, *outp;
    int *ctl, *state, *done;
};

}  // namespace

static void persist_layout(const Overflow& e, Arena& ar, int B, int Tt, Persist& p) {
    const auto& c = e.c;
    int omax = 0;
    for (int l = 0; l < c.outputnet_n_layers; ++l) omax = std::max(omax, c.outputnet_size[l]);
    const int N = Tt * c.state_per_phone, M = c.memory_rnn_dim;
    p.zc = ar.f32((size_t)B * e.O1 * N);
    p.ctl = (int*)ar.f32(2 + B);
    p.state = (int*)ar.f32(B);
    p.done = (int*)ar.f32(B);
    p.quant = ar.f32(B);
    p.hm = ar.f32((size_t)2 * B * M);
    p.cm = ar.f32((size_t)B * M);
    p.pin = ar.f32((size_t)B * c.ar_order * c.out_channels);
    p.pb = ar.f32((size_t)2 * B * c.prenet_dim);
    p.hid = ar.f32((size_t)2 * B * omax);
    p.outp = ar.f32((size_t)B * (2 * c.out_channels + 1));
}

// encode: the state kept until sample() ends, the encoder's scratch and the transposed encoder states
struct EncodeWs { Persist p; SeqEncoder::Scratch enc; float* encT; };
static EncodeWs encode_carve(const Overflow& e, Arena& ar, int B, int Tt) {
    EncodeWs w;
    persist_layout(e, ar, B, Tt, w.p);
    w.enc = e.enc.carve(ar, B, Tt);
    w.encT = ar.f32((size_t)B * e.c.encoder_dim * Tt * e.c.state_per_phone);
    return w;
}

// decode (Overflow only), from the start of the workspace once sampling is done: the squeezed latent, its mask, the
// decoder's mel and the Glow decoder's block
struct DecodeWs { float *za, *msk, *melc; void* dec; size_t dec_bytes; };
static DecodeWs decode_carve(const Overflow& e, Arena& ar, int B, int Tq) {
    const int C = e.c.out_channels, nsq = e.c.num_squeeze;
    DecodeWs w;
    w.za = ar.f32((size_t)B * C * nsq * Tq);
    w.msk = ar.f32((size_t)B * Tq);
    w.melc = ar.f32((size_t)B * C * Tq * nsq);
    w.dec_bytes = e.dec.workspace_bytes(B, Tq);
    w.dec = ar.bytes(w.dec_bytes);
    return w;
}

int Overflow::init(const b200tts_overflow_config& cfg, const float* const* w, int nw) {
    c = cfg;
    const int E = c.encoder_dim, C = c.out_channels, P = c.prenet_dim, M = c.memory_rnn_dim, nL = c.outputnet_n_layers;
    B200_REQUIRE(c.n_vocab > 0 && E > 0 && E % 2 == 0 && c.n_convs >= 1 && c.n_convs <= 8 && c.state_per_phone >= 1 &&
                     C > 0 && c.ar_order >= 1 && P > 0 && c.prenet_n_layers >= 1 && c.prenet_n_layers <= 8 && M > 0 &&
                     nL >= 1 && nL <= 8,
                 "overflow: unsupported config");
    H = E / 2 * c.state_per_phone;
    O1 = c.outputnet_size[0];
    for (int l = 0; l < nL; ++l)
        B200_REQUIRE(c.outputnet_size[l] > 0, "overflow: outputnet_size[%d] = %d", l, c.outputnet_size[l]);
    WeightList wl(w, nw);
    int rc;
    if ((rc = enc.init(c.n_vocab, E, H, c.n_convs, wl))) return rc;
    if ((rc = upload(go, wl.take(), (size_t)c.ar_order))) return rc;
    prenet_w.resize(c.prenet_n_layers);
    for (int l = 0; l < c.prenet_n_layers; ++l)
        if ((rc = upload(prenet_w[l], wl.take(), (size_t)P * (l ? P : c.ar_order * C)))) return rc;
    if ((rc = upload(mem_wih, wl.take(), (size_t)4 * M * P))) return rc;
    if ((rc = upload(mem_whh, wl.take(), (size_t)4 * M * M))) return rc;
    {
        const float *b_ih = wl.take(), *b_hh = wl.take();
        B200_REQUIRE(b_ih && b_hh, "overflow: null memory LSTM bias");
        std::vector<float> b((size_t)4 * M);
        for (int r = 0; r < 4 * M; ++r) b[r] = b_ih[r] + b_hh[r];
        if ((rc = upload(mem_b, b.data(), b.size()))) return rc;
    }
    out_w.resize(nL + 1);
    out_b.resize(nL + 1);
    for (int l = 0; l <= nL; ++l) {
        const int rows = l < nL ? c.outputnet_size[l] : 2 * C + 1;
        const int in = l == 0 ? M + E : c.outputnet_size[l - 1];
        const float *ow = wl.take(), *ob = wl.take();
        if (l == 0) {   // cat(h, z): the h columns per frame, the z columns hoisted into zproj (with the bias)
            B200_REQUIRE(ow, "overflow: null output net weight");
            std::vector<float> wh((size_t)rows * M), wz((size_t)rows * E);
            for (int r = 0; r < rows; ++r) {
                memcpy(wh.data() + (size_t)r * M, ow + (size_t)r * in, sizeof(float) * M);
                memcpy(wz.data() + (size_t)r * E, ow + (size_t)r * in + M, sizeof(float) * E);
            }
            if ((rc = upload(out_w[l], wh.data(), wh.size()))) return rc;
            if ((rc = pack_conv(zproj, wz.data(), ob, rows, E, 1, 1, 0))) return rc;
        } else {
            if ((rc = upload(out_w[l], ow, (size_t)rows * in))) return rc;
            if ((rc = upload(out_b[l], ob, (size_t)rows))) return rc;
        }
    }
    if ((rc = upload(mean, wl.take(), (size_t)C))) return rc;
    if ((rc = upload(std_, wl.take(), (size_t)C))) return rc;
    if (c.has_decoder) {
        B200_REQUIRE(c.num_squeeze >= 1 && c.hidden_channels_dec > 0 && c.kernel_size_dec % 2 == 1 &&
                         c.num_flow_blocks >= 1 && c.num_block_layers >= 1 && c.dilation_rate >= 1,
                     "overflow: unsupported decoder config");
        if ((rc = dec.init(C, c.hidden_channels_dec, c.kernel_size_dec, c.dilation_rate, c.num_flow_blocks,
                           c.num_block_layers, 0, c.num_splits, c.num_squeeze, c.sigmoid_scale, wl)))
            return rc;
    }
    return wl.finish("overflow");
}

size_t Overflow::workspace_bytes(int B, int Tt, int F) const {
    const size_t encb = arena_size([&](Arena& ar) { encode_carve(*this, ar, B, Tt); });
    if (!c.has_decoder || F <= 0) return encb;
    return std::max(encb, arena_size([&](Arena& ar) { decode_carve(*this, ar, B, tq(F)); }));
}

int Overflow::encode(const long long* tokens, const long long* lengths, int B, int Tt, float* states, void* ws,
                     size_t ws_bytes, cudaStream_t st) const {
    B200_REQUIRE(tokens && lengths && states && ws, "overflow_encode: null pointer");
    B200_REQUIRE(B >= 1 && Tt >= 1, "overflow_encode: empty batch");
    const size_t need = workspace_bytes(B, Tt, 0);
    B200_REQUIRE(ws_bytes >= need, "overflow_encode: workspace of %zu bytes, %zu needed", ws_bytes, need);
    const int E = c.encoder_dim, N = Tt * c.state_per_phone;
    Arena ar(ws, ws_bytes);
    const EncodeWs w = encode_carve(*this, ar, B, Tt);
    const Persist& p = w.p;
    float* encT = w.encT;
    int rc;
    // the [B, Tt, 2H] LSTM output is the [B, Tt*spp, E] state tensor
    if ((rc = enc.encode(tokens, lengths, B, Tt, states, w.enc, st))) return rc;
    if ((rc = launch_transpose(states, encT, B, N, E, st))) return rc;
    {   // hoisted: zc[b, r, n] = W_z[r] . state[b, n] + b_0[r] for every state n
        ConvIO io;
        io.x = dense(encT, E, N); io.Tin = N;
        io.y = dense(p.zc, O1, N); io.Tout = N; io.B = B;
        if ((rc = launch_conv(zproj, io, st))) return rc;
    }
    return 0;
}

int Overflow::sample(const long long* lengths, int B, int Tt, float temp, int max_frames, float threshold,
                     const float* noise, const unsigned char* drop, int chunk_frames, float* hmm_out,
                     int* states_travelled, int* frames, void* ws, size_t ws_bytes, cudaStream_t st) const {
    B200_REQUIRE(lengths && hmm_out && states_travelled && frames && ws, "overflow_sample: null pointer");
    B200_REQUIRE(B >= 1 && Tt >= 1 && max_frames >= 1, "overflow_sample: B, Tt and max_frames must be >= 1");
    B200_REQUIRE(temp <= 0.f || noise, "overflow_sample: sampling_temp > 0 needs noise");
    B200_REQUIRE(chunk_frames >= 2 && chunk_frames % 2 == 0, "overflow_sample: chunk_frames must be even and >= 2");
    const size_t need = workspace_bytes(B, Tt, 0);
    B200_REQUIRE(ws_bytes >= need, "overflow_sample: workspace of %zu bytes, %zu needed", ws_bytes, need);
    const int C = c.out_channels, P = c.prenet_dim, M = c.memory_rnn_dim, nL = c.outputnet_n_layers;
    const int N = Tt * c.state_per_phone;
    Arena ar(ws, ws_bytes);
    Persist p;
    persist_layout(*this, ar, B, Tt, p);
    int omax = 0;
    for (int l = 0; l < nL; ++l) omax = std::max(omax, c.outputnet_size[l]);
    B200_CUDA_OK(cudaMemsetAsync(hmm_out, 0, sizeof(float) * (size_t)B * max_frames * C, st));
    hmm_reset_kernel<<<B, 256, 0, st>>>(p.hm, p.cm, M, p.pin, go, c.ar_order, C, p.state, p.quant, p.done, p.ctl,
                                        states_travelled, max_frames, B);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    const unsigned char* dmask = c.prenet_dropout ? drop : nullptr;
    // one frame: prenet layers, LSTMCell, output-net layers, last layer, epilogue -- parity = frame index within the
    // chunk (h is double-buffered; chunk_frames is even, so every replay starts on buffer 0)
    auto frame = [&](cudaStream_t cs, int par, bool note) -> int {
        const float* in = p.pin;
        int K = c.ar_order * C;
        for (int l = 0; l < c.prenet_n_layers; ++l) {
            LinArgs a;
            a.W = prenet_w[l]; a.K = K; a.R = P; a.x = in; a.x_bs = K;
            a.y = p.pb + (size_t)(l & 1) * B * P; a.y_bs = P; a.relu = 1;
            a.drop = dmask; a.drop_layer = l; a.drop_L = c.prenet_n_layers; a.drop_F = max_frames; a.ctl = p.ctl;
            a.done = p.done; a.B = B;
            int rc;
            if ((rc = launch_linear(a, cs, note))) return rc;
            in = a.y; K = P;
        }
        {
            LstmArgs a;   // W_hh h first, then W_ih x
            a.seg[0].W = mem_whh; a.seg[0].ldw = M; a.seg[0].K = M; a.seg[0].x = p.hm + (size_t)par * B * M;
            a.seg[0].x_bs = M;
            a.seg[1].W = mem_wih; a.seg[1].ldw = P; a.seg[1].K = P; a.seg[1].x = in; a.seg[1].x_bs = P;
            a.nseg = 2;
            a.H = M; a.h_out = p.hm + (size_t)(par ^ 1) * B * M; a.h_bs = M;
            a.c = p.cm; a.bias = mem_b; a.done = p.done; a.B = B;
            int rc;
            if ((rc = launch_lstm(a, 1, 8, DISPATCH_LSTM_CELL, cs, note))) return rc;
        }
        in = p.hm + (size_t)(par ^ 1) * B * M;
        K = M;
        for (int l = 0; l <= nL; ++l) {
            const int R = l < nL ? c.outputnet_size[l] : 2 * C + 1;
            LinArgs a;
            a.W = out_w[l]; a.bias = out_b[l]; a.K = K; a.R = R; a.x = in; a.x_bs = K;
            a.y = l < nL ? p.hid + (size_t)(l & 1) * B * omax : p.outp; a.y_bs = l < nL ? omax : 2 * C + 1;
            if (l == 0) { a.add = p.zc; a.add_bs = (long long)O1 * N; a.add_rs = N; a.state = p.state; }
            a.relu = l < nL; a.done = p.done; a.B = B;
            int rc;
            if ((rc = launch_linear(a, cs, note))) return rc;
            in = a.y; K = R;
        }
        StepArgs s;
        s.o = p.outp; s.C = C; s.ar = c.ar_order; s.noise = noise; s.temp = temp; s.floor_ = c.std_floor;
        s.thr = threshold; s.max_frames = max_frames; s.hmm_out = hmm_out; s.pin = p.pin; s.st_tr = states_travelled;
        s.state = p.state; s.quant = p.quant; s.done = p.done; s.ctl = p.ctl; s.lens = lengths;
        s.spp = c.state_per_phone; s.B = B;
        hmm_step_kernel<<<1, 256, 0, cs>>>(s);
        if (note) dispatch_note(DISPATCH_HMM_STEP);
        B200_CUDA_OK(cudaGetLastError());
        return 0;
    };
    const int per_frame = c.prenet_n_layers + 1 + nL + 1 + 1;
    std::vector<int> host;
    int rc;
    if ((rc = run_step_graph("overflow_sample", chunk_frames, max_frames, per_frame, frame, p.ctl, B, host, st)))
        return rc;
    for (int b = 0; b < B; ++b) frames[b] = host[2 + b];
    return 0;
}

int Overflow::decode(const float* hmm_out, const int* frames, int B, int F, int Fpitch, float* mel, void* ws,
                     size_t ws_bytes, cudaStream_t st) const {
    B200_REQUIRE(hmm_out && frames && mel && ws, "overflow_decode: null pointer");
    B200_REQUIRE(F >= 0 && F <= Fpitch, "overflow_decode: F must be in [0, Fpitch]");
    const int C = c.out_channels;
    if (B == 0 || F == 0) return 0;
    if (!c.has_decoder) {   // Neural-HMM: inverse_normalize(hmm_outputs)
        dim3 grid((F * C + 255) / 256, B);
        denorm_kernel<<<grid, 256, 0, st>>>(hmm_out, (long long)Fpitch * C, C, 1, mean, std_, mel, F, C);
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
        return 0;
    }
    const size_t need = workspace_bytes(B, 1, F);
    B200_REQUIRE(ws_bytes >= need, "overflow_decode: workspace of %zu bytes, %zu needed", ws_bytes, need);
    const int nsq = c.num_squeeze, Tv = F / nsq, Tq = tq(F), Cs = C * nsq;
    if (Tv == 0) return 0;
    Arena ar(ws, ws_bytes);
    const DecodeWs w = decode_carve(*this, ar, B, Tq);
    float *za = w.za, *msk = w.msk, *melc = w.melc;
    {
        dim3 grid((Tq + 127) / 128, Cs, B);
        squeeze_hmm_kernel<<<grid, 128, 0, st>>>(hmm_out, Fpitch, frames, za, msk, C, nsq, Tq);
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
    }
    int rc;
    if ((rc = dec.reverse(za, msk, nullptr, B, Tq, Tv, melc, w.dec, w.dec_bytes, st))) return rc;
    const int T = Tv * nsq;
    dim3 grid((T * C + 255) / 256, B);
    denorm_kernel<<<grid, 256, 0, st>>>(melc, (long long)C * T, 1, T, mean, std_, mel, T, C);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace b200tts
