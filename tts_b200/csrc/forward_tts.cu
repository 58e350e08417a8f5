// ForwardTTS inference (FastPitch / FastSpeech / FastSpeech2): text -> mel spectrogram.
// Reference: TTS/tts/models/forward_tts.py:672-714 (inference), :374-415 (_forward_encoder), :353-372
//            (format_durations), :310-351 (generate_attn / expand_encoder_outputs), :417-451 (_forward_decoder),
//            :453-523 (pitch / energy predictors), TTS/tts/layers/generic/transformer.py:6-69 (FFTransformer, -Block),
//            feed_forward/encoder.py:154-162, feed_forward/decoder.py:94-122, generic/pos_encoding.py:38-69,
//            glow_tts/duration_predictor.py (the predictors).
// The text side runs on the exact FP32 FMA conv (durations must be bit-stable); the decoder's convs on the 3xTF32
// tensor-core engine and its attention on attention_tc3.cu.  Each FFTransformer layer in eval is
//   x = norm1((x + a) + a), a = out_proj(attn(in_proj(x)))     (the attention output is added twice, :25-26)
//   x = norm2(x + conv2(relu(conv1(x))))                       (k3 convs, zero padding, LayerNorm eps 1e-5)
// Batched rows: encoder keys and conv inputs stop at the row's token count, decoder keys and conv inputs at its frame
// count; a padded token gets no frame.  Row b thereby computes the single-utterance inference of x[b, :len[b]].
#include <math.h>

#include "engines.cuh"

namespace b200tts {

namespace {

// out[b,:,t] = LayerNorm_c(twice ? (x + y) + y : x + y) * gamma + beta where mask[b,t] != 0, else 0 (a select: the
// columns beyond a decoder row's end hold stale scratch, which must not leak NaN).  block (32 t) x (8 channel groups)
__global__ void __launch_bounds__(256) fft_add_norm_kernel(const float* x, const float* y, int twice, const float* gamma,
                                                           const float* beta, const float* mask, float* out, int C,
                                                           int T, float eps) {
    __shared__ float red[8][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int t = blockIdx.x * 32 + tx, b = blockIdx.y;
    const bool ok = t < T && mask[(size_t)b * T + t] != 0.f;
    const size_t base = (size_t)b * C * T + t;
    auto val = [&](int c) {
        const float yv = y[base + (size_t)c * T];
        const float s = __fadd_rn(x[base + (size_t)c * T], yv);
        return twice ? __fadd_rn(s, yv) : s;
    };
    float s = 0.f;
    if (ok) for (int c = ty; c < C; c += 8) s += val(c);
    red[ty][tx] = s;
    __syncthreads();
    float mean = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) mean += red[k][tx];
    mean /= (float)C;
    __syncthreads();
    float v = 0.f;
    if (ok) for (int c = ty; c < C; c += 8) {
        const float d = val(c) - mean;
        v += d * d;
    }
    red[ty][tx] = v;
    __syncthreads();
    float var = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) var += red[k][tx];
    var /= (float)C;
    const float rstd = rsqrtf(var + eps);
    if (t >= T) return;
    for (int c = ty; c < C; c += 8)
        out[base + (size_t)c * T] = ok ? (val(c) - mean) * rstd * gamma[c] + beta[c] : 0.f;
}

// o_en[b, c, t] += g[b, c] (forward_tts.py:414: the speaker vector is added at every position)
__global__ void add_speaker_kernel(float* o_en, const float* g, int C, int T) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x, c = blockIdx.y, b = blockIdx.z;
    if (t >= T) return;
    const size_t i = ((size_t)b * C + c) * T + t;
    o_en[i] = __fadd_rn(o_en[i], g[(size_t)b * C + c]);
}

// one thread per decoder column t < Tp: token j = the smallest with cum[j] > t (the one-hot path of generate_path), then
//   x[b, c, t] = o_en[b, c, j] * sqrt(C) + pe[c, t]      (t < y_length; 0 beyond, up to the padded pitch Tp)
//   y_mask[b, t], lens[b] (int32), attn[b, t, :] (t < Ty) = one-hot row of token j
__global__ void expand_decoder_input_kernel(const float* o_en, const float* x_mask, const float* cum,
                                            const long long* y_lengths, const float* pe, int pe_len, float scale,
                                            float* x, float* y_mask, int* lens, float* attn, int C, int Tt, int Ty,
                                            int Tp) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (t >= Tp) return;
    const long long yl = y_lengths[b];
    const bool valid = (long long)t < yl;
    const float* cb = cum + (size_t)b * Tt;
    int lo = 0, hi = Tt;
    const float ft = (float)t;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (cb[mid] > ft) hi = mid; else lo = mid + 1;
    }
    const int j = lo;
    const bool hit = valid && j < Tt && x_mask[(size_t)b * Tt + j] != 0.f;
    y_mask[(size_t)b * Tp + t] = valid ? 1.f : 0.f;
    if (t == 0) lens[b] = (int)yl;
    if (attn && t < Ty) {
        float* ar = attn + ((size_t)b * Ty + t) * Tt;
        for (int k = 0; k < Tt; ++k) ar[k] = (hit && k == j) ? 1.f : 0.f;
    }
    const float* eb = o_en + (size_t)b * C * Tt;
    float* xb = x + (size_t)b * C * Tp + t;
    for (int c = 0; c < C; ++c) {
        float v = 0.f;
        if (valid) {
            v = __fmul_rn(hit ? eb[(size_t)c * Tt + j] : 0.f, scale);
            if (pe) v = __fadd_rn(v, pe[(size_t)c * pe_len + t]);
        }
        xb[(size_t)c * Tp] = v;
    }
}

// mel[b, t, o] = pm[b, o, t] for t < y_length, else 0  (postnet(o) * y_mask, transposed to [B, T, C_out])
__global__ void mel_out_kernel(const float* pm, const long long* y_lengths, float* mel, int Co, int Ty, int Tp) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (i >= (long long)Ty * Co) return;
    const int t = (int)(i / Co), o = (int)(i - (long long)t * Co);
    mel[(size_t)b * Ty * Co + i] = (long long)t < y_lengths[b] ? pm[((size_t)b * Co + o) * Tp + t] : 0.f;
}

int pack_layer(ForwardTTS::Layer& L, WeightList& wl, int C, int F, int prec) {
    int rc;
    L.qkv.tc_prec = L.o.tc_prec = L.ffn1.tc_prec = L.ffn2.tc_prec = prec;
    const float *qw = wl.take(), *qb = wl.take(), *ow = wl.take(), *ob = wl.take(), *f1w = wl.take(), *f1b = wl.take(),
                *f2w = wl.take(), *f2b = wl.take();
    if ((rc = pack_conv(L.qkv, qw, qb, 3 * C, C, 1, 1, 0))) return rc;   // in_proj rows q | k | v
    if ((rc = pack_conv(L.o, ow, ob, C, C, 1, 1, 0))) return rc;
    if ((rc = pack_conv(L.ffn1, f1w, f1b, F, C, 3, 1, 1))) return rc;
    if ((rc = pack_conv(L.ffn2, f2w, f2b, C, F, 3, 1, 1))) return rc;
    if ((rc = upload(L.ln1_g, wl.take(), C))) return rc;
    if ((rc = upload(L.ln1_b, wl.take(), C))) return rc;
    if ((rc = upload(L.ln2_g, wl.take(), C))) return rc;
    return upload(L.ln2_b, wl.take(), C);
}

}  // namespace

int launch_add_norm(const float* x, const float* y, bool twice, const float* g, const float* bta, const float* mask,
                    float* out, int B, int C, int T, cudaStream_t st) {
    if (B == 0 || T == 0) return 0;
    dim3 grid((T + 31) / 32, B);
    fft_add_norm_kernel<<<grid, 256, 0, st>>>(x, y, twice ? 1 : 0, g, bta, mask, out, C, T, 1e-5f);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

int ForwardTTS::init(const b200tts_forward_tts_config& cfg, const float* const* w, int nw) {
    c = cfg;
    const int C = c.hidden_channels;
    B200_REQUIRE(c.n_vocab > 0 && C > 0 && c.out_channels > 0 && c.enc_layers >= 1 && c.dec_layers >= 1 &&
                 c.enc_ffn > 0 && c.dec_ffn > 0 && c.dp_hidden > 0 && c.dp_kernel >= 1 && c.proj_g_in >= 0 &&
                 c.pe_len >= 0, "forward_tts: unsupported config");
    B200_REQUIRE(c.enc_heads >= 1 && C % c.enc_heads == 0 && C / c.enc_heads <= 384,
                 "forward_tts: encoder head dim of %d channels / %d heads not supported (<= 384)", C, c.enc_heads);
    B200_REQUIRE(c.dec_heads >= 1 && C % c.dec_heads == 0 && C / c.dec_heads <= 384,
                 "forward_tts: decoder head dim of %d channels / %d heads not supported (<= 384)", C, c.dec_heads);
    B200_REQUIRE(!c.use_pitch || (c.pitch_hidden > 0 && c.pitch_kernel >= 1 && c.pitch_emb_kernel % 2 == 1),
                 "forward_tts: bad pitch predictor config");
    B200_REQUIRE(!c.use_energy || (c.energy_hidden > 0 && c.energy_kernel >= 1 && c.energy_emb_kernel % 2 == 1),
                 "forward_tts: bad energy predictor config");
    WeightList wl(w, nw);
    int rc;
    if ((rc = upload(emb, wl.take(), (size_t)c.n_vocab * C))) return rc;
    enc.resize(c.enc_layers);
    for (int l = 0; l < c.enc_layers; ++l)
        if ((rc = pack_layer(enc[l], wl, C, c.enc_ffn, TC_NONE))) return rc;
    if (c.proj_g_in > 0) {   // nn.Linear(d_vector_dim, C) as a 1x1 conv over a one-column input
        const float *gw = wl.take(), *gb = wl.take();
        if ((rc = pack_conv(proj_g, gw, gb, C, c.proj_g_in, 1, 1, 0))) return rc;
    }
    {
        b200tts_duration_predictor_config dc{C, c.dp_hidden, c.dp_kernel, 0, 0};
        if ((rc = dp.init(dc, wl))) return rc;
    }
    if (c.use_pitch) {
        b200tts_duration_predictor_config dc{C, c.pitch_hidden, c.pitch_kernel, 0, 0};
        if ((rc = pitch_dp.init(dc, wl))) return rc;
        const int k = c.pitch_emb_kernel;
        const float *ew = wl.take(), *eb = wl.take();
        if ((rc = pack_conv(pitch_emb, ew, eb, C, 1, k, 1, (k - 1) / 2))) return rc;
    }
    if (c.use_energy) {
        b200tts_duration_predictor_config dc{C, c.energy_hidden, c.energy_kernel, 0, 0};
        if ((rc = energy_dp.init(dc, wl))) return rc;
        const int k = c.energy_emb_kernel;
        const float *ew = wl.take(), *eb = wl.take();
        if ((rc = pack_conv(energy_emb, ew, eb, C, 1, k, 1, (k - 1) / 2))) return rc;
    }
    if (c.pe_len > 0 && (rc = upload(pe, wl.take(), (size_t)C * c.pe_len))) return rc;
    dec.resize(c.dec_layers);
    for (int l = 0; l < c.dec_layers; ++l)
        if ((rc = pack_layer(dec[l], wl, C, c.dec_ffn, B200TTS_PRECISION_FP32))) return rc;
    postnet.tc_prec = B200TTS_PRECISION_FP32;
    const float *pw = wl.take(), *pb = wl.take();
    if ((rc = pack_conv(postnet, pw, pb, c.out_channels, C, 1, 1, 0))) return rc;
    return wl.finish("forward_tts");
}

// the encoder layers' scratch, the projected speaker vector and one block the duration, pitch and energy predictors
// take in turn
struct FttsEncWs { float *qkv, *att, *yb, *hb, *gp; void* dp; size_t dp_bytes; };
static FttsEncWs ftts_encode_carve(const ForwardTTS& m, Arena& ar, int B, int Tt) {
    const int C = m.c.hidden_channels;
    FttsEncWs w;
    w.qkv = ar.f32((size_t)B * 3 * C * Tt);
    w.att = ar.f32((size_t)B * C * Tt);
    w.yb = ar.f32((size_t)B * C * Tt);
    w.hb = ar.f32((size_t)B * m.c.enc_ffn * Tt);
    w.gp = ar.f32((size_t)B * C);
    w.dp_bytes = m.dp.workspace_bytes(B, Tt);
    if (m.c.use_pitch) w.dp_bytes = std::max(w.dp_bytes, m.pitch_dp.workspace_bytes(B, Tt));
    if (m.c.use_energy) w.dp_bytes = std::max(w.dp_bytes, m.energy_dp.workspace_bytes(B, Tt));
    w.dp = ar.bytes(w.dp_bytes);
    return w;
}

size_t ForwardTTS::encode_bytes(int B, int Tt) const {
    return arena_size([&](Arena& ar) { ftts_encode_carve(*this, ar, B, Tt); });
}

struct FttsDecWs { float *x, *qkv, *att, *yb, *hb, *pm, *ymask; int* lens; };
static FttsDecWs ftts_decode_carve(const ForwardTTS& m, Arena& ar, int B, int Ty) {
    const size_t C = m.c.hidden_channels, Tp = ForwardTTS::tp(Ty);
    FttsDecWs w;
    w.x = ar.f32(B * C * Tp);
    w.qkv = ar.f32(B * 3 * C * Tp);
    w.att = ar.f32(B * C * Tp);
    w.yb = ar.f32(B * C * Tp);
    w.hb = ar.f32(B * m.c.dec_ffn * Tp);
    w.pm = ar.f32(B * m.c.out_channels * Tp);
    w.ymask = ar.f32(B * Tp);
    w.lens = reinterpret_cast<int*>(ar.f32((size_t)B));
    return w;
}

size_t ForwardTTS::decode_bytes(int B, int Ty) const {
    return arena_size([&](Arena& ar) { ftts_decode_carve(*this, ar, B, Ty); });
}

int ForwardTTS::encode(const long long* tokens, const long long* lengths, const float* g, float length_scale, int B,
                       int Tt, float* o_en, float* logw, float* pitch, float* energy, float* x_mask, float* dur,
                       float* cum, long long* y_lengths, long long* meta, void* ws, size_t ws_bytes,
                       cudaStream_t st) const {
    B200_REQUIRE(tokens && lengths && o_en && logw && x_mask && dur && cum && y_lengths && ws,
                 "forward_tts_encode: null pointer");
    B200_REQUIRE(!c.use_pitch || pitch, "forward_tts_encode: the pitch predictor needs a pitch output");
    B200_REQUIRE(!c.use_energy || energy, "forward_tts_encode: the energy predictor needs an energy output");
    const size_t need = encode_bytes(B, Tt);
    B200_REQUIRE(ws_bytes >= need, "forward_tts_encode: workspace of %zu bytes, %zu needed", ws_bytes, need);
    if (B == 0 || Tt == 0) return 0;
    const int C = c.hidden_channels, F = c.enc_ffn;
    Arena ar(ws, ws_bytes);
    const FttsEncWs w = ftts_encode_carve(*this, ar, B, Tt);
    float *qkv = w.qkv, *att = w.att, *yb = w.yb, *hb = w.hb, *gp = w.gp;
    float* x = o_en;
    int rc;
    // x = emb(tokens), no scale (forward_tts.py:405), masked at the row's length
    if ((rc = launch_embed(tokens, lengths, emb, nullptr, B, Tt, C, C, x, x_mask, st, false))) return rc;
    ConvIO eio;   // what every encoder conv shares: Tt columns in and out
    eio.Tin = eio.Tout = Tt; eio.B = B;
    for (const Layer& L : enc) {
        ConvIO io = eio;
        io.x = dense(x, C, Tt); io.y = dense(qkv, 3 * C, Tt);
        if ((rc = launch_conv(L.qkv, io, st))) return rc;
        // key_padding_mask = ~x_mask (transformer.py:60-63): masked keys get no weight
        if ((rc = launch_attention(qkv, x_mask, nullptr, nullptr, att, B, C, Tt, c.enc_heads, -1, st))) return rc;
        io = eio;
        io.x = dense(att, C, Tt); io.y = dense(yb, C, Tt);
        if ((rc = launch_conv(L.o, io, st))) return rc;
        if ((rc = launch_add_norm(x, yb, true, L.ln1_g, L.ln1_b, x_mask, x, B, C, Tt, st))) return rc;
        io = eio;
        io.x = dense(x, C, Tt); io.xmask = {x_mask, Tt}; io.y = dense(hb, F, Tt); io.act = ACT_RELU;
        if ((rc = launch_conv(L.ffn1, io, st))) return rc;
        io = eio;
        io.x = dense(hb, F, Tt); io.xmask = {x_mask, Tt}; io.y = dense(yb, C, Tt);
        if ((rc = launch_conv(L.ffn2, io, st))) return rc;
        // norm2(x + ffn), masked: Encoder.forward's final o * x_mask (feed_forward/encoder.py:161-162)
        if ((rc = launch_add_norm(x, yb, false, L.ln2_g, L.ln2_b, x_mask, x, B, C, Tt, st))) return rc;
    }
    if (g) {   // o_en + g, g = emb_g(ids) / proj_g(d_vector) / d_vector (forward_tts.py:399-414)
        const float* gv = g;
        if (c.proj_g_in > 0) {
            if ((rc = launch_conv_vec(proj_g, g, gp, C, B, false, st))) return rc;
            gv = gp;
        }
        dim3 grid((Tt + 127) / 128, C, B);
        add_speaker_kernel<<<grid, 128, 0, st>>>(x, gv, C, Tt);
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
    }
    // the duration predictor sees o_en with g, before any pitch (forward_tts.py:691)
    if ((rc = dp.forward(x, x_mask, nullptr, nullptr, B, Tt, logw, w.dp, w.dp_bytes, st))) return rc;
    // pitch, then energy on o_en that already holds the pitch embedding: o_en += emb(pred) (:697-704)
    const DurPred* preds[2] = {c.use_pitch ? &pitch_dp : nullptr, c.use_energy ? &energy_dp : nullptr};
    const ConvLayer* embs[2] = {&pitch_emb, &energy_emb};
    float* outs[2] = {pitch, energy};
    for (int p = 0; p < 2; ++p) {
        if (!preds[p]) continue;
        if ((rc = preds[p]->forward(x, x_mask, nullptr, nullptr, B, Tt, outs[p], w.dp, w.dp_bytes, st))) return rc;
        ConvIO io = eio;
        io.x = dense(outs[p], 1, Tt); io.y = dense(x, C, Tt); io.flags = EPI_ACCUM;
        if ((rc = launch_conv(*embs[p], io, st))) return rc;
    }
    return launch_durations_forward(logw, x_mask, length_scale, B, Tt, dur, cum, y_lengths, meta, st);
}

int ForwardTTS::decode(const float* o_en, const float* x_mask, const float* cum, const long long* y_lengths, int B,
                       int Tt, int Ty, float* attn, float* mel, void* ws, size_t ws_bytes, cudaStream_t st) const {
    B200_REQUIRE(o_en && x_mask && cum && y_lengths && mel && ws, "forward_tts_decode: null pointer");
    B200_REQUIRE(c.pe_len == 0 || Ty <= c.pe_len,
                 "forward_tts_decode: sequence is %d frames but the positional encoding is limited to %d", Ty, c.pe_len);
    const size_t need = decode_bytes(B, Ty);
    B200_REQUIRE(ws_bytes >= need, "forward_tts_decode: workspace of %zu bytes, %zu needed", ws_bytes, need);
    if (B == 0 || Ty == 0) return 0;
    const int C = c.hidden_channels, F = c.dec_ffn, Co = c.out_channels, Tp = tp(Ty);
    Arena ar(ws, ws_bytes);
    const FttsDecWs w = ftts_decode_carve(*this, ar, B, Ty);
    float *x = w.x, *qkv = w.qkv, *att = w.att, *yb = w.yb, *hb = w.hb, *pm = w.pm, *ymask = w.ymask;
    int* lens = w.lens;
    int rc;
    {
        dim3 grid((Tp + 127) / 128, B);
        expand_decoder_input_kernel<<<grid, 128, 0, st>>>(o_en, x_mask, cum, y_lengths, pe, c.pe_len,
                                                          pe ? (float)sqrt((double)C) : 1.f, x, ymask, lens, attn, C, Tt,
                                                          Ty, Tp);
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
    }
    // Ragged rows: the tensor-core convs (Tp >= 128) stop at lens[b] and read the input as zero from there; the FMA conv
    // (short batches) computes every column and reads the input through y_mask instead.
    const bool tc = Tp >= 128;
    const bool attn_tc = attention_tc3_takes(C / c.dec_heads);
    ConvIO dio;   // what every decoder conv shares: Tp columns in and out, ragged rows as above
    dio.Tin = dio.Tout = Tp; dio.B = B;
    if (!tc) dio.xmask = {ymask, Tp};
    else dio.lens = lens;
    for (const Layer& L : dec) {
        ConvIO io = dio;
        io.x = dense(x, C, Tp); io.y = dense(qkv, 3 * C, Tp);
        // the FMA attention fallback reads every column of q|k|v, so it gets them computed in full (from zero inputs)
        if (!attn_tc) io.lens = nullptr;
        if ((rc = launch_conv(L.qkv, io, st))) return rc;
        if (attn_tc) {
            if ((rc = launch_attention_tc3(qkv, (long long)3 * C * Tp, Tp, lens, att, (long long)C * Tp, B, C,
                                           c.dec_heads, Ty, st)))
                return rc;
        } else {
            if ((rc = launch_attention(qkv, ymask, nullptr, nullptr, att, B, C, Tp, c.dec_heads, -1, st))) return rc;
            dispatch_note(DISPATCH_ATTN_FMA);
        }
        io = dio;
        io.x = dense(att, C, Tp); io.y = dense(yb, C, Tp);
        if ((rc = launch_conv(L.o, io, st))) return rc;
        if ((rc = launch_add_norm(x, yb, true, L.ln1_g, L.ln1_b, ymask, x, B, C, Tp, st))) return rc;
        io = dio;
        io.x = dense(x, C, Tp); io.y = dense(hb, F, Tp); io.act = ACT_RELU;
        if ((rc = launch_conv(L.ffn1, io, st))) return rc;
        io = dio;
        io.x = dense(hb, F, Tp); io.y = dense(yb, C, Tp);
        if ((rc = launch_conv(L.ffn2, io, st))) return rc;
        if ((rc = launch_add_norm(x, yb, false, L.ln2_g, L.ln2_b, ymask, x, B, C, Tp, st))) return rc;
    }
    ConvIO io = dio;
    io.x = dense(x, C, Tp); io.y = dense(pm, Co, Tp);
    if ((rc = launch_conv(postnet, io, st))) return rc;
    dim3 grid((unsigned)(((long long)Ty * Co + 255) / 256), B);
    mel_out_kernel<<<grid, 256, 0, st>>>(pm, y_lengths, mel, Co, Ty, Tp);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace b200tts
