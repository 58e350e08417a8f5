// Glow-TTS inference: text -> mel spectrogram.
// Reference: TTS/tts/models/glow_tts.py:342-374 (inference), :138-148 (compute_outputs),
//            TTS/tts/layers/glow_tts/encoder.py:143-179 (Encoder.forward), glow.py:11-67 (prenet),
//            transformer.py:411-432 (RelativePositionTransformer without a relative window),
//            generic/normalization.py:5-28 (LayerNorm type "1", eps 1e-4), :66-101 (ActNorm),
//            decoder.py:8-47,113-137 (squeeze / unsqueeze, reverse pass), glow.py:70-137 (InvConvNear),
//            :144-230 (CouplingBlock).
// The encoder and duration predictor reuse the VITS text path's kernels on the exact FP32 FMA conv (durations must be
// bit-stable); the decoder's WaveNet runs the flow's tensor-core convs.  Squeeze is folded into the kernel that builds
// the latent, unsqueeze into the last block's elementwise pass.
#include <math.h>

#include "engines.cuh"

namespace b200tts {

namespace {

constexpr int MAX_SPLITS = 16;

// xdp[b, c, t] = (c < H ? x[b, c, t] : g[b, c - H]) * mask[b, t]     (encoder.py:166-168, cat on the channel axis)
__global__ void cat_cond_kernel(const float* x, const float* g, const float* mask, float* xdp, int H, int Cg, int T) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x, c = blockIdx.y, b = blockIdx.z;
    if (t >= T) return;
    const float v = c < H ? x[((size_t)b * H + c) * T + t] : g[(size_t)b * Cg + (c - H)];
    xdp[((size_t)b * (H + Cg) + c) * T + t] = v * mask[(size_t)b * T + t];
}

// z = (y_mean + exp(y_log_scale) * noise * noise_scale) * y_mask (glow_tts.py:361), squeezed (decoder.py:8-28):
// zs[b, k*C + c, q] = z[b, c, q*nsq + k] * msk[b, q], msk[b, q] = y_mask[b, q*nsq + nsq - 1].  Columns q >= Tv (the
// frames the squeeze truncates, and the alignment padding up to Tq) are zero.
__global__ void squeeze_prior_kernel(const float* y_mean, const float* y_log_scale, const float* noise, float noise_scale,
                                     const long long* y_lengths, float* zs, float* msk, int C, int Ty, int nsq, int Tv,
                                     int Tq) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x, ck = blockIdx.y, b = blockIdx.z;
    if (q >= Tq) return;
    const int k = ck / C, c = ck - k * C;
    const long long yl = y_lengths[b];
    const float m = (q < Tv && (long long)q * nsq + nsq - 1 < yl) ? 1.f : 0.f;
    float v = 0.f;
    if (q < Tv) {
        const int t = q * nsq + k;
        const size_t i = ((size_t)b * C + c) * Ty + t;
        v = y_mean[i];
        if (noise) v = __fadd_rn(v, __fmul_rn(__fmul_rn(expf(y_log_scale[i]), noise[i]), noise_scale));
        v = __fmul_rn(__fmul_rn(v, (long long)t < yl ? 1.f : 0.f), m);
    }
    zs[((size_t)b * C * nsq + ck) * Tq + q] = v;
    if (ck == 0) msk[(size_t)b * Tq + q] = m;
}

// One decoder block's tail, reverse direction, for the num_splits channels of one InvConvNear group at one frame:
//   coupling (glow.py:210-223): x1 = (x1 - t) * exp(-s) * mask, s = log(1e-6 + sigmoid(s + 2)) with sigmoid_scale,
//     t / s = rows [0, Cs/2) / [Cs/2, Cs) of the end conv's output eo; x0 passes unchanged
//   InvConvNear^-1 (glow.py:108-137): channel a*Cs/2 + g*ns/2 + k is split s = a*ns/2 + k of group g;
//     z_s = sum_s' Winv[s][s'] * x_s', then * mask
//   ActNorm^-1 (normalization.py:96-97): (z - bias) * exp(-logs) * mask
// out_nsq > 0: the last block -- write unsqueezed (decoder.py:31-47) into mel [B, C, Tv * out_nsq] instead of [B, Cs, Tq].
__global__ void flow_step_kernel(const float* __restrict__ x, const float* __restrict__ eo, const float* __restrict__ msk,
                                 const float* __restrict__ mix, const float* __restrict__ an_bias,
                                 const float* __restrict__ an_logs, float* __restrict__ y, int Cs, int Tq, int ns,
                                 int sigmoid_scale, int out_nsq, int Tv) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x, grp = blockIdx.y, b = blockIdx.z;
    if (t >= Tq) return;
    const int Ch = Cs / 2, half = ns / 2;
    const float m = msk[(size_t)b * Tq + t];
    const float* xb = x + (size_t)b * Cs * Tq + t;
    const float* eb = eo + (size_t)b * Cs * Tq + t;
    float xin[MAX_SPLITS];
#pragma unroll
    for (int s = 0; s < MAX_SPLITS; ++s) {
        if (s >= ns) break;
        const int a = s >= half ? 1 : 0;
        const int ch = a * Ch + grp * half + (s - a * half);
        float v = xb[(size_t)ch * Tq];
        if (a) {
            const float tt = eb[(size_t)(ch - Ch) * Tq];
            float ss = eb[(size_t)ch * Tq];
            if (sigmoid_scale) ss = logf(__fadd_rn(1e-6f, 1.f / (1.f + expf(-__fadd_rn(ss, 2.f)))));
            v = __fmul_rn(__fmul_rn(__fsub_rn(v, tt), expf(-ss)), m);
        }
        xin[s] = v;
    }
#pragma unroll
    for (int so = 0; so < MAX_SPLITS; ++so) {
        if (so >= ns) break;
        float acc = 0.f;
#pragma unroll
        for (int si = 0; si < MAX_SPLITS; ++si) {
            if (si >= ns) break;
            acc = fmaf(mix[so * ns + si], xin[si], acc);
        }
        const int a = so >= half ? 1 : 0;
        const int o = a * Ch + grp * half + (so - a * half);
        const float r = __fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(acc, m), an_bias[o]), expf(-an_logs[o])), m);
        if (out_nsq) {
            if (t < Tv) {
                const int C = Cs / out_nsq, k = o / C, c = o - k * C;
                y[((size_t)b * C + c) * ((size_t)Tv * out_nsq) + (size_t)t * out_nsq + k] = r;
            }
        } else {
            y[((size_t)b * Cs + o) * Tq + t] = r;
        }
    }
}

}  // namespace

int GlowDecoder::init(int out_channels, int hidden, int kernel_size, int dilation_rate, int num_blocks, int num_layers,
                      int cond_channels, int num_splits, int num_squeeze, int sigmoid, WeightList& wl) {
    Cs = out_channels * num_squeeze;
    Hd = hidden; ns = num_splits; nsq = num_squeeze; sigmoid_scale = sigmoid;
    B200_REQUIRE(ns >= 2 && ns % 2 == 0 && ns <= MAX_SPLITS && Cs % ns == 0,
                 "glow decoder: num_splits %d must be even, <= %d and divide out_channels * num_squeeze = %d", ns,
                 MAX_SPLITS, Cs);
    int rc;
    blocks.resize(num_blocks);
    for (int n = 0; n < num_blocks; ++n) {
        Block& b = blocks[n];
        if ((rc = upload(b.an_logs, wl.take(), Cs))) return rc;
        if ((rc = upload(b.an_bias, wl.take(), Cs))) return rc;
        if ((rc = upload(b.mix, wl.take(), (size_t)ns * ns))) return rc;
        b.start.tc_prec = b.end.tc_prec = B200TTS_PRECISION_FP32;
        const float *sw = wl.take(), *sb = wl.take();
        if ((rc = pack_conv(b.start, sw, sb, Hd, Cs / 2, 1, 1, 0))) return rc;
        if ((rc = b.wn.init(Hd, kernel_size, dilation_rate, num_layers, cond_channels, wl))) return rc;
        const float *ew = wl.take(), *eb = wl.take();
        if ((rc = pack_conv(b.end, ew, eb, Cs, Hd, 1, 1, 0))) return rc;
    }
    return 0;
}

struct GlowDecWs { float *zb, *eo, *h, *acts, *out, *condv; };
static GlowDecWs glowdec_carve(const GlowDecoder& m, Arena& ar, int B, int Tq) {
    GlowDecWs w;
    w.zb = ar.f32((size_t)B * m.Cs * Tq);
    w.eo = ar.f32((size_t)B * m.Cs * Tq);
    w.h = ar.f32((size_t)B * m.Hd * Tq);
    w.acts = ar.f32((size_t)B * m.Hd * Tq);
    w.out = ar.f32((size_t)B * m.Hd * Tq);
    w.condv = ar.f32((size_t)B * m.blocks[0].wn.cond.RowsPad + 64);
    return w;
}

size_t GlowDecoder::workspace_bytes(int B, int Tq) const {
    return arena_size([&](Arena& ar) { glowdec_carve(*this, ar, B, Tq); });
}

int GlowDecoder::reverse(float* z, const float* msk, const float* g, int B, int Tq, int Tv, float* mel, void* ws,
                         size_t ws_bytes, cudaStream_t st) const {
    Arena ar(ws, ws_bytes);
    const GlowDecWs w = glowdec_carve(*this, ar, B, Tq);
    B200_REQUIRE(ar.ok(), "glow decoder: workspace of %zu bytes is too small", ws_bytes);
    float *zb = w.zb, *eo = w.eo, *h = w.h, *acts = w.acts, *out = w.out, *condv = w.condv;
    int rc;
    float* cur = z;
    float* nxt = zb;
    for (int n = (int)blocks.size() - 1; n >= 0; --n) {   // reversed(flows): coupling, InvConvNear, ActNorm per block
        const Block& bl = blocks[n];
        {   // h = start(x0) * mask, x0 = the first half of cur's channels
            ConvIO io;
            io.x = dense(cur, Cs, Tq); io.Tin = Tq;
            io.y = dense(h, Hd, Tq); io.Tout = Tq; io.B = B;
            io.ymask = {msk, Tq}; io.flags = EPI_MASK_POST;
            if ((rc = launch_conv(bl.start, io, st))) return rc;
        }
        if ((rc = bl.wn.forward(h, out, msk, g, B, Tq, acts, condv, st))) return rc;
        {   // [t | s] = end(WN(h))
            ConvIO io;
            io.x = dense(out, Hd, Tq); io.Tin = Tq;
            io.y = dense(eo, Cs, Tq); io.Tout = Tq; io.B = B;
            if ((rc = launch_conv(bl.end, io, st))) return rc;
        }
        dim3 grid((Tq + 127) / 128, Cs / ns, B);
        flow_step_kernel<<<grid, 128, 0, st>>>(cur, eo, msk, bl.mix, bl.an_bias, bl.an_logs, n > 0 ? nxt : mel, Cs, Tq,
                                               ns, sigmoid_scale, n > 0 ? 0 : nsq, Tv);
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
        std::swap(cur, nxt);
    }
    return 0;
}

int GlowTTS::init(const b200tts_glow_tts_config& cfg, const float* const* w, int nw) {
    c = cfg;
    const int H = c.hidden_channels_enc, C = c.out_channels, F = c.hidden_channels_ffn, K = c.kernel_size_enc;
    const int ns = c.num_splits, nsq = c.num_squeeze, cin = c.c_in_channels, Hd = c.hidden_channels_dec;
    B200_REQUIRE(c.n_vocab > 0 && H > 0 && C > 0 && F > 0 && K >= 1 && c.num_layers_enc >= 1 && Hd > 0 && cin >= 0 &&
                 c.num_flow_blocks >= 1 && c.num_block_layers >= 1 && c.kernel_size_dec % 2 == 1 && c.dilation_rate >= 1,
                 "glow_tts: unsupported config");
    B200_REQUIRE(c.num_heads >= 1 && H % c.num_heads == 0, "glow_tts: channels %d not divisible by heads %d", H,
                 c.num_heads);
    B200_REQUIRE(nsq >= 1, "glow_tts: num_squeeze must be >= 1");
    Cs = C * nsq;
    B200_REQUIRE(ns >= 2 && ns % 2 == 0 && ns <= MAX_SPLITS && Cs % ns == 0,
                 "glow_tts: num_splits %d must be even, <= %d and divide out_channels * num_squeeze = %d", ns, MAX_SPLITS,
                 Cs);
    WeightList wl(w, nw);
    int rc;
    if ((rc = upload(emb, wl.take(), (size_t)c.n_vocab * H))) return rc;
    if (c.use_prenet) {   // ResidualConv1dLayerNormBlock(H, H, H, kernel_size=5, num_layers=3), encoder.py:107-110
        prenet.resize(3);
        for (auto& p : prenet) {
            const float *pw = wl.take(), *pb = wl.take();
            if ((rc = pack_conv(p.conv, pw, pb, H, H, 5, 1, 2))) return rc;
            if ((rc = upload(p.g, wl.take(), H))) return rc;
            if ((rc = upload(p.b, wl.take(), H))) return rc;
        }
        const float *pw = wl.take(), *pb = wl.take();
        if ((rc = pack_conv(prenet_proj, pw, pb, H, H, 1, 1, 0))) return rc;
    }
    if ((rc = tf.init(H, F, K, c.num_heads, -1, 1e-4f, c.num_layers_enc, wl))) return rc;
    {   // [proj_m | proj_s]: with mean_only the log-scale rows are zero weights and bias, i.e. zeros_like(x_m) (:176)
        std::vector<float> wp((size_t)2 * C * H, 0.f), bp((size_t)2 * C, 0.f);
        for (int s = 0; s < (c.mean_only ? 1 : 2); ++s) {
            const float *sw = wl.take(), *sb = wl.take();
            B200_REQUIRE(sw && sb, "glow_tts: null proj_m / proj_s weight or bias");
            memcpy(wp.data() + (size_t)s * C * H, sw, sizeof(float) * C * H);
            memcpy(bp.data() + (size_t)s * C, sb, sizeof(float) * C);
        }
        if ((rc = pack_conv(proj, wp.data(), bp.data(), 2 * C, H, 1, 1, 0))) return rc;
    }
    {   // DurationPredictor(H + c_in, hidden_channels_dp, 3): the speaker vector is concatenated, not added (:139-141)
        b200tts_duration_predictor_config dc{H + cin, c.hidden_channels_dp, 3, 0, 0};
        if ((rc = dp.init(dc, wl))) return rc;
    }
    if ((rc = dec.init(C, Hd, c.kernel_size_dec, c.dilation_rate, c.num_flow_blocks, c.num_block_layers, cin, ns, nsq,
                       c.sigmoid_scale, wl)))
        return rc;
    return wl.finish("glow_tts");
}

// x, cat(x, g), the duration predictor's and the transformer's blocks; the prenet runs before the transformer, so its
// two buffers are the transformer's scratch (which holds q|k|v alone, 3 B H Tt floats)
struct GlowEncWs { float *x, *xdp, *pre[2]; void *dp, *tf; size_t dp_bytes, tf_bytes; };
static GlowEncWs glow_encode_carve(const GlowTTS& m, Arena& ar, int B, int Tt) {
    const int H = m.c.hidden_channels_enc;
    GlowEncWs w;
    w.x = ar.f32((size_t)B * H * Tt);
    w.xdp = ar.f32((size_t)B * (H + m.c.c_in_channels) * Tt);
    w.dp_bytes = m.dp.workspace_bytes(B, Tt);
    w.dp = ar.bytes(w.dp_bytes);
    w.tf_bytes = m.tf.workspace_bytes(B, Tt);
    w.tf = ar.bytes(w.tf_bytes);
    Arena pa(w.tf, w.tf_bytes);
    w.pre[0] = pa.f32((size_t)B * H * Tt);
    w.pre[1] = pa.f32((size_t)B * H * Tt);
    return w;
}

size_t GlowTTS::encode_bytes(int B, int Tt) const {
    return arena_size([&](Arena& ar) { glow_encode_carve(*this, ar, B, Tt); });
}

// the squeezed latent, its mask and the Glow decoder's block
struct GlowDecodeWs { float *za, *msk; void* dec; size_t dec_bytes; };
static GlowDecodeWs glow_decode_carve(const GlowTTS& m, Arena& ar, int B, int Tq) {
    GlowDecodeWs w;
    w.za = ar.f32((size_t)B * m.Cs * Tq);
    w.msk = ar.f32((size_t)B * Tq);
    w.dec_bytes = m.dec.workspace_bytes(B, Tq);
    w.dec = ar.bytes(w.dec_bytes);
    return w;
}

size_t GlowTTS::decode_bytes(int B, int Ty) const {
    return arena_size([&](Arena& ar) { glow_decode_carve(*this, ar, B, tq(Ty)); });
}

int GlowTTS::encode(const long long* tokens, const long long* lengths, const float* g, float length_scale, int B,
                    int Tt, float* o_stats, float* logw, float* x_mask, float* w_ceil, float* cum, float* dur_log,
                    long long* y_lengths, long long* meta, void* ws, size_t ws_bytes, cudaStream_t st) const {
    B200_REQUIRE(tokens && lengths && o_stats && logw && x_mask && w_ceil && cum && dur_log && y_lengths && ws,
                 "glow_tts_encode: null pointer");
    B200_REQUIRE((c.c_in_channels > 0) == (g != nullptr), "glow_tts_encode: g must be given iff c_in_channels > 0");
    const size_t need = encode_bytes(B, Tt);
    B200_REQUIRE(ws_bytes >= need, "glow_tts_encode: workspace of %zu bytes, %zu needed", ws_bytes, need);
    if (B == 0 || Tt == 0) return 0;
    const int H = c.hidden_channels_enc, Cg = H + c.c_in_channels;
    Arena ar(ws, ws_bytes);
    const GlowEncWs w = glow_encode_carve(*this, ar, B, Tt);
    float *x = w.x, *xdp = w.xdp;
    int rc;
    // x = emb(tokens) * sqrt(H), masked: the prenet and the transformer both start with x * x_mask
    if ((rc = launch_embed(tokens, lengths, emb, nullptr, B, Tt, H, H, x, x_mask, st))) return rc;
    if (c.use_prenet) {   // glow.py:55-67: 3 x (conv(x * mask) -> LayerNorm(. * mask) -> ReLU), x = (x + proj(.)) * mask
        const float* in = x;
        for (int l = 0; l < 3; ++l) {
            float* out = w.pre[l & 1];
            ConvIO io;
            io.x = dense(in, H, Tt); io.Tin = Tt; io.xmask = {x_mask, Tt};
            if (l > 0) io.in_slope = 0.f;   // the previous layer's ReLU, applied to its masked output
            io.y = dense(out, H, Tt); io.Tout = Tt; io.B = B;
            io.ymask = {x_mask, Tt}; io.flags = EPI_MASK_POST;
            if ((rc = launch_conv(prenet[l].conv, io, st))) return rc;
            if ((rc = launch_add_layernorm(out, nullptr, prenet[l].g, prenet[l].b, nullptr, out, B, H, Tt, 1e-4f, st)))
                return rc;
            in = out;
        }
        ConvIO io;
        io.x = dense(in, H, Tt); io.Tin = Tt; io.xmask = {x_mask, Tt}; io.in_slope = 0.f;
        io.y = dense(x, H, Tt); io.Tout = Tt; io.B = B;
        io.ymask = {x_mask, Tt}; io.flags = EPI_ACCUM | EPI_MASK_POST;
        if ((rc = launch_conv(prenet_proj, io, st))) return rc;
    }
    if ((rc = tf.forward(x, x_mask, B, Tt, w.tf, w.tf_bytes, st))) return rc;
    {   // o_mean = proj_m(x) * mask, o_log_scale = proj_s(x) * mask (encoder.py:172-176)
        ConvIO io;
        io.x = dense(x, H, Tt); io.Tin = Tt;
        io.y = dense(o_stats, 2 * c.out_channels, Tt); io.Tout = Tt; io.B = B;
        io.ymask = {x_mask, Tt}; io.flags = EPI_MASK_POST;
        if ((rc = launch_conv(proj, io, st))) return rc;
    }
    const float* dp_in = x;
    if (c.c_in_channels > 0) {
        dim3 grid((Tt + 127) / 128, Cg, B);
        cat_cond_kernel<<<grid, 128, 0, st>>>(x, g, x_mask, xdp, H, c.c_in_channels, Tt);
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
        dp_in = xdp;
    }
    if ((rc = dp.forward(dp_in, x_mask, nullptr, nullptr, B, Tt, logw, w.dp, w.dp_bytes, st))) return rc;
    return launch_durations_glow(logw, x_mask, length_scale, B, Tt, w_ceil, cum, y_lengths, dur_log, meta, st);
}

int GlowTTS::decode(const float* o_stats, const float* x_mask, const float* cum, const long long* y_lengths,
                    const float* g, const float* noise, float noise_scale, int B, int Tt, int Ty, float* attn,
                    float* y_mean, float* y_log_scale, float* mel, void* ws, size_t ws_bytes, cudaStream_t st) const {
    B200_REQUIRE(o_stats && x_mask && cum && y_lengths && y_mean && y_log_scale && mel && ws,
                 "glow_tts_decode: null pointer");
    B200_REQUIRE((c.c_in_channels > 0) == (g != nullptr), "glow_tts_decode: g must be given iff c_in_channels > 0");
    const size_t need = decode_bytes(B, Ty);
    B200_REQUIRE(ws_bytes >= need, "glow_tts_decode: workspace of %zu bytes, %zu needed", ws_bytes, need);
    if (B == 0 || Ty == 0) return 0;
    const int C = c.out_channels, nsq = c.num_squeeze;
    const int Tv = Ty / nsq, Tq = tq(Ty);
    Arena ar(ws, ws_bytes);
    const GlowDecodeWs w = glow_decode_carve(*this, ar, B, Tq);
    int rc;
    // path and expanded prior (:355-359): attn, y_mean = attn^T o_mean, y_log_scale = attn^T o_log_scale
    if ((rc = launch_expand_prior(cum, x_mask, y_lengths, o_stats, nullptr, 0.f, B, Tt, Ty, C, attn, y_mean, y_log_scale,
                                  nullptr, nullptr, st)))
        return rc;
    if (Tv == 0) return 0;
    {
        dim3 grid((Tq + 127) / 128, Cs, B);
        squeeze_prior_kernel<<<grid, 128, 0, st>>>(y_mean, y_log_scale, noise_scale != 0.f ? noise : nullptr,
                                                   noise_scale, y_lengths, w.za, w.msk, C, Ty, nsq, Tv, Tq);
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
    }
    return dec.reverse(w.za, w.msk, g, B, Tq, Tv, mel, w.dec, w.dec_bytes, st);
}

}  // namespace b200tts
