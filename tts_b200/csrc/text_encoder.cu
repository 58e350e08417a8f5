// VITS TextEncoder: embedding -> 6x [relative-position MHA, add+LayerNorm, conv-FFN, add+LayerNorm] -> 1x1 proj; the
// layer stack is RelPosTransformer, which Glow-TTS shares.
// Reference: TTS/tts/layers/vits/networks.py:80-100 (TextEncoder.forward),
//            TTS/tts/layers/glow_tts/transformer.py:109-163,196-241 (attention with the pad/reshape
//            "skew" tricks, here in closed form -- SURVEY appendix A1), :290-295 (FFN), :411-432 (stack),
//            TTS/tts/layers/generic/normalization.py:31-53 (LayerNorm2, eps 1e-5).
// All dense contractions (QKV, O, FFN k3, proj) go through the fused conv1d kernel; this file adds
// the three small kernels around them.  Tensors stay [B, C, T].
#include <math.h>

#include "engines.cuh"

namespace b200tts {

namespace {

// x[b,c,t] = (c < hidden ? emb[tok]*sqrt(hidden) : lang[b,c-hidden]) * (t < len[b]);  mask[b,t]
__global__ void embed_kernel(const long long* tok, const long long* len, const float* emb, const float* lang,
                             float* x, float* mask, int T, int hidden, int C, float scale) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x, c = blockIdx.y, b = blockIdx.z;
    if (t >= T) return;
    const float m = (t < len[b]) ? 1.f : 0.f;
    float v;
    if (c < hidden) v = emb[tok[(size_t)b * T + t] * hidden + c] * scale;
    else v = lang[(size_t)b * (C - hidden) + (c - hidden)];
    x[((size_t)b * C + c) * T + t] = v * m;
    if (c == 0) mask[(size_t)b * T + t] = m;
}

constexpr int ATT_Q = 8;        // queries per CTA (one warp each)
constexpr int ATT_KT = 32;      // keys per tile
constexpr int ATT_MAXD = 256;   // max head dim of the VITS / Glow-TTS instantiation (8 values per lane)
constexpr int ATT_MAXD_WIDE = 384;   // ForwardTTS's text encoder: one head of 384 channels (12 values per lane)

// qkv [B, 3C, T] (q rows 0..C, k rows C..2C, v rows 2C..3C), head h owns channels [h*d, (h+1)*d); MAXD bounds d.
// Every column below T of q, k and v is read: a padded key is masked by its score (-1e4, as the reference's
// masked_fill), not skipped, and its value still enters P.V with probability 0.  So the outputs of valid queries do not
// depend on padded columns only as long as those are finite (0 * NaN = NaN); callers keep them finite (zero or computed
// from zero inputs).  A padded query row is the reference's uniform softmax over all T keys, padded ones included.
template <int MAXD>
__global__ void __launch_bounds__(32 * ATT_Q) rel_attention_kernel(const float* __restrict__ qkv, const float* __restrict__ mask,
                                                                  const float* __restrict__ emb_rel_k, const float* __restrict__ emb_rel_v,
                                                                  float* __restrict__ out, int C, int T, int d, int window,
                                                                  float inv_sqrt_d) {
    extern __shared__ float sm[];
    const int Tp = (T + 31) & ~31;
    const int nrel = 2 * window + 1;
    float* qs = sm;                              // [ATT_Q][d]
    float* sc = qs + ATT_Q * d;                  // [ATT_Q][Tp]
    float* kt = sc + ATT_Q * Tp;                 // [d][ATT_KT+1]  (reused as vt [ATT_KT][d+1])
    float* ek = kt + (ATT_KT + 1) * (d + 1);     // [nrel][d]
    float* ev = ek + nrel * d;                   // [nrel][d]
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.z, h = blockIdx.y, i0 = blockIdx.x * ATT_Q;
    const float* qb = qkv + ((size_t)b * 3 * C + h * d) * T;
    const float* kb = qb + (size_t)C * T;
    const float* vb = kb + (size_t)C * T;
    const float* mb = mask + (size_t)b * T;
    for (int idx = tid; idx < ATT_Q * d; idx += blockDim.x) {
        const int qi = idx / d, c = idx - qi * d, i = i0 + qi;
        qs[idx] = (i < T) ? qb[(size_t)c * T + i] : 0.f;
    }
    if (window >= 0)
        for (int idx = tid; idx < nrel * d; idx += blockDim.x) { ek[idx] = emb_rel_k[idx]; ev[idx] = emb_rel_v[idx]; }
    const int i = i0 + warp;
    const bool active = i < T;
    // ---- scores = q.k / sqrt(d)
    for (int j0 = 0; j0 < T; j0 += ATT_KT) {
        __syncthreads();
        // all global loads of a batch are issued before the first shared store (in-order issue would otherwise
        // expose one full memory latency per element)
        for (int i0b = 0; i0b < d * ATT_KT; i0b += 8 * 32 * ATT_Q) {
            float tmp[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int idx = i0b + u * 32 * ATT_Q + tid;
                const int c = idx / ATT_KT, jj = idx - c * ATT_KT, j = j0 + jj;
                tmp[u] = (idx < d * ATT_KT && j < T) ? kb[(size_t)c * T + j] : 0.f;
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int idx = i0b + u * 32 * ATT_Q + tid;
                const int c = idx / ATT_KT, jj = idx - c * ATT_KT;
                if (idx < d * ATT_KT) kt[c * (ATT_KT + 1) + jj] = tmp[u];
            }
        }
        __syncthreads();
        if (active) {
            float dot = 0.f;
            const float* q = qs + warp * d;
            for (int c = 0; c < d; ++c) dot = fmaf(q[c], kt[c * (ATT_KT + 1) + lane], dot);
            sc[warp * Tp + j0 + lane] = dot * inv_sqrt_d;
        }
    }
    __syncwarp();
    const float mi = active ? mb[i] : 0.f;
    float outv[MAXD / 32];
#pragma unroll
    for (int u = 0; u < MAXD / 32; ++u) outv[u] = 0.f;
    if (active) {
        // ---- relative-key logits on the +-window band (transformer.py:132-138)
        if (window >= 0 && lane < nrel) {
            const int j = i + lane - window;
            if (j >= 0 && j < T) {
                float dot = 0.f;
                const float* q = qs + warp * d;
                const float* e = ek + lane * d;
                for (int c = 0; c < d; ++c) dot = fmaf(q[c], e[c], dot);
                sc[warp * Tp + j] += dot * inv_sqrt_d;
            }
        }
        __syncwarp();
        // ---- masked_fill(mask == 0, -1e4), softmax over keys (transformer.py:144-149)
        float mx = -INFINITY;
        for (int j = lane; j < T; j += 32) {
            float s = sc[warp * Tp + j];
            if (mi * mb[j] == 0.f) s = -1e4f;
            sc[warp * Tp + j] = s;
            mx = fmaxf(mx, s);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        float sum = 0.f;
        for (int j = lane; j < T; j += 32) {
            const float e = expf(sc[warp * Tp + j] - mx);
            sc[warp * Tp + j] = e;
            sum += e;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        const float inv = 1.f / sum;
        for (int j = lane; j < Tp; j += 32) sc[warp * Tp + j] = (j < T) ? sc[warp * Tp + j] * inv : 0.f;
        __syncwarp();
    }
    // ---- out = p.v (+ relative values)
    float* vt = kt;  // [ATT_KT][d+1]
    for (int j0 = 0; j0 < T; j0 += ATT_KT) {
        __syncthreads();
        for (int i0b = 0; i0b < d * ATT_KT; i0b += 8 * 32 * ATT_Q) {
            float tmp[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int idx = i0b + u * 32 * ATT_Q + tid;
                const int c = idx / ATT_KT, jj = idx - c * ATT_KT, j = j0 + jj;
                tmp[u] = (idx < d * ATT_KT && j < T) ? vb[(size_t)c * T + j] : 0.f;
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int idx = i0b + u * 32 * ATT_Q + tid;
                const int c = idx / ATT_KT, jj = idx - c * ATT_KT;
                if (idx < d * ATT_KT) vt[jj * (d + 1) + c] = tmp[u];
            }
        }
        __syncthreads();
        if (active) {
            const float* p = sc + warp * Tp + j0;
#pragma unroll
            for (int u = 0; u < MAXD / 32; ++u) {
                const int c = lane + 32 * u;
                if (c < d) {
                    float a = outv[u];
                    for (int jj = 0; jj < ATT_KT; ++jj) a = fmaf(p[jj], vt[jj * (d + 1) + c], a);
                    outv[u] = a;
                }
            }
        }
    }
    if (active) {
#pragma unroll
        for (int u = 0; u < MAXD / 32; ++u) {
            const int c = lane + 32 * u;
            if (c < d) {
                float a = outv[u];
                if (window >= 0)
                    for (int r = 0; r < nrel; ++r) {
                        const int j = i + r - window;
                        if (j >= 0 && j < T) a = fmaf(sc[warp * Tp + j], ev[r * d + c], a);
                    }
                out[((size_t)b * C + h * d + c) * T + i] = a;
            }
        }
    }
}

// out[b,:,t] = LayerNorm_c(x[b,:,t] + y[b,:,t]) * gamma + beta  (* mask[b,t]);  block (32 t) x (8 channel groups)
__global__ void __launch_bounds__(256) add_layernorm_kernel(const float* x, const float* y, const float* gamma,
                                                            const float* beta, const float* mask, float* out, int C,
                                                            int T, float eps) {
    __shared__ float red[8][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int t = blockIdx.x * 32 + tx, b = blockIdx.y;
    const bool ok = t < T;
    const size_t base = (size_t)b * C * T + t;
    float s = 0.f;
    if (ok) for (int c = ty; c < C; c += 8) s += x[base + (size_t)c * T] + (y ? y[base + (size_t)c * T] : 0.f);
    red[ty][tx] = s;
    __syncthreads();
    float mean = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) mean += red[k][tx];
    mean /= (float)C;
    __syncthreads();
    float v = 0.f;
    if (ok) for (int c = ty; c < C; c += 8) {
        const float d = x[base + (size_t)c * T] + (y ? y[base + (size_t)c * T] : 0.f) - mean;
        v += d * d;
    }
    red[ty][tx] = v;
    __syncthreads();
    float var = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) var += red[k][tx];
    var /= (float)C;
    const float rstd = rsqrtf(var + eps);
    if (!ok) return;
    const float m = mask ? mask[(size_t)b * T + t] : 1.f;
    for (int c = ty; c < C; c += 8) {
        const float d = x[base + (size_t)c * T] + (y ? y[base + (size_t)c * T] : 0.f) - mean;
        out[base + (size_t)c * T] = (d * rstd * gamma[c] + beta[c]) * m;
    }
}

}  // namespace

int launch_add_layernorm(const float* x, const float* y, const float* gamma, const float* beta, const float* mask,
                         float* out, int B, int C, int T, float eps, cudaStream_t st) {
    if (B == 0 || T == 0) return 0;
    dim3 grid((T + 31) / 32, B);
    add_layernorm_kernel<<<grid, 256, 0, st>>>(x, y, gamma, beta, mask, out, C, T, eps);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

int launch_embed(const long long* tokens, const long long* lengths, const float* emb, const float* lang_emb, int B,
                 int T, int hidden, int C, float* x, float* x_mask, cudaStream_t st, bool scale_sqrt_hidden) {
    dim3 grid((T + 127) / 128, C, B);
    embed_kernel<<<grid, 128, 0, st>>>(tokens, lengths, emb, lang_emb, x, x_mask, T, hidden, C,
                                       scale_sqrt_hidden ? sqrtf((float)hidden) : 1.f);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

int launch_attention(const float* qkv, const float* x_mask, const float* rel_k, const float* rel_v, float* out, int B,
                     int C, int T, int num_heads, int window, cudaStream_t st) {
    B200_REQUIRE(num_heads >= 1 && C >= num_heads, "attention: %d channels in %d heads", C, num_heads);
    const int d = C / num_heads;
    B200_REQUIRE(C % num_heads == 0 && d <= ATT_MAXD_WIDE, "attention: head dim %d (C=%d, %d heads) not supported", d, C,
                 num_heads);
    B200_REQUIRE(window < 0 || (rel_k && rel_v && 2 * window + 1 <= 32), "attention: bad relative window");
    if (B == 0 || T == 0) return 0;
    const int Tp = (T + 31) & ~31;
    const int nrel = window < 0 ? 0 : 2 * window + 1;
    const size_t att_smem = sizeof(float) * ((size_t)ATT_Q * d + (size_t)ATT_Q * Tp + (size_t)(ATT_KT + 1) * (d + 1) +
                                             (size_t)2 * nrel * d);
    B200_REQUIRE(att_smem <= 200 * 1024, "attention: T=%d too long for the attention kernel", T);
    static DeviceOnce attr_once;
    if (int rc0 = device_once(attr_once, nullptr, [](int) -> int {
            B200_CUDA_OK(cudaFuncSetAttribute(rel_attention_kernel<ATT_MAXD>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                              200 * 1024));
            B200_CUDA_OK(cudaFuncSetAttribute(rel_attention_kernel<ATT_MAXD_WIDE>,
                                              cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
            return 0;
        })) return rc0;
    dim3 grid((T + ATT_Q - 1) / ATT_Q, num_heads, B);
    // heads up to 256 channels keep the narrow instantiation (fewer registers per lane)
    auto kern = d <= ATT_MAXD ? rel_attention_kernel<ATT_MAXD> : rel_attention_kernel<ATT_MAXD_WIDE>;
    kern<<<grid, 32 * ATT_Q, att_smem, st>>>(qkv, x_mask, rel_k, rel_v, out, C, T, d, window, 1.f / sqrtf((float)d));
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

int RelPosTransformer::init(int channels, int ffn_channels, int kernel_size, int num_heads, int window_size,
                            float ln_eps, int num_layers, WeightList& wl) {
    C = channels; F = ffn_channels; heads = num_heads; window = window_size; eps = ln_eps;
    const int K = kernel_size, d = C / heads;
    const int nrel = 2 * window + 1;
    int rc;
    layers.resize(num_layers);
    for (int l = 0; l < num_layers; ++l) {
        Layer& L = layers[l];
        if (window >= 0) {
            if ((rc = upload(L.rel_k, wl.take(), (size_t)nrel * d))) return rc;
            if ((rc = upload(L.rel_v, wl.take(), (size_t)nrel * d))) return rc;
        }
        // fused QKV: rows [q | k | v]
        std::vector<float> wq((size_t)3 * C * C), bq((size_t)3 * C);
        for (int s = 0; s < 3; ++s) {
            const float *sw = wl.take(), *sb = wl.take();
            B200_REQUIRE(sw && sb, "rel_pos_transformer: null q / k / v weight or bias");
            memcpy(wq.data() + (size_t)s * C * C, sw, sizeof(float) * C * C);
            memcpy(bq.data() + (size_t)s * C, sb, sizeof(float) * C);
        }
        if ((rc = pack_conv(L.qkv, wq.data(), bq.data(), 3 * C, C, 1, 1, 0))) return rc;
        const float *ow = wl.take(), *ob = wl.take();
        if ((rc = pack_conv(L.o, ow, ob, C, C, 1, 1, 0))) return rc;
        if ((rc = upload(L.ln1_g, wl.take(), C))) return rc;
        if ((rc = upload(L.ln1_b, wl.take(), C))) return rc;
        // FeedForwardNetwork._same_padding: pad_l = (k-1)//2 (transformer.py:307-313)
        const float *f1w = wl.take(), *f1b = wl.take();
        if ((rc = pack_conv(L.ffn1, f1w, f1b, F, C, K, 1, (K - 1) / 2))) return rc;
        const float *f2w = wl.take(), *f2b = wl.take();
        if ((rc = pack_conv(L.ffn2, f2w, f2b, C, F, K, 1, (K - 1) / 2))) return rc;
        if ((rc = upload(L.ln2_g, wl.take(), C))) return rc;
        if ((rc = upload(L.ln2_b, wl.take(), C))) return rc;
    }
    return 0;
}

struct RelPosWs { float *qkv, *att, *yb, *hb; };
static RelPosWs relpos_carve(const RelPosTransformer& m, Arena& ar, int B, int T) {
    RelPosWs w;
    w.qkv = ar.f32((size_t)B * 3 * m.C * T);
    w.att = ar.f32((size_t)B * m.C * T);
    w.yb = ar.f32((size_t)B * m.C * T);
    w.hb = ar.f32((size_t)B * m.F * T);
    return w;
}

size_t RelPosTransformer::workspace_bytes(int B, int T) const {
    return arena_size([&](Arena& ar) { relpos_carve(*this, ar, B, T); });
}

int RelPosTransformer::forward(float* x, const float* x_mask, int B, int T, void* ws, size_t ws_bytes,
                               cudaStream_t st) const {
    Arena ar(ws, ws_bytes);
    const RelPosWs w = relpos_carve(*this, ar, B, T);
    B200_REQUIRE(ar.ok(), "rel_pos_transformer: workspace of %zu bytes is too small", ws_bytes);
    float *qkv = w.qkv, *att = w.att, *yb = w.yb, *hb = w.hb;
    int rc;
    for (const Layer& L : layers) {
        {   // q,k,v = conv_{q,k,v}(x)       (x is already masked: the caller / previous norm2 epilogue)
            ConvIO io;
            io.x = dense(x, C, T); io.Tin = T;
            io.y = dense(qkv, 3 * C, T); io.Tout = T; io.B = B;
            if ((rc = launch_conv(L.qkv, io, st))) return rc;
        }
        if ((rc = launch_attention(qkv, x_mask, L.rel_k, L.rel_v, att, B, C, T, heads, window, st))) return rc;
        {   // y = conv_o(att)
            ConvIO io;
            io.x = dense(att, C, T); io.Tin = T;
            io.y = dense(yb, C, T); io.Tout = T; io.B = B;
            if ((rc = launch_conv(L.o, io, st))) return rc;
        }
        if ((rc = launch_add_layernorm(x, yb, L.ln1_g, L.ln1_b, nullptr, x, B, C, T, eps, st))) return rc;
        {   // h = relu(conv_1(pad(x * mask)))
            ConvIO io;
            io.x = dense(x, C, T); io.Tin = T; io.xmask = {x_mask, T};
            io.y = dense(hb, F, T); io.Tout = T; io.B = B;
            io.act = ACT_RELU;
            if ((rc = launch_conv(L.ffn1, io, st))) return rc;
        }
        {   // y = conv_2(pad(h * mask)) * mask
            ConvIO io;
            io.x = dense(hb, F, T); io.Tin = T; io.xmask = {x_mask, T};
            io.y = dense(yb, C, T); io.Tout = T; io.B = B;
            io.ymask = {x_mask, T}; io.flags = EPI_MASK_POST;
            if ((rc = launch_conv(L.ffn2, io, st))) return rc;
        }
        // x = norm2(x + y); the next layer and the stack's output (transformer.py:419, :431) use x * mask -> fold the
        // mask here
        if ((rc = launch_add_layernorm(x, yb, L.ln2_g, L.ln2_b, x_mask, x, B, C, T, eps, st))) return rc;
    }
    return 0;
}

// weights: emb [V,hidden]; per layer: see RelPosTransformer::init (window w); proj.w [2*out,C,1], proj.b
int TextEncoder::init(const b200tts_text_encoder_config& cfg, const float* const* w, int nw) {
    c = cfg;
    C = c.hidden_channels + c.language_emb_dim;
    B200_REQUIRE(c.num_heads >= 1 && C % c.num_heads == 0, "text_encoder: channels %d not divisible by heads %d", C,
                 c.num_heads);
    const int d = C / c.num_heads;
    B200_REQUIRE(d <= ATT_MAXD, "text_encoder: head dim %d > %d", d, ATT_MAXD);
    B200_REQUIRE(c.rel_attn_window_size >= 0 && 2 * c.rel_attn_window_size + 1 <= 32, "text_encoder: bad window");
    WeightList wl(w, nw);
    int rc;
    if ((rc = upload(emb, wl.take(), (size_t)c.n_vocab * c.hidden_channels))) return rc;
    if ((rc = tf.init(C, c.hidden_channels_ffn, c.kernel_size, c.num_heads, c.rel_attn_window_size, 1e-5f,
                      c.num_layers, wl)))
        return rc;
    const float *pw = wl.take(), *pb = wl.take();
    if ((rc = pack_conv(proj, pw, pb, 2 * c.out_channels, C, 1, 1, 0))) return rc;
    return wl.finish("text_encoder");
}

// the whole workspace is the transformer's
size_t TextEncoder::workspace_bytes(int B, int T) const { return tf.workspace_bytes(B, T); }

int TextEncoder::forward(const long long* tokens, const long long* lengths, const float* lang_emb, int B, int T,
                         float* x, float* stats, float* x_mask, void* ws, size_t ws_bytes, cudaStream_t st) const {
    B200_REQUIRE(tokens && lengths && x && stats && x_mask && ws, "text_encoder_forward: null pointer");
    B200_REQUIRE((c.language_emb_dim > 0) == (lang_emb != nullptr), "text_encoder_forward: lang_emb mismatch");
    const size_t need = workspace_bytes(B, T);
    B200_REQUIRE(ws_bytes >= need, "text_encoder_forward: workspace of %zu bytes, %zu needed", ws_bytes, need);
    if (B == 0 || T == 0) return 0;
    int rc;
    if ((rc = launch_embed(tokens, lengths, emb, lang_emb, B, T, c.hidden_channels, C, x, x_mask, st))) return rc;
    if ((rc = tf.forward(x, x_mask, B, T, ws, ws_bytes, st))) return rc;
    {   // stats = proj(x) * mask  -> [m_p | logs_p]
        ConvIO io;
        io.x = dense(x, C, T); io.Tin = T;
        io.y = dense(stats, 2 * c.out_channels, T); io.Tout = T; io.B = B;
        io.ymask = {x_mask, T}; io.flags = EPI_MASK_POST;
        if ((rc = launch_conv(proj, io, st))) return rc;
    }
    return 0;
}

}  // namespace b200tts
