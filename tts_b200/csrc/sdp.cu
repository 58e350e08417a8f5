// Stochastic duration predictor, reverse (inference) direction.
// Reference: TTS/tts/layers/vits/stochastic_duration_predictor.py:222-239,285-294 (SDP.forward reverse),
//            :46-63 (DilatedDepthSeparableConv), :66-84 (ElementwiseAffine), :120-147 (ConvFlow),
//            TTS/tts/layers/vits/transforms.py:51-184 (unconstrained rational-quadratic spline, inverse).
// FLOP-wise negligible (1 MFLOP/token) but ~40 tiny library kernels per spline call in the reference;
// here: one fused kernel per DDSConv half-layer and ONE kernel for the whole spline inverse.
#include <math.h>

#include "engines.cuh"

namespace b200tts {

namespace {

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752440f)); }

// block = 32 time steps x 8 channel groups; per-column LayerNorm statistics reduced through shared memory
__device__ __forceinline__ void column_stats(float partial_sum, float (*red)[33], int tx, int ty, int C, float& mean) {
    red[ty][tx] = partial_sum;
    __syncthreads();
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) s += red[k][tx];
    mean = s / (float)C;
    __syncthreads();
}

// y = GELU(LN(depthwise_conv_k(x * mask)))          (DDSConv first half, sdp.py:55-57)
// Each thread owns one time step and every 8th channel; its <= DDS_MAXC values stay in registers between the conv,
// the two LayerNorm reductions and the store (all global loads of a pass are issued before the first use: with 64
// CTAs per launch this kernel is pure load latency).
constexpr int DDS_MAXC = 32;   // channels per thread (C <= 256)

__global__ void __launch_bounds__(256) dds_sep_ln_gelu_kernel(const float* __restrict__ x, const float* __restrict__ mask,
                                                             const float* __restrict__ w, const float* __restrict__ bias,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta,
                                                             float* __restrict__ y, int C, int T, int K, int dil) {
    __shared__ float red[8][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int t = blockIdx.x * 32 + tx, b = blockIdx.y;
    const bool ok = t < T;
    const size_t base = (size_t)b * C * T;
    const float* mb = mask + (size_t)b * T;
    const int pad = (K * dil - dil) / 2;
    float av[DDS_MAXC];
#pragma unroll
    for (int u = 0; u < DDS_MAXC; ++u) av[u] = 0.f;
    if (ok) {
#pragma unroll
        for (int u = 0; u < DDS_MAXC; ++u) { const int c = ty + 8 * u; if (c < C) av[u] = bias[c]; }
        for (int k = 0; k < K; ++k) {            // same accumulation order as before: taps outer-to-inner per channel
            const int ti = t + k * dil - pad;
            if (ti < 0 || ti >= T) continue;
            const float mk = mb[ti];
            float xv[DDS_MAXC];
#pragma unroll
            for (int u = 0; u < DDS_MAXC; ++u) { const int c = ty + 8 * u; xv[u] = (c < C) ? x[base + (size_t)c * T + ti] : 0.f; }
#pragma unroll
            for (int u = 0; u < DDS_MAXC; ++u) { const int c = ty + 8 * u; if (c < C) av[u] = fmaf(w[c * K + k], xv[u] * mk, av[u]); }
        }
    }
    float s = 0.f;
#pragma unroll
    for (int u = 0; u < DDS_MAXC; ++u) if (ty + 8 * u < C) s += av[u];
    float mean, var;
    column_stats(s, red, tx, ty, C, mean);
    float v = 0.f;
#pragma unroll
    for (int u = 0; u < DDS_MAXC; ++u) if (ty + 8 * u < C) { const float d = av[u] - mean; v += d * d; }
    column_stats(v, red, tx, ty, C, var);
    if (!ok) return;
    const float rstd = rsqrtf(var + 1e-5f);
#pragma unroll
    for (int u = 0; u < DDS_MAXC; ++u) {
        const int c = ty + 8 * u;
        if (c < C) y[base + (size_t)c * T + t] = gelu_erf((av[u] - mean) * rstd * gamma[c] + beta[c]);
    }
}

// x = x + GELU(LN(y))  (* mask after the last layer)        (DDSConv second half, sdp.py:59-63)
__global__ void __launch_bounds__(256) dds_ln_gelu_res_kernel(float* __restrict__ x, const float* __restrict__ y,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta,
                                                             const float* __restrict__ mask, int C, int T, int apply_mask) {
    __shared__ float red[8][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int t = blockIdx.x * 32 + tx, b = blockIdx.y;
    const bool ok = t < T;
    const size_t base = (size_t)b * C * T + t;
    float yv[DDS_MAXC], xv[DDS_MAXC];
#pragma unroll
    for (int u = 0; u < DDS_MAXC; ++u) {
        const int c = ty + 8 * u;
        const bool in = ok && c < C;
        yv[u] = in ? y[base + (size_t)c * T] : 0.f;
        xv[u] = in ? x[base + (size_t)c * T] : 0.f;
    }
    float s = 0.f;
#pragma unroll
    for (int u = 0; u < DDS_MAXC; ++u) if (ty + 8 * u < C) s += yv[u];
    float mean, var;
    column_stats(s, red, tx, ty, C, mean);
    float v = 0.f;
#pragma unroll
    for (int u = 0; u < DDS_MAXC; ++u) if (ty + 8 * u < C) { const float d = yv[u] - mean; v += d * d; }
    column_stats(v, red, tx, ty, C, var);
    if (!ok) return;
    const float rstd = rsqrtf(var + 1e-5f);
    const float m = apply_mask ? mask[(size_t)b * T + t] : 1.f;
#pragma unroll
    for (int u = 0; u < DDS_MAXC; ++u) {
        const int c = ty + 8 * u;
        if (c < C) x[base + (size_t)c * T] = (xv[u] + gelu_erf((yv[u] - mean) * rstd * gamma[c] + beta[c])) * m;
    }
}

// h[b,c,t] = w[c]*z0[b,t] + bias[c] + g[b,c,t]        (ConvFlow.pre on one channel, fused with DDSConv's x+g)
__global__ void convflow_pre_kernel(const float* z, int ch0, const float* w, const float* bias, const float* g,
                                    float* h, int C, int T) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x, c = blockIdx.y, b = blockIdx.z;
    if (t >= T) return;
    const float z0 = z[((size_t)b * 2 + ch0) * T + t];
    const size_t i = ((size_t)b * C + c) * T + t;
    h[i] = fmaf(w[c], z0, bias[c]) + g[i];
}

__global__ void scale_copy_kernel(const float* src, float* dst, float scale, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = src[i] * scale;
}

// ElementwiseAffine reverse after a channel flip (sdp.py:83): logical channel l lives in physical ch[l]
__global__ void affine_reverse_kernel(float* z, const float* mask, const float* translation, const float* log_scale,
                                      int ch0, int ch1, int T) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (t >= T) return;
    const float m = mask[(size_t)b * T + t];
    float* z0 = z + ((size_t)b * 2 + ch0) * T + t;
    float* z1 = z + ((size_t)b * 2 + ch1) * T + t;
    *z0 = (*z0 - translation[0]) * expf(-log_scale[0]) * m;
    *z1 = (*z1 - translation[1]) * expf(-log_scale[1]) * m;
}

constexpr int NB_MAX = 16;

// Inverse rational-quadratic spline with linear tails, one thread per (b,t); hp [B, 3*nb-1, T] = proj(h)*mask.
// Follows transforms.py:62-74 (tails), :118-140 (knots), :45-47,142 (bin search), :159-171 (quadratic root).
__global__ void spline_inverse_kernel(float* z, const float* hp, const float* mask, int ch0, int ch1, int T, int nb,
                                      float sqrt_h, float tail_bound, float deriv_const, int* err_flag) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (t >= T) return;
    const float m = mask[(size_t)b * T + t];
    float* z0 = z + ((size_t)b * 2 + ch0) * T + t;
    float* z1 = z + ((size_t)b * 2 + ch1) * T + t;
    const float x = *z1;
    float outv = x;
    if (x >= -tail_bound && x <= tail_bound) {
        const float* p = hp + (size_t)b * (3 * nb - 1) * T + t;
        // constants evaluated like the reference (python doubles rounded to fp32); mul/add kept unfused
        const float min_w = 1e-3f, min_h = 1e-3f, min_d = 1e-3f;
        const float sc_w = (float)(1.0 - 1e-3 * (double)nb), sc_h = sc_w;
        const float span = 2.f * tail_bound;
        float cw[NB_MAX + 1], chh[NB_MAX + 1];
        {   // widths: softmax -> floor -> cumsum -> affine to [-tb, tb], end points forced
            float u[NB_MAX], mx = -INFINITY, sum = 0.f;
            for (int i = 0; i < nb; ++i) { u[i] = p[(size_t)i * T] / sqrt_h; mx = fmaxf(mx, u[i]); }
            for (int i = 0; i < nb; ++i) { u[i] = expf(u[i] - mx); sum += u[i]; }
            float run = 0.f;
            cw[0] = -tail_bound;
            for (int i = 0; i < nb; ++i) {
                const float wi = __fadd_rn(min_w, __fmul_rn(sc_w, u[i] / sum));
                run = __fadd_rn(run, wi);
                cw[i + 1] = __fadd_rn(__fmul_rn(span, run), -tail_bound);
            }
            cw[nb] = tail_bound;
        }
        {
            float u[NB_MAX], mx = -INFINITY, sum = 0.f;
            for (int i = 0; i < nb; ++i) { u[i] = p[(size_t)(nb + i) * T] / sqrt_h; mx = fmaxf(mx, u[i]); }
            for (int i = 0; i < nb; ++i) { u[i] = expf(u[i] - mx); sum += u[i]; }
            float run = 0.f;
            chh[0] = -tail_bound;
            for (int i = 0; i < nb; ++i) {
                const float hi = __fadd_rn(min_h, __fmul_rn(sc_h, u[i] / sum));
                run = __fadd_rn(run, hi);
                chh[i + 1] = __fadd_rn(__fmul_rn(span, run), -tail_bound);
            }
            chh[nb] = tail_bound;
        }
        int bin = -1;
        for (int i = 0; i <= nb; ++i) {
            const float loc = (i == nb) ? chh[i] + 1e-6f : chh[i];
            bin += (x >= loc) ? 1 : 0;
        }
        bin = min(max(bin, 0), nb - 1);
        auto deriv = [&](int i) {  // padded unnormalised derivatives: index 0 and nb are the tail constant
            const float ud = (i == 0 || i == nb) ? deriv_const : p[(size_t)(2 * nb + i - 1) * T];
            const float sp = (ud > 20.f) ? ud : log1pf(expf(ud));
            return min_d + sp;
        };
        const float in_cw = cw[bin], in_w = cw[bin + 1] - cw[bin];
        const float in_ch = chh[bin], in_h = chh[bin + 1] - chh[bin];
        const float delta = in_h / in_w;
        const float d0 = deriv(bin), d1 = deriv(bin + 1);
        const float dx = x - in_ch;
        const float s2 = __fadd_rn(__fadd_rn(d0, d1), -__fmul_rn(2.f, delta));
        const float qa = __fadd_rn(__fmul_rn(dx, s2), __fmul_rn(in_h, __fadd_rn(delta, -d0)));
        const float qb = __fadd_rn(__fmul_rn(in_h, d0), -__fmul_rn(dx, s2));
        const float qc = __fmul_rn(-delta, dx);
        const float disc = __fadd_rn(__fmul_rn(qb, qb), -__fmul_rn(__fmul_rn(4.f, qa), qc));
        if (!(disc >= 0.f)) atomicExch(err_flag, 1);   // the reference asserts here (transforms.py:168)
        const float root = (2.f * qc) / (-qb - sqrtf(fmaxf(disc, 0.f)));
        outv = __fadd_rn(__fmul_rn(root, in_w), in_cw);
    }
    *z0 = *z0 * m;       // torch.cat([x0, x1], 1) * x_mask  (sdp.py:143)
    *z1 = outv * m;
}

}  // namespace

// ------------------------------------------------------------------ deterministic duration predictor (use_sdp=False)
// Reference: TTS/tts/layers/glow_tts/duration_predictor.py:44-69 (LayerNorm eps 1e-4: generic/normalization.py:5-28)
namespace {
__global__ void add_chan_bias_kernel(const float* x, const float* cb, long long cb_bs, float* out, int C, int T) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x, c = blockIdx.y, b = blockIdx.z;
    if (t >= T) return;
    const size_t i = ((size_t)b * C + c) * T + t;
    out[i] = x[i] + cb[(size_t)b * cb_bs + c];
}
}  // namespace

// weights: conv_1.w [F,Cin,k], .b, norm_1.gamma [1,F,1], .beta, conv_2.w [F,F,k], .b, norm_2.gamma, .beta,
//          proj.w [1,F,1], .b, [cond.w [Cin,cond,1], .b], [cond_lang.w, .b]
int DurPred::init(const b200tts_duration_predictor_config& cfg, const float* const* w, int nw) {
    WeightList wl(w, nw);
    if (int rc = init(cfg, wl)) return rc;
    return wl.finish("duration_predictor");
}

int DurPred::init(const b200tts_duration_predictor_config& cfg, WeightList& wl) {
    c = cfg;
    const int Cin = c.in_channels + c.language_emb_dim, F = c.hidden_channels, K = c.kernel_size;
    int rc;
    const float *c1w = wl.take(), *c1b = wl.take();
    if ((rc = pack_conv(conv1, c1w, c1b, F, Cin, K, 1, K / 2))) return rc;
    if ((rc = upload(g1, wl.take(), F))) return rc;
    if ((rc = upload(b1, wl.take(), F))) return rc;
    const float *c2w = wl.take(), *c2b = wl.take();
    if ((rc = pack_conv(conv2, c2w, c2b, F, F, K, 1, K / 2))) return rc;
    if ((rc = upload(g2, wl.take(), F))) return rc;
    if ((rc = upload(b2, wl.take(), F))) return rc;
    const float *pw = wl.take(), *pb = wl.take();
    if ((rc = pack_conv(proj, pw, pb, 1, F, 1, 1, 0))) return rc;
    if (c.cond_channels > 0) {
        const float *gw = wl.take(), *gb = wl.take();
        if ((rc = pack_conv(cond, gw, gb, Cin, c.cond_channels, 1, 1, 0))) return rc;
    }
    if (c.language_emb_dim > 0) {
        const float *lw = wl.take(), *lb = wl.take();
        if ((rc = pack_conv(cond_lang, lw, lb, Cin, c.language_emb_dim, 1, 1, 0))) return rc;
    }
    return 0;
}

// the conditioned input, the two hidden tensors and the per-utterance bias (row pitch cpad)
struct DurPredWs { float *xin, *h1, *h2, *cv; int cpad; };
static DurPredWs durpred_carve(const DurPred& m, Arena& ar, int B, int T) {
    DurPredWs w;
    w.xin = ar.f32((size_t)B * (m.c.in_channels + m.c.language_emb_dim) * T);
    w.h1 = ar.f32((size_t)B * m.c.hidden_channels * T);
    w.h2 = ar.f32((size_t)B * m.c.hidden_channels * T);
    w.cpad = std::max(std::max(m.cond.RowsPad, m.cond_lang.RowsPad), 64);
    w.cv = ar.f32((size_t)B * w.cpad + 64);
    return w;
}

size_t DurPred::workspace_bytes(int B, int T) const {
    return arena_size([&](Arena& ar) { durpred_carve(*this, ar, B, T); });
}

int DurPred::forward(const float* x, const float* mask, const float* g, const float* lang_emb, int B, int T,
                     float* logw, void* ws, size_t ws_bytes, cudaStream_t st) const {
    B200_REQUIRE(x && mask && logw && ws, "duration_predictor: null pointer");
    const size_t need = workspace_bytes(B, T);
    B200_REQUIRE(ws_bytes >= need, "duration_predictor: workspace of %zu bytes, %zu needed", ws_bytes, need);
    if (B == 0 || T == 0) return 0;
    const int Cin = c.in_channels + c.language_emb_dim, F = c.hidden_channels;
    Arena ar(ws, ws_bytes);
    const DurPredWs w = durpred_carve(*this, ar, B, T);
    float *xin = w.xin, *h1 = w.h1, *h2 = w.h2, *cv = w.cv;
    const int cpad = w.cpad;
    int rc;
    const float* cur = x;
    const bool has_g = c.cond_channels > 0 && g, has_l = c.language_emb_dim > 0 && lang_emb;
    if (has_g || has_l) {       // x = x + cond(g) (+ cond_lang(lang_emb)) : per-utterance channel bias on the INPUT
        if (has_g && (rc = launch_conv_vec(cond, g, cv, cpad, B, false, st))) return rc;
        if (has_l && (rc = launch_conv_vec(cond_lang, lang_emb, cv, cpad, B, has_g, st))) return rc;
        dim3 grid((T + 127) / 128, Cin, B);
        add_chan_bias_kernel<<<grid, 128, 0, st>>>(x, cv, cpad, xin, Cin, T);
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
        cur = xin;
    }
    ConvIO io;   // conv1 and conv2 (ReLU, then LayerNorm), then proj: all read their input through the mask
    io.Tin = io.Tout = T; io.B = B; io.xmask = {mask, T}; io.act = ACT_RELU;
    io.x = dense(cur, Cin, T); io.y = dense(h1, F, T);
    if ((rc = launch_conv(conv1, io, st))) return rc;
    if ((rc = launch_add_layernorm(h1, nullptr, g1, b1, nullptr, h1, B, F, T, 1e-4f, st))) return rc;
    io.x = dense(h1, F, T); io.y = dense(h2, F, T);
    if ((rc = launch_conv(conv2, io, st))) return rc;
    if ((rc = launch_add_layernorm(h2, nullptr, g2, b2, nullptr, h2, B, F, T, 1e-4f, st))) return rc;
    io.x = dense(h2, F, T); io.y = dense(logw, 1, T); io.act = ACT_NONE;
    io.ymask = {mask, T}; io.flags = EPI_MASK_POST;
    return launch_conv(proj, io, st);
}

// per layer: sep.w [C,1,K], sep.b, 1x1.w [C,C,1], 1x1.b, norm1.gamma, norm1.beta, norm2.gamma, norm2.beta
int DDSConv::init(int channels, int kernel_size, int num_layers, WeightList& wl) {
    C = channels; K = kernel_size; L = num_layers;
    conv1x1.resize(L);
    sep_w.resize(L); sep_b.resize(L); g1.resize(L); b1.resize(L); g2.resize(L); b2.resize(L);
    int rc;
    for (int l = 0; l < L; ++l) {
        if ((rc = upload(sep_w[l], wl.take(), (size_t)C * K))) return rc;
        if ((rc = upload(sep_b[l], wl.take(), C))) return rc;
        const float *pw = wl.take(), *pb = wl.take();
        if ((rc = pack_conv(conv1x1[l], pw, pb, C, C, 1, 1, 0))) return rc;
        if ((rc = upload(g1[l], wl.take(), C))) return rc;
        if ((rc = upload(b1[l], wl.take(), C))) return rc;
        if ((rc = upload(g2[l], wl.take(), C))) return rc;
        if ((rc = upload(b2[l], wl.take(), C))) return rc;
    }
    return 0;
}

// x [B,C,T] updated in place; y1,y2 scratch [B,C,T]
int DDSConv::forward(float* x, const float* mask, int B, int T, float* y1, float* y2, cudaStream_t st) const {
    B200_REQUIRE(C <= 8 * DDS_MAXC, "DDSConv: %d channels exceed the kernel's register column (%d)", C, 8 * DDS_MAXC);
    dim3 grid((T + 31) / 32, B);
    int dil = 1, rc;
    for (int l = 0; l < L; ++l) {
        dds_sep_ln_gelu_kernel<<<grid, 256, 0, st>>>(x, mask, sep_w[l], sep_b[l], g1[l], b1[l], y1, C, T, K, dil);
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
        ConvIO io;
        io.x = dense(y1, C, T); io.Tin = T;
        io.y = dense(y2, C, T); io.Tout = T; io.B = B;
        if ((rc = launch_conv(conv1x1[l], io, st))) return rc;
        dds_ln_gelu_res_kernel<<<grid, 256, 0, st>>>(x, y2, g2[l], b2[l], mask, C, T, l == L - 1 ? 1 : 0);
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
        dil *= K;
    }
    return 0;
}

// weights: pre.w [H,in,1], pre.b, [cond.w,cond.b], [cond_lang.w,cond_lang.b], convs(3 layers x 8), proj.w, proj.b,
//          flows.0.translation [2], flows.0.log_scale [2],
//          for f = 1..num_flows: pre.w [H,1,1], pre.b, convs(3 x 8), proj.w [3*nb-1, H, 1], proj.b
int SDP::init(const b200tts_sdp_config& cfg, const float* const* w, int nw) {
    c = cfg;
    B200_REQUIRE(c.num_bins >= 1 && c.num_bins <= NB_MAX, "sdp: num_bins %d unsupported", c.num_bins);
    const int H = c.hidden_channels;
    WeightList wl(w, nw);
    int rc;
    const float *pw = wl.take(), *pb = wl.take();
    if ((rc = pack_conv(pre, pw, pb, H, c.in_channels + c.language_emb_dim, 1, 1, 0))) return rc;
    if (c.cond_channels > 0) {
        const float *gw = wl.take(), *gb = wl.take();
        if ((rc = pack_conv(cond, gw, gb, H, c.cond_channels, 1, 1, 0))) return rc;
    }
    if (c.language_emb_dim > 0) {
        const float *lw = wl.take(), *lb = wl.take();
        if ((rc = pack_conv(cond_lang, lw, lb, H, c.language_emb_dim, 1, 1, 0))) return rc;
    }
    if ((rc = convs.init(H, c.kernel_size, 3, wl))) return rc;
    const float *qw = wl.take(), *qb = wl.take();
    if ((rc = pack_conv(proj, qw, qb, H, H, 1, 1, 0))) return rc;
    if ((rc = upload(ea_t, wl.take(), 2))) return rc;
    if ((rc = upload(ea_ls, wl.take(), 2))) return rc;
    flows.resize(c.num_flows);
    for (int f = 0; f < c.num_flows; ++f) {
        CFlow& F = flows[f];
        if ((rc = upload(F.pre_w, wl.take(), H))) return rc;
        if ((rc = upload(F.pre_b, wl.take(), H))) return rc;
        if ((rc = F.convs.init(H, c.kernel_size, 3, wl))) return rc;
        const float *fw = wl.take(), *fb = wl.take();
        if ((rc = pack_conv(F.proj, fw, fb, 3 * c.num_bins - 1, H, 1, 1, 0))) return rc;
    }
    return wl.finish("sdp");
}

struct SdpWs { float *xc, *h, *y1, *y2, *z, *hp, *condv; };
static SdpWs sdp_carve(const SDP& m, Arena& ar, int B, int T) {
    const size_t bh = (size_t)B * m.c.hidden_channels * T;
    SdpWs w;
    w.xc = ar.f32(bh);
    w.h = ar.f32(bh);
    w.y1 = ar.f32(bh);
    w.y2 = ar.f32(bh);
    w.z = ar.f32((size_t)B * 2 * T);
    w.hp = ar.f32((size_t)B * (3 * m.c.num_bins - 1) * T);
    w.condv = ar.f32((size_t)B * std::max(std::max(m.cond.RowsPad, m.cond_lang.RowsPad), 64) + 64);
    return w;
}

size_t SDP::workspace_bytes(int B, int T) const {
    return arena_size([&](Arena& ar) { sdp_carve(*this, ar, B, T); });
}

int SDP::reverse(const float* x, const float* mask, const float* noise, const float* g, const float* lang_emb,
                 float noise_scale, int B, int T, float* logw, int* err_flag, void* ws, size_t ws_bytes,
                 cudaStream_t st) const {
    B200_REQUIRE(x && mask && noise && logw && ws, "sdp_reverse: null pointer");
    const size_t need = workspace_bytes(B, T);
    B200_REQUIRE(ws_bytes >= need, "sdp_reverse: workspace of %zu bytes, %zu needed", ws_bytes, need);
    if (B == 0 || T == 0) return 0;
    const int H = c.hidden_channels, nproj = 3 * c.num_bins - 1;
    Arena ar(ws, ws_bytes);
    const SdpWs w = sdp_carve(*this, ar, B, T);
    float *xc = w.xc, *h = w.h, *y1 = w.y1, *y2 = w.y2, *z = w.z, *hp = w.hp, *condv = w.condv;
    float* cv = nullptr;
    int rc;
    const bool has_g = c.cond_channels > 0 && g != nullptr;
    const bool has_l = c.language_emb_dim > 0 && lang_emb != nullptr;
    const int cpad = has_g ? cond.RowsPad : cond_lang.RowsPad;
    if (has_g || has_l) {   // per-utterance bias: cond(g) (+ cond_lang(lang_emb)) -> [B, H]
        cv = condv;
        if (has_g && (rc = launch_conv_vec(cond, g, cv, cpad, B, false, st))) return rc;
        if (has_l && (rc = launch_conv_vec(cond_lang, lang_emb, cv, cpad, B, has_g, st))) return rc;
    }
    {   // xc = pre(x) + cond
        ConvIO io;
        io.x = dense(x, pre.Cin, T); io.Tin = T;
        io.y = dense(xc, H, T); io.Tout = T; io.B = B;
        if (cv) io.cond = {cv, cpad};
        if ((rc = launch_conv(pre, io, st))) return rc;
    }
    if ((rc = convs.forward(xc, mask, B, T, y1, y2, st))) return rc;
    {   // xc = proj(xc) * mask     (into h, then swap roles)
        ConvIO io;
        io.x = dense(xc, H, T); io.Tin = T;
        io.y = dense(h, H, T); io.Tout = T; io.B = B;
        io.ymask = {mask, T}; io.flags = EPI_MASK_POST;
        if ((rc = launch_conv(proj, io, st))) return rc;
        float* tmp = xc; xc = h; h = tmp;
    }
    {
        const size_t n = (size_t)B * 2 * T;
        scale_copy_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(noise, z, noise_scale, n);
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
    }
    // flows = reversed(self.flows); drop the second-to-last (sdp.py:285-286): [F_n, ..., F_2, EA]
    int ch0 = 0, ch1 = 1;
    std::vector<int> order;
    for (int f = c.num_flows; f >= 2; --f) order.push_back(f);
    order.push_back(0);
    const float dconst = (float)log(exp(1.0 - 1e-3) - 1.0);
    for (int f : order) {
        { const int t = ch0; ch0 = ch1; ch1 = t; }  // z = torch.flip(z, [1])
        if (f == 0) {
            dim3 grid((T + 127) / 128, B);
            affine_reverse_kernel<<<grid, 128, 0, st>>>(z, mask, ea_t, ea_ls, ch0, ch1, T);
            count_launch();
            B200_CUDA_OK(cudaGetLastError());
            continue;
        }
        const CFlow& F = flows[f - 1];
        {
            dim3 grid((T + 127) / 128, H, B);
            convflow_pre_kernel<<<grid, 128, 0, st>>>(z, ch0, F.pre_w, F.pre_b, xc, h, H, T);
            count_launch();
            B200_CUDA_OK(cudaGetLastError());
        }
        if ((rc = F.convs.forward(h, mask, B, T, y1, y2, st))) return rc;
        {
            ConvIO io;
            io.x = dense(h, H, T); io.Tin = T;
            io.y = dense(hp, nproj, T); io.Tout = T; io.B = B;
            io.ymask = {mask, T}; io.flags = EPI_MASK_POST;
            if ((rc = launch_conv(F.proj, io, st))) return rc;
        }
        {
            dim3 grid((T + 127) / 128, B);
            spline_inverse_kernel<<<grid, 128, 0, st>>>(z, hp, mask, ch0, ch1, T, c.num_bins,
                                                        sqrtf((float)H), c.tail_bound, dconst, err_flag);
            count_launch();
            B200_CUDA_OK(cudaGetLastError());
        }
    }
    // logw = z[:, 0]  (logical channel 0)
    B200_CUDA_OK(cudaMemcpy2DAsync(logw, sizeof(float) * T, z + (size_t)ch0 * T, sizeof(float) * 2 * T,
                                   sizeof(float) * T, B, cudaMemcpyDeviceToDevice, st));
    return 0;
}

}  // namespace b200tts
