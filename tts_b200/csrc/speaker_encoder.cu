// H/ASP ResNet speaker encoder: waveform (or mel) windows -> d-vectors.
// Reference: TTS/encoder/models/resnet.py:8-198 (SELayer, SEBasicBlock, ResNetSpeakerEncoder.forward),
//            TTS/encoder/models/base_encoder.py:12-96 (PreEmphasis, MelSpectrogram front end, compute_embedding).
//
// Layout (see engines.cuh): every stage keeps its activations freq-major as [H + 2][C][L] with zero rows 0 and H + 1.
// The windows of a batch sit side by side on the time axis: window b owns columns [b*P, b*P + T) of its stage and the
// columns up to (b+1)*P are zero, so a conv's zero padding at a window's edge is the neighbour's zero gap.  Output row h
// of a 3x3 conv reads rows h-1..h+1, i.e. 3C consecutive channel rows: one launch of the 1D conv engine with
// Cin = 3C, K = 3, pad 1, batch index h and batch stride C*L.  Columns in the gaps are computed and then zeroed by the
// element-wise kernel that follows each conv.
//
// Stride 2 (first block of stages 2..4): freq stride 2 is a doubled batch stride.  Time stride 2 is a polyphase split:
// the last block of the previous stage writes its output as [H + 2][2][C][L'] (even columns, then odd columns, L' the
// next stage's row length), and out[q] = w0*odd[q-1] + w1*even[q] + w2*odd[q] is a K = 2, pad 1 conv over 6C channel
// rows.  P halves from stage to stage (P4 = T4 + 1), so window b's columns stay at b*P in every stage.
//
// BatchNorm: bn2 and downsample.1 follow a conv directly and are folded into it.  bn1 (stem and blocks) follows the
// ReLU, so it stays a per-channel affine after the activation; the zero padding the next conv reads is zero after
// that affine, which is why it cannot be folded forward either.  The head's BatchNorm1d also follows a ReLU, but the
// next layer is a 1x1 conv with no padding, into which it folds exactly.
//
// All reductions (instance norm, SE squeeze, attention pooling, l2 norm, window mean) run in a fixed order without
// atomics, so repeated runs are bit-identical.
#include <math.h>

#include "engines.cuh"

namespace b200tts {

namespace {

constexpr int NT = 256;

__device__ __forceinline__ float warp_sum(float v) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// deterministic block sum (NT threads); every thread gets the result
__device__ float block_sum(float v, float* red) {
    v = warp_sum(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) red[w] = v;
    __syncthreads();
    float s = 0.f;
    for (int i = 0; i < NT / 32; ++i) s += red[i];
    return s;
}

inline unsigned grid_for(long long n) { return (unsigned)std::max(1LL, std::min((n + NT - 1) / NT, 1LL << 30)); }

// pre-emphasis of each window at its own edges (reflect pad of one sample on the left): y[0] = p0*x[1] + p1*x[0]
__global__ void preemph_kernel(const float* x, const int* starts, int B, int N, float p0, float p1, float* y) {
    const long long n = (long long)B * N;
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < n; i += (long long)gridDim.x * NT) {
        const int b = (int)(i / N), t = (int)(i - (long long)b * N);
        const float* xb = x + starts[b];
        y[i] = p0 * xb[t == 0 ? 1 : t - 1] + p1 * xb[t];
    }
}

// log(x + 1e-6) (optional), InstanceNorm1d (biased variance, eps 1e-5) per (window, mel) row, written into row 1 + m,
// columns [b*P, b*P + T) of the stem input [H + 2][1][L].  One CTA per row.
__global__ void __launch_bounds__(NT) front_norm_kernel(const float* src, long long src_bs, const int* starts, int chan_stride,
                                                        int T, int log_input, float* out, int L, int P) {
    __shared__ float red[NT / 32];
    const int m = blockIdx.x, b = blockIdx.y;
    const float* s = src + (starts ? (long long)starts[b] : (long long)b * src_bs) + (long long)m * chan_stride;
    float acc = 0.f;
    for (int t = threadIdx.x; t < T; t += NT) {
        float v = s[t];
        if (log_input) v = logf(v + 1e-6f);
        acc += v;
    }
    const float mean = block_sum(acc, red) / (float)T;
    float acc2 = 0.f;
    for (int t = threadIdx.x; t < T; t += NT) {
        float v = s[t];
        if (log_input) v = logf(v + 1e-6f);
        acc2 += (v - mean) * (v - mean);
    }
    const float var = block_sum(acc2, red) / (float)T;
    const float inv = 1.f / sqrtf(var + 1e-5f);
    float* o = out + (long long)(1 + m) * L + (long long)b * P;
    for (int t = threadIdx.x; t < T; t += NT) {
        float v = s[t];
        if (log_input) v = logf(v + 1e-6f);
        o[t] = (v - mean) * inv;
    }
}

// in place over the interior rows of [H + 2][C][L]: y = relu(y) * s[c] + t[c] in the windows, 0 in the gaps
__global__ void relu_affine_kernel(float* y, int H, int C, int L, int P, int T, int B, const float* sc, const float* sh) {
    const long long n = (long long)H * C * L;
    float* base = y + (long long)C * L;
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < n; i += (long long)gridDim.x * NT) {
        const int col = (int)(i % L), c = (int)((i / L) % C);
        const bool valid = col < B * P && (col % P) < T;
        base[i] = valid ? fmaxf(base[i], 0.f) * sc[c] + sh[c] : 0.f;
    }
}

// SE squeeze, pass 1: part[(h*C + c)*B + b] = sum over the window's T columns of row (h, c).  One CTA per (h, c), one
// warp per window.
__global__ void __launch_bounds__(NT) se_partial_kernel(const float* y, int C, int L, int P, int T, int B, float* part) {
    const int hc = blockIdx.x, w = threadIdx.x >> 5, l = threadIdx.x & 31;
    const float* row = y + (long long)C * L + (long long)hc * L;
    for (int b = w; b < B; b += NT / 32) {
        float acc = 0.f;
        for (int t = l; t < T; t += 32) acc += row[(long long)b * P + t];
        acc = warp_sum(acc);
        if (l == 0) part[(long long)hc * B + b] = acc;
    }
}

// SE squeeze pass 2 + excitation MLP: scale[b][c] = sigmoid(W2 relu(W1 mean + b1) + b2).  One CTA per window.
__global__ void __launch_bounds__(NT) se_mlp_kernel(const float* part, int H, int C, int Cr, int T, int B, const float* w1,
                                                    const float* b1, const float* w2, const float* b2, float* scale) {
    extern __shared__ float sm[];
    float* s = sm;        // [C]
    float* z = sm + C;    // [Cr]
    const int b = blockIdx.x;
    const float inv = 1.f / ((float)H * (float)T);
    for (int c = threadIdx.x; c < C; c += NT) {
        float acc = 0.f;
        for (int h = 0; h < H; ++h) acc += part[((long long)h * C + c) * B + b];
        s[c] = acc * inv;
    }
    __syncthreads();
    for (int j = threadIdx.x; j < Cr; j += NT) {
        float acc = b1[j];
        for (int c = 0; c < C; ++c) acc += w1[(long long)j * C + c] * s[c];
        z[j] = fmaxf(acc, 0.f);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += NT) {
        float acc = b2[c];
        for (int j = 0; j < Cr; ++j) acc += w2[(long long)c * Cr + j] * z[j];
        scale[(long long)b * C + c] = 1.f / (1.f + expf(-acc));
    }
}

// block output: relu(y * scale[b][c] + res) in the windows, 0 in the gaps.  y / res: interior rows of [H + 2][C][L].
// Ln == 0: written in the same layout to out (may alias res).  Ln > 0: written polyphase to out [H + 2][2][C][Ln]
// (column 2j + p -> phase p, column j), the input layout of the next stage's stride-2 convs.
__global__ void block_out_kernel(const float* y, const float* res, const float* scale, int H, int C, int L, int P, int T,
                                 int B, float* out, int Ln) {
    const float* yb = y + (long long)C * L;
    const float* rb = res + (long long)C * L;
    if (Ln == 0) {
        const long long n = (long long)H * C * L;
        float* ob = out + (long long)C * L;
        for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < n; i += (long long)gridDim.x * NT) {
            const int col = (int)(i % L), c = (int)((i / L) % C);
            const int b = col / P;
            const bool valid = col < B * P && col - b * P < T;
            ob[i] = valid ? fmaxf(yb[i] * scale[(long long)b * C + c] + rb[i], 0.f) : 0.f;
        }
        return;
    }
    const long long n = (long long)H * 2 * C * Ln;
    float* ob = out + 2LL * C * Ln;
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < n; i += (long long)gridDim.x * NT) {
        const int j = (int)(i % Ln);
        long long r = i / Ln;
        const int c = (int)(r % C);
        r /= C;
        const int p = (int)(r & 1), h = (int)(r >> 1);
        const int col = 2 * j + p, b = col / P;
        const bool valid = col < B * P && col - b * P < T;
        float v = 0.f;
        if (valid) {
            const long long k = ((long long)h * C + c) * L + col;
            v = fmaxf(yb[k] * scale[(long long)b * C + c] + rb[k], 0.f);
        }
        ob[i] = v;
    }
}

// attention pooling: per (channel j = h*C + c, window b) softmax over the window's T columns of logits row c*Hf + h, then
// mu = sum x w and (ASP) sg = sqrt(max(sum x^2 w - mu^2, 1e-5)).  Written to pooled [out_dim][Bp] at the reference's
// channel index c*Hf + h (mu) and Hf*C + c*Hf + h (sg).  One warp per (j, b).
__global__ void __launch_bounds__(NT) attn_pool_kernel(const float* logits, const float* x, int Hf, int C, int L, int P,
                                                       int T, int B, int asp, float* pooled, int Bp) {
    const int j = blockIdx.x, b = blockIdx.y * (NT / 32) + (threadIdx.x >> 5), l = threadIdx.x & 31;
    if (b >= B) return;
    const int h = j / C, c = j - h * C, r = c * Hf + h;
    const float* lg = logits + (long long)r * L + (long long)b * P;   // the attention conv's rows are in reference order
    const float* xv = x + (long long)j * L + (long long)b * P;
    float m = -INFINITY;
    for (int t = l; t < T; t += 32) m = fmaxf(m, lg[t]);
    m = warp_max(m);
    float den = 0.f;
    for (int t = l; t < T; t += 32) den += expf(lg[t] - m);
    den = warp_sum(den);
    float mu = 0.f, s2 = 0.f;
    for (int t = l; t < T; t += 32) {
        const float w = expf(lg[t] - m) / den, v = xv[t];
        mu += v * w;
        s2 += v * v * w;
    }
    mu = warp_sum(mu);
    s2 = warp_sum(s2);
    if (l == 0) {
        pooled[(long long)r * Bp + b] = mu;
        if (asp) pooled[((long long)Hf * C + r) * Bp + b] = sqrtf(fmaxf(s2 - mu * mu, 1e-5f));
    }
}

// optional l2 norm of each window's embedding (F.normalize: x / max(|x|, 1e-12)), then the mean over each group of
// nw = B / groups consecutive windows.  y [D][Bp]; emb [groups][D].  One CTA per group.
__global__ void __launch_bounds__(NT) l2_mean_kernel(const float* y, int D, int Bp, int nw, int l2, float* emb) {
    extern __shared__ float den[];   // [nw]
    __shared__ float red[NT / 32];
    const int g = blockIdx.x;
    for (int w = 0; w < nw; ++w) {
        const int b = g * nw + w;
        float acc = 0.f;
        for (int k = threadIdx.x; k < D; k += NT) {
            const float v = y[(long long)k * Bp + b];
            acc += v * v;
        }
        const float ss = block_sum(acc, red);
        if (threadIdx.x == 0) den[w] = l2 ? fmaxf(sqrtf(ss), 1e-12f) : 1.f;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < D; k += NT) {
        float acc = 0.f;
        for (int w = 0; w < nw; ++w) {
            const float v = y[(long long)k * Bp + g * nw + w];
            acc += l2 ? v / den[w] : v;
        }
        emb[(long long)g * D + k] = acc / (float)nw;
    }
}

// dense copy of a stage's windows out of the padded layout: out [B][C][H][T].  Ln > 0: the source is polyphase.
__global__ void gather_kernel(const float* src, int H, int C, int L, int P, int T, int B, int Ln, float* out) {
    const long long n = (long long)B * C * H * T;
    for (long long i = blockIdx.x * (long long)NT + threadIdx.x; i < n; i += (long long)gridDim.x * NT) {
        const int t = (int)(i % T);
        long long r = i / T;
        const int h = (int)(r % H);
        r /= H;
        const int c = (int)(r % C), b = (int)(r / C);
        const int col = b * P + t;
        out[i] = Ln ? src[(((long long)(1 + h) * 2 + (col & 1)) * C + c) * Ln + (col >> 1)]
                    : src[((long long)(1 + h) * C + c) * L + col];
    }
}

struct BN { std::vector<double> s, t; };
BN bn_affine(const float* w, const float* b, const float* mean, const float* var, int C) {
    BN r;
    r.s.resize(C);
    r.t.resize(C);
    for (int c = 0; c < C; ++c) {
        r.s[c] = (double)w[c] / sqrt((double)var[c] + 1e-5);
        r.t[c] = (double)b[c] - (double)mean[c] * r.s[c];
    }
    return r;
}
int upload_d(DevBuf<float>& dst, const std::vector<double>& v) {
    std::vector<float> f(v.begin(), v.end());
    return upload(dst, f.data(), f.size());
}

// 3x3 conv (stride 1) as a 1D conv over 3 freq rows: W'[co][dy*Cin + ci][dx]
std::vector<float> repack3x3(const float* w, int Cout, int Cin, const std::vector<double>* fold) {
    std::vector<float> r((size_t)Cout * 3 * Cin * 3);
    for (int co = 0; co < Cout; ++co)
        for (int ci = 0; ci < Cin; ++ci)
            for (int dy = 0; dy < 3; ++dy)
                for (int dx = 0; dx < 3; ++dx) {
                    const double v = w[(((size_t)co * Cin + ci) * 3 + dy) * 3 + dx];
                    r[(((size_t)co * 3 + dy) * Cin + ci) * 3 + dx] = (float)(fold ? v * (*fold)[co] : v);
                }
    return r;
}
// 3x3 conv, stride (2, 2), over the polyphase input: channel ((dy*2 + p)*Cin + ci), K = 2, pad 1:
// even phase: tap 1 = dx 1 (tap 0 zero); odd phase: tap 0 = dx 0, tap 1 = dx 2
std::vector<float> repack3x3_s2(const float* w, int Cout, int Cin) {
    std::vector<float> r((size_t)Cout * 6 * Cin * 2, 0.f);
    for (int co = 0; co < Cout; ++co)
        for (int ci = 0; ci < Cin; ++ci)
            for (int dy = 0; dy < 3; ++dy) {
                const float* k = w + (((size_t)co * Cin + ci) * 3 + dy) * 3;
                float* e = &r[(((size_t)co * 6 + dy * 2 + 0) * Cin + ci) * 2];
                float* o = &r[(((size_t)co * 6 + dy * 2 + 1) * Cin + ci) * 2];
                e[1] = k[1];
                o[0] = k[0];
                o[1] = k[2];
            }
    return r;
}

struct Geo {   // per-stage geometry for B windows
    int H[5], C[5], T[5], P[5], L[5];   // index 1..4 = stages; 0 = stem input (H = input_dim, C = 1)
};
Geo geometry(const b200tts_speaker_encoder_config& c, int B, int T1) {
    Geo g;
    g.T[1] = T1;
    for (int s = 2; s <= 4; ++s) g.T[s] = (g.T[s - 1] + 1) / 2;
    g.P[4] = g.T[4] + 1;
    for (int s = 3; s >= 1; --s) g.P[s] = 2 * g.P[s + 1];
    g.H[1] = c.input_dim;
    for (int s = 2; s <= 4; ++s) g.H[s] = (g.H[s - 1] + 1) / 2;
    for (int s = 1; s <= 4; ++s) {
        g.C[s] = c.num_filters[s - 1];
        g.L[s] = (B * g.P[s] + 3) / 4 * 4;
    }
    g.H[0] = c.input_dim; g.C[0] = 1; g.T[0] = T1; g.P[0] = g.P[1]; g.L[0] = g.L[1];
    return g;
}

int frames_of(const b200tts_speaker_encoder_config& c, int T) {
    return c.use_torch_spec ? T / c.hop_length + 1 : T;
}

struct Ws {
    float *pre, *spec, *mel, *x0, *buf[4], *part, *scale, *atth, *logits, *pooled, *fco;
    int Bp;
};
Ws ws_carve(const b200tts_speaker_encoder_config& c, Arena& a, int B, int T) {
    const Geo g = geometry(c, B, frames_of(c, T));
    const int F = c.fft_size / 2 + 1, T1 = g.T[1];
    size_t big = 0, part = 0;
    for (int s = 1; s <= 4; ++s) {
        big = std::max(big, (size_t)(g.H[s] + 2) * g.C[s] * g.L[s]);
        if (s < 4) big = std::max(big, (size_t)(g.H[s] + 2) * 2 * g.C[s] * g.L[s + 1]);
        part = std::max(part, (size_t)g.H[s] * g.C[s] * B);
    }
    const int Hf = c.input_dim / 8, C4 = c.num_filters[3], Bp = (B + 3) / 4 * 4;
    const int out_dim = (c.encoder_type ? 2 : 1) * Hf * C4;
    Ws w;
    w.pre = a.f32(c.use_torch_spec ? (size_t)B * T : 0);
    w.spec = a.f32(c.use_torch_spec ? (size_t)B * F * T1 : 0);
    w.mel = a.f32(c.use_torch_spec ? (size_t)B * c.input_dim * T1 : 0);
    w.x0 = a.f32((size_t)(g.H[0] + 2) * g.L[0]);
    for (int i = 0; i < 4; ++i) w.buf[i] = a.f32(big);
    w.part = a.f32(part);
    w.scale = a.f32((size_t)B * 256 * 4);   // C <= 1024
    w.atth = a.f32((size_t)128 * g.L[4]);
    w.logits = a.f32((size_t)Hf * C4 * g.L[4]);
    w.pooled = a.f32((size_t)out_dim * Bp);
    w.fco = a.f32((size_t)c.proj_dim * Bp);
    w.Bp = Bp;
    return w;
}

int zero_rows(float* buf, int H, size_t row, cudaStream_t st) {   // rows 0 and H + 1 of [H + 2][row]
    B200_CUDA_OK(cudaMemsetAsync(buf, 0, row * sizeof(float), st));
    B200_CUDA_OK(cudaMemsetAsync(buf + (size_t)(H + 1) * row, 0, row * sizeof(float), st));
    return 0;
}

}  // namespace

int SpeakerEncoder::init(const b200tts_speaker_encoder_config& cfg, const float* const* w, int nw) {
    c = cfg;
    B200_REQUIRE(c.input_dim >= 8 && c.input_dim % 8 == 0, "speaker_encoder: input_dim=%d must be a multiple of 8", c.input_dim);
    B200_REQUIRE(c.proj_dim >= 1 && (c.encoder_type == 0 || c.encoder_type == 1), "speaker_encoder: bad proj_dim / encoder_type");
    for (int s = 0; s < 4; ++s)
        B200_REQUIRE(c.layers[s] >= 1 && c.num_filters[s] >= 8 && c.num_filters[s] <= 1024,
                     "speaker_encoder: stage %d needs >= 1 block and 8..1024 filters", s + 1);
    WeightList wl(w, nw);
    int rc;
    if (c.use_torch_spec) {
        B200_REQUIRE(c.win_length >= 1 && c.win_length <= c.fft_size && c.hop_length >= 1, "speaker_encoder: bad STFT sizes");
        const float* filt = wl.take();
        const float* win = wl.take();
        const float* fb = wl.take();
        B200_REQUIRE(filt && win && fb, "speaker_encoder: missing front-end weights");
        pre0 = filt[0]; pre1 = filt[1];
        const int F = c.fft_size / 2 + 1, left = (c.fft_size - c.win_length) / 2;
        std::vector<float> wp(c.fft_size, 0.f), basis((size_t)c.input_dim * F);
        for (int k = 0; k < c.win_length; ++k) wp[left + k] = win[k];
        for (int f = 0; f < F; ++f)
            for (int m = 0; m < c.input_dim; ++m) basis[(size_t)m * F + f] = fb[(size_t)f * c.input_dim + m];
        if ((rc = stft.init(c.fft_size, c.hop_length, wp.data(), basis.data(), c.input_dim))) return rc;
    }
    auto bn = [&](int C, BN& out) -> int {
        const float *bw = wl.take(), *bb = wl.take(), *bm = wl.take(), *bv = wl.take();
        B200_REQUIRE(bw && bb && bm && bv, "speaker_encoder: missing BatchNorm tensors");
        out = bn_affine(bw, bb, bm, bv, C);
        return 0;
    };
    // stem: conv1 (1 -> F0, bias) -> ReLU -> bn1
    const int F0 = c.num_filters[0];
    {
        const float *cw = wl.take(), *cb = wl.take();
        B200_REQUIRE(cw && cb, "speaker_encoder: missing conv1");
        BN b;
        if ((rc = bn(F0, b))) return rc;
        std::vector<float> r = repack3x3(cw, F0, 1, nullptr);
        conv1.tc_prec = B200TTS_PRECISION_FP32;
        if ((rc = pack_conv(conv1, r.data(), cb, F0, 3, 3, 1, 1))) return rc;
        if ((rc = upload_d(s0, b.s)) || (rc = upload_d(t0, b.t))) return rc;
    }
    int Cprev = F0;
    blocks.reserve(c.layers[0] + c.layers[1] + c.layers[2] + c.layers[3]);
    for (int s = 0; s < 4; ++s) {
        stage_first[s] = (int)blocks.size();
        for (int k = 0; k < c.layers[s]; ++k) {
            blocks.emplace_back();
            Block& b = blocks.back();
            b.C = c.num_filters[s]; b.Cin = (k == 0) ? Cprev : b.C; b.Cr = b.C / 8; b.down = (k == 0 && s > 0);
            const float* w1 = wl.take();
            BN b1, b2;
            if ((rc = bn(b.C, b1))) return rc;
            const float* w2 = wl.take();
            if ((rc = bn(b.C, b2))) return rc;
            const float *f1w = wl.take(), *f1b = wl.take(), *f2w = wl.take(), *f2b = wl.take();
            B200_REQUIRE(w1 && w2 && f1w && f1b && f2w && f2b, "speaker_encoder: missing block weights");
            b.c1.tc_prec = b.c2.tc_prec = B200TTS_PRECISION_FP32;
            if (b.down) {
                std::vector<float> r = repack3x3_s2(w1, b.C, b.Cin);
                if ((rc = pack_conv(b.c1, r.data(), nullptr, b.C, 6 * b.Cin, 2, 1, 1))) return rc;
            } else {
                B200_REQUIRE(b.Cin == b.C, "speaker_encoder: stage 1 keeps its width");
                std::vector<float> r = repack3x3(w1, b.C, b.Cin, nullptr);
                if ((rc = pack_conv(b.c1, r.data(), nullptr, b.C, 3 * b.Cin, 3, 1, 1))) return rc;
            }
            {
                std::vector<float> r = repack3x3(w2, b.C, b.C, &b2.s), bias(b2.t.begin(), b2.t.end());
                if ((rc = pack_conv(b.c2, r.data(), bias.data(), b.C, 3 * b.C, 3, 1, 1))) return rc;
            }
            if ((rc = upload_d(b.s1, b1.s)) || (rc = upload_d(b.t1, b1.t))) return rc;
            if ((rc = upload(b.fc1w, f1w, (size_t)b.Cr * b.C)) || (rc = upload(b.fc1b, f1b, b.Cr)) ||
                (rc = upload(b.fc2w, f2w, (size_t)b.C * b.Cr)) || (rc = upload(b.fc2b, f2b, b.C)))
                return rc;
            if (b.down) {
                const float* dw = wl.take();
                B200_REQUIRE(dw, "speaker_encoder: missing downsample weight");
                BN bd;
                if ((rc = bn(b.C, bd))) return rc;
                std::vector<float> r((size_t)b.C * b.Cin), bias(bd.t.begin(), bd.t.end());
                for (int co = 0; co < b.C; ++co)
                    for (int ci = 0; ci < b.Cin; ++ci) r[(size_t)co * b.Cin + ci] = (float)(dw[(size_t)co * b.Cin + ci] * bd.s[co]);
                b.ds.tc_prec = B200TTS_PRECISION_FP32;
                if ((rc = pack_conv(b.ds, r.data(), bias.data(), b.C, b.Cin, 1, 1, 0))) return rc;
            }
        }
        Cprev = c.num_filters[s];
    }
    stage_first[4] = (int)blocks.size();
    // head: attention conv 1x1 (input channels permuted from the reference's c*Hf + h to this layout's h*C + c)
    const int Hf = c.input_dim / 8, C4 = c.num_filters[3], Ca = Hf * C4;
    {
        const float *aw = wl.take(), *ab = wl.take();
        BN ba;
        if ((rc = bn(128, ba))) return rc;
        const float *a3w = wl.take(), *a3b = wl.take();
        B200_REQUIRE(aw && ab && a3w && a3b, "speaker_encoder: missing attention weights");
        std::vector<int> perm(Ca);
        for (int cc = 0; cc < C4; ++cc)
            for (int h = 0; h < Hf; ++h) perm[cc * Hf + h] = h * C4 + cc;
        att1.tc_prec = att2.tc_prec = B200TTS_PRECISION_FP32;
        if ((rc = pack_conv(att1, aw, ab, 128, Ca, 1, 1, 0, 0, perm.data()))) return rc;
        // BatchNorm1d after the ReLU folded into the following 1x1 conv: W3 (s x + t) + b3
        std::vector<float> r((size_t)Ca * 128), bias(Ca);
        for (int o = 0; o < Ca; ++o) {
            double acc = a3b[o];
            for (int k = 0; k < 128; ++k) {
                r[(size_t)o * 128 + k] = (float)(a3w[(size_t)o * 128 + k] * ba.s[k]);
                acc += (double)a3w[(size_t)o * 128 + k] * ba.t[k];
            }
            bias[o] = (float)acc;
        }
        if ((rc = pack_conv(att2, r.data(), bias.data(), Ca, 128, 1, 1, 0))) return rc;
    }
    {
        const float *fw = wl.take(), *fb = wl.take();
        B200_REQUIRE(fw && fb, "speaker_encoder: missing fc");
        fc.tc_prec = B200TTS_PRECISION_FP32;
        if ((rc = pack_conv(fc, fw, fb, c.proj_dim, (c.encoder_type ? 2 : 1) * Ca, 1, 1, 0))) return rc;
    }
    return wl.finish("speaker_encoder");
}

size_t SpeakerEncoder::workspace_bytes(int B, int T) const {
    if (B <= 0 || T <= 0) return 0;
    return arena_size([&](Arena& ar) { ws_carve(c, ar, B, T); });
}

int SpeakerEncoder::run(const float* x, const int* starts, int B, int T, int groups, int l2_norm, float* emb, int stop,
                        float* feat, void* ws, size_t ws_bytes, cudaStream_t st) const {
    B200_REQUIRE(x && starts && ws, "speaker_encoder: null pointer");
    B200_REQUIRE(B >= 1 && T >= 1, "speaker_encoder: B=%d, T=%d", B, T);
    B200_REQUIRE(stop <= 4, "speaker_encoder: stage %d does not exist", stop);
    B200_REQUIRE(stop >= 0 ? feat != nullptr : (emb && groups >= 1 && B % groups == 0 && B / groups <= 8192),
                 "speaker_encoder: B=%d windows do not split into %d groups of at most 8192 (or null output)", B, groups);
    const size_t need = workspace_bytes(B, T);
    B200_REQUIRE(ws_bytes >= need, "speaker_encoder: workspace of %zu bytes, %zu needed", ws_bytes, need);
    Arena ar(ws, ws_bytes);
    const Ws W = ws_carve(c, ar, B, T);
    const int T1 = frames_of(c, T);
    const Geo g = geometry(c, B, T1);
    // ---- front end -> stem input [H0 + 2][1][L1]
    B200_CUDA_OK(cudaMemsetAsync(W.x0, 0, sizeof(float) * (size_t)(g.H[0] + 2) * g.L[0], st));
    if (c.use_torch_spec) {
        B200_REQUIRE(T >= 2 && c.fft_size / 2 < T, "speaker_encoder: a window of %d samples is too short for the "
                     "centred STFT (needs more than %d)", T, c.fft_size / 2);
        preemph_kernel<<<grid_for((long long)B * T), NT, 0, st>>>(x, starts, B, T, pre0, pre1, W.pre);
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
        int rc;
        if ((rc = stft.magnitude(W.pre, B, T, 0, c.fft_size / 2, 2, 1.f, W.spec, T1, st))) return rc;
        if ((rc = stft.mel_project(W.spec, B, T1, 0.f, W.mel, st))) return rc;
        front_norm_kernel<<<dim3(c.input_dim, B), NT, 0, st>>>(W.mel, (long long)c.input_dim * T1, nullptr, T1, T1,
                                                               c.log_input, W.x0, g.L[0], g.P[0]);
    } else {
        front_norm_kernel<<<dim3(c.input_dim, B), NT, 0, st>>>(x, 0, starts, T, T, c.log_input, W.x0, g.L[0], g.P[0]);
    }
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    auto gather = [&](const float* src, int s, int Ln) -> int {
        gather_kernel<<<grid_for((long long)B * g.C[s] * g.H[s] * g.T[s]), NT, 0, st>>>(src, g.H[s], g.C[s], g.L[s], g.P[s],
                                                                                      g.T[s], B, Ln, feat);
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
        return 0;
    };
    if (stop == 0) return gather(W.x0, 0, 0);
    float *X = W.buf[0], *A = W.buf[1], *T1b = W.buf[2], *T2b = W.buf[3];
    int rc;
    // ---- stem: conv1 -> ReLU -> bn1 into A (stage 1 layout)
    {
        const int H = g.H[1], C = g.C[1], L = g.L[1];
        if ((rc = zero_rows(A, H, (size_t)C * L, st)) || (rc = zero_rows(T1b, H, (size_t)C * L, st))) return rc;
        ConvIO io;
        io.x = dense(W.x0, 1, L); io.Tin = L;
        io.y = dense(A + (size_t)C * L, C, L); io.Tout = L; io.B = H;
        if ((rc = launch_conv(conv1, io, st))) return rc;
        relu_affine_kernel<<<grid_for((long long)H * C * L), NT, 0, st>>>(A, H, C, L, g.P[1], g.T[1], B, s0, t0);
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
    }
    for (int s = 1; s <= 4; ++s) {
        const int H = g.H[s], C = g.C[s], L = g.L[s], P = g.P[s], Ts = g.T[s];
        const size_t row = (size_t)C * L;
        if (s > 1 && ((rc = zero_rows(A, H, row, st)) || (rc = zero_rows(T1b, H, row, st)))) return rc;
        for (int k = stage_first[s - 1]; k < stage_first[s]; ++k) {
            const Block& b = blocks[k];
            const bool last = (k == stage_first[s] - 1);
            // conv1 (-> ReLU -> bn1 in place)
            ConvIO io;
            if (b.down) {   // from the polyphase output of the previous stage: rows 2h .. 2h+2, K = 2
                const size_t prow = (size_t)2 * b.Cin * L;
                io.x = {X, (long long)(2 * prow), L}; io.Tin = L;
            } else {
                io.x = dense(A, C, L); io.Tin = L;
            }
            io.y = dense(T1b + row, C, L); io.Tout = L; io.B = H;
            if ((rc = launch_conv(b.c1, io, st))) return rc;
            relu_affine_kernel<<<grid_for((long long)H * row), NT, 0, st>>>(T1b, H, C, L, P, Ts, B, b.s1, b.t1);
            count_launch();
            B200_CUDA_OK(cudaGetLastError());
            // conv2 + bn2
            ConvIO io2;
            io2.x = dense(T1b, C, L); io2.Tin = L;
            io2.y = dense(T2b + row, C, L); io2.Tout = L; io2.B = H;
            if ((rc = launch_conv(b.c2, io2, st))) return rc;
            // SE
            se_partial_kernel<<<H * C, NT, 0, st>>>(T2b, C, L, P, Ts, B, W.part);
            se_mlp_kernel<<<B, NT, sizeof(float) * (C + b.Cr), st>>>(W.part, H, C, b.Cr, Ts, B, b.fc1w, b.fc1b, b.fc2w,
                                                                      b.fc2b, W.scale);
            count_launch(2);
            B200_CUDA_OK(cudaGetLastError());
            // residual: downsample (1x1, stride 2, bn folded) of the even phase of rows 2h+1 into A
            if (b.down) {
                const size_t prow = (size_t)2 * b.Cin * L;
                ConvIO iod;
                iod.x = {X + prow, (long long)(2 * prow), L}; iod.Tin = L;
                iod.y = dense(A + row, C, L); iod.Tout = L; iod.B = H;
                if ((rc = launch_conv(b.ds, iod, st))) return rc;
            }
            // relu(se(y) + residual): in place into A, or polyphase into X at the end of stages 1..3
            int Ln = 0;
            float* out = A;
            if (last && s < 4) {
                Ln = g.L[s + 1];
                out = X;
                if ((rc = zero_rows(X, H, (size_t)2 * C * Ln, st))) return rc;
            }
            block_out_kernel<<<grid_for((long long)H * C * (Ln ? 2LL * Ln : (long long)L)), NT, 0, st>>>(
                T2b, A, W.scale, H, C, L, P, Ts, B, out, Ln);
            count_launch();
            B200_CUDA_OK(cudaGetLastError());
        }
        if (stop == s) return gather(s < 4 ? X : A, s, s < 4 ? g.L[s + 1] : 0);
    }
    // ---- head
    const int Hf = g.H[4], C4 = g.C[4], L4 = g.L[4], Ca = Hf * C4;
    B200_REQUIRE(Hf == c.input_dim / 8, "speaker_encoder: input_dim=%d does not reduce to %d rows", c.input_dim, c.input_dim / 8);
    {
        ConvIO io;
        io.x = {A + (size_t)C4 * L4, 0, L4}; io.Tin = L4;
        io.y = {W.atth, 0, L4}; io.Tout = L4; io.B = 1; io.act = ACT_RELU;
        if ((rc = launch_conv(att1, io, st))) return rc;
        ConvIO io2;
        io2.x = {W.atth, 0, L4}; io2.Tin = L4;
        io2.y = {W.logits, 0, L4}; io2.Tout = L4; io2.B = 1;
        if ((rc = launch_conv(att2, io2, st))) return rc;
    }
    attn_pool_kernel<<<dim3(Ca, (B + NT / 32 - 1) / (NT / 32)), NT, 0, st>>>(W.logits, A + (size_t)C4 * L4, Hf, C4, L4, g.P[4],
                                                                            g.T[4], B, c.encoder_type, W.pooled, W.Bp);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    {
        ConvIO io;
        io.x = {W.pooled, 0, W.Bp}; io.Tin = B;
        io.y = {W.fco, 0, W.Bp}; io.Tout = B; io.B = 1;
        if ((rc = launch_conv(fc, io, st))) return rc;
    }
    const int nw = B / groups;
    l2_mean_kernel<<<groups, NT, sizeof(float) * nw, st>>>(W.fco, c.proj_dim, W.Bp, nw, l2_norm, emb);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace b200tts
