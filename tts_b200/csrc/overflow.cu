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

constexpr int NB = 8;          // batch rows per block in the LSTM / GEMV kernels (one weight read serves NB rows)
constexpr int UNITS = 8;       // LSTM units (4 gate rows each) or GEMV rows per 256-thread block: one per warp

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

template <int N>
__device__ __forceinline__ void warp_sum(float (&v)[N]) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int i = 0; i < N; ++i) v[i] += __shfl_xor_sync(0xffffffffu, v[i], o);
    }
}

// One LSTM time step for UNITS hidden units x NB batch rows per block; warp w owns unit j and its gate rows
// (i, f, g, o) = (j, H + j, 2H + j, 3H + j) of the torch layout.
//   gates = Wx x + Wh h_in + bias            (LSTMCell: x = prenet output, bias = b_ih + b_hh; rows that are done skip)
//   gates = Wh h_in + pre[b, d*4H + row, t]  (BiLSTM: pre = W_ih x + b_ih + b_hh for every token; direction d = blockIdx.y;
//                                             forward t = step, backward t = len_b - 1 - step; rows with step >= len_b skip)
//   c = f c + i g, h = o tanh(c) -> c (in place), h_out, out[b, t, d*H + j] (BiLSTM)
struct LstmArgs {
    const float* Wx = nullptr; int Kx = 0; const float* x = nullptr; int x_bs = 0;
    const float* Wh = nullptr; long long Wh_ds = 0; int H = 0;
    const float* h_in = nullptr; float* h_out = nullptr; float* c = nullptr; long long st_ds = 0;
    const float* bias = nullptr;
    const float* pre = nullptr; long long pre_bs = 0; int pre_cs = 0;
    float* out = nullptr; long long out_bs = 0; int out_ts = 0;
    const long long* lens = nullptr; int step = 0;
    const int* done = nullptr;
    int B = 0;
};

__global__ void __launch_bounds__(256) lstm_kernel(LstmArgs a) {
    extern __shared__ float sm[];
    const int H = a.H, d = blockIdx.y, b0 = blockIdx.z * NB, nb = min(NB, a.B - b0);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, j = blockIdx.x * UNITS + warp;
    float* xs = sm;                       // [NB][Kx]
    float* hs = sm + NB * a.Kx;           // [NB][H]
    const float* hin = a.h_in + d * a.st_ds;
    for (int i = threadIdx.x; i < nb * H; i += blockDim.x) hs[i] = hin[(size_t)(b0 + i / H) * H + i % H];
    for (int i = threadIdx.x; i < nb * a.Kx; i += blockDim.x) xs[i] = a.x[(size_t)(b0 + i / a.Kx) * a.x_bs + i % a.Kx];
    __syncthreads();
    if (j >= H) return;
    float acc[4 * NB];
#pragma unroll
    for (int i = 0; i < 4 * NB; ++i) acc[i] = 0.f;
    const float* Wh = a.Wh + d * a.Wh_ds;
    for (int k = lane; k < H; k += 32) {
#pragma unroll
        for (int g = 0; g < 4; ++g) {
            const float w = Wh[(size_t)(g * H + j) * H + k];
#pragma unroll
            for (int bb = 0; bb < NB; ++bb) acc[g * NB + bb] = fmaf(w, hs[(bb < nb ? bb : 0) * H + k], acc[g * NB + bb]);
        }
    }
    for (int k = lane; k < a.Kx; k += 32) {
#pragma unroll
        for (int g = 0; g < 4; ++g) {
            const float w = a.Wx[(size_t)(g * H + j) * a.Kx + k];
#pragma unroll
            for (int bb = 0; bb < NB; ++bb)
                acc[g * NB + bb] = fmaf(w, xs[(bb < nb ? bb : 0) * a.Kx + k], acc[g * NB + bb]);
        }
    }
    warp_sum(acc);
    float gv[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int bb = 0; bb < NB; ++bb)
        if (lane == bb) {
#pragma unroll
            for (int g = 0; g < 4; ++g) gv[g] = acc[g * NB + bb];
        }
    if (lane >= nb) return;
    const int b = b0 + lane;
    int t = 0;
    if (a.lens) {
        const int len = (int)a.lens[b];
        if (a.step >= len) return;
        t = d ? len - 1 - a.step : a.step;
#pragma unroll
        for (int g = 0; g < 4; ++g) gv[g] += a.pre[(size_t)b * a.pre_bs + (size_t)(d * 4 * H + g * H + j) * a.pre_cs + t];
    } else {
        if (a.done[b]) return;
#pragma unroll
        for (int g = 0; g < 4; ++g) gv[g] += a.bias[g * H + j];
    }
    float* cp = a.c + d * a.st_ds + (size_t)b * H + j;
    const float cn = sigmoidf_(gv[1]) * *cp + sigmoidf_(gv[0]) * tanhf(gv[2]);
    const float h = sigmoidf_(gv[3]) * tanhf(cn);
    *cp = cn;
    a.h_out[d * a.st_ds + (size_t)b * H + j] = h;
    if (a.out) a.out[(size_t)b * a.out_bs + (size_t)t * a.out_ts + d * H + j] = h;
}

// y[b, r] = act(W[r] . x[b] + bias[r] + add[b, r, state[b]]), then the prenet dropout (drop[b, f, layer, r] ? 2v : 0
// with f the loop's frame counter); rows that are done skip.  One warp per row r, NB batch rows per block.
struct LinArgs {
    const float* W = nullptr; const float* bias = nullptr; int K = 0, R = 0;
    const float* x = nullptr; int x_bs = 0;
    float* y = nullptr; int y_bs = 0;
    const float* add = nullptr; long long add_bs = 0; int add_rs = 0; const int* state = nullptr;
    int relu = 0;
    const unsigned char* drop = nullptr; int drop_layer = 0, drop_L = 0, drop_F = 0; const int* ctl = nullptr;
    const int* done = nullptr;
    int B = 0;
};

__global__ void __launch_bounds__(256) hmm_linear_kernel(LinArgs a) {
    extern __shared__ float xs[];     // [NB][K]
    const int b0 = blockIdx.y * NB, nb = min(NB, a.B - b0);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, r = blockIdx.x * UNITS + warp;
    for (int i = threadIdx.x; i < nb * a.K; i += blockDim.x) xs[i] = a.x[(size_t)(b0 + i / a.K) * a.x_bs + i % a.K];
    __syncthreads();
    if (r >= a.R) return;
    float acc[NB];
#pragma unroll
    for (int i = 0; i < NB; ++i) acc[i] = 0.f;
    const float* w = a.W + (size_t)r * a.K;
    for (int k = lane; k < a.K; k += 32) {
        const float wv = w[k];
#pragma unroll
        for (int bb = 0; bb < NB; ++bb) acc[bb] = fmaf(wv, xs[(bb < nb ? bb : 0) * a.K + k], acc[bb]);
    }
    warp_sum(acc);
    float v = 0.f;
#pragma unroll
    for (int bb = 0; bb < NB; ++bb)
        if (lane == bb) v = acc[bb];
    if (lane >= nb) return;
    const int b = b0 + lane;
    if (a.done[b]) return;
    if (a.bias) v += a.bias[r];
    if (a.add) v += a.add[(size_t)b * a.add_bs + (size_t)r * a.add_rs + a.state[b]];
    if (a.relu) v = fmaxf(v, 0.f);
    if (a.drop) {
        const int f = a.ctl[1];
        v = a.drop[(((size_t)b * a.drop_F + f) * a.drop_L + a.drop_layer) * a.R + r] ? v * 2.f : 0.f;
    }
    a.y[(size_t)b * a.y_bs + r] = v;
}

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

// y[b, c, n] = x[b, n, c]   ([B, N, E] encoder states -> channel-major for the hoisted conv)
__global__ void transpose_kernel(const float* x, float* y, int N, int E) {
    __shared__ float tile[32][33];
    const int b = blockIdx.z, n0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int n = n0 + i, c = c0 + threadIdx.x;
        tile[i][threadIdx.x] = (n < N && c < E) ? x[((size_t)b * N + n) * E + c] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int c = c0 + i, n = n0 + threadIdx.x;
        if (n < N && c < E) y[((size_t)b * E + c) * N + n] = tile[threadIdx.x][i];
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

static int lin_smem(int K) { return NB * K * (int)sizeof(float); }

static bool persist_layout(const Overflow& e, Arena& ar, int B, int Tt, Persist& p) {
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
    return p.zc && p.ctl && p.state && p.done && p.quant && p.hm && p.cm && p.pin && p.pb && p.hid && p.outp;
}

Overflow::~Overflow() {
    if (emb) cudaFree(emb);
    for (auto& L : convs) free_conv(L);
    free_conv(lstm_in);
    free_conv(zproj);
    for (float* p : prenet_w) cudaFree(p);
    for (float* p : out_w) if (p) cudaFree(p);
    for (float* p : out_b) if (p) cudaFree(p);
    for (float* p : {whh, mem_wih, mem_whh, mem_b, go, mean, std_}) if (p) cudaFree(p);
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
    const int max_k = 48 * 1024 / (NB * (int)sizeof(float));
    B200_REQUIRE(H <= max_k && P + M <= max_k && c.ar_order * C <= max_k,
                 "overflow: layer widths above %d inputs are not supported", max_k);
    for (int l = 0; l < nL; ++l)
        B200_REQUIRE(c.outputnet_size[l] > 0 && c.outputnet_size[l] <= max_k, "overflow: outputnet_size[%d] = %d", l,
                     c.outputnet_size[l]);
    const int per_block = 3 + 2 + 4 * c.num_block_layers + 2;
    const int expect = 1 + 6 * c.n_convs + 8 + 1 + c.prenet_n_layers + 4 + 2 * nL + 2 + 2 +
                       (c.has_decoder ? per_block * c.num_flow_blocks : 0);
    B200_REQUIRE(nw == expect, "overflow: expected %d weight tensors, got %d", expect, nw);
    int rc, i = 0;
    if ((rc = upload(&emb, w[i++], (size_t)c.n_vocab * E))) return rc;
    for (int l = 0; l < c.n_convs; ++l, i += 6) {   // ConvBNBlock: BatchNorm1d (eps 1e-5) folded into the conv
        std::vector<float> wf((size_t)E * E * 5), bf(E);
        for (int o = 0; o < E; ++o) {
            const double s = (double)w[i + 2][o] / sqrt((double)w[i + 5][o] + 1e-5);
            for (size_t k = 0; k < (size_t)E * 5; ++k) wf[(size_t)o * E * 5 + k] = (float)(w[i][(size_t)o * E * 5 + k] * s);
            bf[o] = (float)(((double)w[i + 1][o] - w[i + 4][o]) * s + w[i + 3][o]);
        }
        if ((rc = pack_conv(convs[l], wf.data(), bf.data(), E, E, 5, 1, 2))) return rc;
    }
    {   // LSTM: both directions' input projections as one 1x1 conv (rows [fwd 4H | bwd 4H]), bias b_ih + b_hh
        std::vector<float> wi((size_t)8 * H * E), bi((size_t)8 * H), wh((size_t)8 * H * H);
        for (int d = 0; d < 2; ++d) {
            const float* const* p = w + i + 4 * d;
            memcpy(wi.data() + (size_t)d * 4 * H * E, p[0], sizeof(float) * 4 * H * E);
            memcpy(wh.data() + (size_t)d * 4 * H * H, p[1], sizeof(float) * 4 * H * H);
            for (int r = 0; r < 4 * H; ++r) bi[(size_t)d * 4 * H + r] = p[2][r] + p[3][r];
        }
        if ((rc = pack_conv(lstm_in, wi.data(), bi.data(), 8 * H, E, 1, 1, 0))) return rc;
        if ((rc = upload(&whh, wh.data(), wh.size()))) return rc;
        i += 8;
    }
    if ((rc = upload(&go, w[i++], (size_t)c.ar_order))) return rc;
    for (int l = 0; l < c.prenet_n_layers; ++l) {
        float* p = nullptr;
        if ((rc = upload(&p, w[i++], (size_t)P * (l ? P : c.ar_order * C)))) return rc;
        prenet_w.push_back(p);
    }
    if ((rc = upload(&mem_wih, w[i], (size_t)4 * M * P))) return rc;
    if ((rc = upload(&mem_whh, w[i + 1], (size_t)4 * M * M))) return rc;
    {
        std::vector<float> b((size_t)4 * M);
        for (int r = 0; r < 4 * M; ++r) b[r] = w[i + 2][r] + w[i + 3][r];
        if ((rc = upload(&mem_b, b.data(), b.size()))) return rc;
    }
    i += 4;
    for (int l = 0; l <= nL; ++l, i += 2) {
        const int rows = l < nL ? c.outputnet_size[l] : 2 * C + 1;
        const int in = l == 0 ? M + E : c.outputnet_size[l - 1];
        float *pw = nullptr, *pbias = nullptr;
        if (l == 0) {   // cat(h, z): the h columns per frame, the z columns hoisted into zproj (with the bias)
            std::vector<float> wh((size_t)rows * M), wz((size_t)rows * E);
            for (int r = 0; r < rows; ++r) {
                memcpy(wh.data() + (size_t)r * M, w[i] + (size_t)r * in, sizeof(float) * M);
                memcpy(wz.data() + (size_t)r * E, w[i] + (size_t)r * in + M, sizeof(float) * E);
            }
            if ((rc = upload(&pw, wh.data(), wh.size()))) return rc;
            if ((rc = pack_conv(zproj, wz.data(), w[i + 1], rows, E, 1, 1, 0))) return rc;
        } else {
            if ((rc = upload(&pw, w[i], (size_t)rows * in))) return rc;
            if ((rc = upload(&pbias, w[i + 1], (size_t)rows))) return rc;
        }
        out_w.push_back(pw);
        out_b.push_back(pbias);
    }
    if ((rc = upload(&mean, w[i], (size_t)C))) return rc;
    if ((rc = upload(&std_, w[i + 1], (size_t)C))) return rc;
    i += 2;
    if (c.has_decoder) {
        B200_REQUIRE(c.num_squeeze >= 1 && c.hidden_channels_dec > 0 && c.kernel_size_dec % 2 == 1 &&
                         c.num_flow_blocks >= 1 && c.num_block_layers >= 1 && c.dilation_rate >= 1,
                     "overflow: unsupported decoder config");
        int used = 0;
        if ((rc = dec.init(C, c.hidden_channels_dec, c.kernel_size_dec, c.dilation_rate, c.num_flow_blocks,
                           c.num_block_layers, 0, c.num_splits, c.num_squeeze, c.sigmoid_scale, w + i, &used)))
            return rc;
    }
    return 0;
}

size_t Overflow::persist_bytes(int B, int Tt) const {
    int omax = 0;
    for (int l = 0; l < c.outputnet_n_layers; ++l) omax = std::max(omax, c.outputnet_size[l]);
    const int N = Tt * c.state_per_phone, M = c.memory_rnn_dim;
    return arena_bytes((size_t)B * O1 * N) + 3 * arena_bytes(B) + arena_bytes(2 + B) + arena_bytes((size_t)2 * B * M) +
           arena_bytes((size_t)B * M) + arena_bytes((size_t)B * c.ar_order * c.out_channels) +
           arena_bytes((size_t)2 * B * c.prenet_dim) + arena_bytes((size_t)2 * B * omax) +
           arena_bytes((size_t)B * (2 * c.out_channels + 1));
}

size_t Overflow::workspace_bytes(int B, int Tt, int F) const {
    const int E = c.encoder_dim, N = Tt * c.state_per_phone;
    const size_t enc = persist_bytes(B, Tt) + 2 * arena_bytes((size_t)B * E * Tt) + arena_bytes((size_t)B * Tt) +
                       arena_bytes((size_t)B * 8 * H * Tt) + arena_bytes((size_t)4 * B * H) +
                       arena_bytes((size_t)2 * B * H) + arena_bytes((size_t)B * E * N);
    size_t decb = 0;
    if (c.has_decoder && F > 0) {
        const int Tq = tq(F), Cs = c.out_channels * c.num_squeeze;
        decb = arena_bytes((size_t)B * Cs * Tq) + arena_bytes((size_t)B * Tq) +
               arena_bytes((size_t)B * c.out_channels * Tq * c.num_squeeze) + dec.workspace_bytes(B, Tq);
    }
    return std::max(enc, decb) + 1024;
}

int Overflow::encode(const long long* tokens, const long long* lengths, int B, int Tt, float* states, void* ws,
                     size_t ws_bytes, cudaStream_t st) const {
    B200_REQUIRE(tokens && lengths && states && ws, "overflow_encode: null pointer");
    B200_REQUIRE(B >= 1 && Tt >= 1, "overflow_encode: empty batch");
    B200_REQUIRE(ws_bytes >= workspace_bytes(B, Tt, 0), "overflow_encode: workspace too small");
    const int E = c.encoder_dim, N = Tt * c.state_per_phone;
    Arena ar(ws, ws_bytes);
    Persist p;
    B200_REQUIRE(persist_layout(*this, ar, B, Tt, p), "overflow_encode: arena exhausted");
    float* x = ar.f32((size_t)B * E * Tt);
    float* y = ar.f32((size_t)B * E * Tt);
    float* xmask = ar.f32((size_t)B * Tt);
    float* pre = ar.f32((size_t)B * 8 * H * Tt);
    float* hb = ar.f32((size_t)4 * B * H);
    float* cb = ar.f32((size_t)2 * B * H);
    float* encT = ar.f32((size_t)B * E * N);
    B200_REQUIRE(x && y && xmask && pre && hb && cb && encT, "overflow_encode: arena exhausted");
    int rc;
    // emb(x) without a scale, zero past each row's length (the reference runs each row at its own length)
    if ((rc = launch_embed(tokens, lengths, emb, nullptr, B, Tt, E, E, x, xmask, st, false))) return rc;
    const long long bs = (long long)E * Tt;
    for (int l = 0; l < c.n_convs; ++l) {   // conv -> BN (folded) -> ReLU -> Dropout (eval: identity), masked
        ConvIO io;
        io.x = x; io.x_bs = bs; io.x_cs = Tt; io.Tin = Tt;
        io.y = y; io.y_bs = bs; io.y_cs = Tt; io.Tout = Tt; io.B = B;
        io.act = ACT_RELU; io.ymask = xmask; io.ymask_bs = Tt; io.flags = EPI_MASK_POST;
        if ((rc = launch_conv(convs[l], io, st))) return rc;
        std::swap(x, y);
    }
    {   // pre[b, d*4H + row, t] = W_ih x + b_ih + b_hh, both directions
        ConvIO io;
        io.x = x; io.x_bs = bs; io.x_cs = Tt; io.Tin = Tt;
        io.y = pre; io.y_bs = (long long)8 * H * Tt; io.y_cs = Tt; io.Tout = Tt; io.B = B;
        if ((rc = launch_conv(lstm_in, io, st))) return rc;
    }
    B200_CUDA_OK(cudaMemsetAsync(hb, 0, sizeof(float) * 2 * B * H, st));
    B200_CUDA_OK(cudaMemsetAsync(cb, 0, sizeof(float) * 2 * B * H, st));
    B200_CUDA_OK(cudaMemsetAsync(states, 0, sizeof(float) * (size_t)B * N * E, st));
    const int smem = NB * H * (int)sizeof(float);
    for (int s = 0; s < Tt; ++s) {   // the [B, Tt, 2H] LSTM output is the [B, Tt*spp, E] state tensor
        LstmArgs a;
        a.Wh = whh; a.Wh_ds = (long long)4 * H * H; a.H = H;
        a.h_in = hb + (size_t)(s & 1) * 2 * B * H; a.h_out = hb + (size_t)((s + 1) & 1) * 2 * B * H;
        a.c = cb; a.st_ds = (long long)B * H;
        a.pre = pre; a.pre_bs = (long long)8 * H * Tt; a.pre_cs = Tt;
        a.out = states; a.out_bs = (long long)Tt * 2 * H; a.out_ts = 2 * H;
        a.lens = lengths; a.step = s; a.B = B;
        dim3 grid((H + UNITS - 1) / UNITS, 2, (B + NB - 1) / NB);
        lstm_kernel<<<grid, 256, smem, st>>>(a);
        count_launch();
        dispatch_note(DISPATCH_LSTM_BI);
        B200_CUDA_OK(cudaGetLastError());
    }
    {
        dim3 grid((N + 31) / 32, (E + 31) / 32, B);
        transpose_kernel<<<grid, dim3(32, 8), 0, st>>>(states, encT, N, E);
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
    }
    {   // hoisted: zc[b, r, n] = W_z[r] . state[b, n] + b_0[r] for every state n
        ConvIO io;
        io.x = encT; io.x_bs = (long long)E * N; io.x_cs = N; io.Tin = N;
        io.y = p.zc; io.y_bs = (long long)O1 * N; io.y_cs = N; io.Tout = N; io.B = B;
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
    B200_REQUIRE(ws_bytes >= workspace_bytes(B, Tt, 0), "overflow_sample: workspace too small");
    const int C = c.out_channels, P = c.prenet_dim, M = c.memory_rnn_dim, nL = c.outputnet_n_layers;
    const int N = Tt * c.state_per_phone;
    Arena ar(ws, ws_bytes);
    Persist p;
    B200_REQUIRE(persist_layout(*this, ar, B, Tt, p), "overflow_sample: arena exhausted");
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
            dim3 grid((P + UNITS - 1) / UNITS, (B + NB - 1) / NB);
            hmm_linear_kernel<<<grid, 256, lin_smem(K), cs>>>(a);
            if (note) dispatch_note(DISPATCH_HMM_LINEAR);
            in = a.y; K = P;
        }
        {
            LstmArgs a;
            a.Wx = mem_wih; a.Kx = P; a.x = in; a.x_bs = P;
            a.Wh = mem_whh; a.H = M; a.h_in = p.hm + (size_t)par * B * M; a.h_out = p.hm + (size_t)(par ^ 1) * B * M;
            a.c = p.cm; a.bias = mem_b; a.done = p.done; a.B = B;
            dim3 grid((M + UNITS - 1) / UNITS, 1, (B + NB - 1) / NB);
            lstm_kernel<<<grid, 256, NB * (P + M) * (int)sizeof(float), cs>>>(a);
            if (note) dispatch_note(DISPATCH_LSTM_CELL);
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
            dim3 grid((R + UNITS - 1) / UNITS, (B + NB - 1) / NB);
            hmm_linear_kernel<<<grid, 256, lin_smem(K), cs>>>(a);
            if (note) dispatch_note(DISPATCH_HMM_LINEAR);
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
    cudaStream_t cs = nullptr;
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    B200_CUDA_OK(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
    int rc = 0;
    if (cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal) != cudaSuccess) {
        cudaStreamDestroy(cs);
        set_error("overflow_sample: cannot capture the frame graph");
        return 2;
    }
    for (int f = 0; f < chunk_frames && rc == 0; ++f) rc = frame(cs, f & 1, f == 0);
    const cudaError_t ce = cudaStreamEndCapture(cs, &graph);
    cudaStreamDestroy(cs);
    if (rc || ce != cudaSuccess) {
        if (graph) cudaGraphDestroy(graph);
        if (!rc) set_error("overflow_sample: frame graph capture failed: %s", cudaGetErrorString(ce));
        return rc ? rc : 2;
    }
    const cudaError_t ie = cudaGraphInstantiate(&exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ie != cudaSuccess) {
        set_error("overflow_sample: cannot instantiate the frame graph: %s", cudaGetErrorString(ie));
        return 2;
    }
    // replay until no row runs: every row is done by frame max_frames - 1, so frames past it do no work
    std::vector<int> host(2 + B);
    for (int done_frames = 0; done_frames < max_frames; done_frames += chunk_frames) {
        cudaError_t e = cudaGraphLaunch(exec, st);
        count_launch(per_frame * chunk_frames);
        if (e == cudaSuccess) e = cudaMemcpyAsync(host.data(), p.ctl, sizeof(int) * (2 + B), cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) {
            cudaGraphExecDestroy(exec);
            set_error("overflow_sample: %s", cudaGetErrorString(e));
            return 2;
        }
        if (host[0] == 0) break;
    }
    cudaGraphExecDestroy(exec);
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
    B200_REQUIRE(ws_bytes >= workspace_bytes(B, 1, F), "overflow_decode: workspace too small");
    const int nsq = c.num_squeeze, Tv = F / nsq, Tq = tq(F), Cs = C * nsq;
    if (Tv == 0) return 0;
    Arena ar(ws, ws_bytes);
    float* za = ar.f32((size_t)B * Cs * Tq);
    float* msk = ar.f32((size_t)B * Tq);
    float* melc = ar.f32((size_t)B * C * Tq * nsq);
    B200_REQUIRE(za && msk && melc, "overflow_decode: arena exhausted");
    {
        dim3 grid((Tq + 127) / 128, Cs, B);
        squeeze_hmm_kernel<<<grid, 128, 0, st>>>(hmm_out, Fpitch, frames, za, msk, C, nsq, Tq);
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
    }
    int rc;
    if ((rc = dec.reverse(za, msk, nullptr, B, Tq, Tv, melc, ar.base + ar.off, ar.cap - ar.off, st))) return rc;
    const int T = Tv * nsq;
    dim3 grid((T * C + 255) / 256, B);
    denorm_kernel<<<grid, 256, 0, st>>>(melc, (long long)C * T, 1, T, mean, std_, mel, T, C);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace b200tts
