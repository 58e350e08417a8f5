// UnivNet generator engine.
// Reference semantics: TTS/vocoder/models/univnet_generator.py (UnivnetGenerator), TTS/vocoder/layers/lvc_block.py
// (KernelPredictor, LVCBlock).
//
// Per call, with h_n = u_0 ... u_n the cumulative hop of block n:
//   x = first_conv(noise)                                        conv engine, k7
//   per block n:
//     H = KPnet(mel)                                             conv engine at frame rate: input_conv + lrelu 0.1, six
//                                                                residual convs + lrelu 0.1, the last one + H_in (the
//                                                                engine's leaky-ReLU / residual epilogue)
//     P = [kernel_conv | bias_conv](H)                           univnet_predict_kernel: one split-fp16 tensor-core GEMM,
//                                                                written frame-major (layout below)
//     x = upsample(lrelu(x, 0.2))                                conv engine, ConvTranspose1d
//     per layer i: x = x + sigmoid(o[:32]) tanh(o[32:]),
//                  o = LVC_P(lrelu(conv_i(lrelu(x, 0.2)), 0.2))  univnet_lvc_kernel, one launch per layer
//   out = tanh(last_conv(lrelu(x, 0.1)))                         conv engine, k7
//
// Predicted-kernel layout.  Per frame (b, f) one row of MP = L * (64 * 96 + 64) floats, frame-major ([B * T][MP]):
//   kernels  [l][co 64][tap * 32 + ci]      (the LVC MMA's A operand, row-major, K = 96 = 3 taps x 32 channels)
//   biases   [l][co 64]                     after all L kernels
// The reference's channel of kernel_conv for (l, ci, co, tap) is ((l * 32 + ci) * 64 + co) * 3 + tap; init() permutes
// the GEMM rows so that the GEMM writes this layout directly.
//
// Both kernels use mma.sync.m16n8k16 with fp16 operands and fp32 accumulation, split-fp16 in three products as the conv
// engine's PREC_F16X3: v = hi + lo / 2048 for each operand, A B = A_hi B_hi + (A_hi B_lo + A_lo B_hi) / 2048, the large
// and the small terms in separate accumulators.  Every operand is data split at run time (the predicted kernels are
// activations), so a value with |v| >= 65504 sets the device's range flag and the next launch fails.
#include <cuda_fp16.h>

#include <cmath>

#include "conv_tc.cuh"
#include "engines.cuh"

namespace b200tts {

namespace uv {
constexpr int C = 32;                 // hidden_channels the kernels take
constexpr int CO = 2 * C;             // LVC output channels (sigmoid | tanh halves)
constexpr int KK = 3 * C;             // LVC / conv_i reduction: 3 taps x 32 channels
constexpr int KSZ = CO * KK;          // one layer's kernel per frame: 6144 floats
constexpr int NT = 128;               // LVC output samples per CTA
constexpr int YW = NT + 2;            // y columns a tile needs: one each side for the LVC taps
constexpr int XW = 136;               // conv_i columns computed (17 MMA n-tiles >= YW)
constexpr int XS = 148;               // row stride of the staged x windows (== 4 mod 16: conflict-free B fragments)
constexpr int YS = 132;               // row stride of y (== 4 mod 16)
constexpr int SMEM = (3 * C * XS + C * YS) * 4;
constexpr int PT_M = 128, PT_N = 64;  // prediction GEMM tile: 128 rows x 64 frames, 8 warps of 32 x 32
}  // namespace uv

__device__ __forceinline__ void mma_f16(float* d, const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// the three products of one split-fp16 m16n8k16 step: big += A_hi B_hi, small += A_hi B_lo + A_lo B_hi
__device__ __forceinline__ void mma_x3(float* big, float* small, const uint32_t (&ah)[4], const uint32_t (&al)[4],
                                       const uint32_t (&bh)[2], const uint32_t (&bl)[2]) {
    mma_f16(small, ah, bl[0], bl[1]);
    mma_f16(small, al, bh[0], bh[1]);
    mma_f16(big, ah, bh[0], bh[1]);
}

// A fragment of a row-major fp32 matrix (row stride ld) at rows r, r + 8 and columns k, k + 8 (k = 16 s + 2 (lane % 4)):
// split into hi / lo
__device__ __forceinline__ void load_a(const float* __restrict__ p, int ld, uint32_t (&ah)[4], uint32_t (&al)[4],
                                       float& amax) {
    const float2 v0 = __ldg(reinterpret_cast<const float2*>(p));
    const float2 v1 = __ldg(reinterpret_cast<const float2*>(p + 8 * ld));
    const float2 v2 = __ldg(reinterpret_cast<const float2*>(p + 8));
    const float2 v3 = __ldg(reinterpret_cast<const float2*>(p + 8 * ld + 8));
    amax = fmaxf(amax, fmaxf(fmaxf(fmaxf(fabsf(v0.x), fabsf(v0.y)), fmaxf(fabsf(v1.x), fabsf(v1.y))),
                             fmaxf(fmaxf(fabsf(v2.x), fabsf(v2.y)), fmaxf(fabsf(v3.x), fabsf(v3.y)))));
    tc::split_f16x2(v0.x, v0.y, ah[0], al[0]);
    tc::split_f16x2(v1.x, v1.y, ah[1], al[1]);
    tc::split_f16x2(v2.x, v2.y, ah[2], al[2]);
    tc::split_f16x2(v3.x, v3.y, ah[3], al[3]);
}

// B fragment from four reduction rows (2t, 2t + 1, 2t + 8, 2t + 9) of one column, split into hi / lo
__device__ __forceinline__ void split_b(float r0, float r1, float r8, float r9, uint32_t (&bh)[2], uint32_t (&bl)[2],
                                        float& amax) {
    amax = fmaxf(amax, fmaxf(fmaxf(fabsf(r0), fabsf(r1)), fmaxf(fabsf(r8), fabsf(r9))));
    tc::split_f16x2(r0, r1, bh[0], bl[0]);
    tc::split_f16x2(r8, r9, bh[1], bl[1]);
}

__device__ __forceinline__ void flag_range(float amax, int* err) {
    if (amax >= tc::F16X3_MAX && err) { *reinterpret_cast<volatile int*>(err + tc::ERR_RANGE) = 1; __threadfence_system(); }
}

__device__ __forceinline__ float lrelu(float v, float s) { return v > 0.f ? v : v * s; }

// ------------------------------------------------------------------ the kernel-prediction GEMM
// P[(b T + f) MP + m] = bias[m] + sum_{tap, ch} W[m][tap * Ch + ch] H[b][ch][f + tap - pad]   (zero outside [0, T))
// A = W (rows m, row stride Kd = Kp Ch), B = the k-tap window of H (one column per frame of the batch, N = B T), so one
// weight tile serves 64 frames.  Ch % 16 == 0: a 16-wide reduction step stays inside one tap.
__global__ void __launch_bounds__(256) univnet_predict_kernel(const float* __restrict__ H, long long h_bs, int h_cs, int Ch,
                                                              int Kp, int T, int B, const float* __restrict__ W,
                                                              const float* __restrict__ bias, int MP,
                                                              float* __restrict__ P, int* err) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const int m0 = blockIdx.y * uv::PT_M + (warp & 3) * 32;
    if (m0 >= MP) return;                     // MP is a multiple of 32 (one warp's rows), not always of 128
    const long long n0 = (long long)blockIdx.x * uv::PT_N + (warp >> 2) * 32;
    const long long N = (long long)B * T;
    const int Kd = Kp * Ch, pad = (Kp - 1) / 2;
    const float* hrow[4];
    int fcol[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {             // this lane's B column (frame) of n-tile j
        const long long n = n0 + 8 * j + g;
        const int b = (int)(n / T);
        fcol[j] = n < N ? (int)(n - (long long)b * T) : -(1 << 30);
        hrow[j] = H + (n < N ? b : 0) * h_bs;
    }
    float big[2][4][4], small[2][4][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) big[i][j][e] = small[i][j][e] = 0.f;
    float amax = 0.f;
    const float* wrow0 = W + (size_t)(m0 + g) * Kd + 2 * t;
#pragma unroll 1
    for (int k0 = 0; k0 < Kd; k0 += 16) {
        const int tap = k0 / Ch, ci = k0 - tap * Ch + 2 * t;
        uint32_t bh[4][2], bl[4][2];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int f = fcol[j] + tap - pad;
            const bool in = f >= 0 && f < T;
            const float* hp = hrow[j] + (size_t)ci * h_cs + f;
            const float r0 = in ? __ldg(hp) : 0.f, r1 = in ? __ldg(hp + h_cs) : 0.f;
            const float r8 = in ? __ldg(hp + 8 * h_cs) : 0.f, r9 = in ? __ldg(hp + 9 * h_cs) : 0.f;
            split_b(r0, r1, r8, r9, bh[j], bl[j], amax);
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            uint32_t ah[4], al[4];
            load_a(wrow0 + (size_t)(16 * i) * Kd + k0, Kd, ah, al, amax);
#pragma unroll
            for (int j = 0; j < 4; ++j) mma_x3(big[i][j], small[i][j], ah, al, bh[j], bl[j]);
        }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = m0 + 16 * i + g + 8 * h;
            const float bm = __ldg(bias + m);
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const long long n = n0 + 8 * j + 2 * t + e;
                    if (n < N) P[n * MP + m] = big[i][j][2 * h + e] + small[i][j][2 * h + e] * (1.f / 2048.f) + bm;
                }
        }
    flag_range(amax, err);
}

// ------------------------------------------------------------------ the fused LVC layer
struct UvLayerArgs {
    const float* x;          // [B][32][pitch], read (also the residual)
    float* xn;               // [B][32][pitch], written (never the buffer x is)
    long long bs;            // batch stride of x / xn
    int pitch, Ts, hop, dil, T;
    const float* cw;         // conv_i [32 co][96 = tap * 32 + ci]
    const float* cb;         // conv_i bias [32]
    const float* P;          // predicted kernels of this block, frame-major [B * T][MP]
    int MP, koff, boff;      // this layer's kernel / bias offset within a frame's row
    int* err;
};

// One CTA: NT output samples of one row.  (1) the three tap windows of lrelu(x, 0.2) at dilation dil, staged fp32;
// (2) y = lrelu(conv_i + bias, 0.2) on the 130 columns the LVC reads (zero outside the row: the LVC's zero padding),
// kept in shared memory; (3) per 8-column n-tile and frame, the LVC as M = 64 (co) x K = 96 MMAs with the frame's
// predicted kernel as A and the y window as B (columns of other frames masked to zero, so a tile may span frames of any
// hop); (4) bias, gate and residual, one store of x.
__global__ void __launch_bounds__(256) univnet_lvc_kernel(const UvLayerArgs a) {
    using namespace uv;
    extern __shared__ __align__(16) float usm[];
    float* const xs = usm;                     // [3][32][XS]: column j <-> sample t0 - 1 + j + (tap - 1) dil
    float* const ys = usm + 3 * C * XS;        // [32][YS]: column j <-> sample t0 - 1 + j
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const int b = blockIdx.y, t0 = blockIdx.x * NT;
    const float* xb = a.x + b * a.bs;
    float amax = 0.f;
    for (int i = tid; i < 3 * C * XW; i += blockDim.x) {
        const int tap = i / (C * XW), r = i - tap * C * XW, ci = r / XW, j = r - ci * XW;
        const int n = t0 - 1 + j + (tap - 1) * a.dil;
        xs[(tap * C + ci) * XS + j] = (n >= 0 && n < a.Ts) ? lrelu(__ldg(xb + (size_t)ci * a.pitch + n), 0.2f) : 0.f;
    }
    __syncthreads();
    // ---- conv_i: 2 m-tiles (32 co) x 17 n-tiles, n-tiles spread over the warps
    for (int nt = warp; nt < XW / 8; nt += 8) {
        const int c0 = nt * 8;
        float big[2][4], small[2][4];
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int e = 0; e < 4; ++e) big[i][e] = small[i][e] = 0.f;
#pragma unroll
        for (int s = 0; s < 6; ++s) {
            const int tap = s >> 1, ci = (s & 1) * 16 + 2 * t;
            const float* xp = xs + (tap * C + ci) * XS + c0 + g;
            uint32_t bh[2], bl[2];
            split_b(xp[0], xp[XS], xp[8 * XS], xp[9 * XS], bh, bl, amax);
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                uint32_t ah[4], al[4];
                load_a(a.cw + (16 * i + g) * KK + 16 * s + 2 * t, KK, ah, al, amax);
                mma_x3(big[i], small[i], ah, al, bh, bl);
            }
        }
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int co = 16 * i + g + 8 * h;
                const float bc = __ldg(a.cb + co);
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int j = c0 + 2 * t + e, n = t0 - 1 + j;
                    if (j < YW)
                        ys[co * YS + j] = (n >= 0 && n < a.Ts)
                                              ? lrelu(big[i][2 * h + e] + small[i][2 * h + e] * (1.f / 2048.f) + bc, 0.2f)
                                              : 0.f;
                }
            }
    }
    __syncthreads();
    // ---- the LVC: 4 m-tiles (64 co) x 16 n-tiles; this lane's B column is tile column c0 + g
    for (int nt = warp; nt < NT / 8; nt += 8) {
        const int c0 = nt * 8, s0 = t0 + c0;
        if (s0 >= a.Ts) break;
        uint32_t bh[6][2], bl[6][2];
#pragma unroll
        for (int s = 0; s < 6; ++s) {
            const int tap = s >> 1, ci = (s & 1) * 16 + 2 * t;
            const float* yp = ys + ci * YS + c0 + g + tap;   // y[s + tap - 1] for output sample s = t0 + c0 + g
            split_b(yp[0], yp[YS], yp[8 * YS], yp[9 * YS], bh[s], bl[s], amax);
        }
        float big[4][4], small[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int e = 0; e < 4; ++e) big[i][e] = small[i][e] = 0.f;
        const int my_s = s0 + g;
        const int my_f = my_s < a.Ts ? my_s / a.hop : -1;
        const int f_lo = s0 / a.hop, f_hi = (min(s0 + 7, a.Ts - 1)) / a.hop;
        const float* Pb = a.P + (size_t)b * a.T * a.MP;
#pragma unroll 1
        for (int f = f_lo; f <= f_hi; ++f) {
            const bool mine = my_f == f;
            const float* K = Pb + (size_t)f * a.MP + a.koff + g * KK + 2 * t;
#pragma unroll
            for (int s = 0; s < 6; ++s) {
                const uint32_t mh[2] = {mine ? bh[s][0] : 0u, mine ? bh[s][1] : 0u};
                const uint32_t ml[2] = {mine ? bl[s][0] : 0u, mine ? bl[s][1] : 0u};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    uint32_t ah[4], al[4];
                    load_a(K + 16 * i * KK + 16 * s, KK, ah, al, amax);
                    mma_x3(big[i], small[i], ah, al, mh, ml);
                }
            }
        }
        // rows of m-tiles 0 / 1 (co < 32, the sigmoid half) and 2 / 3 (their tanh partners) sit in the same thread
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int ch = 16 * i + g + 8 * h;
                const float* xr = xb + (size_t)ch * a.pitch;
                float* yr = a.xn + b * a.bs + (size_t)ch * a.pitch;
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int s = s0 + 2 * t + e;
                    if (s >= a.Ts) continue;
                    const float* bias = Pb + (size_t)(s / a.hop) * a.MP + a.boff;
                    const float os = big[i][2 * h + e] + small[i][2 * h + e] * (1.f / 2048.f) + __ldg(bias + ch);
                    const float ot = big[i + 2][2 * h + e] + small[i + 2][2 * h + e] * (1.f / 2048.f) + __ldg(bias + C + ch);
                    yr[s] = xr[s] + (1.f / (1.f + expf(-os))) * tanhf(ot);
                }
            }
    }
    flag_range(amax, a.err);
}

static DeviceOnce g_uv_once;

// ------------------------------------------------------------------ engine
static inline int round4(int v) { return (v + 3) / 4 * 4; }

int Univnet::init(const b200tts_univnet_config& cfg, const float* const* w, int nw) {
    using namespace uv;
    c = cfg;
    const int S = c.num_upsamples, L = c.lvc_layers, Ch = c.kpnet_hidden_channels, Kp = c.kpnet_conv_size;
    B200_REQUIRE(c.hidden_channels == C && c.lvc_kernel_size == 3,
                 "univnet: the kernels take hidden_channels = 32 and lvc_kernel_size = 3 (got %d, %d)", c.hidden_channels,
                 c.lvc_kernel_size);
    B200_REQUIRE(S >= 1 && S <= 8 && L >= 1 && L <= 8 && c.in_channels >= 1 && c.out_channels >= 1 && c.cond_channels >= 1,
                 "univnet: unsupported config (%d upsample factors, %d LVC layers)", S, L);
    B200_REQUIRE(Ch >= 16 && Ch % 16 == 0 && Kp >= 1 && Kp % 2 == 1,
                 "univnet: kpnet_hidden_channels must be a multiple of 16 and kpnet_conv_size odd (got %d, %d)", Ch, Kp);
    hop_total = 1;
    for (int s = 0; s < S; ++s) {
        B200_REQUIRE(c.upsample_factors[s] >= 1 && c.upsample_factors[s] <= 64, "univnet: upsample factor %d",
                     c.upsample_factors[s]);
        hop_total *= c.upsample_factors[s];
    }
    B200_REQUIRE(hop_total <= 4096, "univnet: %d samples per frame (at most 4096)", hop_total);
    for (int i = 0; i < nw; ++i) B200_REQUIRE(w[i] != nullptr, "univnet: weight tensor %d is null", i);
    MP = L * (KSZ + CO);
    WeightList wl(w, nw);
    int rc;
    first.tc_prec = B200TTS_PRECISION_FP32;
    const float *fw = wl.take(), *fb = wl.take();
    if ((rc = pack_conv(first, fw, fb, C, c.in_channels, 7, 1, 3))) return rc;
    blocks.resize(S);
    int hop = 1;
    const int Kd = Kp * Ch, kpad = (Kp - 1) / 2;
    for (int s = 0; s < S; ++s) {
        Block& bl = blocks[s];
        const int u = c.upsample_factors[s];
        hop *= u;
        bl.hop = hop;
        bl.up.tc_prec = B200TTS_PRECISION_FP32;
        const float *uw = wl.take(), *ub = wl.take();
        if ((rc = pack_conv_transpose(bl.up, uw, ub, C, C, 2 * u, u, u / 2 + u % 2, u % 2))) return rc;
        bl.kin.tc_prec = B200TTS_PRECISION_FP32;
        const float *iw = wl.take(), *ib = wl.take();
        if ((rc = pack_conv(bl.kin, iw, ib, Ch, c.cond_channels, 5, 1, 2))) return rc;
        bl.kres.resize(6);
        for (auto& l : bl.kres) {
            l.tc_prec = B200TTS_PRECISION_FP32;
            const float *rw = wl.take(), *rb = wl.take();
            if ((rc = pack_conv(l, rw, rb, Ch, Ch, Kp, 1, kpad))) return rc;
        }
        // kernel_conv | bias_conv as one GEMM, rows permuted into the frame-major layout (see the top of this file)
        const float *kw = wl.take(), *kb = wl.take(), *bw = wl.take(), *bb = wl.take();
        B200_REQUIRE(kw && kb && bw && bb, "univnet: null kernel_conv / bias_conv weight or bias");
        std::vector<float> W((size_t)MP * Kd), bias(MP);
        auto put = [&](int m, const float* src, float bsrc) {   // src: [Ch][Kp] of one reference output channel
            for (int tap = 0; tap < Kp; ++tap)
                for (int ch = 0; ch < Ch; ++ch) W[(size_t)m * Kd + tap * Ch + ch] = src[ch * Kp + tap];
            bias[m] = bsrc;
        };
        for (int l = 0; l < L; ++l)
            for (int co = 0; co < CO; ++co)
                for (int tap = 0; tap < 3; ++tap)
                    for (int ci = 0; ci < C; ++ci) {
                        const int ref = ((l * C + ci) * CO + co) * 3 + tap;
                        put(l * KSZ + co * KK + tap * C + ci, kw + (size_t)ref * Ch * Kp, kb[ref]);
                    }
        for (int l = 0; l < L; ++l)
            for (int co = 0; co < CO; ++co) put(L * KSZ + l * CO + co, bw + (size_t)(l * CO + co) * Ch * Kp, bb[l * CO + co]);
        if (upload(bl.pw, W.data(), W.size()) || upload(bl.pb, bias.data(), bias.size())) return 2;
        // conv_i: [layer][co][tap * 32 + ci]
        std::vector<float> cw((size_t)L * C * KK), cb((size_t)L * C);
        for (int l = 0; l < L; ++l) {
            const float *lw = wl.take(), *lb = wl.take();
            B200_REQUIRE(lw && lb, "univnet: null conv_i weight or bias");
            for (int co = 0; co < C; ++co) {
                for (int ci = 0; ci < C; ++ci)
                    for (int tap = 0; tap < 3; ++tap)
                        cw[((size_t)l * C + co) * KK + tap * C + ci] = lw[((size_t)co * C + ci) * 3 + tap];
                cb[(size_t)l * C + co] = lb[co];
            }
        }
        if (upload(bl.cw, cw.data(), cw.size()) || upload(bl.cb, cb.data(), cb.size())) return 2;
    }
    last.tc_prec = B200TTS_PRECISION_FP32;
    const float *lw = wl.take(), *lb = wl.take();
    if ((rc = pack_conv(last, lw, lb, c.out_channels, C, 7, 1, 3))) return rc;
    return wl.finish("univnet");
}

// the KPnet hidden state (3 tensors); forward() also takes the predicted kernels of one block (P) and two x tensors at
// the final rate
struct UnivnetWs { float *P, *H[3], *X0, *X1; };
static UnivnetWs univnet_carve(const Univnet& m, Arena& ar, int B, int T, bool whole) {
    const size_t Tp = (size_t)round4(T), Ts = (size_t)round4(T * m.hop_total);
    UnivnetWs w{};
    if (whole) w.P = ar.f32((size_t)B * T * m.MP);
    for (float*& h : w.H) h = ar.f32((size_t)B * m.c.kpnet_hidden_channels * Tp);
    if (whole) {
        w.X0 = ar.f32((size_t)B * uv::C * Ts);
        w.X1 = ar.f32((size_t)B * uv::C * Ts);
    }
    return w;
}

size_t Univnet::workspace_bytes(int B, int T) const {
    return arena_size([&](Arena& ar) { univnet_carve(*this, ar, B, T, true); });
}

int Univnet::check_call(const char* who, int B, int T) const {
    B200_REQUIRE(B >= 0 && B <= 65535 && T >= 1, "%s: B = %d, T = %d", who, B, T);
    B200_REQUIRE((long long)T * hop_total < (1LL << 30) && (long long)B * T * MP < (1LL << 40), "%s: %d frames is too long",
                 who, T);
    return 0;
}

static int uv_device(int** err) {
    int num_sms = 0;
    size_t max_smem = 0;
    if (int rc = tc_device(err, &num_sms, &max_smem)) return rc;
    B200_REQUIRE(max_smem >= (size_t)uv::SMEM, "univnet: the LVC kernel needs %d B of shared memory per block", uv::SMEM);
    return device_once(g_uv_once, nullptr, [](int) -> int {
        B200_CUDA_OK(cudaFuncSetAttribute(univnet_lvc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, uv::SMEM));
        return 0;
    });
}

// H = KPnet(mel) [B][Ch][Tp] and P = [kernel_conv | bias_conv](H), frame-major
int Univnet::launch_predict(int blk, const float* mel, int B, int T, float* P, float* H0, float* H1, float* H2, int* err,
                            cudaStream_t st) const {
    const Block& bl = blocks[blk];
    const int Ch = c.kpnet_hidden_channels, Tp = round4(T);
    const long long hbs = (long long)Ch * Tp;
    ConvIO io;
    io.x = dense(mel, c.cond_channels, T); io.Tin = T;
    io.y = dense(H0, Ch, Tp); io.Tout = T; io.B = B;
    io.flags = EPI_WAVEGRAD; io.act = ACT_LRELU; io.act_param = 0.1f;   // input_conv + LeakyReLU(0.1)
    if (int rc = launch_conv(bl.kin, io, st)) return rc;
    const float* in = H0;
    float* outs[2] = {H1, H2};
    for (int k = 0; k < 6; ++k) {   // residual_conv; the last conv's epilogue adds the block input: H = H0 + r
        io.x = dense(in, Ch, Tp);
        io.y = dense(outs[k & 1], Ch, Tp);
        if (k == 5) io.res = dense(H0, Ch, Tp);
        if (int rc = launch_conv(bl.kres[k], io, st)) return rc;
        in = outs[k & 1];
    }
    const long long N = (long long)B * T;
    const dim3 grid((unsigned)((N + uv::PT_N - 1) / uv::PT_N), (unsigned)((MP + uv::PT_M - 1) / uv::PT_M));
    univnet_predict_kernel<<<grid, 256, 0, st>>>(H2, hbs, Tp, Ch, c.kpnet_conv_size, T, B, bl.pw, bl.pb, MP, P, err);
    count_launch();
    dispatch_note(DISPATCH_UNIVNET_PREDICT);
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

int Univnet::launch_lvc(int blk, int l, const float* x, float* xn, int B, int T, int pitch, const float* P, int* err,
                        cudaStream_t st) const {
    using namespace uv;
    const Block& bl = blocks[blk];
    UvLayerArgs a;
    memset(&a, 0, sizeof(a));
    a.x = x; a.xn = xn; a.bs = (long long)C * pitch; a.pitch = pitch;
    a.Ts = T * bl.hop; a.hop = bl.hop; a.T = T;
    int d = 1;
    for (int k = 0; k < l; ++k) d *= 3;
    a.dil = d;
    a.cw = bl.cw + (size_t)l * C * KK; a.cb = bl.cb + (size_t)l * C;
    a.P = P; a.MP = MP; a.koff = l * KSZ; a.boff = c.lvc_layers * KSZ + l * CO;
    a.err = err;
    const dim3 grid((unsigned)((a.Ts + NT - 1) / NT), (unsigned)B);
    univnet_lvc_kernel<<<grid, 256, SMEM, st>>>(a);
    count_launch();
    dispatch_note(DISPATCH_UNIVNET_LVC);
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

int Univnet::forward(const float* mel, const float* noise, int B, int T, float* out, void* ws, size_t ws_bytes,
                     cudaStream_t st) const {
    using namespace uv;
    B200_REQUIRE(mel && noise && out && ws, "univnet_forward: null pointer");
    if (int rc = check_call("univnet_forward", B, T)) return rc;
    if (B == 0) return 0;
    const size_t need = workspace_bytes(B, T);
    B200_REQUIRE(ws_bytes >= need, "univnet_forward: workspace of %zu bytes, %zu needed", ws_bytes, need);
    Arena ar(ws, ws_bytes);
    const UnivnetWs w = univnet_carve(*this, ar, B, T, true);
    float *P = w.P, *X0 = w.X0, *X1 = w.X1;
    int* err = nullptr;
    if (int rc = uv_device(&err)) return rc;
    const int Tp = round4(T);
    int rc;
    {   // first_conv(noise)
        ConvIO io;
        io.x = dense(noise, c.in_channels, T); io.Tin = T;
        io.y = dense(X0, C, Tp); io.Tout = T; io.B = B;
        if ((rc = launch_conv(first, io, st))) return rc;
    }
    float *x = X0, *xo = X1;
    int len = T, pitch = Tp;
    for (int s = 0; s < c.num_upsamples; ++s) {
        const Block& bl = blocks[s];
        if ((rc = launch_predict(s, mel, B, T, P, w.H[0], w.H[1], w.H[2], err, st))) return rc;
        const int Ls = T * bl.hop, Lp = round4(Ls);
        {   // x = upsample(lrelu(x, 0.2))
            ConvIO io;
            io.x = dense(x, C, pitch); io.Tin = len; io.in_slope = 0.2f;
            io.y = dense(xo, C, Lp); io.Tout = Ls; io.B = B;
            if ((rc = launch_conv(bl.up, io, st))) return rc;
        }
        std::swap(x, xo);
        len = Ls; pitch = Lp;
        for (int l = 0; l < c.lvc_layers; ++l) {
            if ((rc = launch_lvc(s, l, x, xo, B, T, pitch, P, err, st))) return rc;
            std::swap(x, xo);
        }
    }
    ConvIO io;   // tanh(last_conv(lrelu(x, 0.1)))
    io.x = dense(x, C, pitch); io.Tin = len; io.in_slope = 0.1f;
    io.y = dense(out, c.out_channels, len); io.Tout = len; io.B = B;
    io.act = ACT_TANH;
    return launch_conv(last, io, st);
}

int Univnet::predict(int blk, const float* mel, int B, int T, float* P, void* ws, size_t ws_bytes, cudaStream_t st) const {
    B200_REQUIRE(mel && P && ws, "univnet_predict: null pointer");
    B200_REQUIRE(blk >= 0 && blk < c.num_upsamples, "univnet_predict: block %d of %d", blk, c.num_upsamples);
    if (int rc = check_call("univnet_predict", B, T)) return rc;
    if (B == 0) return 0;
    const size_t need = arena_size([&](Arena& ar) { univnet_carve(*this, ar, B, T, false); });
    B200_REQUIRE(ws_bytes >= need, "univnet_predict: workspace of %zu bytes, %zu needed", ws_bytes, need);
    Arena ar(ws, ws_bytes);
    const UnivnetWs w = univnet_carve(*this, ar, B, T, false);
    int* err = nullptr;
    if (int rc = uv_device(&err)) return rc;
    return launch_predict(blk, mel, B, T, P, w.H[0], w.H[1], w.H[2], err, st);
}

int Univnet::lvc_layer(int blk, int l, const float* x, const float* P, int B, int T, float* x_new, int pitch,
                       cudaStream_t st) const {
    B200_REQUIRE(x && P && x_new, "univnet_lvc_layer: null pointer");
    B200_REQUIRE(blk >= 0 && blk < c.num_upsamples && l >= 0 && l < c.lvc_layers, "univnet_lvc_layer: block %d layer %d",
                 blk, l);
    B200_REQUIRE(x != x_new, "univnet_lvc_layer: x_new must not be the buffer x is (neighbouring tiles still read x)");
    if (int rc = check_call("univnet_lvc_layer", B, T)) return rc;
    B200_REQUIRE(pitch >= T * blocks[blk].hop, "univnet_lvc_layer: row pitch %d < %d samples", pitch, T * blocks[blk].hop);
    if (B == 0) return 0;
    int* err = nullptr;
    if (int rc = uv_device(&err)) return rc;
    return launch_lvc(blk, l, x, x_new, B, T, pitch, P, err, st);
}

}  // namespace b200tts
