// Durations -> monotonic path -> expanded prior, replacing the glue at TTS/tts/models/vits.py:1140-1155:
//   w = exp(logw) * x_mask * length_scale ; w_ceil = ceil(w) ; y_lengths = clamp_min(sum(w_ceil), 1)
//   attn = generate_path(w_ceil, mask)                (TTS/tts/utils/helpers.py:154-169)
//   m_p, logs_p = matmul(attn^T, .)                   (a gather, exact because attn is one-hot)
//   z_p = m_p + noise * exp(logs_p) * inference_noise_scale
// Stage 1 runs before the one unavoidable host sync (max y_length fixes T_dec); stage 2 after it.
#include <limits.h>
#include "engines.cuh"

namespace b200tts {

namespace {

// one warp per utterance (one CTA, warps stride over the batch): inclusive scan of integral-valued fp32 durations
// (exact below 2^24).  The same CTA reduces max(y_lengths) and forwards the duration predictor's error flag into
// `meta` = {max y_length, flag}, so the caller's one host read fetches both (no second synchronisation); the FORWARD rule
// has no flag and reports the shortest row's y_length instead (SpeedySpeech's convs need a minimum length).
// GLOW: the Glow-TTS rule (glow_tts.py:350-352), w = (exp(logw) - 1) * x_mask * length_scale and w_ceil =
// clamp_min(ceil(w), 1) -- the clamp gives every padded token one frame too -- plus dur_log = log(1 + sum(attn, -1)) *
// x_mask of compute_outputs (:147): a valid token's path row holds w_ceil ones, a padded token's none.
// FORWARD: the ForwardTTS rule (forward_tts.py:369-371), w = (exp(logw) - 1) * x_mask * length_scale, values below 1
// become 1, then round half to even (torch.round); a padded token gets 0 frames.  exp is evaluated in double and
// rounded once, so the exactly representable ties (2.5, 3.5, ...) come out as the reference's.
enum : int { RULE_VITS = 0, RULE_GLOW = 1, RULE_FORWARD = 2 };
template <int RULE>
__global__ void durations_kernel(const float* logw, const float* x_mask, float length_scale, float* w_ceil,
                                 float* cum, long long* y_lengths, int B, int T, const int* err_flag, long long* meta,
                                 float* dur_log) {
    __shared__ long long wmax[32], wmin[32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    long long mymax = 0, mymin = LLONG_MAX;
    for (int b = warp; b < B; b += nwarps) {
        float carry = 0.f;
        for (int t0 = 0; t0 < T; t0 += 32) {
            const int t = t0 + lane;
            float wc = 0.f;
            if (t < T) {
                const float m = x_mask[(size_t)b * T + t];
                if (RULE == RULE_GLOW) {
                    const float w = __fmul_rn(__fmul_rn(__fsub_rn(expf(logw[(size_t)b * T + t]), 1.f), m), length_scale);
                    wc = fmaxf(ceilf(w), 1.f);
                    dur_log[(size_t)b * T + t] = __fmul_rn(logf(__fadd_rn(1.f, __fmul_rn(wc, m))), m);
                } else if (RULE == RULE_FORWARD) {
                    const float e = (float)exp((double)logw[(size_t)b * T + t]);
                    const float w = __fmul_rn(__fmul_rn(__fsub_rn(e, 1.f), m), length_scale);
                    wc = m != 0.f ? rintf(w < 1.f ? 1.f : w) : 0.f;
                } else {
                    const float w = __fmul_rn(__fmul_rn(expf(logw[(size_t)b * T + t]), m), length_scale);
                    wc = ceilf(w);
                }
                w_ceil[(size_t)b * T + t] = wc;
            }
            float s = wc;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const float n = __shfl_up_sync(0xffffffffu, s, o);
                if (lane >= o) s += n;
            }
            s += carry;
            if (t < T) cum[(size_t)b * T + t] = s;
            carry = __shfl_sync(0xffffffffu, s, 31);
        }
        const long long yl = RULE == RULE_FORWARD ? (long long)carry : (long long)fmaxf(carry, 1.f);
        if (lane == 0) y_lengths[b] = yl;
        mymax = yl > mymax ? yl : mymax;
        mymin = yl < mymin ? yl : mymin;
    }
    if (meta) {
        if (lane == 0) { wmax[warp] = mymax; wmin[warp] = mymin; }
        __syncthreads();
        if (threadIdx.x == 0) {
            long long m = 0, n = LLONG_MAX;
            for (int i = 0; i < nwarps; ++i) {
                m = wmax[i] > m ? wmax[i] : m;
                n = wmin[i] < n ? wmin[i] : n;
            }
            meta[0] = m;
            meta[1] = RULE == RULE_FORWARD ? n : err_flag ? (long long)err_flag[0] : 0;
        }
    }
}

// one thread per decoder frame: token index by binary search over the cumulative durations
__global__ void expand_prior_kernel(const float* cum, const float* x_mask, const long long* y_lengths,
                                    const float* stats, const float* noise, float noise_scale, float* attn,
                                    float* m_p, float* logs_p, float* z_p, float* y_mask, int Tx, int Ty, int C) {
    const int y = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (y >= Ty) return;
    const float* cb = cum + (size_t)b * Tx;
    const bool yvalid = (long long)y < y_lengths[b];
    int lo = 0, hi = Tx;   // smallest j with cum[j] > y
    const float fy = (float)y;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (cb[mid] > fy) hi = mid; else lo = mid + 1;
    }
    const int j = lo;
    // path[x,y] = [cum[x-1] <= y < cum[x]] * x_mask[x] * y_mask[y]   (helpers.py:163-168)
    const bool hit = yvalid && j < Tx && x_mask[(size_t)b * Tx + j] != 0.f;
    if (y_mask) y_mask[(size_t)b * Ty + y] = yvalid ? 1.f : 0.f;
    if (attn) {
        float* ab = attn + (size_t)b * Tx * Ty + y;
        for (int x = 0; x < Tx; ++x) ab[(size_t)x * Ty] = (hit && x == j) ? 1.f : 0.f;
    }
    const float* sm = stats + (size_t)b * 2 * C * Tx;          // [m_p | logs_p], each [C, Tx]
    const size_t ob = (size_t)b * C * Ty + y;
    for (int c = 0; c < C; ++c) {
        const float m = hit ? sm[(size_t)c * Tx + j] : 0.f;
        const float s = hit ? sm[(size_t)(C + c) * Tx + j] : 0.f;
        m_p[ob + (size_t)c * Ty] = m;
        logs_p[ob + (size_t)c * Ty] = s;
        // m_p + noise * exp(logs_p) * scale, evaluated left to right like the reference
        if (z_p) z_p[ob + (size_t)c * Ty] = __fadd_rn(m, __fmul_rn(__fmul_rn(noise[ob + (size_t)c * Ty], expf(s)), noise_scale));
    }
}

}  // namespace

int launch_durations(const float* logw, const float* x_mask, float length_scale, int B, int T, float* w_ceil,
                     float* cum, long long* y_lengths, const int* err_flag, long long* meta, cudaStream_t st) {
    B200_REQUIRE(logw && x_mask && w_ceil && cum && y_lengths, "durations: null pointer");
    if (B == 0) return 0;
    durations_kernel<RULE_VITS><<<1, 32 * (B < 32 ? B : 32), 0, st>>>(logw, x_mask, length_scale, w_ceil, cum, y_lengths,
                                                                 B, T, err_flag, meta, nullptr);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

int launch_durations_glow(const float* logw, const float* x_mask, float length_scale, int B, int T, float* w_ceil,
                          float* cum, long long* y_lengths, float* dur_log, long long* meta, cudaStream_t st) {
    B200_REQUIRE(logw && x_mask && w_ceil && cum && y_lengths && dur_log, "durations_glow: null pointer");
    if (B == 0) return 0;
    durations_kernel<RULE_GLOW><<<1, 32 * (B < 32 ? B : 32), 0, st>>>(logw, x_mask, length_scale, w_ceil, cum, y_lengths,
                                                                B, T, nullptr, meta, dur_log);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

int launch_durations_forward(const float* logw, const float* x_mask, float length_scale, int B, int T, float* dur,
                             float* cum, long long* y_lengths, long long* meta, cudaStream_t st) {
    B200_REQUIRE(logw && x_mask && dur && cum && y_lengths, "durations_forward: null pointer");
    if (B == 0) return 0;
    durations_kernel<RULE_FORWARD><<<1, 32 * (B < 32 ? B : 32), 0, st>>>(logw, x_mask, length_scale, dur, cum,
                                                                        y_lengths, B, T, nullptr, meta, nullptr);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

int launch_expand_prior(const float* cum, const float* x_mask, const long long* y_lengths, const float* stats,
                        const float* noise, float noise_scale, int B, int Tx, int Ty, int C, float* attn, float* m_p,
                        float* logs_p, float* z_p, float* y_mask, cudaStream_t st) {
    B200_REQUIRE(cum && x_mask && y_lengths && stats && m_p && logs_p && (noise || !z_p), "expand_prior: null pointer");
    if (B == 0 || Ty == 0) return 0;
    dim3 grid((Ty + 127) / 128, B);
    expand_prior_kernel<<<grid, 128, 0, st>>>(cum, x_mask, y_lengths, stats, noise, noise_scale, attn, m_p, logs_p,
                                              z_p, y_mask, Tx, Ty, C);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------ latent upsampling (VitsArgs.encoder_sample_rate)
// z' = F.interpolate(z, scale_factor=[f], mode="linear") (vits.py:952; align_corners=False): source position
// (t + 0.5)/f - 0.5 clamped at 0, neighbours t1 and min(t1+1, Tin-1), weights (1-l, l).
namespace {
__global__ void upsample_linear_kernel(const float* __restrict__ x, float* __restrict__ y, int rows, int Tin, int Tout,
                                       float rscale) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= Tout) return;
    float src = fmaf(rscale, (float)t + 0.5f, -0.5f);   // one rounding, like the reference build's contracted expression
    src = src < 0.f ? 0.f : src;
    const int t1 = (int)src;
    const int t1p = (t1 < Tin - 1) ? 1 : 0;
    const float l1 = src - (float)t1, l0 = 1.f - l1;
    for (size_t row = blockIdx.y; row < (size_t)rows; row += gridDim.y) {
        const float* xr = x + row * Tin;
        y[row * Tout + t] = fmaf(l1, xr[t1 + t1p], __fmul_rn(l0, xr[t1]));
    }
}
}  // namespace

int launch_upsample_linear(const float* x, int rows, int Tin, float scale_factor, float* y, int Tout, cudaStream_t st) {
    B200_REQUIRE(x && y && scale_factor > 0.f, "upsample_linear: bad arguments");
    if (rows == 0 || Tout == 0) return 0;
    dim3 grid((Tout + 255) / 256, rows < 65535 ? rows : 65535);
    upsample_linear_kernel<<<grid, 256, 0, st>>>(x, y, rows, Tin, Tout, (float)(1.0 / (double)scale_factor));
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace b200tts
