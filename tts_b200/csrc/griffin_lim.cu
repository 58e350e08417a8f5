// Griffin-Lim phase reconstruction and the reference's inverse-spectrogram chain, batched on the device:
// AudioProcessor.inv_spectrogram / inv_melspectrogram (TTS/utils/audio/processor.py:444-458) and
// numpy_transforms.griffin_lim (TTS/utils/audio/numpy_transforms.py:220-230).
//
//  gl_prepare_kernel : denormalize -> db_to_amp (base ** (x / spec_gain)) -> [clamp 1e-10] -> ** power -> |.|, through a
//      32 x 32 shared-memory tile, so the strided model output is read and the result written coalesced.  Linear input
//      goes straight to the magnitudes; mel input runs it twice around the pseudo-inverse GEMM (FP32 conv engine):
//      first denormalize + db_to_amp into [B, n_mels, T], then clamp + power out of [B, F, T].  The magnitudes are
//      frame-major [B, T, F]: an iteration reads one contiguous row per frame.
//  gl_iter_kernel    : one Griffin-Lim iteration, y_next = istft(|S| exp(i angle(stft(y_prev)))), librosa's transforms
//      (center, reflect padding, window-sum-square normalisation, output length hop (T - 1)).  A CTA owns a run of
//      output samples of one row and recomputes every frame that overlaps it, two real frames per complex FFT, so no
//      sample is written by two CTAs and nothing is accumulated across CTAs.  The first launch builds the spectrum from
//      the phase draws instead (angles = exp(2 pi i u)) and flags a row whose waveform is not finite.
//  gl_deemphasis_kernel : scipy.signal.lfilter([1], [1, -coef]) over each row's valid samples as a chunked scan (a plain
//      copy for coef 0), the tail zeroed; a flagged row becomes the reference's np.array([0.0]).
// Every row is computed from its own data on a frame grid anchored at its start, so row b of a batch is bit-identical
// to the same row alone.
#include <float.h>
#include <math.h>

#include "audio_norm.cuh"
#include "engines.cuh"
#include "fft.cuh"

namespace b200tts {

namespace {

constexpr int GL_NT = 256;
constexpr int GL_SCAN_NT = 1024;
constexpr int GL_SAMPLES = 4096;   // output samples per CTA (at least one hop)
enum : int { GL_DENORM_AMP = 1, GL_CLAMP = 2, GL_POWER = 4 };

// frames of row b: lens[b] clamped to [1, T] (the host checks lengths >= 2 before they reach the device)
__device__ __forceinline__ int row_frames(const int* lens, int b, int T) { return lens ? min(max(lens[b], 1), T) : T; }

__device__ __forceinline__ int floor_div(int a, int b) { return (a >= 0) ? a / b : -((-a + b - 1) / b); }

// out[b, c, t] = f(x[b, c, t]) for c < C, t < T_b.  out addressed with (out_cs, out_ts): one of them is 1.
__global__ void __launch_bounds__(256) gl_prepare_kernel(const float* __restrict__ x, long long x_bs, int x_cs, int x_ts,
                                                         int C, int T, const int* __restrict__ lens, NormParams np, float base,
                                                         float gain, float power, int ops, float* __restrict__ out,
                                                         long long out_bs, int out_cs, int out_ts) {
    __shared__ float tile[32][33];
    const int b = blockIdx.z, c0 = blockIdx.y * 32, t0 = blockIdx.x * 32, tx = threadIdx.x, ty = threadIdx.y;
    const int Tb = row_frames(lens, b, T);
    if (t0 >= Tb) return;
    const float* xb = x + (long long)b * x_bs;
    for (int i = 0; i < 32; i += 8) {
        const int c = c0 + ty + i, t = t0 + tx;
        float v = 0.f;
        if (c < C && t < Tb) {
            v = xb[(long long)c * x_cs + (long long)t * x_ts];
            if (ops & GL_DENORM_AMP) {
                v = denorm_one(np, v, c);
                if (base > 0.f) {
                    v = __fdiv_rn(v, gain);
                    v = (base == 10.f) ? exp10f(v) : (base == (float)M_E) ? expf(v) : powf(base, v);
                }
            }
            if (ops & GL_CLAMP) v = fmaxf(v, 1e-10f);
            if (ops & GL_POWER) v = fabsf(power == 1.f ? v : powf(v, power));
        }
        tile[ty + i][tx] = v;
    }
    __syncthreads();
    float* ob = out + (long long)b * out_bs;
    for (int i = 0; i < 32; i += 8) {
        if (out_ts == 1) {      // time-contiguous
            const int c = c0 + ty + i, t = t0 + tx;
            if (c < C && t < Tb) ob[(long long)c * out_cs + t] = tile[ty + i][tx];
        } else {                // frame-major
            const int c = c0 + tx, t = t0 + ty + i;
            if (c < C && t < Tb) ob[(long long)t * out_ts + c] = tile[tx][ty + i];
        }
    }
}

// (re, im) <- s * X / |X|, and (s, 0) where X = 0 (numpy's angle(0) = 0).  Where re^2 + im^2 overflows (|X| > 1.8e19,
// which unclipped dB inputs reach) or underflows, X is scaled by its larger component first.
__device__ __forceinline__ void project(float& re, float& im, float s) {
    const float p = re * re + im * im;
    if (p >= FLT_MIN && p <= FLT_MAX) {
        const float n = sqrtf(p);
        re = s * (re / n); im = s * (im / n);
        return;
    }
    const float m = fmaxf(fabsf(re), fabsf(im));
    if (m == 0.f) { re = s; im = 0.f; return; }
    const float r = re / m, i = im / m, n = sqrtf(r * r + i * i);
    re = s * (r / n); im = s * (i / n);
}

// mag [B, T, F] frame-major; u [B, F, T] phase draws (FIRST only); y rows of pitch y_pitch, L_b = hop (T_b - 1) valid.
// Shared memory: re, im [n_fft] (two frames per transform: frame ta real, frame ta + 1 imaginary), acc, wss [S].
template <bool FIRST>
__global__ void __launch_bounds__(GL_NT) gl_iter_kernel(const float* __restrict__ mag, const float* __restrict__ u,
                                                        const float* __restrict__ yin, float* __restrict__ yout,
                                                        long long y_pitch, const int* __restrict__ lens, int T,
                                                        const float* __restrict__ window, const float2* __restrict__ tw,
                                                        int n_fft, int log2n, int hop, int win_lo, int win_hi, int S,
                                                        int* __restrict__ bad) {
    extern __shared__ float sm[];
    float* re = sm;
    float* im = sm + n_fft;
    float* acc = sm + 2 * n_fft;
    float* wss = acc + S;
    const int b = blockIdx.y, tid = threadIdx.x, half = n_fft / 2, F = half + 1;
    const int Tb = row_frames(lens, b, T);
    const int L = hop * (Tb - 1);
    const int s0 = blockIdx.x * S;
    if (s0 >= L) return;
    if (!FIRST && bad[b]) return;           // a non-finite row: its output is discarded
    const int s1 = min(s0 + S, L);
    for (int j = tid; j < s1 - s0; j += GL_NT) { acc[j] = 0.f; wss[j] = 0.f; }
    // frame t reaches output sample j iff win_lo <= j + half - t hop < win_hi
    const int t_lo = max(0, floor_div(s0 + half - win_hi, hop) + 1);
    const int t_hi = min(Tb - 1, floor_div(s1 - 1 + half - win_lo, hop));
    const float* mb = mag + (long long)b * T * F;
    const float* yb = yin + (long long)b * y_pitch;
    const float inv_n = 1.f / (float)n_fft;
    for (int ta = t_lo; ta <= t_hi; ta += 2) {
        const bool two = ta + 1 <= t_hi;
        const float* ma = mb + (long long)ta * F;
        const float* mbb = ma + F;
        __syncthreads();                    // the previous pair's overlap-add has read re / im
        if (FIRST) {
            const float* ub = u + (long long)b * F * T;
            for (int k = tid; k <= half; k += GL_NT) {
                float sa, ca, sb = 0.f, cb = 0.f;
                sincospif(2.f * ub[(long long)k * T + ta], &sa, &ca);
                float ar = ma[k] * ca, ai = ma[k] * sa, br = 0.f, bi = 0.f;
                if (two) {
                    sincospif(2.f * ub[(long long)k * T + ta + 1], &sb, &cb);
                    br = mbb[k] * cb; bi = mbb[k] * sb;
                }
                if (k == 0 || k == half) { ai = 0.f; bi = 0.f; }   // irfft ignores their imaginary parts
                // C = A + i B is the spectrum of frame ta + i frame ta+1:  C[k] = A[k] + i B[k], C[n-k] = conj(A[k]) + i conj(B[k])
                re[k] = ar - bi; im[k] = ai + br;
                if (k > 0 && k < half) { re[n_fft - k] = ar + bi; im[n_fft - k] = br - ai; }
            }
        } else {
            for (int n = tid; n < n_fft; n += GL_NT) {
                const float w = window[n];
                const int r = fft_brev(n, log2n);
                re[r] = w * yb[reflect_index(ta * hop + n - half, L)];
                im[r] = two ? w * yb[reflect_index((ta + 1) * hop + n - half, L)] : 0.f;
            }
            __syncthreads();
            fft_dit<false>(re, im, tw, n_fft, log2n, tid, GL_NT);
            // split Z = FFT(a + i b) into A = FFT(a), B = FFT(b); project onto |S| with the phase of A / B (angle(0) = 0);
            // thread k owns bins k and n - k, so the in-place rewrite needs no barrier
            for (int k = tid; k <= half; k += GL_NT) {
                const int kn = (n_fft - k) & (n_fft - 1);
                const float zr = re[k], zi = im[k], wr = re[kn], wi = im[kn];
                float ar = 0.5f * (zr + wr), ai = 0.5f * (zi - wi);
                float br = 0.5f * (zi + wi), bi = 0.5f * (wr - zr);
                const float sa = ma[k];
                project(ar, ai, sa);
                if (two) {
                    project(br, bi, mbb[k]);
                } else {
                    br = 0.f; bi = 0.f;
                }
                if (k == 0 || k == half) { ai = 0.f; bi = 0.f; }
                re[k] = ar - bi; im[k] = ai + br;
                if (k > 0 && k < half) { re[kn] = ar + bi; im[kn] = br - ai; }
            }
        }
        __syncthreads();
        fft_dif<true>(re, im, tw, n_fft, log2n, tid, GL_NT);   // bit-reversed output: sample n at fft_brev(n)
        // overlap-add of the two frames, in frame order, onto the owned samples
        const int j_lo = max(s0, ta * hop - half + win_lo);
        const int j_hi = min(s1, (two ? ta + 1 : ta) * hop - half + win_hi);
        for (int j = j_lo + tid; j < j_hi; j += GL_NT) {
            float v = acc[j - s0], q = wss[j - s0];
            const int na = j + half - ta * hop;
            if (na >= win_lo && na < win_hi) {
                const float w = window[na];
                v += w * (re[fft_brev(na, log2n)] * inv_n);
                q += w * w;
            }
            const int nb = na - hop;
            if (two && nb >= win_lo && nb < win_hi) {
                const float w = window[nb];
                v += w * (im[fft_brev(nb, log2n)] * inv_n);
                q += w * w;
            }
            acc[j - s0] = v; wss[j - s0] = q;
        }
    }
    __syncthreads();
    float* ob = yout + (long long)b * y_pitch;
    bool finite = true;
    for (int j = tid; j < s1 - s0; j += GL_NT) {
        const float q = wss[j];
        const float v = (q > FLT_MIN) ? acc[j] / q : acc[j];
        ob[s0 + j] = v;
        finite = finite && isfinite(v);
    }
    if (FIRST && !finite) bad[b] = 1;      // every writer stores the same value
}

// y[n] = x[n] + coef y[n - 1] over the row's L samples: each thread filters its chunk from zero, the chunks' affine maps
// y -> coef^len y + e are scanned across the CTA, and each chunk is filtered again from its carry.
__global__ void __launch_bounds__(GL_SCAN_NT) gl_deemphasis_kernel(const float* __restrict__ y, long long y_pitch,
                                                                   const int* __restrict__ lens, int T, int hop, float coef,
                                                                   const int* __restrict__ bad, float* __restrict__ out,
                                                                   long long out_pitch, int* __restrict__ wav_lengths) {
    __shared__ float sa[GL_SCAN_NT], sb[GL_SCAN_NT];
    const int b = blockIdx.x, tid = threadIdx.x;
    const int Tb = row_frames(lens, b, T);
    const int L = bad[b] ? 1 : hop * (Tb - 1);
    const float* xb = y + (long long)b * y_pitch;
    float* ob = out + (long long)b * out_pitch;
    if (tid == 0) wav_lengths[b] = L;
    for (long long j = L + tid; j < out_pitch; j += GL_SCAN_NT) ob[j] = 0.f;
    if (bad[b]) {
        if (tid == 0) ob[0] = 0.f;
        return;
    }
    if (coef == 0.f) {
        for (int j = tid; j < L; j += GL_SCAN_NT) ob[j] = xb[j];
        return;
    }
    const int chunk = (L + GL_SCAN_NT - 1) / GL_SCAN_NT;
    const int lo = min(L, tid * chunk), hi = min(L, lo + chunk);
    float a = 1.f, e = 0.f;
    for (int j = lo; j < hi; ++j) { e = fmaf(coef, e, xb[j]); a *= coef; }
    sa[tid] = a; sb[tid] = e;
    __syncthreads();
    for (int d = 1; d < GL_SCAN_NT; d <<= 1) {   // inclusive scan: map[k] = map[k] o map[k - d]
        float pa = 1.f, pb = 0.f;
        if (tid >= d) { pa = sa[tid - d]; pb = sb[tid - d]; }
        __syncthreads();
        if (tid >= d) { sb[tid] = fmaf(sa[tid], pb, sb[tid]); sa[tid] *= pa; }
        __syncthreads();
    }
    e = tid > 0 ? sb[tid - 1] : 0.f;
    for (int j = lo; j < hi; ++j) {
        e = fmaf(coef, e, xb[j]);
        ob[j] = e;
    }
}

int gl_samples_per_cta(int hop) { return hop >= GL_SAMPLES ? hop : (GL_SAMPLES / hop) * hop; }

}  // namespace

int GriffinLim::init(int n_fft_, int hop_, const float* window_host, const float* pinv_host, int n_mels_) {
    n_fft = n_fft_; hop = hop_; n_mels = pinv_host ? n_mels_ : 0;
    log2n = 0;
    while ((1 << log2n) < n_fft) ++log2n;
    B200_REQUIRE((1 << log2n) == n_fft && n_fft >= 32 && n_fft <= 8192,
                 "griffin_lim: n_fft=%d must be a power of two in [32, 8192]", n_fft);
    B200_REQUIRE(window_host && hop >= 1 && hop <= n_fft, "griffin_lim: bad window / hop_length=%d", hop);
    B200_REQUIRE(!pinv_host || n_mels_ >= 1, "griffin_lim: n_mels=%d", n_mels_);
    win_lo = n_fft; win_hi = 0;
    for (int n = 0; n < n_fft; ++n)
        if (window_host[n] != 0.f) { win_lo = std::min(win_lo, n); win_hi = n + 1; }
    B200_REQUIRE(win_hi > win_lo, "griffin_lim: the window is zero everywhere");
    int rc;
    if ((rc = upload(window, window_host, n_fft))) return rc;
    const std::vector<float2> tw = fft_twiddles(n_fft);
    if ((rc = upload(twiddle, tw.data(), tw.size()))) return rc;
    // |S| = pinv(mel_basis) [F, n_mels] @ mel  ==  1x1 conv with Cin = n_mels, on the FP32 FMA kernel
    if (pinv_host && (rc = pack_conv(pinv, pinv_host, nullptr, n_fft / 2 + 1, n_mels, 1, 1, 0))) return rc;
    return 0;
}

// the magnitudes, two waveforms, the non-finite row flags; mel input also takes the denormalised mel (amp) and its
// linear projection (lin)
struct GlWs { float *mag, *y[2], *amp, *lin; int* bad; };
static GlWs gl_carve(const GriffinLim& m, Arena& ar, int B, int T) {
    const size_t F = m.n_fft / 2 + 1, BT = (size_t)B * T, L = (size_t)m.hop * (size_t)std::max(T - 1, 0);
    GlWs w{};
    w.mag = ar.f32(BT * F);
    w.y[0] = ar.f32((size_t)B * L);
    w.y[1] = ar.f32((size_t)B * L);
    w.bad = (int*)ar.f32(B);
    if (m.n_mels) {
        w.amp = ar.f32(BT * m.n_mels);
        w.lin = ar.f32(BT * F);
    }
    return w;
}

size_t GriffinLim::workspace_bytes(int B, int T) const {
    return arena_size([&](Arena& ar) { gl_carve(*this, ar, B, T); });
}

int GriffinLim::forward(const float* x, long long x_bs, int x_cs, int x_ts, int B, int C, int T, const int* lens,
                        const b200tts_audio_norm& norm, float base, float spec_gain, float power, int num_iter,
                        float preemphasis, const float* u, float* wav, long long wav_pitch, int* wav_lengths, void* ws,
                        size_t ws_bytes, cudaStream_t st) const {
    const int F = n_fft / 2 + 1;
    B200_REQUIRE(x && u && wav && wav_lengths, "griffin_lim_forward: null pointer");
    B200_REQUIRE(C == (n_mels ? n_mels : F), "griffin_lim_forward: %d channels, the handle takes %d (%s)", C,
                 n_mels ? n_mels : F, n_mels ? "mel" : "linear");
    B200_REQUIRE(B >= 1 && B <= 65535 && T >= 2 && num_iter >= 0, "griffin_lim_forward: B=%d T=%d num_iter=%d", B, T,
                 num_iter);
    B200_REQUIRE((long long)hop * (T - 1) <= 0x7fffffffLL && wav_pitch >= (long long)hop * (T - 1),
                 "griffin_lim_forward: output pitch %lld < %lld samples", wav_pitch, (long long)hop * (T - 1));
    B200_REQUIRE(base >= 0.f && spec_gain != 0.f, "griffin_lim_forward: base=%f spec_gain=%f", (double)base,
                 (double)spec_gain);
    const size_t need = workspace_bytes(B, T);
    B200_REQUIRE(ws_bytes >= need, "griffin_lim_forward: workspace of %zu bytes, %zu needed", ws_bytes, need);
    const long long L = (long long)hop * (T - 1);
    Arena ar(ws, ws_bytes);
    const GlWs w = gl_carve(*this, ar, B, T);
    float *mag = w.mag, *amp = w.amp, *lin = w.lin;
    float* const* y = w.y;
    int* bad = w.bad;
    const NormParams np = to_params(norm);
    const dim3 tblk(32, 8);
    if (!n_mels) {
        dispatch_note(DISPATCH_GL_PREPARE);
        gl_prepare_kernel<<<dim3((T + 31) / 32, (C + 31) / 32, B), tblk, 0, st>>>(
            x, x_bs, x_cs, x_ts, C, T, lens, np, base, spec_gain, power, GL_DENORM_AMP | GL_POWER, mag, (long long)T * F, 1, F);
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
    } else {
        dispatch_note(DISPATCH_GL_PREPARE);
        gl_prepare_kernel<<<dim3((T + 31) / 32, (C + 31) / 32, B), tblk, 0, st>>>(
            x, x_bs, x_cs, x_ts, C, T, lens, np, base, spec_gain, power, GL_DENORM_AMP, amp, (long long)n_mels * T, T, 1);
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
        ConvIO io;
        io.x = dense(amp, n_mels, T); io.Tin = T;
        io.y = dense(lin, F, T); io.Tout = T; io.B = B;
        if (int rc = launch_conv(pinv, io, st)) return rc;
        dispatch_note(DISPATCH_GL_PREPARE);
        gl_prepare_kernel<<<dim3((T + 31) / 32, (F + 31) / 32, B), tblk, 0, st>>>(
            lin, (long long)F * T, T, 1, F, T, lens, np, 0.f, 1.f, power, GL_CLAMP | GL_POWER, mag, (long long)T * F, 1, F);
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
    }
    B200_CUDA_OK(cudaMemsetAsync(bad, 0, sizeof(int) * B, st));
    const int S = gl_samples_per_cta(hop);
    const size_t smem = sizeof(float) * (2 * (size_t)n_fft + 2 * (size_t)S);
    static DeviceOnce attr_once;
    if (int rc = device_once(attr_once, nullptr, [](int) -> int {
            B200_CUDA_OK(cudaFuncSetAttribute(gl_iter_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
            B200_CUDA_OK(cudaFuncSetAttribute(gl_iter_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
            return 0;
        })) return rc;
    const dim3 grid((unsigned)((L + S - 1) / S), B);
    for (int it = 0; it <= num_iter; ++it) {
        dispatch_note(DISPATCH_GL_ITER);
        if (it == 0)
            gl_iter_kernel<true><<<grid, GL_NT, smem, st>>>(mag, u, nullptr, y[0], L, lens, T, window, twiddle, n_fft, log2n,
                                                           hop, win_lo, win_hi, S, bad);
        else
            gl_iter_kernel<false><<<grid, GL_NT, smem, st>>>(mag, nullptr, y[(it - 1) & 1], y[it & 1], L, lens, T, window,
                                                            twiddle, n_fft, log2n, hop, win_lo, win_hi, S, bad);
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
    }
    dispatch_note(DISPATCH_GL_DEEMPHASIS);
    gl_deemphasis_kernel<<<B, GL_SCAN_NT, 0, st>>>(y[num_iter & 1], L, lens, T, hop, preemphasis, bad, wav, wav_pitch,
                                                   wav_lengths);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace b200tts
