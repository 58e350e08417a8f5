// STFT magnitude + mel projection front end.
// Reference: TTS/tts/models/vits.py:96-138 (wav_to_spec: reflect pad (n_fft-hop)/2, hann STFT center=False,
//            sqrt(re^2+im^2+1e-6)), :141-157 (spec_to_mel: mel_basis @ spec, log(clamp(.,1e-5))), :160-208 (wav_to_mel);
//            TTS/utils/audio/torch_transforms.py:104-145 (TorchSTFT.__call__: center=True, sqrt(clamp(.,1e-8))).
// One CTA transforms FR consecutive frames of one utterance: windowed frame -> shared memory (bit-reversed),
// radix-2 FFT in shared memory with a precomputed twiddle table, magnitudes staged in shared memory and written
// as FR-wide runs per frequency bin (the [B, F, frames] layout is frame-contiguous).  The mel projection is a
// 1x1 "conv" over the frequency axis through the fused conv1d kernel with a log-clamp epilogue.
#include <math.h>

#include "engines.cuh"

namespace b200tts {

namespace {

constexpr int STFT_FR = 8;
constexpr int STFT_NT = 256;

__device__ __forceinline__ int reflect_index(int i, int n) {   // torch 'reflect' padding (no edge repeat)
    if (n == 1) return 0;
    const int period = 2 * (n - 1);
    i %= period;
    if (i < 0) i += period;
    return (i < n) ? i : period - i;
}

__global__ void __launch_bounds__(STFT_NT) stft_mag_kernel(const float* wav, const float* window, const float2* twiddle,
                                                          float* spec, int T, int n_fft, int log2n, int hop, int pad1,
                                                          int pad2, int n_frames, int mode, float power) {
    extern __shared__ float sm[];
    float* re = sm;                     // [n_fft]
    float* im = sm + n_fft;             // [n_fft]
    float* mag = sm + 2 * n_fft;        // [STFT_FR][F]
    const int F = n_fft / 2 + 1;
    const int b = blockIdx.y, frame0 = blockIdx.x * STFT_FR, tid = threadIdx.x;
    const float* wb = wav + (size_t)b * T;
    const int len1 = T + 2 * pad1;      // length after the first (inner) reflect pad
    for (int fr = 0; fr < STFT_FR; ++fr) {
        const int frame = frame0 + fr;
        if (frame >= n_frames) break;
        for (int n = tid; n < n_fft; n += STFT_NT) {
            int i = frame * hop + n - pad2;            // index into the once-padded signal
            if (pad2 > 0) i = reflect_index(i, len1);
            i -= pad1;                                  // index into the raw signal
            if (pad1 > 0) i = reflect_index(i, T);
            const float v = (i >= 0 && i < T) ? wb[i] * window[n] : 0.f;
            const int r = (int)(__brev((unsigned)n) >> (32 - log2n));
            re[r] = v;
            im[r] = 0.f;
        }
        __syncthreads();
        for (int s = 1; s <= log2n; ++s) {
            const int half = 1 << (s - 1), tstride = n_fft >> s;
            for (int k = tid; k < n_fft / 2; k += STFT_NT) {
                const int j = k & (half - 1);
                const int i0 = ((k >> (s - 1)) << s) + j, i1 = i0 + half;
                const float2 w = twiddle[j * tstride];  // (cos, -sin)(2 pi j tstride / n_fft)
                const float xr = re[i1], xi = im[i1];
                const float tr = w.x * xr - w.y * xi, ti = w.x * xi + w.y * xr;
                const float ur = re[i0], ui = im[i0];
                re[i0] = ur + tr; im[i0] = ui + ti;
                re[i1] = ur - tr; im[i1] = ui - ti;
            }
            __syncthreads();
        }
        for (int f = tid; f < F; f += STFT_NT) {
            const float p = re[f] * re[f] + im[f] * im[f];
            float m = (mode == 0) ? sqrtf(p + 1e-6f) : (mode == 2) ? p : sqrtf(fmaxf(p, 1e-8f));   // 2: power spectrum
            if (power != 1.f) m = powf(m, power);
            mag[fr * F + f] = m;
        }
        __syncthreads();
    }
    const int nfr = min(STFT_FR, n_frames - frame0);
    for (int idx = tid; idx < F * STFT_FR; idx += STFT_NT) {
        const int f = idx / STFT_FR, fr = idx - f * STFT_FR;
        if (fr < nfr) spec[((size_t)b * F + f) * n_frames + frame0 + fr] = mag[fr * F + f];
    }
}

}  // namespace

Stft::~Stft() {
    if (window) cudaFree(window);
    if (twiddle) cudaFree(twiddle);
    free_conv(mel);
}

int Stft::init(int n_fft_, int hop_, const float* window_host, const float* mel_basis_host, int n_mels_) {
    n_fft = n_fft_; hop = hop_; n_mels = n_mels_;
    log2n = 0;
    while ((1 << log2n) < n_fft) ++log2n;
    B200_REQUIRE((1 << log2n) == n_fft && n_fft >= 32 && n_fft <= 8192, "stft: n_fft=%d must be a power of two in [32, 8192]", n_fft);
    B200_REQUIRE(hop >= 1 && window_host, "stft: bad arguments");
    int rc;
    if ((rc = upload(&window, window_host, n_fft))) return rc;
    std::vector<float> tw(n_fft);  // n_fft/2 float2 entries
    for (int k = 0; k < n_fft / 2; ++k) {
        const double a = -2.0 * M_PI * (double)k / (double)n_fft;
        tw[2 * k] = (float)cos(a);
        tw[2 * k + 1] = (float)sin(a);
    }
    if ((rc = upload(&twiddle, tw.data(), n_fft))) return rc;
    if (mel_basis_host && n_mels > 0) {
        // mel = basis [n_mels, F] @ spec [F, frames]  ==  1x1 conv with Cin = F
        if ((rc = pack_conv(mel, mel_basis_host, nullptr, n_mels, n_fft / 2 + 1, 1, 1, 0))) return rc;
    }
    return 0;
}

int Stft::magnitude(const float* wav, int B, int T, int pad1, int pad2, int mode, float power, float* spec,
                    int n_frames, cudaStream_t st) const {
    B200_REQUIRE(wav && spec, "stft_magnitude: null pointer");
    if (B == 0 || n_frames <= 0) return 0;
    B200_REQUIRE(pad1 < T && pad2 < T + 2 * pad1, "stft_magnitude: reflect padding needs pad < length");
    B200_REQUIRE((long long)(n_frames - 1) * hop + n_fft <= (long long)T + 2LL * pad1 + 2LL * pad2,
                 "stft_magnitude: n_frames=%d exceeds the padded signal", n_frames);
    const int F = n_fft / 2 + 1;
    const size_t smem = sizeof(float) * (2 * (size_t)n_fft + (size_t)STFT_FR * F);
    static DeviceOnce attr_once;
    if (int rc = device_once(attr_once, nullptr, [](int) -> int {
            B200_CUDA_OK(cudaFuncSetAttribute(stft_mag_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
            return 0;
        })) return rc;
    dim3 grid((n_frames + STFT_FR - 1) / STFT_FR, B);
    stft_mag_kernel<<<grid, STFT_NT, smem, st>>>(wav, window, reinterpret_cast<const float2*>(twiddle), spec, T, n_fft,
                                                 log2n, hop, pad1, pad2, n_frames, mode, power);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

int Stft::mel_project(const float* spec, int B, int n_frames, float log_clamp, float* out, cudaStream_t st) const {
    B200_REQUIRE(mel.w, "mel_project: handle was created without a mel basis");
    const int F = n_fft / 2 + 1;
    ConvIO io;
    io.x = spec; io.x_bs = (long long)F * n_frames; io.x_cs = n_frames; io.Tin = n_frames;
    io.y = out; io.y_bs = (long long)n_mels * n_frames; io.y_cs = n_frames; io.Tout = n_frames; io.B = B;
    if (log_clamp > 0.f) { io.act = ACT_LOGCLAMP; io.act_param = log_clamp; }
    return launch_conv(mel, io, st);
}

}  // namespace b200tts
