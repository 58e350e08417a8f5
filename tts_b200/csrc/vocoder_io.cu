// The hand-off kernels either side of the HiFiGAN generator on the reference's public path (SURVEY 8 f1 / f3):
//
//  vocoder_input_kernel : what Synthesizer.tts does between the TTS model and a standalone vocoder
//      (TTS/utils/synthesizer.py:412-429): tts_ap.denormalize -> vocoder_ap.normalize
//      (TTS/utils/audio/processor.py:259-337, all four branches: mean-var, symmetric, asymmetric, clip) ->
//      interpolate_vocoder_input (TTS/vocoder/utils/generic_utils.py:11-29: bilinear, align_corners=False,
//      recompute_scale_factor=True, scale [1, sr_voc/sr_tts]) -> the replicate padding of HifiganGenerator.inference
//      (TTS/vocoder/models/hifigan_generator.py:281) -- fused into ONE pass that writes conv_pre's input with a
//      16-byte aligned row pitch.  The reference does this in numpy on the host, one sentence at a time.
//  absmax / to_int16    : save_wav's peak normalisation, wav * (32767 / max(0.01, max|wav|)) truncated to int16
//      (TTS/utils/audio/numpy_transforms.py:439-441), on the device: the conv_post kernel already folds max|wav| into a
//      device word while it stores the waveform (conv1d.cu), to_int16 scales and converts.
#include "audio_norm.cuh"
#include "engines.cuh"

namespace b200tts {

namespace {

// out[b, c, j] for j in [0, Tmid + 2*pad): source column jj = clamp(j - pad, 0, Tmid - 1) of the interpolated
// spectrogram; interpolation (Tmid != T): src = (jj + 0.5) * (T / Tmid) - 0.5 clamped at 0, neighbours t0, min(t0+1, T-1).
__global__ void vocoder_input_kernel(const float* __restrict__ x, int x_bs, int x_cs, int x_ts, NormParams dn, NormParams nm,
                                     int C, int T, int Tmid, float rscale, int pad, float* __restrict__ y, int Tout,
                                     int y_pitch) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= Tout) return;
    const int jj = min(max(j - pad, 0), Tmid - 1);
    int t0 = jj, t1 = jj;
    float l1 = 0.f;
    if (Tmid != T) {
        float src = fmaf(rscale, (float)jj + 0.5f, -0.5f);
        src = src < 0.f ? 0.f : src;
        t0 = (int)src;
        t1 = t0 + ((t0 < T - 1) ? 1 : 0);
        l1 = src - (float)t0;
    }
    const float l0 = 1.f - l1;
    const int b = blockIdx.z;
    for (int c = blockIdx.y; c < C; c += gridDim.y) {
        const float* xr = x + (long long)b * x_bs + (long long)c * x_cs;
        const float v0 = norm_one(nm, denorm_one(dn, xr[(long long)t0 * x_ts], c), c);
        float v = v0;
        if (Tmid != T) {
            const float v1 = norm_one(nm, denorm_one(dn, xr[(long long)t1 * x_ts], c), c);
            v = __fadd_rn(__fmul_rn(l0, v0), __fmul_rn(l1, v1));      // the order upsample_bilinear2d uses: w0*x0 + w1*x1
        }
        y[((long long)b * C + c) * y_pitch + j] = v;
    }
}

__global__ void absmax_kernel(const float* __restrict__ x, long long n, unsigned* __restrict__ out) {
    float m = 0.f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        m = fmaxf(m, fabsf(x[i]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(out, __float_as_uint(m));   // non-negative floats order like uints
}

// columns [lo, hi) of `rows` rows of `pitch` floats (a streaming window of the waveform)
__global__ void absmax_window_kernel(const float* __restrict__ x, long long pitch, int lo, int hi, unsigned* __restrict__ out) {
    float m = 0.f;
    const float* xr = x + (long long)blockIdx.y * pitch;
    for (int i = lo + (int)(blockIdx.x * blockDim.x + threadIdx.x); i < hi; i += (int)(gridDim.x * blockDim.x))
        m = fmaxf(m, fabsf(xr[i]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(out, __float_as_uint(m));
}

// wav * (32767 / max(0.01, peak)) truncated toward zero (numpy astype(int16) of an in-range float)
__global__ void to_int16_kernel(const float* __restrict__ x, long long n, const unsigned* __restrict__ peak_bits,
                                short* __restrict__ out) {
    const float peak = __uint_as_float(*peak_bits);
    const float s = __fdiv_rn(32767.f, fmaxf(0.01f, peak));
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        out[i] = (short)__float2int_rz(__fmul_rn(x[i], s));
}

}  // namespace

int vocoder_input_len(int T, float scale_factor, int pad) {
    const int Tmid = (scale_factor == 1.f) ? T : (int)floor((double)T * (double)scale_factor);
    return Tmid + 2 * pad;
}

int launch_vocoder_input(const float* x, long long x_bs, int x_cs, int x_ts, int B, int C, int T,
                         const b200tts_audio_norm* denorm, const b200tts_audio_norm* norm, float scale_factor, int pad,
                         float* y, int y_pitch, cudaStream_t st) {
    B200_REQUIRE(x && y && denorm && norm, "vocoder_input: null pointer");
    B200_REQUIRE(scale_factor > 0.f && pad >= 0, "vocoder_input: bad scale_factor / padding");
    if (B == 0 || C == 0 || T == 0) return 0;
    const int Tmid = (scale_factor == 1.f) ? T : (int)floor((double)T * (double)scale_factor);
    B200_REQUIRE(Tmid >= 1, "vocoder_input: scale_factor %f leaves no frames", (double)scale_factor);
    const int Tout = Tmid + 2 * pad;
    B200_REQUIRE(y_pitch >= Tout, "vocoder_input: output pitch %d < %d columns", y_pitch, Tout);
    dim3 grid((Tout + 127) / 128, C < 65535 ? C : 65535, B);
    B200_REQUIRE(B <= 65535, "vocoder_input: batch too large");
    // recompute_scale_factor=True: coordinates use the size ratio, not the requested factor
    const float rscale = (float)((double)T / (double)Tmid);
    vocoder_input_kernel<<<grid, 128, 0, st>>>(x, (int)x_bs, x_cs, x_ts, to_params(*denorm), to_params(*norm), C, T, Tmid,
                                               rscale, pad, y, Tout, y_pitch);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

// grid-stride kernels: eight CTAs per SM of the current device
static int stride_grid(long long n) {
    int dev = 0, sms = 132;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
        sms = 132;
    return (int)std::min<long long>((n + 1023) / 1024, (long long)sms * 8);
}

int launch_absmax(const float* x, long long n, unsigned* peak_bits, cudaStream_t st) {
    B200_REQUIRE(peak_bits && (x || n == 0), "absmax: null pointer");
    if (n == 0) return 0;
    const int blocks = stride_grid(n);
    absmax_kernel<<<blocks, 256, 0, st>>>(x, n, peak_bits);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

int launch_absmax_window(const float* x, int rows, long long pitch, int lo, int hi, unsigned* peak_bits, cudaStream_t st) {
    B200_REQUIRE(peak_bits && (x || rows == 0), "absmax: null pointer");
    if (rows <= 0 || hi <= lo) return 0;
    B200_REQUIRE(rows <= 65535, "absmax: too many rows");
    const dim3 grid((unsigned)std::min((hi - lo + 255) / 256, 64), (unsigned)rows);
    absmax_window_kernel<<<grid, 256, 0, st>>>(x, pitch, lo, hi, peak_bits);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

int launch_to_int16(const float* x, long long n, const unsigned* peak_bits, short* out, cudaStream_t st) {
    B200_REQUIRE(peak_bits && (n == 0 || (x && out)), "to_int16: null pointer");
    if (n == 0) return 0;
    const int blocks = stride_grid(n);
    to_int16_kernel<<<blocks, 256, 0, st>>>(x, n, peak_bits, out);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace b200tts
