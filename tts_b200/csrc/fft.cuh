// Shared-memory power-of-two FFTs for one CTA, over separate real / imaginary arrays of n = 2^log2n points.
//
//   reflect_index       where sample i of a signal of n samples, reflect-padded on both sides, comes from
//   fft_twiddles        host: the table tw[k] = exp(-2 pi i k / n), k < n / 2, computed in double
//   fft_brev            bit reversal of an index (where a decimation-in-time input goes)
//   fft_dit_radix2      one radix-2 decimation-in-time stage s (span 2^s): STFT's whole transform, stage by stage
//   fft_dit             bit-reversed input -> natural output, stages paired into radix-4 butterflies
//   fft_dif             natural input -> bit-reversed output, the decimation-in-frequency mirror of fft_dit
// INV = true uses the conjugate twiddles (an unscaled inverse transform).  Each stage is followed by a barrier, so
// every thread of the CTA must call these with the same arguments; tid / nt are the caller's thread index and count.
#pragma once
#include <math.h>
#include <vector>

namespace b200tts {

inline std::vector<float2> fft_twiddles(int n) {
    std::vector<float2> tw(n / 2);
    for (int k = 0; k < n / 2; ++k) {
        const double a = -2.0 * M_PI * (double)k / (double)n;
        tw[k] = make_float2((float)cos(a), (float)sin(a));
    }
    return tw;
}

// 'reflect' padding without edge repeat (numpy's np.pad, torch's within one length): periodic with period 2 (n - 1),
// so a pad longer than the signal keeps reflecting as numpy's does.
__device__ __forceinline__ int reflect_index(int i, int n) {
    if (n == 1) return 0;
    const int period = 2 * (n - 1);
    i %= period;
    if (i < 0) i += period;
    return (i < n) ? i : period - i;
}

__device__ __forceinline__ int fft_brev(int i, int log2n) { return (int)(__brev((unsigned)i) >> (32 - log2n)); }

template <bool INV>
__device__ __forceinline__ float2 fft_tw(const float2* tw, int k) {
    const float2 w = tw[k];
    return INV ? make_float2(w.x, -w.y) : w;
}

__device__ __forceinline__ void cmul(float ar, float ai, float2 w, float& r, float& i) {
    r = w.x * ar - w.y * ai;
    i = w.x * ai + w.y * ar;
}

template <bool INV = false>
__device__ __forceinline__ void fft_dit_radix2(float* re, float* im, const float2* tw, int n, int s, int tid, int nt) {
    const int half = 1 << (s - 1), tstride = n >> s;
    for (int k = tid; k < n / 2; k += nt) {
        const int j = k & (half - 1);
        const int i0 = ((k >> (s - 1)) << s) + j, i1 = i0 + half;
        const float2 w = fft_tw<INV>(tw, j * tstride);   // (cos, -sin)(2 pi j tstride / n)
        const float xr = re[i1], xi = im[i1];
        const float tr = w.x * xr - w.y * xi, ti = w.x * xi + w.y * xr;
        const float ur = re[i0], ui = im[i0];
        re[i0] = ur + tr; im[i0] = ui + ti;
        re[i1] = ur - tr; im[i1] = ui - ti;
    }
}

// Radix-2 stages s and s + 1 in one pass: the same products as the two radix-2 stages, with the second stage's
// odd twiddle W^(j + half) taken as W^j * (-/+ i) exactly instead of from the table.
template <bool INV>
__device__ __forceinline__ void fft_dit_radix4(float* re, float* im, const float2* tw, int n, int s, int tid, int nt) {
    const int half = 1 << (s - 1);
    for (int q = tid; q < n / 4; q += nt) {
        const int j = q & (half - 1);
        const int i0 = ((q >> (s - 1)) << (s + 1)) + j, i1 = i0 + half, i2 = i1 + half, i3 = i2 + half;
        const float2 w1 = fft_tw<INV>(tw, j * (n >> s)), w2 = fft_tw<INV>(tw, j * (n >> (s + 1)));
        const float2 w3 = INV ? make_float2(-w2.y, w2.x) : make_float2(w2.y, -w2.x);
        float ar, ai, br, bi;
        cmul(re[i1], im[i1], w1, ar, ai);
        cmul(re[i3], im[i3], w1, br, bi);
        const float y0r = re[i0] + ar, y0i = im[i0] + ai, y1r = re[i0] - ar, y1i = im[i0] - ai;
        const float y2r = re[i2] + br, y2i = im[i2] + bi, y3r = re[i2] - br, y3i = im[i2] - bi;
        cmul(y2r, y2i, w2, ar, ai);
        cmul(y3r, y3i, w3, br, bi);
        re[i0] = y0r + ar; im[i0] = y0i + ai; re[i2] = y0r - ar; im[i2] = y0i - ai;
        re[i1] = y1r + br; im[i1] = y1i + bi; re[i3] = y1r - br; im[i3] = y1i - bi;
    }
}

template <bool INV>
__device__ __forceinline__ void fft_dit(float* re, float* im, const float2* tw, int n, int log2n, int tid, int nt) {
    int s = 1;
    if (log2n & 1) {
        fft_dit_radix2<INV>(re, im, tw, n, 1, tid, nt);
        __syncthreads();
        s = 2;
    }
    for (; s < log2n; s += 2) {
        fft_dit_radix4<INV>(re, im, tw, n, s, tid, nt);
        __syncthreads();
    }
}

// Decimation in frequency, stages s and s - 1 (spans 2^s and 2^(s-1)) in one radix-4 pass.
template <bool INV>
__device__ __forceinline__ void fft_dif_radix4(float* re, float* im, const float2* tw, int n, int s, int tid, int nt) {
    const int qs = 1 << (s - 2);
    for (int q = tid; q < n / 4; q += nt) {
        const int j = q & (qs - 1);
        const int i0 = ((q >> (s - 2)) << s) + j, i1 = i0 + qs, i2 = i1 + qs, i3 = i2 + qs;
        const float2 wa = fft_tw<INV>(tw, j * (n >> s)), wc = fft_tw<INV>(tw, j * (n >> (s - 1)));
        const float2 wb = INV ? make_float2(-wa.y, wa.x) : make_float2(wa.y, -wa.x);
        const float x0r = re[i0], x0i = im[i0], x1r = re[i1], x1i = im[i1];
        const float x2r = re[i2], x2i = im[i2], x3r = re[i3], x3i = im[i3];
        const float y0r = x0r + x2r, y0i = x0i + x2i, y1r = x1r + x3r, y1i = x1i + x3i;
        float y2r, y2i, y3r, y3i;
        cmul(x0r - x2r, x0i - x2i, wa, y2r, y2i);
        cmul(x1r - x3r, x1i - x3i, wb, y3r, y3i);
        re[i0] = y0r + y1r; im[i0] = y0i + y1i;
        cmul(y0r - y1r, y0i - y1i, wc, re[i1], im[i1]);
        re[i2] = y2r + y3r; im[i2] = y2i + y3i;
        cmul(y2r - y3r, y2i - y3i, wc, re[i3], im[i3]);
    }
}

template <bool INV>
__device__ __forceinline__ void fft_dif(float* re, float* im, const float2* tw, int n, int log2n, int tid, int nt) {
    int s = log2n;
    for (; s >= 2; s -= 2) {
        fft_dif_radix4<INV>(re, im, tw, n, s, tid, nt);
        __syncthreads();
    }
    if (s == 1) {   // odd log2n: the last span-2 stage, twiddle 1
        for (int k = tid; k < n / 2; k += nt) {
            const float ar = re[2 * k], ai = im[2 * k], br = re[2 * k + 1], bi = im[2 * k + 1];
            re[2 * k] = ar + br; im[2 * k] = ai + bi;
            re[2 * k + 1] = ar - br; im[2 * k + 1] = ai - bi;
        }
        __syncthreads();
    }
}

}  // namespace b200tts
