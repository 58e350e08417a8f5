// MelGAN generator engine (plain, full-band, multi-band) and the PQMF synthesis kernel.
// Reference semantics: TTS/vocoder/models/melgan_generator.py:9-74 (MelganGenerator), TTS/vocoder/layers/melgan.py:6-36
// (ResidualStack), TTS/vocoder/layers/pqmf.py:9-53 (PQMF.synthesis), multiband_melgan_generator.py:36-43.
//
// Every layer but the PQMF filter runs on the shared conv engine: reflection padding is an input addressing mode of its
// kernels (ConvIO::reflect), so no padded copy of any activation is made.  Per residual block three launches:
//   h = conv_dil(lrelu(x, 0.2))            reflect-padded by (res_kernel - 1) / 2 * dilation
//   y = shortcut(x)                        1x1, no prologue
//   y += conv1x1(lrelu(h, 0.2))            EPI_ACCUM: (acc + bias) + shortcut, the reference's shortcut(x) + block(x)
// and x / y swap.  conv_pre, the upsamplers and the residual-stack convs request the 3xTF32 tensor-core kernels;
// conv_post (1 or 4 output rows) stays FP32 (single-row streaming kernel or the FMA tile kernel).
#include "engines.cuh"

namespace b200tts {

// ------------------------------------------------------------------ PQMF synthesis
// synthesis(x) = conv1d(conv_transpose1d(x, N * I, stride N), G, padding = taps / 2) as one polyphase filter:
//   y[n] = sum_k sum_j N G[k, j] x[k, (n + j - taps/2) / N]    over the j with n + j - taps/2 a multiple of N whose
// quotient lies in [0, Tb) (zero padding).  A CTA produces PQ_TB band steps (N * PQ_TB samples); its band window
// [N][PQ_TB + 2 halo] and N * G sit in shared memory, so every x element is read from global memory once per CTA (plus
// the halo).  HBM-bound: 4 B read per band sample, 4 B written per output sample.  y has N * Tb - taps % 2 samples.
constexpr int PQ_TB = 256;

__global__ void __launch_bounds__(256) pqmf_synthesis_kernel(const float* __restrict__ x, long long x_bs, int x_cs, int N,
                                                             int Tb, const float* __restrict__ G, int taps, int halo,
                                                             float* __restrict__ y, unsigned* __restrict__ peak_bits) {
    extern __shared__ float sm[];
    const int K1 = taps + 1, W = PQ_TB + 2 * halo;
    float* gs = sm;                 // [N][taps + 1], scaled by N (the updown filter's factor)
    float* xs = sm + N * K1;        // [N][W], column j <-> band step t0 - halo + j
    const int b = blockIdx.y, t0 = blockIdx.x * PQ_TB;
    for (int i = threadIdx.x; i < N * K1; i += blockDim.x) gs[i] = (float)N * G[i];
    const float* xb = x + b * x_bs;
    for (int i = threadIdx.x; i < N * W; i += blockDim.x) {
        const int k = i / W, j = i - k * W, t = t0 - halo + j;
        xs[i] = (t >= 0 && t < Tb) ? __ldg(xb + (long long)k * x_cs + t) : 0.f;
    }
    __syncthreads();
    const int P = taps / 2;
    const long long Ty = (long long)N * Tb - (taps & 1);   // conv1d(padding = taps / 2) drops one sample for odd taps
    float m = 0.f;
    for (int r = 0; r < N; ++r) {
        const long long n = (long long)N * t0 + r * PQ_TB + threadIdx.x;
        if (n >= Ty) continue;
        const int e = (int)(n - (long long)N * t0) - P;        // n - P relative to the CTA's first sample (a multiple of N)
        const int j0 = ((-e) % N + N) % N;                      // first tap with e + j a multiple of N
        float acc = 0.f;
        for (int k = 0; k < N; ++k) {
            const float* g = gs + k * K1;
            const float* xr = xs + k * W + halo;
            for (int j = j0; j <= taps; j += N) acc = fmaf(g[j], xr[(e + j) / N], acc);
        }
        y[b * Ty + n] = acc;
        m = fmaxf(m, fabsf(acc));
    }
    if (peak_bits) {   // save_wav's max|wav| folded into the store, one atomic per warp (as conv_post does for HiFiGAN)
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
        if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(peak_bits, __float_as_uint(m));
    }
}

int launch_pqmf_synthesis(const float* x, long long x_bs, int x_cs, int B, int N, int Tb, const float* G, int taps, float* y,
                          unsigned* peak_bits, cudaStream_t st) {
    B200_REQUIRE(x && G && y, "pqmf_synthesis: null pointer");
    B200_REQUIRE(N >= 1 && N <= 64 && taps >= 0 && taps <= 1024 && B >= 0 && B <= 65535 && Tb >= 0,
                 "pqmf_synthesis: unsupported shape (N %d, taps %d, B %d, Tb %d)", N, taps, B, Tb);
    if (B == 0 || Tb == 0) return 0;
    const int P = taps / 2;
    // (n + j - P) / N stays within [-ceil(P / N), PQ_TB - 1 + ceil((taps - P) / N)] of the CTA's first band step
    const int halo = (std::max(P, taps - P) + N - 1) / N + 1;
    const size_t smem = ((size_t)N * (taps + 1) + (size_t)N * (PQ_TB + 2 * halo)) * sizeof(float);
    B200_REQUIRE(smem <= 48 * 1024, "pqmf_synthesis: %zu B of shared memory", smem);
    const dim3 grid((unsigned)((Tb + PQ_TB - 1) / PQ_TB), (unsigned)B);
    pqmf_synthesis_kernel<<<grid, 256, smem, st>>>(x, x_bs, x_cs, N, Tb, G, taps, halo, y, peak_bits);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------ engine
static inline int round4(int v) { return (v + 3) / 4 * 4; }

Melgan::~Melgan() {
    free_conv(conv_pre);
    free_conv(conv_post);
    for (auto& l : ups) free_conv(l);
    for (auto& st : blocks)
        for (auto& b : st) { free_conv(b.dil); free_conv(b.c1x1); free_conv(b.shortcut); }
    if (G) cudaFree(G);
}

int Melgan::init(const b200tts_melgan_config& cfg, const float* const* w, int nw) {
    c = cfg;
    const int S = c.num_upsamples, nb = c.num_res_blocks;
    B200_REQUIRE(S >= 1 && S <= 8 && nb >= 1 && nb <= 8 && c.in_channels > 0 && c.out_channels > 0 &&
                     c.proj_kernel >= 1 && c.proj_kernel % 2 == 1 && c.res_kernel >= 1 && c.res_kernel % 2 == 1 &&
                     c.base_channels >= (1 << S) && c.base_channels % (1 << S) == 0,
                 "melgan: unsupported config (proj_kernel and res_kernel must be odd, base_channels divisible by 2^stages)");
    for (int s = 0; s < S; ++s) B200_REQUIRE(c.upsample_factors[s] >= 1, "melgan: upsample factor %d", c.upsample_factors[s]);
    B200_REQUIRE(c.pqmf_bands == 0 || (c.pqmf_bands == c.out_channels && c.pqmf_taps >= 0 && c.pqmf_taps <= 1024),
                 "melgan: pqmf_bands must be 0 or equal out_channels (%d), with pqmf_taps >= 0", c.out_channels);
    const int expect = 2 + S * (2 + 6 * nb) + 2 + (c.pqmf_bands > 0 ? 1 : 0);
    B200_REQUIRE(nw == expect, "melgan: expected %d weight tensors, got %d", expect, nw);
    int i = 0, rc;
    const int ppad = (c.proj_kernel - 1) / 2;
    conv_pre.tc_prec = B200TTS_PRECISION_FP32;
    if ((rc = pack_conv(conv_pre, w[i], w[i + 1], c.base_channels, c.in_channels, c.proj_kernel, 1, ppad))) return rc;
    i += 2;
    ups.resize(S);
    blocks.assign(S, std::vector<Block>(nb));
    int ch = c.base_channels;
    for (int s = 0; s < S; ++s) {
        const int u = c.upsample_factors[s], Cs = ch / 2;
        ups[s].tc_prec = B200TTS_PRECISION_FP32;
        if ((rc = pack_conv_transpose(ups[s], w[i], w[i + 1], ch, Cs, 2 * u, u, u / 2 + u % 2, u % 2))) return rc;
        i += 2;
        int d = 1;
        for (int m = 0; m < nb; ++m, d *= c.res_kernel) {
            Block& bl = blocks[s][m];
            bl.dil.tc_prec = bl.c1x1.tc_prec = bl.shortcut.tc_prec = B200TTS_PRECISION_FP32;
            if ((rc = pack_conv(bl.dil, w[i], w[i + 1], Cs, Cs, c.res_kernel, d, (c.res_kernel - 1) / 2 * d))) return rc;
            if ((rc = pack_conv(bl.c1x1, w[i + 2], w[i + 3], Cs, Cs, 1, 1, 0))) return rc;
            if ((rc = pack_conv(bl.shortcut, w[i + 4], w[i + 5], Cs, Cs, 1, 1, 0))) return rc;
            i += 6;
        }
        ch = Cs;
    }
    if ((rc = pack_conv(conv_post, w[i], w[i + 1], c.out_channels, ch, c.proj_kernel, 1, ppad))) return rc;
    i += 2;
    if (c.pqmf_bands > 0) {
        B200_REQUIRE(w[i] != nullptr, "melgan: null PQMF filter");
        if (upload(&G, w[i], (size_t)c.pqmf_bands * (c.pqmf_taps + 1))) return 2;
    }
    return 0;
}

void Melgan::stage_dims(int T, std::vector<int>& C, std::vector<int>& L) const {
    C.resize(c.num_upsamples);
    L.resize(c.num_upsamples);
    int ch = c.base_channels, len = T;
    for (int s = 0; s < c.num_upsamples; ++s) {
        ch /= 2;
        len = conv_transpose_out_len(ups[s], len);   // = len * u (output_padding u % 2)
        C[s] = ch;
        L[s] = len;
    }
}

// floats per row of the scratch H: a residual block's hidden tensor, and (synthesis) conv_post's band signals
// [out_channels][L_last] -- which exceed the stage tensors when out_channels > the last stage's channels
static size_t h_floats(const b200tts_melgan_config& c, const std::vector<int>& C, const std::vector<int>& L) {
    size_t mx = (size_t)c.out_channels * (size_t)L.back();
    for (size_t s = 0; s < C.size(); ++s) mx = std::max(mx, (size_t)C[s] * (size_t)round4(L[s]));
    return mx;
}

int Melgan::out_len(int T) const {
    std::vector<int> C, L;
    stage_dims(T, C, L);
    return L.back();
}

size_t Melgan::workspace_bytes(int B, int T) const {
    std::vector<int> C, L;
    stage_dims(T, C, L);
    size_t mx = 0;
    for (size_t s = 0; s < C.size(); ++s) mx = std::max(mx, (size_t)C[s] * (size_t)round4(L[s]));
    const size_t Tp = (size_t)round4(T);
    return arena_bytes((size_t)B * c.in_channels * Tp) + arena_bytes((size_t)B * c.base_channels * Tp) +
           2 * arena_bytes((size_t)B * mx) + arena_bytes((size_t)B * h_floats(c, C, L));
}

int Melgan::check_len(int T) const {
    B200_REQUIRE(T >= 1, "melgan_forward: T = %d", T);
    const int ppad = (c.proj_kernel - 1) / 2;
    B200_REQUIRE(ppad <= T - 1, "melgan_forward: conv_pre reflect-pads %d columns; needs at least %d frames, got %d", ppad,
                 ppad + 1, T);
    std::vector<int> C, L;
    stage_dims(T, C, L);
    for (int s = 0; s < c.num_upsamples; ++s) {
        const int pad = blocks[s].back().dil.pad;   // the largest dilation
        B200_REQUIRE(pad <= L[s] - 1, "melgan_forward: stage %d reflect-pads %d columns; needs at least %d, got %d (T = %d)",
                     s, pad, pad + 1, L[s], T);
    }
    B200_REQUIRE(ppad <= L.back() - 1, "melgan_forward: conv_post reflect-pads %d columns; needs at least %d, got %d", ppad,
                 ppad + 1, L.back());
    return 0;
}

int Melgan::forward(const float* x, int B, int T, int synthesize, float* out, unsigned* peak_bits, void* ws,
                    size_t ws_bytes, cudaStream_t st) const {
    B200_REQUIRE(x && out && ws, "melgan_forward: null pointer");
    B200_REQUIRE(!synthesize || c.pqmf_bands > 0, "melgan_forward: synthesis needs a multi-band generator (pqmf_bands > 0)");
    B200_REQUIRE(B >= 0, "melgan_forward: B = %d", B);
    if (B == 0) return 0;
    if (int rc = check_len(T)) return rc;
    B200_REQUIRE(ws_bytes >= workspace_bytes(B, T), "melgan_forward: workspace too small");
    std::vector<int> C, L;
    stage_dims(T, C, L);
    size_t mx = 0;
    for (size_t s = 0; s < C.size(); ++s) mx = std::max(mx, (size_t)C[s] * (size_t)round4(L[s]));
    const int Tp = round4(T), C0 = c.base_channels;
    Arena ar(ws, ws_bytes);
    float* Xp = ar.f32((size_t)B * c.in_channels * Tp);
    float* P = ar.f32((size_t)B * C0 * Tp);
    float* X = ar.f32((size_t)B * mx);
    float* Y = ar.f32((size_t)B * mx);
    float* H = ar.f32((size_t)B * h_floats(c, C, L));
    B200_REQUIRE(Xp && P && X && Y && H, "melgan_forward: arena exhausted");
    // 16-byte aligned input rows for the tensor-core producers: re-pitch an unaligned input once (B x in x T floats)
    const float* xin = x;
    int x_pitch = T;
    if (Tp != T || (reinterpret_cast<uintptr_t>(x) & 15) != 0) {
        B200_CUDA_OK(cudaMemcpy2DAsync(Xp, (size_t)Tp * sizeof(float), x, (size_t)T * sizeof(float), (size_t)T * sizeof(float),
                                       (size_t)B * c.in_channels, cudaMemcpyDeviceToDevice, st));
        xin = Xp;
        x_pitch = Tp;
    }
    int rc;
    {   // conv_pre(reflect_pad(x))   (melgan_generator.py:32-35)
        ConvIO io;
        io.x = xin; io.x_bs = (long long)c.in_channels * x_pitch; io.x_cs = x_pitch; io.Tin = T;
        io.y = P; io.y_bs = (long long)C0 * Tp; io.y_cs = Tp; io.Tout = T; io.B = B;
        io.reflect = 1;
        if ((rc = launch_conv(conv_pre, io, st))) return rc;
    }
    const float* cur = P;
    int curC = C0, curL = T, curP = Tp;
    for (int s = 0; s < c.num_upsamples; ++s) {
        const int Cs = C[s], Ls = L[s], Lp = round4(Ls);
        const long long bs = (long long)Cs * Lp;
        float* xa = (cur == X) ? Y : X;    // never the buffer the upsampler reads
        float* ya = (xa == X) ? Y : X;
        {   // x = ups(lrelu(x, 0.2))   (:44-57)
            ConvIO io;
            io.x = cur; io.x_bs = (long long)curC * curP; io.x_cs = curP; io.Tin = curL; io.in_slope = 0.2f;
            io.y = xa; io.y_bs = bs; io.y_cs = Lp; io.Tout = Ls; io.B = B;
            if ((rc = launch_conv(ups[s], io, st))) return rc;
        }
        for (const Block& bl : blocks[s]) {   // x = shortcut(x) + block(x)   (melgan.py:33-36)
            ConvIO io;
            io.x = xa; io.x_bs = bs; io.x_cs = Lp; io.Tin = Ls; io.in_slope = 0.2f;
            io.y = H; io.y_bs = bs; io.y_cs = Lp; io.Tout = Ls; io.B = B;
            io.reflect = 1;
            if ((rc = launch_conv(bl.dil, io, st))) return rc;
            io.in_slope = 1.f; io.reflect = 0; io.y = ya;
            if ((rc = launch_conv(bl.shortcut, io, st))) return rc;
            io.x = H; io.in_slope = 0.2f; io.flags = EPI_ACCUM;
            if ((rc = launch_conv(bl.c1x1, io, st))) return rc;
            std::swap(xa, ya);
        }
        cur = xa; curC = Cs; curL = Ls; curP = Lp;
    }
    {   // tanh(conv_post(reflect_pad(lrelu(x, 0.2))))   (:62-70); the band signals go to H when they are synthesised
        ConvIO io;
        io.x = cur; io.x_bs = (long long)curC * curP; io.x_cs = curP; io.Tin = curL; io.in_slope = 0.2f;
        io.y = synthesize ? H : out; io.y_bs = (long long)c.out_channels * curL; io.y_cs = curL; io.Tout = curL; io.B = B;
        io.act = ACT_TANH;
        io.reflect = 1;
        io.peak_bits = synthesize ? nullptr : peak_bits;
        if ((rc = launch_conv(conv_post, io, st))) return rc;
    }
    if (synthesize)   // PQMF.synthesis (pqmf.py:50-53)
        return launch_pqmf_synthesis(H, (long long)c.out_channels * curL, curL, B, c.pqmf_bands, curL, G, c.pqmf_taps, out,
                                     peak_bits, st);
    return 0;
}

}  // namespace b200tts
