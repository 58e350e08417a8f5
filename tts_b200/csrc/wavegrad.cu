// WaveGrad refinement network (engines.cuh: Wavegrad).  Reference semantics: TTS/vocoder/models/wavegrad.py:106-145
// (forward and the refinement loop), TTS/vocoder/layers/wavegrad.py:19-154 (PositionalEncoding, FiLM, UBlock, DBlock).
//
// Every conv but out_conv runs on the shared conv engine.  Per FiLM two launches:
//   h = input_conv(x)   epilogue (lrelu(acc + bias, 0.2) + noise_level[b]) + pe[c, t] / 5000   (the table as `res`)
//   F = output_conv(h)  -> the [shift | scale] tensor, kept for the UBlock of the same rate
// per DBlock four (the decimation x[..., ::f] is the nearest-resampling input mode; the 1x1 res_block commutes with it):
//   R = res_block(x[::f]);  A = main0(lrelu(x[::f]));  B = main1(lrelu(A));  out = main2(lrelu(B)) + R
// per UBlock five (x_inter = nearest upsampling of x, read through the same input mode, never written):
//   R = res_block(x_inter)
//   O = film(main0(lrelu(x_inter)))
//   H = film(res2), R = res2 = R + main1(lrelu(O))          one launch: res2 to y2 = R (element for element), film to H
//   O = film(out0(lrelu(H)))
//   H = out1(lrelu(O)) + R
// and out_conv (128 -> 1, k3) is a single-row kernel here whose epilogue is either the plain output (forward) or the
// refinement update (step).  The same (shift, scale) serves all three FiLMs of a UBlock.
#include "engines.cuh"

namespace b200tts {

static inline int round4(int v) { return (v + 3) / 4 * 4; }
constexpr float WG_SLOPE = 0.2f;

// ------------------------------------------------------------------ out_conv (+ refinement update)
// eps[b, t] = bias + sum_ci sum_k w[ci, k] x[b, ci, t + k - 1] (zero padding); each thread owns 4 consecutive samples.
// update = 0: out[b, t] = eps.  update = 1: y[b, t] = clamp(c1 * (y - c2 * eps) + sigma * z, -1, 1) in place (z nullable),
// every product and sum rounded on its own as the reference's separate tensor ops do.  HBM-bound by the x read.
__global__ void __launch_bounds__(256) wavegrad_out_kernel(const float* __restrict__ x, long long x_bs, int x_cs, int Cin,
                                                           int L, const float* __restrict__ w, const float* __restrict__ bias,
                                                           float* y, const float* __restrict__ z, float c1, float c2,
                                                           float sigma, int update) {
    extern __shared__ float ws[];
    for (int i = threadIdx.x; i < Cin * 3; i += blockDim.x) ws[i] = w[i];
    __syncthreads();
    const int b = blockIdx.y;
    const int t0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (t0 >= L) return;
    const float* xb = x + b * x_bs;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int ci = 0; ci < Cin; ++ci) {
        const float* xr = xb + (long long)ci * x_cs;
        float win[6];
#pragma unroll
        for (int i = 0; i < 6; ++i) {
            const int t = t0 - 1 + i;
            win[i] = (t >= 0 && t < L) ? __ldg(xr + t) : 0.f;
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float wk = ws[ci * 3 + k];
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[j] = fmaf(wk, win[j + k], acc[j]);
        }
    }
    const float bv = bias[0];
    float* yb = y + (long long)b * L;
    const float* zb = z ? z + (long long)b * L : nullptr;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int t = t0 + j;
        if (t >= L) break;
        const float eps = __fadd_rn(acc[j], bv);
        if (!update) { yb[t] = eps; continue; }
        float u = __fmul_rn(c1, __fsub_rn(yb[t], __fmul_rn(c2, eps)));
        if (zb) u = __fadd_rn(u, __fmul_rn(sigma, zb[t]));
        yb[t] = fminf(fmaxf(u, -1.f), 1.f);
    }
}

// ------------------------------------------------------------------ engine
int Wavegrad::hop() const {
    int h = 1;
    for (int i = 0; i < c.num_upsamples; ++i) h *= c.upsample_factors[i];
    return h;
}

void Wavegrad::lengths(int T, std::vector<int>& L) const {
    const int n = c.num_upsamples;
    L.assign(n, 0);
    L[0] = hop() * T;
    for (int i = 0; i + 1 < n; ++i) L[i + 1] = L[i] / c.upsample_factors[n - 1 - i];
}

int Wavegrad::init(const b200tts_wavegrad_config& cfg, const float* const* w, int nw) {
    c = cfg;
    const int n = c.num_upsamples;
    B200_REQUIRE(n >= 1 && n <= 8 && c.in_channels > 0 && c.out_channels == 1 && c.y_conv_channels > 0 &&
                     c.x_conv_channels > 0,
                 "wavegrad: unsupported config (1 to 8 upsample factors, out_channels 1)");
    for (int i = 0; i < n; ++i) {
        B200_REQUIRE(c.upsample_factors[i] >= 1 && c.ublock_out_channels[i] > 0, "wavegrad: upsample factor / channels");
        for (int k = 0; k < 4; ++k) B200_REQUIRE(c.upsample_dilations[i][k] >= 1, "wavegrad: dilation");
        // FiLM i + 1 reads DBlock i's output and is built for ublock_out_channels[n - 1 - i] input channels
        if (i + 1 < n)
            B200_REQUIRE(c.dblock_out_channels[i] > 0 && c.dblock_out_channels[i] == c.ublock_out_channels[n - 1 - i],
                         "wavegrad: dblock_out_channels[%d] = %d must equal ublock_out_channels[%d] = %d", i,
                         c.dblock_out_channels[i], n - 1 - i, c.ublock_out_channels[n - 1 - i]);
    }
    for (int i = 0; i < nw; ++i) B200_REQUIRE(w[i] != nullptr, "wavegrad: null weight %d", i);
    WeightList wl(w, nw);
    int rc;
    // split-fp16 operands where Cin % 16 == 0 (pack_rows falls back to 3xTF32 otherwise; y_conv's Cin 1 runs on FMA)
    auto conv = [&](ConvLayer& L, int Cout, int Cin, int K, int dil) -> int {
        L.tc_prec = B200TTS_PRECISION_F16X3;
        const float *cw = wl.take(), *cb = wl.take();
        return pack_conv(L, cw, cb, Cout, Cin, K, dil, (K - 1) / 2 * dil);
    };
    if ((rc = conv(y_conv, c.y_conv_channels, 1, 5, 1))) return rc;
    db.resize(n - 1);
    int ic = c.y_conv_channels;
    for (int d = 0; d + 1 < n; ++d) {
        const int oc = c.dblock_out_channels[d];
        db[d].f = c.upsample_factors[n - 1 - d];
        if ((rc = conv(db[d].res, oc, ic, 1, 1)) || (rc = conv(db[d].m0, oc, ic, 3, 1)) || (rc = conv(db[d].m1, oc, oc, 3, 2)) ||
            (rc = conv(db[d].m2, oc, oc, 3, 4)))
            return rc;
        ic = oc;
    }
    film.resize(n);
    ic = c.y_conv_channels;
    for (int f = 0; f < n; ++f) {
        const int oc = c.ublock_out_channels[n - 1 - f];
        if ((rc = conv(film[f].in, ic, ic, 3, 1)) || (rc = conv(film[f].out, 2 * oc, ic, 3, 1))) return rc;
        if (f + 1 < n) ic = c.dblock_out_channels[f];
    }
    ub.resize(n);
    ic = c.x_conv_channels;
    for (int u = 0; u < n; ++u) {
        const int hc = c.ublock_out_channels[u];
        const int* d = c.upsample_dilations[u];
        ub[u].f = c.upsample_factors[u];
        if ((rc = conv(ub[u].res, hc, ic, 1, 1)) || (rc = conv(ub[u].m0, hc, ic, 3, d[0])) || (rc = conv(ub[u].m1, hc, hc, 3, d[1])) ||
            (rc = conv(ub[u].o0, hc, hc, 3, d[2])) || (rc = conv(ub[u].o1, hc, hc, 3, d[3])))
            return rc;
        ic = hc;
    }
    if ((rc = conv(x_conv, c.x_conv_channels, c.in_channels, 3, 1))) return rc;
    if ((rc = upload(out_w, wl.take(), (size_t)ic * 3)) || (rc = upload(out_b, wl.take(), 1))) return rc;
    return wl.finish("wavegrad");
}

// per-batch-row floats: [0] conditioning, [1 .. n] FiLM tensors, [n + 1] one stage buffer (five are used)
static void wg_sizes(const Wavegrad& m, int T, std::vector<size_t>& s) {
    const auto& c = m.c;
    const int n = c.num_upsamples;
    std::vector<int> L;
    m.lengths(T, L);
    s.assign(n + 2, 0);
    s[0] = (size_t)c.x_conv_channels * round4(T);
    size_t mx = (size_t)c.y_conv_channels * round4(L[0]);
    int ic = c.y_conv_channels;
    for (int i = 0; i < n; ++i) {
        s[1 + i] = (size_t)2 * c.ublock_out_channels[n - 1 - i] * round4(L[i]);
        mx = std::max(mx, (size_t)ic * round4(L[i]));                                   // FiLM input_conv output
        if (i + 1 < n) {
            mx = std::max(mx, (size_t)c.dblock_out_channels[i] * round4(L[i + 1]));    // DBlock tensors
            ic = c.dblock_out_channels[i];
        }
        mx = std::max(mx, (size_t)c.ublock_out_channels[n - 1 - i] * round4(L[i]));   // UBlock n-1-i tensors
    }
    s[n + 1] = mx;
}

namespace {
struct WgBufs {
    float* xc = nullptr;
    std::vector<float*> F;
    float* P[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
};
// x_conv's output comes first, so condition() and step() find it at the same offset
WgBufs wg_carve(const Wavegrad& m, Arena& ar, int B, int T) {
    std::vector<size_t> s;
    wg_sizes(m, T, s);
    const int n = m.c.num_upsamples;
    WgBufs o;
    o.xc = ar.f32((size_t)B * s[0]);
    o.F.resize(n);
    for (int i = 0; i < n; ++i) o.F[i] = ar.f32((size_t)B * s[1 + i]);
    for (auto& p : o.P) p = ar.f32((size_t)B * s[n + 1]);
    return o;
}
// a stage buffer that is none of the given ones
float* wg_pick(const WgBufs& o, const float* a, const float* b = nullptr, const float* c = nullptr, const float* d = nullptr) {
    for (float* p : o.P)
        if (p != a && p != b && p != c && p != d) return p;
    return nullptr;
}
}  // namespace

size_t Wavegrad::workspace_bytes(int B, int T) const {
    return arena_size([&](Arena& ar) { wg_carve(*this, ar, B, T); });
}

int Wavegrad::condition(const float* x, int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) const {
    B200_REQUIRE(x, "wavegrad_condition: null input");
    B200_REQUIRE(B >= 1 && T >= 1, "wavegrad_condition: B = %d, T = %d", B, T);
    const size_t need = workspace_bytes(B, T);
    B200_REQUIRE(ws && ws_bytes >= need, "wavegrad: workspace of %zu bytes, %zu needed", ws_bytes, need);
    Arena ar(ws, ws_bytes);
    const WgBufs o = wg_carve(*this, ar, B, T);
    ConvIO io;   // x_conv (wavegrad.py:115)
    io.x = dense(x, c.in_channels, T); io.Tin = T;
    io.y = dense(o.xc, c.x_conv_channels, round4(T)); io.Tout = T; io.B = B;
    return launch_conv(x_conv, io, st);
}

int Wavegrad::network(const float* y, const float* noise_level, const float* const* pe, int pe_frames, int B, int T,
                      float* out, float c1, float c2, float sigma, const float* z, int update, void* ws, size_t ws_bytes,
                      cudaStream_t st) const {
    B200_REQUIRE(y && noise_level && pe && out, "wavegrad: null pointer");
    B200_REQUIRE(B >= 1 && B <= 65535 && T >= 1, "wavegrad: B = %d, T = %d", B, T);
    B200_REQUIRE(pe_frames >= T, "wavegrad: positional-encoding tables for %d frames, the input has %d", pe_frames, T);
    const int n = c.num_upsamples;
    for (int i = 0; i < n; ++i) B200_REQUIRE(pe[i], "wavegrad: null positional-encoding table %d", i);
    const size_t need = workspace_bytes(B, T);
    B200_REQUIRE(ws && ws_bytes >= need, "wavegrad: workspace of %zu bytes, %zu needed", ws_bytes, need);
    Arena ar(ws, ws_bytes);
    const WgBufs o = wg_carve(*this, ar, B, T);
    std::vector<int> L, Lpe;
    lengths(T, L);
    lengths(pe_frames, Lpe);
    int rc;
    // ---- down path (wavegrad.py:108-113)
    float* cur = o.P[0];
    int curC = c.y_conv_channels;
    {   // y_conv(y): y is the caller's dense [B, 1, L0]
        ConvIO io;
        io.x = dense(y, 1, L[0]); io.Tin = L[0];
        io.y = dense(cur, curC, round4(L[0])); io.Tout = L[0]; io.B = B;
        if ((rc = launch_conv(y_conv, io, st))) return rc;
    }
    for (int i = 0; i < n; ++i) {
        const int Li = L[i], Lp = round4(Li), oc = c.ublock_out_channels[n - 1 - i];
        {   // FiLM i (layers/wavegrad.py:50-54)
            float* h = wg_pick(o, cur);
            ConvIO io;
            io.x = dense(cur, curC, Lp); io.y = dense(h, curC, Lp); io.Tin = io.Tout = Li; io.B = B;
            io.flags = EPI_WAVEGRAD; io.act = ACT_LRELU; io.act_param = WG_SLOPE; io.act_add = noise_level;
            io.res = {pe[i], 0, Lpe[i]};                          // PositionalEncoding: + pe[:, :T] / 5000
            if ((rc = launch_conv(film[i].in, io, st))) return rc;
            io = ConvIO();
            io.x = dense(h, curC, Lp); io.y = dense(o.F[i], 2 * oc, Lp); io.Tin = io.Tout = Li; io.B = B;
            if ((rc = launch_conv(film[i].out, io, st))) return rc;
        }
        if (i + 1 == n) break;
        const DBlock& d = db[i];   // DBlock i (layers/wavegrad.py:141-148)
        const int Ld = L[i + 1], Ldp = round4(Ld), dc = c.dblock_out_channels[i];
        float* R = wg_pick(o, cur);
        float* A = wg_pick(o, cur, R);
        float* Bb = wg_pick(o, cur, R, A);
        float* D = wg_pick(o, cur, R, A, Bb);
        ConvIO io;
        io.x = dense(cur, curC, Lp); io.y = dense(R, dc, Ldp); io.Tin = io.Tout = Ld; io.B = B;
        io.near_src = Li;                                                       // x[..., ::f]
        if ((rc = launch_conv(d.res, io, st))) return rc;
        io.y = dense(A, dc, Ldp); io.in_slope = WG_SLOPE;
        if ((rc = launch_conv(d.m0, io, st))) return rc;
        io = ConvIO();
        io.x = dense(A, dc, Ldp); io.y = dense(Bb, dc, Ldp); io.Tin = io.Tout = Ld; io.B = B;
        io.in_slope = WG_SLOPE;
        if ((rc = launch_conv(d.m1, io, st))) return rc;
        io.x = dense(Bb, dc, Ldp); io.y = dense(D, dc, Ldp); io.res = dense(R, dc, Ldp);   // o + res
        if ((rc = launch_conv(d.m2, io, st))) return rc;
        cur = D;
        curC = dc;
    }
    // ---- up path (wavegrad.py:115-118)
    const float* xu = o.xc;
    int xC = c.x_conv_channels, xL = T;
    for (int u = 0; u < n; ++u) {
        const UBlock& b = ub[u];   // layers/wavegrad.py:90-104
        const int k = n - 1 - u, Lu = L[k], Lup = round4(Lu), hc = c.ublock_out_channels[u];
        float* R = wg_pick(o, xu);
        float* O = wg_pick(o, xu, R);
        float* H = wg_pick(o, xu, R, O);
        const InView film_k = dense(o.F[k], 2 * hc, Lup);                     // [shift | scale] of FiLM k
        ConvIO io;
        io.x = dense(xu, xC, round4(xL)); io.y = dense(R, hc, Lup); io.Tin = io.Tout = Lu; io.B = B;
        io.near_src = xL;                                                       // x_inter
        if ((rc = launch_conv(b.res, io, st))) return rc;
        io.y = dense(O, hc, Lup); io.in_slope = WG_SLOPE;
        io.flags = EPI_WAVEGRAD; io.film = film_k; io.film_half = hc;
        if ((rc = launch_conv(b.m0, io, st))) return rc;
        ConvIO f;
        f.x = dense(O, hc, Lup); f.y = dense(H, hc, Lup); f.Tin = f.Tout = Lu; f.B = B;
        f.in_slope = WG_SLOPE;
        f.flags = EPI_WAVEGRAD; f.film = film_k; f.film_half = hc;
        f.res = dense(R, hc, Lup);                                              // res2 = res + main1(...)
        f.y2 = dense(R, hc, Lup);
        if ((rc = launch_conv(b.m1, f, st))) return rc;
        f.x = dense(H, hc, Lup); f.y = dense(O, hc, Lup); f.res = InView(); f.y2 = OutView();
        if ((rc = launch_conv(b.o0, f, st))) return rc;
        ConvIO p;
        p.x = dense(O, hc, Lup); p.y = dense(H, hc, Lup); p.Tin = p.Tout = Lu; p.B = B;
        p.in_slope = WG_SLOPE;
        p.res = dense(R, hc, Lup);                                              // out_block[1](...) + res2
        if ((rc = launch_conv(b.o1, p, st))) return rc;
        xu = H; xC = hc; xL = Lu;
    }
    // ---- out_conv (wavegrad.py:119), alone or fused into the update (:139-145)
    const int L0 = L[0];
    const size_t smem = (size_t)xC * 3 * sizeof(float);
    B200_REQUIRE(smem <= 48 * 1024, "wavegrad: out_conv with %d input channels", xC);
    const dim3 grid((unsigned)((L0 + 1023) / 1024), (unsigned)B);
    wavegrad_out_kernel<<<grid, 256, smem, st>>>(xu, (long long)xC * round4(L0), round4(L0), xC, L0, out_w, out_b, out, z, c1,
                                                 c2, sigma, update);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

int Wavegrad::forward(const float* y, const float* x, const float* noise_scale, const float* const* pe, int pe_frames, int B,
                      int T, float* eps, void* ws, size_t ws_bytes, cudaStream_t st) const {
    if (int rc = condition(x, B, T, ws, ws_bytes, st)) return rc;
    return network(y, noise_scale, pe, pe_frames, B, T, eps, 1.f, 0.f, 0.f, nullptr, 0, ws, ws_bytes, st);
}

int Wavegrad::step(float* y, const float* noise_level, const float* const* pe, int pe_frames, float c1, float c2, float sigma,
                   const float* z, int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) const {
    return network(y, noise_level, pe, pe_frames, B, T, y, c1, c2, sigma, z, 1, ws, ws_bytes, st);
}

}  // namespace b200tts
