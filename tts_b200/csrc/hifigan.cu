// HiFiGAN generator engine: launch schedule over the fused conv1d kernel.
// Reference semantics: TTS/vocoder/models/hifigan_generator.py:236-265 (HifiganGenerator.forward),
// :84-99 (ResBlock1.forward), :150-155 (ResBlock2.forward), ctor :163-234.
#include "engines.cuh"

namespace b200tts {

// weights: host pointers, canonical order (see include/tts_b200.h).  precision (B200TTS_PRECISION_*): the tensor-core
// operand type of conv_pre, the upsamplers and every resblock conv -- the layers that run on the wgmma kernels (~97% of
// the FLOPs); cond and conv_post stay fp32, and so does every margin, workspace size and launch window.  FP32 runs
// them as the split-fp16 product (F16X3: 3 fp16 MMAs where 3xTF32 needs 6 tf32 ones, same operand accuracy);
// TF32X3 keeps 3xTF32 for models whose activations leave fp16's range.
int Hifigan::init(const b200tts_hifigan_config& cfg, const float* const* w, int nw, int precision) {
    c = cfg;
    B200_REQUIRE(precision == B200TTS_PRECISION_FP32 || precision == B200TTS_PRECISION_BF16 ||
                     precision == B200TTS_PRECISION_FP16 || precision == B200TTS_PRECISION_TF32X3 ||
                     precision == B200TTS_PRECISION_F16X3,
                 "hifigan: unknown precision %d", precision);
    prec = precision;
    const int lp = precision == B200TTS_PRECISION_FP32     ? B200TTS_PRECISION_F16X3
                   : precision == B200TTS_PRECISION_TF32X3 ? B200TTS_PRECISION_FP32
                                                           : precision;   // ConvLayer::tc_prec of the layers above
    B200_REQUIRE(c.num_upsamples >= 1 && c.num_upsamples <= 8 && c.num_kernels >= 1 && c.num_kernels <= 8 &&
                     c.num_dilations >= 1 && c.num_dilations <= 8,
                 "hifigan: unsupported config");
    const int type1 = (c.resblock_type == 1);
    WeightList wl(w, nw);
    conv_pre.tc_prec = lp;
    const float *pw = wl.take(), *pb = wl.take();
    int rc = pack_conv(conv_pre, pw, pb, c.upsample_initial_channel, c.in_channels, 7, 1, 3);
    if (rc) return rc;
    if (c.cond_channels > 0) {
        const float *cw = wl.take(), *cb = wl.take();
        rc = pack_conv(cond, cw, cb, c.upsample_initial_channel, c.cond_channels, 1, 1, 0);
        if (rc) return rc;
    }
    ups.resize(c.num_upsamples);
    rb_c1.resize(c.num_upsamples * c.num_kernels);
    rb_c2.resize(c.num_upsamples * c.num_kernels);
    int ch = c.upsample_initial_channel;
    for (int s = 0; s < c.num_upsamples; ++s) {
        const int u = c.upsample_factors[s], k = c.upsample_kernel_sizes[s];
        ups[s].tc_prec = lp;
        const float *uw = wl.take(), *ub = wl.take();
        rc = pack_conv_transpose(ups[s], uw, ub, ch, ch / 2, k, u, (k - u) / 2);
        if (rc) return rc;
        ch /= 2;
        for (int j = 0; j < c.num_kernels; ++j) {
            const int rk = c.resblock_kernel_sizes[j];
            auto& v1 = rb_c1[s * c.num_kernels + j];
            auto& v2 = rb_c2[s * c.num_kernels + j];
            v1.resize(c.num_dilations);
            if (type1) v2.resize(c.num_dilations);
            for (int n = 0; n < c.num_dilations; ++n) {
                const int d = c.resblock_dilations[j][n];
                v1[n].tc_prec = lp;
                const float *w1 = wl.take(), *b1 = wl.take();
                rc = pack_conv(v1[n], w1, b1, ch, ch, rk, d, (rk * d - d) / 2);
                if (rc) return rc;
                if (type1) {
                    v2[n].tc_prec = lp;
                    const float *w2 = wl.take(), *b2 = wl.take();
                    rc = pack_conv(v2[n], w2, b2, ch, ch, rk, 1, (rk - 1) / 2);
                    if (rc) return rc;
                }
            }
        }
    }
    const float *qw = wl.take(), *qb = wl.take();
    rc = pack_conv(conv_post, qw, qb, c.out_channels, ch, 7, 1, 3);
    if (rc == 0) rc = wl.finish("hifigan");
    if (rc == 0) plan_margins();
    return rc;
}

// Ragged batches: how far past a row's last valid sample must each tensor be exact so that the waveform below the
// row's end is bit-identical to the dense computation?  Walk the schedule backwards adding each layer's one-sided reach.
void Hifigan::plan_margins() {
    const int S = c.num_upsamples, nk = c.num_kernels, nd = c.num_dilations;
    const bool type1 = c.resblock_type == 1;
    need_OUT.assign(S, 0); need_U.assign(S, 0); need_q_ups.assign(S, 0); rate.assign(S, 1);
    need_T1.assign(S * nk, std::vector<int>(nd, 0));
    need_X.assign(S * nk, std::vector<int>(nd, 0));
    int r = 1;
    for (int s = 0; s < S; ++s) { r *= c.upsample_factors[s]; rate[s] = r; }
    int need_next = std::max(conv_post.pad, conv_post.K - 1 - conv_post.pad);     // what conv_post reads past a sample
    for (int s = S - 1; s >= 0; --s) {
        need_OUT[s] = need_next;
        int worst = 0;
        for (int j = 0; j < nk; ++j) {
            int cur = need_OUT[s];
            for (int n = nd - 1; n >= 0; --n) {
                const ConvLayer& c1 = rb_c1[s * nk + j][n];
                const int r1 = std::max(c1.pad, (c1.K - 1) * c1.dil - c1.pad);
                need_X[s * nk + j][n] = cur;                       // output of this dilation step (R, or OUT for the last)
                if (type1) {
                    const ConvLayer& c2 = rb_c2[s * nk + j][n];
                    const int r2 = std::max(c2.pad, (c2.K - 1) * c2.dil - c2.pad);
                    need_T1[s * nk + j][n] = cur + r2;
                    cur += r2 + r1;
                } else {
                    cur += r1;
                }
            }
            worst = std::max(worst, cur);
        }
        need_U[s] = worst;
        const ConvLayer& u = ups[s];                               // polyphase: GEMM columns are input steps
        need_q_ups[s] = (need_U[s] + u.ups - 1) / u.ups;
        need_next = need_q_ups[s] + std::max(u.pad, (u.K - 1) * u.dil - u.pad);
    }
    need_P = need_next;
}

void Hifigan::stage_dims(int T, std::vector<int>& C, std::vector<int>& L) const {
    C.resize(c.num_upsamples);
    L.resize(c.num_upsamples);
    int ch = c.upsample_initial_channel, len = T;
    for (int s = 0; s < c.num_upsamples; ++s) {
        ch /= 2;
        len = conv_transpose_out_len(ups[s], len);
        C[s] = ch;
        L[s] = len;
    }
}

struct HifiganWs { float *P, *Xp, *U, *T1, *R, *OUT, *condv; };

// P: conv_pre's output, Xp: the re-pitched input, U / T1 / R / OUT: the stage tensors (the largest stage each)
static HifiganWs hifigan_carve(const Hifigan& m, Arena& ar, int B, int T) {
    std::vector<int> C, L;
    m.stage_dims(T, C, L);
    size_t mx = 0;
    for (size_t s = 0; s < C.size(); ++s) mx = std::max(mx, (size_t)C[s] * (size_t)L[s]);
    const size_t Tp = (size_t)(T + 3) / 4 * 4;    // 16-byte aligned row pitch for the stage-0 tensors
    HifiganWs w;
    w.P = ar.f32((size_t)B * m.c.upsample_initial_channel * Tp);
    w.Xp = ar.f32((size_t)B * m.c.in_channels * Tp);
    w.U = ar.f32((size_t)B * mx);
    w.T1 = ar.f32((size_t)B * mx);
    w.R = ar.f32((size_t)B * mx);
    w.OUT = ar.f32((size_t)B * mx);
    w.condv = ar.f32((size_t)B * m.cond.RowsPad + 64);
    return w;
}

size_t Hifigan::workspace_bytes(int B, int T) const {
    return arena_size([&](Arena& ar) { hifigan_carve(*this, ar, B, T); });
}

int Hifigan::out_len(int T) const {
    std::vector<int> C, L;
    stage_dims(T, C, L);
    return L.back();
}

// samples [lo, hi) of every row of wav that lie past the row's end (lens[b] * rate)
__global__ void zero_past_end_kernel(float* __restrict__ wav, int C, int Tout, const int* __restrict__ lens, int rate,
                                     int lo, int hi) {
    const int b = blockIdx.y;
    const long long e = (long long)lens[b] * rate;
    const int from = (int)max((long long)lo, min(e, (long long)hi));
    for (int c = 0; c < C; ++c) {
        float* row = wav + ((long long)b * C + c) * Tout;
        for (int t = from + (int)(blockIdx.x * blockDim.x + threadIdx.x); t < hi; t += (int)(gridDim.x * blockDim.x)) row[t] = 0.f;
    }
}

int Hifigan::forward(const float* x, const float* g, int B, int T, float* wav, void* ws, size_t ws_bytes,
                     cudaStream_t st, unsigned* peak_bits, const int* lens, int frame_begin, int frame_end) const {
    B200_REQUIRE(x && wav && ws, "hifigan_forward: null pointer");
    B200_REQUIRE((c.cond_channels > 0) == (g != nullptr) || c.cond_channels == 0,
                 "hifigan_forward: model has cond_channels=%d but g is null", c.cond_channels);
    const size_t need = workspace_bytes(B, T);
    B200_REQUIRE(ws_bytes >= need, "hifigan_forward: workspace of %zu bytes, %zu needed", ws_bytes, need);
    if (frame_end < 0) frame_end = T;
    const bool windowed = frame_begin != 0 || frame_end != T;
    B200_REQUIRE(!windowed || (0 <= frame_begin && frame_begin < frame_end && frame_end <= T),
                 "hifigan_forward: frame window [%d, %d) is not inside [0, %d)", frame_begin, frame_end, T);
    if (B == 0 || T == 0) return 0;
    std::vector<int> C, L;
    stage_dims(T, C, L);
    // a window is sample-aligned only when every stage multiplies the length exactly (k - u even for each upsampler)
    B200_REQUIRE(!windowed || L.back() == T * (rate.empty() ? 1 : rate.back()),
                 "hifigan_forward: frame windows need out_len(T) == T * prod(upsample_factors) (got %d for T = %d)",
                 L.back(), T);
    // each launch's column window: its margin `need` either side of the frames' span at its own rate, and its input's
    // data start (the producing launch's window start)
    const long long fb = frame_begin, fe = frame_end;
    auto window = [&](ConvIO& io) {
        if (!windowed) return;             // the whole tensor (also for lengths that are not T * hop)
        io.q_lo = (int)std::max(0LL, fb * io.rate_out - io.need_out);
        io.q_hi = (int)std::min(0x7fffffffLL, fe * io.rate_out + io.need_out);
        io.in_lo = (int)std::max(0LL, fb * io.rate_in - io.need_in);
        io.in_hi = (int)std::min(0x7fffffffLL, fe * io.rate_in + io.need_in);
    };
    Arena ar(ws, ws_bytes);
    const HifiganWs w = hifigan_carve(*this, ar, B, T);
    float *P = w.P, *Xp = w.Xp, *U = w.U, *T1 = w.T1, *R = w.R, *OUT = w.OUT, *condv = w.condv;
    const int C0 = c.upsample_initial_channel;
    // The tensor-core kernels stage activation rows with 16-byte cp.async: rows must start 16-byte aligned.  T (decoder frames)
    // is arbitrary, so the stage-0 tensors use a row pitch rounded up to 4 floats and an unaligned input is re-pitched
    // once (B x Cin x T floats, tiny) -- otherwise conv_pre / ups[0] would silently take the FP32-FMA kernel for 3 of 4 T.
    const int Tp = (T + 3) / 4 * 4;
    const float* xin0 = x;
    int x_pitch = T;
    if (Tp != T || (reinterpret_cast<uintptr_t>(x) & 15) != 0) {
        B200_CUDA_OK(cudaMemcpy2DAsync(Xp, (size_t)Tp * sizeof(float), x, (size_t)T * sizeof(float), (size_t)T * sizeof(float),
                                       (size_t)B * c.in_channels, cudaMemcpyDeviceToDevice, st));
        xin0 = Xp;
        x_pitch = Tp;
    }
    int rc;
    const bool has_cond = c.cond_channels > 0 && g != nullptr;
    // cond_layer(g): [B, cond, 1] -> [B, C0]
    if (has_cond && (rc = launch_conv_vec(cond, g, condv, cond.RowsPad, B, false, st))) return rc;
    {  // conv_pre (+ cond broadcast over T)
        ConvIO io;
        io.x = dense(xin0, c.in_channels, x_pitch); io.Tin = T;
        io.y = dense(P, C0, Tp); io.Tout = T; io.B = B;
        if (has_cond) io.cond = {condv, cond.RowsPad};
        io.lens = lens; io.rate_out = 1; io.need_out = need_P; io.rate_in = 1; io.need_in = T;   // z is defined everywhere
        window(io);
        if ((rc = launch_conv(conv_pre, io, st))) return rc;
    }
    const float* cur = P;
    int curC = C0, curL = T, curPitch = Tp;
    const bool type1 = c.resblock_type == 1;
    for (int s = 0; s < c.num_upsamples; ++s) {
        const int Cs = C[s], Ls = L[s];
        {  // o = ups(leaky_relu(o, 0.1))
            ConvIO io;
            io.x = dense(cur, curC, curPitch); io.Tin = curL; io.in_slope = 0.1f;
            io.y = dense(U, Cs, Ls); io.Tout = Ls; io.B = B;
            io.lens = lens; io.rate_in = (s == 0) ? 1 : rate[s - 1]; io.need_in = (s == 0) ? need_P : need_OUT[s - 1];
            io.rate_out = io.rate_in; io.need_out = need_q_ups[s];      // tiles run over GEMM columns = input steps
            window(io);
            if ((rc = launch_conv(ups[s], io, st))) return rc;
        }
        for (int j = 0; j < c.num_kernels; ++j) {
            const auto& c1 = rb_c1[s * c.num_kernels + j];
            const auto& c2 = rb_c2[s * c.num_kernels + j];
            const float* xin = U;
            int need_xin = need_U[s];
            float* pp[2] = {R, T1};  // ping-pong for ResBlock2
            for (int n = 0; n < c.num_dilations; ++n) {
                const bool last = (n == c.num_dilations - 1);
                const float* convin = xin;
                const ConvLayer* lastconv = &c1[n];
                if (type1) {  // T1 = c1(lrelu(xin))
                    ConvIO io;
                    io.x = dense(xin, Cs, Ls); io.Tin = Ls; io.in_slope = 0.1f;
                    io.y = dense(T1, Cs, Ls); io.Tout = Ls; io.B = B;
                    io.lens = lens; io.rate_in = io.rate_out = rate[s];
                    io.need_in = need_xin; io.need_out = need_T1[s * c.num_kernels + j][n];
                    window(io);
                    if ((rc = launch_conv(c1[n], io, st))) return rc;
                    convin = T1;
                    lastconv = &c2[n];
                }
                ConvIO io;  // xnew = conv(lrelu(convin)) + xin ; MRF: OUT (+)= xnew, mean on the last resblock
                io.x = dense(convin, Cs, Ls); io.Tin = Ls; io.in_slope = 0.1f;
                io.res = dense(xin, Cs, Ls);
                io.B = B; io.Tout = Ls;
                float* dst;
                if (last) {
                    dst = OUT;
                    if (j > 0) io.flags |= EPI_ACCUM;
                    if (j == c.num_kernels - 1) io.post_div = (float)c.num_kernels;
                } else {
                    dst = type1 ? R : pp[n & 1];
                }
                io.y = dense(dst, Cs, Ls);
                io.lens = lens; io.rate_in = io.rate_out = rate[s];
                io.need_in = type1 ? need_T1[s * c.num_kernels + j][n] : need_xin;
                io.need_out = need_X[s * c.num_kernels + j][n];
                window(io);
                if ((rc = launch_conv(*lastconv, io, st))) return rc;
                xin = dst;
                need_xin = io.need_out;
            }
        }
        cur = OUT;
        curC = Cs;
        curL = Ls;
        curPitch = Ls;
        // the next stage's ups reads OUT and writes U; OUT is only rewritten by later launches
        // on the same stream, after that read has completed.
    }
    {  // tanh(conv_post(leaky_relu(o)))  -- default slope 0.01 (hifigan_generator.py:262)
        ConvIO io;
        io.x = dense(cur, curC, curPitch); io.Tin = curL; io.in_slope = 0.01f;
        io.y = dense(wav, c.out_channels, curL); io.Tout = curL; io.B = B;
        io.act = ACT_TANH;
        io.peak_bits = peak_bits;
        io.lens = lens; io.rate_in = io.rate_out = rate.empty() ? 1 : rate.back(); io.need_in = need_OUT.empty() ? 0 : need_OUT.back();
        io.need_out = 0;
        window(io);       // exactly the window's samples: [frame_begin * hop, frame_end * hop)
        if (lens) {       // the window's samples past each row's end are zero (other windows' samples are left alone)
            B200_REQUIRE(B <= 65535, "hifigan_forward: batch too large");
            const int lo = io.q_lo, hi = std::min(io.q_hi, curL);
            const dim3 grid((unsigned)std::max(1, std::min((hi - lo + 255) / 256, 64)), (unsigned)B);
            zero_past_end_kernel<<<grid, 256, 0, st>>>(wav, c.out_channels, curL, lens, io.rate_out, lo, hi);
            count_launch();
            B200_CUDA_OK(cudaGetLastError());
        }
        if ((rc = launch_conv(conv_post, io, st))) return rc;
    }
    return 0;
}

}  // namespace b200tts
