// WaveNet stack + residual-coupling flow (reverse) + posterior encoder on top of the fused conv1d kernel.
// Reference: TTS/tts/layers/generic/wavenet.py:94-115 (WN.forward, gate :6-13),
//            TTS/tts/layers/vits/networks.py:138-166 (ResidualCouplingBlock.forward, mean_only),
//            :214-232 (ResidualCouplingBlocks.forward, reverse branch with channel flips).
// The torch.flip between blocks is folded into the packing of `pre` (input-channel order) and
// `post` (output-row order): the latent stays in place in HBM and is never permuted.
#include "engines.cuh"

namespace b200tts {

// wl: [cond.w, cond.b] (if cond_channels) then per layer: in.w, in.b, rs.w, rs.b
int WaveNet::init(int hidden, int kernel_size, int dilation_rate, int num_layers, int cond_channels, WeightList& wl) {
    H = hidden; K = kernel_size; L = num_layers; cond_ch = cond_channels;
    int rc;
    if (cond_ch > 0) {
        // rows of cond_layer are sliced per layer (wavenet.py:104-105) and must follow the gate interleave
        std::vector<int> perm(2 * H * L);
        for (int l = 0; l < L; ++l)
            for (int r = 0; r < 2 * H; ++r) perm[l * 2 * H + r] = l * 2 * H + (r < H ? 2 * r : 2 * (r - H) + 1);
        const float *cw = wl.take(), *cb = wl.take();
        if ((rc = pack_conv(cond, cw, cb, 2 * H * L, cond_ch, 1, 1, 0, 0, nullptr, perm.data()))) return rc;
    }
    in_layers.resize(L);
    res_skip.resize(L);
    int d = 1;
    for (int l = 0; l < L; ++l) {
        in_layers[l].tc_prec = res_skip[l].tc_prec = B200TTS_PRECISION_FP32;   // ~85% of the flow FLOPs (k5, 192 -> 384)
        const float *iw = wl.take(), *ib = wl.take();
        if ((rc = pack_conv(in_layers[l], iw, ib, 2 * H, H, K, d, (K * d - d) / 2, /*gate_half=*/H))) return rc;
        const int rows = (l < L - 1) ? 2 * H : H;
        const float *rw = wl.take(), *rb = wl.take();
        if ((rc = pack_conv(res_skip[l], rw, rb, rows, H, 1, 1, 0))) return rc;
        d *= dilation_rate;
    }
    return 0;
}

// h [B,H,T] (masked, updated in place), out [B,H,T] <- WN(h) * mask
int WaveNet::forward(float* h, float* out, const float* mask, const float* g, int B, int T, float* acts,
                     float* condv, cudaStream_t st, const int* lens) const {
    int rc;
    const bool has_g = cond_ch > 0 && g != nullptr;
    if (has_g && (rc = launch_conv_vec(cond, g, condv, cond.RowsPad, B, false, st))) return rc;
    for (int l = 0; l < L; ++l) {
        {   // acts = tanh(a[:H]) * sigmoid(a[H:]),  a = in_layer(h) + g_l
            ConvIO io;
            io.x = dense(h, H, T); io.Tin = T;
            io.y = dense(acts, H, T); io.Tout = T; io.B = B;
            io.flags = EPI_GATE;
            io.lens = lens;      // everything in the WaveNet is re-masked: rows end exactly at their length (need = 0)
            if (has_g) io.cond = {condv + (size_t)l * 2 * H, cond.RowsPad};
            if ((rc = launch_conv(in_layers[l], io, st))) return rc;
        }
        ConvIO io;
        io.x = dense(acts, H, T); io.Tin = T; io.Tout = T; io.B = B;
        io.ymask = {mask, T};
        io.lens = lens;
        if (l < L - 1) {  // h = (h + rs[:H]) * mask ; out (+)= rs[H:]
            io.y = dense(h, H, T);
            io.y2 = dense(out, H, T); io.split = H;
            io.flags = EPI_SPLIT | (l > 0 ? EPI_ACCUM2 : 0);
        } else {          // out = (out + rs) * mask
            io.y = dense(out, H, T);
            io.flags = EPI_MASK_POST | (l > 0 ? EPI_ACCUM : 0);
        }
        if ((rc = launch_conv(res_skip[l], io, st))) return rc;
    }
    return 0;
}

// ------------------------------------------------------------------ residual coupling blocks (reverse)
int Flow::init(const b200tts_flow_config& cfg, const float* const* w, int nw, int forward_direction) {
    c = cfg;
    fwd = forward_direction != 0;
    B200_REQUIRE(c.channels % 2 == 0 && c.num_flows >= 1 && c.num_layers >= 1, "flow: unsupported config");
    WeightList wl(w, nw);
    const int half = c.channels / 2;
    std::vector<int> rev(half);
    for (int i = 0; i < half; ++i) rev[i] = half - 1 - i;
    blocks.resize(c.num_flows);
    for (int n = 0; n < c.num_flows; ++n) {
        Block& b = blocks[n];
        // reverse pass applies flows F-1 .. 0, each after one more flip: block n sees (F - n) flips;
        // the forward pass (networks.py:223-227) flips after each block: block n sees n flips
        b.odd = fwd ? (n % 2) == 1 : ((c.num_flows - n) % 2) == 1;
        int rc;
        b.pre.tc_prec = b.post.tc_prec = B200TTS_PRECISION_FP32;
        const float *pw = wl.take(), *pb = wl.take();
        if ((rc = pack_conv(b.pre, pw, pb, c.hidden_channels, half, 1, 1, 0, 0, b.odd ? rev.data() : nullptr, nullptr)))
            return rc;
        if ((rc = b.wn.init(c.hidden_channels, c.kernel_size, c.dilation_rate, c.num_layers, c.cond_channels, wl)))
            return rc;
        const float *qw = wl.take(), *qb = wl.take();
        if ((rc = pack_conv(b.post, qw, qb, half, c.hidden_channels, 1, 1, 0, 0, nullptr, b.odd ? rev.data() : nullptr)))
            return rc;
    }
    return wl.finish("flow");
}

// the scratch of a hidden-width stage around one WaveNet (Flow, PosteriorEnc): its input h, the gated activations, its
// output and the per-utterance cond vector
struct WnWs { float *h, *acts, *out, *condv; };
static WnWs wn_carve(const WaveNet& wn, Arena& ar, int B, int T) {
    WnWs w;
    w.h = ar.f32((size_t)B * wn.H * T);
    w.acts = ar.f32((size_t)B * wn.H * T);
    w.out = ar.f32((size_t)B * wn.H * T);
    w.condv = ar.f32((size_t)B * wn.cond.RowsPad + 64);
    return w;
}

size_t Flow::workspace_bytes(int B, int T) const {
    return arena_size([&](Arena& ar) { wn_carve(blocks[0].wn, ar, B, T); });
}

int Flow::reverse(float* z, const float* mask, const float* g, int B, int T, void* ws, size_t ws_bytes,
                  cudaStream_t st, const int* lens) const {
    B200_REQUIRE(z && mask && ws, "flow_reverse: null pointer");
    // (also runs the forward direction when the handle was packed for it: same kernels, opposite block order,
    //  x1 = m + x1*mask instead of x1 = (x1 - m)*mask)
    B200_REQUIRE(c.cond_channels == 0 || g != nullptr, "flow_reverse: model has cond_channels=%d but g is null",
                 c.cond_channels);
    const size_t need = workspace_bytes(B, T);
    B200_REQUIRE(ws_bytes >= need, "flow_reverse: workspace of %zu bytes, %zu needed", ws_bytes, need);
    if (B == 0 || T == 0) return 0;
    Arena ar(ws, ws_bytes);
    const WnWs w = wn_carve(blocks[0].wn, ar, B, T);
    float *h = w.h, *acts = w.acts, *out = w.out, *condv = w.condv;
    const int H = c.hidden_channels, half = c.channels / 2;
    const long long zbs = (long long)c.channels * T;
    int rc;
    for (int step = 0; step < c.num_flows; ++step) {
        const int n = fwd ? step : c.num_flows - 1 - step;
        const Block& b = blocks[n];
        // logical x0 / x1 live in the upper / lower physical half when an odd number of flips is pending
        float* x0 = z + (b.odd ? (size_t)half * T : 0);
        float* x1 = z + (b.odd ? 0 : (size_t)half * T);
        {   // h = pre(x0) * mask
            ConvIO io;
            io.x = {x0, zbs, T}; io.Tin = T;
            io.y = dense(h, H, T); io.Tout = T; io.B = B;
            io.ymask = {mask, T}; io.flags = EPI_MASK_POST;
            io.lens = lens;
            if ((rc = launch_conv(b.pre, io, st))) return rc;
        }
        if ((rc = b.wn.forward(h, out, mask, g, B, T, acts, condv, st, lens))) return rc;
        {   // m = post(out) * mask ; x1 = (x1 - m) * mask     (mean_only: log_scale = 0)
            ConvIO io;
            io.x = dense(out, H, T); io.Tin = T;
            io.y = {x1, zbs, T}; io.Tout = T; io.B = B;
            io.ymask = {mask, T};
            io.scale = fwd ? 1.f : -1.f;   // forward: x1 = m + x1*mask ; reverse: x1 = (x1 - m)*mask
            io.flags = EPI_MASK_PRE | EPI_ACCUM | EPI_MASK_POST;
            io.lens = lens;
            if ((rc = launch_conv(b.post, io, st))) return rc;
        }
    }
    return 0;
}

// ------------------------------------------------------------------ posterior encoder (training / voice conversion)
// Reference: TTS/tts/layers/vits/networks.py:275-288: pre 1x1 -> WN (16 layers) -> proj 1x1 -> z = (m + eps*exp(logs))*mask
namespace {
__global__ void sample_posterior_kernel(const float* stats, const float* noise, const float* mask, float* z, int C,
                                        int T) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x, c = blockIdx.y, b = blockIdx.z;
    if (t >= T) return;
    const float m = stats[((size_t)b * 2 * C + c) * T + t];
    const float ls = stats[((size_t)b * 2 * C + C + c) * T + t];
    const size_t o = ((size_t)b * C + c) * T + t;
    z[o] = __fmul_rn(__fadd_rn(m, __fmul_rn(noise[o], expf(ls))), mask[(size_t)b * T + t]);
}
}  // namespace

// weights: pre.w [H,Cin,1], pre.b, enc.* (WaveNet order), proj.w [2*out,H,1], proj.b
int PosteriorEnc::init(const b200tts_posterior_config& cfg, const float* const* w, int nw) {
    c = cfg;
    WeightList wl(w, nw);
    int rc;
    pre.tc_prec = proj.tc_prec = B200TTS_PRECISION_FP32;
    const float *pw = wl.take(), *pb = wl.take();
    if ((rc = pack_conv(pre, pw, pb, c.hidden_channels, c.in_channels, 1, 1, 0))) return rc;
    if ((rc = wn.init(c.hidden_channels, c.kernel_size, c.dilation_rate, c.num_layers, c.cond_channels, wl))) return rc;
    const float *qw = wl.take(), *qb = wl.take();
    if ((rc = pack_conv(proj, qw, qb, 2 * c.out_channels, c.hidden_channels, 1, 1, 0))) return rc;
    return wl.finish("posterior_encoder");
}

size_t PosteriorEnc::workspace_bytes(int B, int T) const {
    return arena_size([&](Arena& ar) { wn_carve(wn, ar, B, T); });
}

int PosteriorEnc::forward(const float* x, const float* mask, const float* g, const float* noise, int B, int T, float* z,
                          float* stats, void* ws, size_t ws_bytes, cudaStream_t st) const {
    B200_REQUIRE(x && mask && noise && z && stats && ws, "posterior_encoder: null pointer");
    B200_REQUIRE(c.cond_channels == 0 || g != nullptr, "posterior_encoder: model has cond_channels=%d but g is null", c.cond_channels);
    const size_t need = workspace_bytes(B, T);
    B200_REQUIRE(ws_bytes >= need, "posterior_encoder: workspace of %zu bytes, %zu needed", ws_bytes, need);
    if (B == 0 || T == 0) return 0;
    Arena ar(ws, ws_bytes);
    const WnWs w = wn_carve(wn, ar, B, T);
    float *h = w.h, *acts = w.acts, *out = w.out, *condv = w.condv;
    const int H = c.hidden_channels;
    int rc;
    {
        ConvIO io;
        io.x = dense(x, c.in_channels, T); io.Tin = T;
        io.y = dense(h, H, T); io.Tout = T; io.B = B;
        io.ymask = {mask, T}; io.flags = EPI_MASK_POST;
        if ((rc = launch_conv(pre, io, st))) return rc;
    }
    if ((rc = wn.forward(h, out, mask, g, B, T, acts, condv, st, nullptr))) return rc;
    {
        ConvIO io;
        io.x = dense(out, H, T); io.Tin = T;
        io.y = dense(stats, 2 * c.out_channels, T); io.Tout = T; io.B = B;
        io.ymask = {mask, T}; io.flags = EPI_MASK_POST;
        if ((rc = launch_conv(proj, io, st))) return rc;
    }
    dim3 grid((T + 127) / 128, c.out_channels, B);
    sample_posterior_kernel<<<grid, 128, 0, st>>>(stats, noise, mask, z, c.out_channels, T);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace b200tts
