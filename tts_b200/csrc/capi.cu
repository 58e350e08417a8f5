// extern "C" surface of libtts_b200.so -- see include/tts_b200.h for the contract.
#include <new>
#include <type_traits>

#include "engines.cuh"

using namespace b200tts;

struct b200tts_hifigan { Hifigan impl; };
struct b200tts_flow { Flow impl; };
struct b200tts_text_encoder { TextEncoder impl; };
struct b200tts_sdp { SDP impl; };
struct b200tts_stft { Stft impl; };
struct b200tts_posterior { PosteriorEnc impl; };
struct b200tts_duration_predictor { DurPred impl; };
struct b200tts_speaker_encoder { SpeakerEncoder impl; };
struct b200tts_glow_tts { GlowTTS impl; };
struct b200tts_melgan { Melgan impl; };
struct b200tts_forward_tts { ForwardTTS impl; };
struct b200tts_wavegrad { Wavegrad impl; };
struct b200tts_overflow { Overflow impl; };
struct b200tts_tacotron2 { Tacotron2 impl; };
struct b200tts_tacotron { Tacotron impl; };
struct b200tts_pwgan { Pwgan impl; };
struct b200tts_univnet { Univnet impl; };
struct b200tts_griffin_lim { GriffinLim impl; };

// A handle owns its device buffers through DevBuf members: copying one would free them twice, so it must not compile.
static_assert(!std::is_copy_constructible_v<ConvLayer>);
static_assert(!std::is_copy_constructible_v<Hifigan>);
static_assert(!std::is_copy_constructible_v<Flow>);
static_assert(!std::is_copy_constructible_v<TextEncoder>);
static_assert(!std::is_copy_constructible_v<SDP>);
static_assert(!std::is_copy_constructible_v<Stft>);
static_assert(!std::is_copy_constructible_v<PosteriorEnc>);
static_assert(!std::is_copy_constructible_v<DurPred>);
static_assert(!std::is_copy_constructible_v<SpeakerEncoder>);
static_assert(!std::is_copy_constructible_v<GlowTTS>);
static_assert(!std::is_copy_constructible_v<Melgan>);
static_assert(!std::is_copy_constructible_v<ForwardTTS>);
static_assert(!std::is_copy_constructible_v<Wavegrad>);
static_assert(!std::is_copy_constructible_v<Overflow>);
static_assert(!std::is_copy_constructible_v<Tacotron2>);
static_assert(!std::is_copy_constructible_v<Tacotron>);
static_assert(!std::is_copy_constructible_v<Pwgan>);
static_assert(!std::is_copy_constructible_v<Univnet>);
static_assert(!std::is_copy_constructible_v<GriffinLim>);

extern "C" {

const char* b200tts_last_error(void) { return last_error(); }
unsigned long long b200tts_launch_count(void) { return g_launch_count; }
int b200tts_version(void) { return 100; }
int b200tts_debug_tc_error(void) { return conv_tc_error_flag(); }
long long b200tts_debug_device_buffers(void) { return g_device_buffers.load(); }
void b200tts_debug_dispatch_begin(void) { dispatch_begin(); }
int b200tts_debug_dispatch_end(int32_t* ids, int cap) { return dispatch_end(ids, cap); }

struct b200tts_conv1d {
    ConvLayer L; b200tts_conv1d_config c; int reflect = 0;   // reflect: B200TTS_PAD_REFLECT
};

static bool valid_precision(int p) {
    return p == B200TTS_PRECISION_FP32 || p == B200TTS_PRECISION_BF16 || p == B200TTS_PRECISION_FP16 ||
           p == B200TTS_PRECISION_TF32X3 || p == B200TTS_PRECISION_F16X3;
}

static int conv1d_create_impl(const b200tts_conv1d_config* cfg, const float* weight, const float* bias, int allow_tensor_cores,
                              int precision, b200tts_conv1d** out, int padding_mode = B200TTS_PAD_ZEROS, int gate_half = 0,
                              const int* in_perm = nullptr, const int* out_perm = nullptr) {
    if (!cfg || !weight || !out) { set_error("conv1d_create: null argument"); return 1; }
    *out = nullptr;
    if (cfg->transposed && (gate_half || in_perm || out_perm)) {
        set_error("conv1d_create: gate / channel permutations need a non-transposed conv");
        return 1;
    }
    if (!valid_precision(precision)) { set_error("conv1d_create: unknown precision %d", precision); return 1; }
    if (padding_mode != B200TTS_PAD_ZEROS && padding_mode != B200TTS_PAD_REFLECT) {
        set_error("conv1d_create: unknown padding mode %d", padding_mode);
        return 1;
    }
    if (padding_mode == B200TTS_PAD_REFLECT && (cfg->transposed || 2 * cfg->padding != cfg->dilation * (cfg->kernel_size - 1))) {
        set_error("conv1d_create: reflection padding needs a non-transposed conv with padding = dilation * (kernel_size - 1) / 2");
        return 1;
    }
    b200tts_conv1d* h = new (std::nothrow) b200tts_conv1d();
    if (!h) { set_error("conv1d_create: out of host memory"); return 1; }
    h->c = *cfg;
    h->reflect = padding_mode == B200TTS_PAD_REFLECT;
    // FP32 and TF32X3 are both the 3xTF32 images (ConvLayer::tc_prec never holds TF32X3)
    const int lp = precision == B200TTS_PRECISION_TF32X3 ? B200TTS_PRECISION_FP32 : precision;
    h->L.tc_prec = allow_tensor_cores ? lp : TC_NONE;
    int rc = cfg->transposed
                 ? pack_conv_transpose(h->L, weight, bias, cfg->in_channels, cfg->out_channels, cfg->kernel_size,
                                       cfg->stride, cfg->padding)
                 : pack_conv(h->L, weight, bias, cfg->out_channels, cfg->in_channels, cfg->kernel_size, cfg->dilation,
                             cfg->padding, gate_half, in_perm, out_perm);
    if (rc) { delete h; return rc; }
    *out = h;
    return 0;
}
int b200tts_conv1d_create(const b200tts_conv1d_config* cfg, const float* weight, const float* bias, int allow_tensor_cores,
                          b200tts_conv1d** out) {
    return conv1d_create_impl(cfg, weight, bias, allow_tensor_cores, B200TTS_PRECISION_FP32, out);
}
int b200tts_conv1d_create_ex(const b200tts_conv1d_config* cfg, const float* weight, const float* bias, int precision,
                             b200tts_conv1d** out) {
    return conv1d_create_impl(cfg, weight, bias, 1, precision, out);
}
int b200tts_conv1d_create_padded(const b200tts_conv1d_config* cfg, const float* weight, const float* bias,
                                 int allow_tensor_cores, int precision, int padding_mode, b200tts_conv1d** out) {
    return conv1d_create_impl(cfg, weight, bias, allow_tensor_cores, precision, out, padding_mode);
}
void b200tts_conv1d_destroy(b200tts_conv1d* h) { delete h; }
int b200tts_conv1d_out_len(const b200tts_conv1d* h, int T) {
    if (!h) return 0;
    if (h->c.transposed) return conv_transpose_out_len(h->L, T);
    return T + 2 * h->c.padding - h->c.dilation * (h->c.kernel_size - 1);
}
int b200tts_conv1d_forward(const b200tts_conv1d* h, const float* x, int B, int T, float in_slope, const float* residual,
                           float scale, int accumulate, float post_div, float* y, void* stream) {
    if (!h) { set_error("conv1d_forward: null handle"); return 1; }
    const int Tout = b200tts_conv1d_out_len(h, T);
    ConvIO io;
    io.x = dense(x, h->c.in_channels, T); io.Tin = T; io.in_slope = in_slope;
    io.y = dense(y, h->c.out_channels, Tout); io.Tout = Tout; io.B = B;
    if (residual) io.res = dense(residual, h->c.out_channels, Tout);
    io.scale = scale; io.post_div = post_div;
    if (accumulate) io.flags |= EPI_ACCUM;
    io.reflect = h->reflect;
    return launch_conv(h->L, io, (cudaStream_t)stream);
}
int b200tts_conv1d_forward_strided(const b200tts_conv1d* h, const float* x, long long x_batch_stride, int x_channel_stride,
                                   int B, int T, float in_slope, const float* residual, float scale, int accumulate,
                                   float post_div, int tanh, float* y, uint32_t* peak_bits, void* stream) {
    if (!h) { set_error("conv1d_forward_strided: null handle"); return 1; }
    if (peak_bits && !tanh) { set_error("conv1d_forward_strided: peak_bits needs the tanh epilogue"); return 1; }
    const int Tout = b200tts_conv1d_out_len(h, T);
    ConvIO io;
    io.x = {x, x_batch_stride, x_channel_stride}; io.Tin = T; io.in_slope = in_slope;
    io.y = dense(y, h->c.out_channels, Tout); io.Tout = Tout; io.B = B;
    if (residual) io.res = dense(residual, h->c.out_channels, Tout);
    io.scale = scale; io.post_div = post_div;
    if (accumulate) io.flags |= EPI_ACCUM;
    if (tanh) { io.act = ACT_TANH; io.peak_bits = peak_bits; }
    io.reflect = h->reflect;
    return launch_conv(h->L, io, (cudaStream_t)stream);
}

int b200tts_conv1d_forward_wavegrad(const b200tts_conv1d* h, const float* x, long long x_batch_stride, int x_channel_stride,
                                    int B, int T, int near_src, float in_slope, int lrelu, const float* act_add,
                                    const float* residual, long long res_batch_stride, int res_channel_stride,
                                    const float* film, long long film_batch_stride, int film_channel_stride, int film_half,
                                    float* y, long long y_batch_stride, int y_channel_stride, float* y2, void* stream) {
    if (!h) { set_error("conv1d_forward_wavegrad: null handle"); return 1; }
    if (h->c.transposed || h->reflect) { set_error("conv1d_forward_wavegrad: a zero-padded, non-transposed conv only"); return 1; }
    const int Tout = b200tts_conv1d_out_len(h, T);
    ConvIO io;
    io.x = {x, x_batch_stride, x_channel_stride}; io.Tin = T; io.in_slope = in_slope;
    io.y = {y, y_batch_stride, y_channel_stride}; io.Tout = Tout; io.B = B;
    if (y2) io.y2 = {y2, y_batch_stride, y_channel_stride};
    if (residual) io.res = {residual, res_batch_stride, res_channel_stride};
    io.flags = EPI_WAVEGRAD;
    io.near_src = near_src;
    if (lrelu) { io.act = ACT_LRELU; io.act_param = 0.2f; }
    io.act_add = act_add;
    io.film = {film, film_batch_stride, film_channel_stride}; io.film_half = film_half;
    return launch_conv(h->L, io, (cudaStream_t)stream);
}

int b200tts_debug_conv1d_create(const b200tts_conv1d_config* cfg, const float* weight, const float* bias,
                                int allow_tensor_cores, int precision, int padding_mode, int gate_half,
                                const int32_t* in_perm, const int32_t* out_perm, b200tts_conv1d** out) {
    if (!cfg || !out) { set_error("debug_conv1d_create: null argument"); return 1; }
    *out = nullptr;
    auto is_perm = [](const int32_t* p, int n) {   // pack_conv writes through the permutation: it must be one
        std::vector<char> seen(n > 0 ? n : 0, 0);
        for (int i = 0; i < n; ++i) {
            if (p[i] < 0 || p[i] >= n || seen[p[i]]) return false;
            seen[p[i]] = 1;
        }
        return true;
    };
    if ((in_perm && !is_perm(in_perm, cfg->in_channels)) || (out_perm && !is_perm(out_perm, cfg->out_channels))) {
        set_error("debug_conv1d_create: in_perm / out_perm must be permutations of the channels");
        return 1;
    }
    return conv1d_create_impl(cfg, weight, bias, allow_tensor_cores, precision, out, padding_mode, gate_half, in_perm,
                              out_perm);
}
static_assert(sizeof(b200tts_debug_conv_io) == 216, "tts_b200/_lib.py DebugConvIOC mirrors this layout");
static int debug_conv1d_launch(const b200tts_conv1d* h, const b200tts_debug_conv_io* d, const b200tts_debug_conv_bn* bn,
                               void* stream) {
    if (!h || !d) { set_error("debug_conv1d_launch: null argument"); return 1; }
    ConvIO io;
    io.x = {d->x, d->x_batch_stride, d->x_channel_stride}; io.Tin = d->T;
    io.xmask = {d->xmask, d->xmask_batch_stride}; io.in_slope = d->in_slope;
    io.cond = {d->cond, d->cond_batch_stride};
    io.y = {d->y, d->y_batch_stride, d->y_channel_stride}; io.Tout = b200tts_conv1d_out_len(h, d->T);
    io.res = {d->res, d->res_batch_stride, d->res_channel_stride};
    io.ymask = {d->ymask, d->ymask_batch_stride};
    io.y2 = {d->y2, d->y2_batch_stride, d->y2_channel_stride};
    io.split = d->split; io.scale = d->scale; io.post_div = d->post_div;
    io.act = d->act; io.act_param = d->act_param; io.flags = d->flags; io.B = d->B;
    io.lens = d->lens; io.rate_out = d->rate_out; io.need_out = d->need_out; io.rate_in = d->rate_in; io.need_in = d->need_in;
    io.q_lo = d->q_lo; io.q_hi = d->q_hi; io.in_lo = d->in_lo; io.in_hi = d->in_hi;
    if (bn) { io.edge_lo = bn->edge_lo; io.edge_hi = bn->edge_hi; io.aff_s = bn->aff_s; io.aff_h = bn->aff_h; }
    io.reflect = h->reflect;
    if (io.flags & ~(EPI_GATE | EPI_MASK_PRE | EPI_MASK_POST | EPI_ACCUM | EPI_SPLIT | EPI_ACCUM2 | (bn ? EPI_WINDOW : 0)) ||
        !(io.act >= ACT_NONE && io.act <= ACT_LOGCLAMP)) {
        set_error("debug_conv1d_launch: unknown flags 0x%x or act %d", io.flags, io.act);
        return 1;
    }
    return launch_conv(h->L, io, (cudaStream_t)stream);
}
int b200tts_debug_conv1d_launch(const b200tts_conv1d* h, const b200tts_debug_conv_io* d, void* stream) {
    return debug_conv1d_launch(h, d, nullptr, stream);
}
int b200tts_debug_conv1d_launch_bn(const b200tts_conv1d* h, const b200tts_debug_conv_io* d, const b200tts_debug_conv_bn* bn,
                                   void* stream) {
    if (!bn) { set_error("debug_conv1d_launch_bn: null argument"); return 1; }
    return debug_conv1d_launch(h, d, bn, stream);
}

int b200tts_debug_attention(const float* qkv, const float* mask, const float* rel_k, const float* rel_v, float* out,
                            int B, int C, int T, int num_heads, int window, void* stream) {
    if (!qkv || !mask || !out) { set_error("debug_attention: null argument"); return 1; }
    if (B < 0 || T < 0) { set_error("debug_attention: B=%d, T=%d", B, T); return 1; }
    if (int rc = launch_attention(qkv, mask, window < 0 ? nullptr : rel_k, window < 0 ? nullptr : rel_v, out, B, C, T,
                                  num_heads, window, (cudaStream_t)stream))
        return rc;
    if (B > 0 && T > 0) dispatch_note(DISPATCH_ATTN_FMA);
    return 0;
}

int b200tts_debug_add_layernorm(int kind, const float* x, const float* y, int twice, const float* gamma,
                                const float* beta, const float* mask, float* out, int B, int C, int T, float eps,
                                void* stream) {
    if (!x || !gamma || !beta || !out) { set_error("debug_add_layernorm: null argument"); return 1; }
    if (B < 0 || C < 1 || T < 0) { set_error("debug_add_layernorm: B=%d, C=%d, T=%d", B, C, T); return 1; }
    if (kind == 0) {
        if (twice) { set_error("debug_add_layernorm: kind 0 has no `twice` residual"); return 1; }
        return launch_add_layernorm(x, y, gamma, beta, mask, out, B, C, T, eps, (cudaStream_t)stream);
    }
    if (kind == 1) {
        if (!y || !mask) { set_error("debug_add_layernorm: kind 1 needs y and mask"); return 1; }
        if (eps != 1e-5f) { set_error("debug_add_layernorm: kind 1 has eps 1e-5, not %g", (double)eps); return 1; }
        return launch_add_norm(x, y, twice != 0, gamma, beta, mask, out, B, C, T, (cudaStream_t)stream);
    }
    set_error("debug_add_layernorm: unknown kind %d", kind);
    return 1;
}

size_t b200tts_mas_workspace_bytes(int B, int Tx, int Ty) { return mas_workspace_bytes(B, Tx, Ty); }

int b200tts_mas(const float* value, const float* mask, const int32_t* t_x, const int32_t* t_y, int B, int Tx,
                int Ty, void* path, int path_is_f32, void* workspace, size_t workspace_bytes, void* stream) {
    return mas_forward(value, mask, t_x, t_y, B, Tx, Ty, path, path_is_f32, workspace, workspace_bytes,
                       (cudaStream_t)stream);
}

size_t b200tts_mas_from_stats_workspace_bytes(int B, int Tx, int Ty) { return mas_from_stats_workspace_bytes(B, Tx, Ty); }
int b200tts_mas_from_stats(const float* z_p, const float* m_p, const float* logs_p, const int32_t* t_x, const int32_t* t_y,
                           int B, int C, int Tx, int Ty, void* path, int path_is_f32, float* logp_out, void* workspace,
                           size_t workspace_bytes, void* stream) {
    return mas_from_stats(z_p, m_p, logs_p, t_x, t_y, B, C, Tx, Ty, path, path_is_f32, logp_out, workspace, workspace_bytes,
                          (cudaStream_t)stream);
}

int b200tts_hifigan_create_ex(const b200tts_hifigan_config* cfg, const float* const* weights, int num_weights, int precision,
                              b200tts_hifigan** out) {
    if (!cfg || !weights || !out) { set_error("hifigan_create: null argument"); return 1; }
    *out = nullptr;
    b200tts_hifigan* h = new (std::nothrow) b200tts_hifigan();
    if (!h) { set_error("hifigan_create: out of host memory"); return 1; }
    int rc = h->impl.init(*cfg, weights, num_weights, precision);
    if (rc) { delete h; return rc; }
    *out = h;
    return 0;
}
int b200tts_hifigan_create(const b200tts_hifigan_config* cfg, const float* const* weights, int num_weights,
                           b200tts_hifigan** out) {
    return b200tts_hifigan_create_ex(cfg, weights, num_weights, B200TTS_PRECISION_FP32, out);
}
int b200tts_hifigan_precision(const b200tts_hifigan* h) { return h ? h->impl.prec : -1; }
void b200tts_hifigan_destroy(b200tts_hifigan* h) { delete h; }
size_t b200tts_hifigan_workspace_bytes(const b200tts_hifigan* h, int B, int T) {
    return h ? h->impl.workspace_bytes(B, T) : 0;
}
int b200tts_hifigan_out_len(const b200tts_hifigan* h, int T) { return h ? h->impl.out_len(T) : 0; }
int b200tts_hifigan_forward(const b200tts_hifigan* h, const float* x, const float* g, int B, int T, float* wav,
                            void* workspace, size_t workspace_bytes, void* stream) {
    if (!h) { set_error("hifigan_forward: null handle"); return 1; }
    return h->impl.forward(x, g, B, T, wav, workspace, workspace_bytes, (cudaStream_t)stream);
}

int b200tts_hifigan_forward_ex(const b200tts_hifigan* h, const float* x, const float* g, int B, int T, float* wav,
                               const int32_t* frame_lengths, uint32_t* peak_bits, void* workspace, size_t workspace_bytes,
                               void* stream) {
    if (!h) { set_error("hifigan_forward_ex: null handle"); return 1; }
    return h->impl.forward(x, g, B, T, wav, workspace, workspace_bytes, (cudaStream_t)stream, peak_bits, frame_lengths);
}
int b200tts_hifigan_forward_window(const b200tts_hifigan* h, const float* x, const float* g, int B, int T,
                                   int frame_begin, int frame_end, float* wav, const int32_t* frame_lengths,
                                   uint32_t* peak_bits, void* workspace, size_t workspace_bytes, void* stream) {
    if (!h) { set_error("hifigan_forward_window: null handle"); return 1; }
    if (!(0 <= frame_begin && frame_begin < frame_end && frame_end <= T)) {
        set_error("hifigan_forward_window: frame window [%d, %d) is not inside [0, %d)", frame_begin, frame_end, T);
        return 1;
    }
    const int hop = b200tts_hifigan_out_len(h, 1);
    if (h->impl.out_len(T) != T * hop || h->impl.out_len(1) <= 0) {
        set_error("hifigan_forward_window: the upsamplers do not multiply the length exactly (out_len(%d) = %d)", T,
                  h->impl.out_len(T));
        return 1;
    }
    return h->impl.forward(x, g, B, T, wav, workspace, workspace_bytes, (cudaStream_t)stream, peak_bits, frame_lengths,
                           frame_begin, frame_end);
}
int b200tts_hifigan_margin_frames(const b200tts_hifigan* h) {   // frames past a row's end the ragged schedule still computes
    return h ? h->impl.need_P : 0;
}

int b200tts_vocoder_input_len(int T, float scale_factor, int padding) { return vocoder_input_len(T, scale_factor, padding); }
int b200tts_vocoder_input(const float* x, long long x_batch_stride, int x_channel_stride, int x_time_stride, int B, int C,
                          int T, const b200tts_audio_norm* denormalize, const b200tts_audio_norm* normalize,
                          float scale_factor, int padding, float* y, int y_pitch, void* stream) {
    return launch_vocoder_input(x, x_batch_stride, x_channel_stride, x_time_stride, B, C, T, denormalize, normalize,
                                scale_factor, padding, y, y_pitch, (cudaStream_t)stream);
}
int b200tts_absmax(const float* x, long long n, uint32_t* peak_bits, void* stream) {
    return launch_absmax(x, n, peak_bits, (cudaStream_t)stream);
}
int b200tts_to_int16(const float* x, long long n, const uint32_t* peak_bits, int16_t* out, void* stream) {
    return launch_to_int16(x, n, peak_bits, out, (cudaStream_t)stream);
}

int b200tts_flow_create(const b200tts_flow_config* cfg, const float* const* weights, int num_weights,
                        b200tts_flow** out) {
    if (!cfg || !weights || !out) { set_error("flow_create: null argument"); return 1; }
    *out = nullptr;
    b200tts_flow* h = new (std::nothrow) b200tts_flow();
    if (!h) { set_error("flow_create: out of host memory"); return 1; }
    int rc = h->impl.init(*cfg, weights, num_weights);
    if (rc) { delete h; return rc; }
    *out = h;
    return 0;
}
int b200tts_flow_create_forward(const b200tts_flow_config* cfg, const float* const* weights, int num_weights,
                                b200tts_flow** out) {
    if (!cfg || !weights || !out) { set_error("flow_create_forward: null argument"); return 1; }
    *out = nullptr;
    b200tts_flow* h = new (std::nothrow) b200tts_flow();
    if (!h) { set_error("flow_create_forward: out of host memory"); return 1; }
    int rc = h->impl.init(*cfg, weights, num_weights, 1);
    if (rc) { delete h; return rc; }
    *out = h;
    return 0;
}
void b200tts_flow_destroy(b200tts_flow* h) { delete h; }
size_t b200tts_flow_workspace_bytes(const b200tts_flow* h, int B, int T) {
    return h ? h->impl.workspace_bytes(B, T) : 0;
}
int b200tts_flow_reverse(const b200tts_flow* h, float* z, const float* mask, const float* g, int B, int T,
                         void* workspace, size_t workspace_bytes, void* stream) {
    if (!h) { set_error("flow_reverse: null handle"); return 1; }
    return h->impl.reverse(z, mask, g, B, T, workspace, workspace_bytes, (cudaStream_t)stream);
}
int b200tts_flow_reverse_ragged(const b200tts_flow* h, float* z, const float* mask, const float* g,
                                const int32_t* frame_lengths, int B, int T, void* workspace, size_t workspace_bytes,
                                void* stream) {
    if (!h) { set_error("flow_reverse_ragged: null handle"); return 1; }
    return h->impl.reverse(z, mask, g, B, T, workspace, workspace_bytes, (cudaStream_t)stream, frame_lengths);
}

int b200tts_text_encoder_create(const b200tts_text_encoder_config* cfg, const float* const* weights,
                                int num_weights, b200tts_text_encoder** out) {
    if (!cfg || !weights || !out) { set_error("text_encoder_create: null argument"); return 1; }
    *out = nullptr;
    b200tts_text_encoder* h = new (std::nothrow) b200tts_text_encoder();
    if (!h) { set_error("text_encoder_create: out of host memory"); return 1; }
    int rc = h->impl.init(*cfg, weights, num_weights);
    if (rc) { delete h; return rc; }
    *out = h;
    return 0;
}
void b200tts_text_encoder_destroy(b200tts_text_encoder* h) { delete h; }
size_t b200tts_text_encoder_workspace_bytes(const b200tts_text_encoder* h, int B, int T) {
    return h ? h->impl.workspace_bytes(B, T) : 0;
}
int b200tts_text_encoder_forward(const b200tts_text_encoder* h, const int64_t* tokens, const int64_t* lengths,
                                 const float* lang_emb, int B, int T, float* x, float* stats, float* x_mask,
                                 void* workspace, size_t workspace_bytes, void* stream) {
    if (!h) { set_error("text_encoder_forward: null handle"); return 1; }
    return h->impl.forward((const long long*)tokens, (const long long*)lengths, lang_emb, B, T, x, stats, x_mask,
                           workspace, workspace_bytes, (cudaStream_t)stream);
}

int b200tts_sdp_create(const b200tts_sdp_config* cfg, const float* const* weights, int num_weights,
                       b200tts_sdp** out) {
    if (!cfg || !weights || !out) { set_error("sdp_create: null argument"); return 1; }
    *out = nullptr;
    b200tts_sdp* h = new (std::nothrow) b200tts_sdp();
    if (!h) { set_error("sdp_create: out of host memory"); return 1; }
    int rc = h->impl.init(*cfg, weights, num_weights);
    if (rc) { delete h; return rc; }
    *out = h;
    return 0;
}
void b200tts_sdp_destroy(b200tts_sdp* h) { delete h; }
size_t b200tts_sdp_workspace_bytes(const b200tts_sdp* h, int B, int T) { return h ? h->impl.workspace_bytes(B, T) : 0; }
int b200tts_sdp_reverse(const b200tts_sdp* h, const float* x, const float* mask, const float* noise, const float* g,
                        const float* lang_emb, float noise_scale, int B, int T, float* logw, int32_t* err_flag,
                        void* workspace, size_t workspace_bytes, void* stream) {
    if (!h) { set_error("sdp_reverse: null handle"); return 1; }
    return h->impl.reverse(x, mask, noise, g, lang_emb, noise_scale, B, T, logw, err_flag, workspace, workspace_bytes,
                           (cudaStream_t)stream);
}

int b200tts_durations(const float* logw, const float* x_mask, float length_scale, int B, int T, float* w_ceil,
                      float* cum, int64_t* y_lengths, const int32_t* err_flag, int64_t* meta, void* stream) {
    return launch_durations(logw, x_mask, length_scale, B, T, w_ceil, cum, (long long*)y_lengths, err_flag,
                            (long long*)meta, (cudaStream_t)stream);
}
int b200tts_expand_prior(const float* cum, const float* x_mask, const int64_t* y_lengths, const float* stats,
                         const float* noise, float noise_scale, int B, int Tx, int Ty, int C, float* attn,
                         float* m_p, float* logs_p, float* z_p, float* y_mask, void* stream) {
    return launch_expand_prior(cum, x_mask, (const long long*)y_lengths, stats, noise, noise_scale, B, Tx, Ty, C, attn,
                               m_p, logs_p, z_p, y_mask, (cudaStream_t)stream);
}

int b200tts_upsample_linear(const float* x, int rows, int Tin, float scale_factor, float* y, int Tout, void* stream) {
    return launch_upsample_linear(x, rows, Tin, scale_factor, y, Tout, (cudaStream_t)stream);
}

int b200tts_stft_create(int n_fft, int hop_length, const float* window, const float* mel_basis, int n_mels,
                        b200tts_stft** out) {
    if (!out) { set_error("stft_create: null argument"); return 1; }
    *out = nullptr;
    b200tts_stft* h = new (std::nothrow) b200tts_stft();
    if (!h) { set_error("stft_create: out of host memory"); return 1; }
    int rc = h->impl.init(n_fft, hop_length, window, mel_basis, n_mels);
    if (rc) { delete h; return rc; }
    *out = h;
    return 0;
}
void b200tts_stft_destroy(b200tts_stft* h) { delete h; }
int b200tts_stft_magnitude(const b200tts_stft* h, const float* wav, int B, int T, int pad1, int pad2, int mode,
                           float power, float* spec, int n_frames, void* stream) {
    if (!h) { set_error("stft_magnitude: null handle"); return 1; }
    return h->impl.magnitude(wav, B, T, pad1, pad2, mode, power, spec, n_frames, (cudaStream_t)stream);
}
int b200tts_stft_mel_project(const b200tts_stft* h, const float* spec, int B, int n_frames, float log_clamp,
                             float* mel, void* stream) {
    if (!h) { set_error("stft_mel_project: null handle"); return 1; }
    return h->impl.mel_project(spec, B, n_frames, log_clamp, mel, (cudaStream_t)stream);
}

int b200tts_griffin_lim_create(int n_fft, int hop_length, const float* window, const float* pinv, int n_mels,
                               b200tts_griffin_lim** out) {
    if (!out) { set_error("griffin_lim_create: null argument"); return 1; }
    *out = nullptr;
    b200tts_griffin_lim* h = new (std::nothrow) b200tts_griffin_lim();
    if (!h) { set_error("griffin_lim_create: out of host memory"); return 1; }
    int rc = h->impl.init(n_fft, hop_length, window, pinv, n_mels);
    if (rc) { delete h; return rc; }
    *out = h;
    return 0;
}
void b200tts_griffin_lim_destroy(b200tts_griffin_lim* h) { delete h; }
size_t b200tts_griffin_lim_workspace_bytes(const b200tts_griffin_lim* h, int B, int T) {
    return h ? h->impl.workspace_bytes(B, T) : 0;
}
int b200tts_griffin_lim_forward(const b200tts_griffin_lim* h, const float* x, long long x_batch_stride,
                                int x_channel_stride, int x_time_stride, int B, int C, int T, const int32_t* lengths,
                                const b200tts_audio_norm* norm, float base, float spec_gain, float power, int num_iter,
                                float preemphasis, const float* angles, float* wav, long long wav_pitch,
                                int32_t* wav_lengths, void* workspace, size_t workspace_bytes, void* stream) {
    if (!h || !norm) { set_error("griffin_lim_forward: null handle / norm"); return 1; }
    return h->impl.forward(x, x_batch_stride, x_channel_stride, x_time_stride, B, C, T, lengths, *norm, base, spec_gain,
                           power, num_iter, preemphasis, angles, wav, wav_pitch, wav_lengths, workspace, workspace_bytes,
                           (cudaStream_t)stream);
}

#define B200_HANDLE_API(NAME, TYPE, CFG)                                                                        \
    int b200tts_##NAME##_create(const CFG* cfg, const float* const* weights, int num_weights, TYPE** out) {       \
        if (!cfg || !weights || !out) { set_error(#NAME "_create: null argument"); return 1; }                   \
        *out = nullptr;                                                                                          \
        TYPE* h = new (std::nothrow) TYPE();                                                                     \
        if (!h) { set_error(#NAME "_create: out of host memory"); return 1; }                                    \
        int rc = h->impl.init(*cfg, weights, num_weights);                                                       \
        if (rc) { delete h; return rc; }                                                                         \
        *out = h;                                                                                                \
        return 0;                                                                                                \
    }                                                                                                            \
    void b200tts_##NAME##_destroy(TYPE* h) { delete h; }                                                         \
    size_t b200tts_##NAME##_workspace_bytes(const TYPE* h, int B, int T) { return h ? h->impl.workspace_bytes(B, T) : 0; }

B200_HANDLE_API(posterior, b200tts_posterior, b200tts_posterior_config)
B200_HANDLE_API(duration_predictor, b200tts_duration_predictor, b200tts_duration_predictor_config)

int b200tts_posterior_forward(const b200tts_posterior* h, const float* x, const float* mask, const float* g,
                              const float* noise, int B, int T, float* z, float* stats, void* workspace,
                              size_t workspace_bytes, void* stream) {
    if (!h) { set_error("posterior_forward: null handle"); return 1; }
    return h->impl.forward(x, mask, g, noise, B, T, z, stats, workspace, workspace_bytes, (cudaStream_t)stream);
}
int b200tts_duration_predictor_forward(const b200tts_duration_predictor* h, const float* x, const float* mask,
                                       const float* g, const float* lang_emb, int B, int T, float* logw,
                                       void* workspace, size_t workspace_bytes, void* stream) {
    if (!h) { set_error("duration_predictor_forward: null handle"); return 1; }
    return h->impl.forward(x, mask, g, lang_emb, B, T, logw, workspace, workspace_bytes, (cudaStream_t)stream);
}

B200_HANDLE_API(speaker_encoder, b200tts_speaker_encoder, b200tts_speaker_encoder_config)

int b200tts_speaker_encoder_forward(const b200tts_speaker_encoder* h, const float* x, const int32_t* starts, int B,
                                    int T, int groups, int l2_norm, float* emb, void* workspace, size_t workspace_bytes,
                                    void* stream) {
    if (!h) { set_error("speaker_encoder_forward: null handle"); return 1; }
    return h->impl.run(x, starts, B, T, groups, l2_norm, emb, -1, nullptr, workspace, workspace_bytes,
                       (cudaStream_t)stream);
}
int b200tts_speaker_encoder_features(const b200tts_speaker_encoder* h, const float* x, const int32_t* starts, int B,
                                     int T, int stage, float* out, void* workspace, size_t workspace_bytes,
                                     void* stream) {
    if (!h) { set_error("speaker_encoder_features: null handle"); return 1; }
    if (stage < 0 || stage > 4) { set_error("speaker_encoder_features: stage %d is not in 0..4", stage); return 1; }
    return h->impl.run(x, starts, B, T, 1, 0, nullptr, stage, out, workspace, workspace_bytes, (cudaStream_t)stream);
}

int b200tts_glow_tts_create(const b200tts_glow_tts_config* cfg, const float* const* weights, int num_weights,
                            b200tts_glow_tts** out) {
    if (!cfg || !weights || !out) { set_error("glow_tts_create: null argument"); return 1; }
    *out = nullptr;
    b200tts_glow_tts* h = new (std::nothrow) b200tts_glow_tts();
    if (!h) { set_error("glow_tts_create: out of host memory"); return 1; }
    int rc = h->impl.init(*cfg, weights, num_weights);
    if (rc) { delete h; return rc; }
    *out = h;
    return 0;
}
void b200tts_glow_tts_destroy(b200tts_glow_tts* h) { delete h; }
size_t b200tts_glow_tts_workspace_bytes(const b200tts_glow_tts* h, int B, int Tt, int Ty) {
    return h ? std::max(h->impl.encode_bytes(B, Tt), h->impl.decode_bytes(B, Ty)) : 0;
}
int b200tts_glow_tts_encode(const b200tts_glow_tts* h, const int64_t* tokens, const int64_t* lengths, const float* g,
                            float length_scale, int B, int Tt, float* o_stats, float* logw, float* x_mask, float* w_ceil,
                            float* cum, float* dur_log, int64_t* y_lengths, int64_t* meta, void* workspace,
                            size_t workspace_bytes, void* stream) {
    if (!h) { set_error("glow_tts_encode: null handle"); return 1; }
    return h->impl.encode((const long long*)tokens, (const long long*)lengths, g, length_scale, B, Tt, o_stats, logw,
                          x_mask, w_ceil, cum, dur_log, (long long*)y_lengths, (long long*)meta, workspace,
                          workspace_bytes, (cudaStream_t)stream);
}
int b200tts_glow_tts_decode(const b200tts_glow_tts* h, const float* o_stats, const float* x_mask, const float* cum,
                            const int64_t* y_lengths, const float* g, const float* noise, float noise_scale, int B, int Tt,
                            int Ty, float* attn, float* y_mean, float* y_log_scale, float* mel, void* workspace,
                            size_t workspace_bytes, void* stream) {
    if (!h) { set_error("glow_tts_decode: null handle"); return 1; }
    return h->impl.decode(o_stats, x_mask, cum, (const long long*)y_lengths, g, noise, noise_scale, B, Tt, Ty, attn,
                          y_mean, y_log_scale, mel, workspace, workspace_bytes, (cudaStream_t)stream);
}

int b200tts_forward_tts_create(const b200tts_forward_tts_config* cfg, const float* const* weights, int num_weights,
                               b200tts_forward_tts** out) {
    if (!cfg || !weights || !out) { set_error("forward_tts_create: null argument"); return 1; }
    *out = nullptr;
    b200tts_forward_tts* h = new (std::nothrow) b200tts_forward_tts();
    if (!h) { set_error("forward_tts_create: out of host memory"); return 1; }
    int rc = h->impl.init(*cfg, weights, num_weights);
    if (rc) { delete h; return rc; }
    *out = h;
    return 0;
}
int b200tts_speedy_speech_create(const b200tts_speedy_speech_config* cfg, const float* const* weights, int num_weights,
                                 b200tts_forward_tts** out) {
    if (!cfg || !weights || !out) { set_error("speedy_speech_create: null argument"); return 1; }
    *out = nullptr;
    b200tts_forward_tts* h = new (std::nothrow) b200tts_forward_tts();
    if (!h) { set_error("speedy_speech_create: out of host memory"); return 1; }
    int rc = h->impl.init_conv_bn(*cfg, weights, num_weights);
    if (rc) { delete h; return rc; }
    *out = h;
    return 0;
}
void b200tts_forward_tts_destroy(b200tts_forward_tts* h) { delete h; }
size_t b200tts_forward_tts_encode_workspace_bytes(const b200tts_forward_tts* h, int B, int Tt) {
    return h ? h->impl.encode_bytes(B, Tt) : 0;
}
size_t b200tts_forward_tts_decode_workspace_bytes(const b200tts_forward_tts* h, int B, int Ty) {
    return h ? h->impl.decode_bytes(B, Ty) : 0;
}
int b200tts_forward_tts_encode(const b200tts_forward_tts* h, const int64_t* tokens, const int64_t* lengths,
                               const float* g, float length_scale, int B, int Tt, float* o_en, float* logw, float* pitch,
                               float* energy, float* x_mask, float* dur, float* cum, int64_t* y_lengths, int64_t* meta,
                               void* workspace, size_t workspace_bytes, void* stream) {
    if (!h) { set_error("forward_tts_encode: null handle"); return 1; }
    return h->impl.encode((const long long*)tokens, (const long long*)lengths, g, length_scale, B, Tt, o_en, logw, pitch,
                          energy, x_mask, dur, cum, (long long*)y_lengths, (long long*)meta, workspace, workspace_bytes,
                          (cudaStream_t)stream);
}
int b200tts_forward_tts_decode(const b200tts_forward_tts* h, const float* o_en, const float* x_mask, const float* cum,
                               const int64_t* y_lengths, int B, int Tt, int Ty, float* attn, float* mel, void* workspace,
                               size_t workspace_bytes, void* stream) {
    if (!h) { set_error("forward_tts_decode: null handle"); return 1; }
    return h->impl.decode(o_en, x_mask, cum, (const long long*)y_lengths, B, Tt, Ty, attn, mel, workspace,
                          workspace_bytes, (cudaStream_t)stream);
}
int b200tts_attention_tc3(const float* qkv, const int* lens, int B, int C, int num_heads, int T, int pitch, float* out,
                          void* stream) {
    return launch_attention_tc3(qkv, (long long)3 * C * pitch, pitch, lens, out, (long long)C * pitch, B, C, num_heads, T,
                                (cudaStream_t)stream);
}

B200_HANDLE_API(melgan, b200tts_melgan, b200tts_melgan_config)

int b200tts_melgan_out_len(const b200tts_melgan* h, int T) { return h ? h->impl.out_len(T) : 0; }
int b200tts_melgan_forward(const b200tts_melgan* h, const float* x, int B, int T, int synthesize, float* out,
                           uint32_t* peak_bits, void* workspace, size_t workspace_bytes, void* stream) {
    if (!h) { set_error("melgan_forward: null handle"); return 1; }
    return h->impl.forward(x, B, T, synthesize, out, peak_bits, workspace, workspace_bytes, (cudaStream_t)stream);
}
int b200tts_pqmf_synthesis(const float* x, int B, int N, int Tb, const float* G, int taps, float* y, uint32_t* peak_bits,
                           void* stream) {
    return launch_pqmf_synthesis(x, (long long)N * Tb, Tb, B, N, Tb, G, taps, y, peak_bits, (cudaStream_t)stream);
}

B200_HANDLE_API(wavegrad, b200tts_wavegrad, b200tts_wavegrad_config)

int b200tts_wavegrad_forward(const b200tts_wavegrad* h, const float* y, const float* x, const float* noise_scale,
                             const float* const* pe, int pe_frames, int B, int T, float* eps, void* workspace,
                             size_t workspace_bytes, void* stream) {
    if (!h) { set_error("wavegrad_forward: null handle"); return 1; }
    return h->impl.forward(y, x, noise_scale, pe, pe_frames, B, T, eps, workspace, workspace_bytes, (cudaStream_t)stream);
}
int b200tts_wavegrad_condition(const b200tts_wavegrad* h, const float* x, int B, int T, void* workspace,
                               size_t workspace_bytes, void* stream) {
    if (!h) { set_error("wavegrad_condition: null handle"); return 1; }
    return h->impl.condition(x, B, T, workspace, workspace_bytes, (cudaStream_t)stream);
}
int b200tts_wavegrad_step(const b200tts_wavegrad* h, float* y, const float* noise_level, const float* const* pe,
                          int pe_frames, float c1, float c2, float sigma, const float* z, int B, int T, void* workspace,
                          size_t workspace_bytes, void* stream) {
    if (!h) { set_error("wavegrad_step: null handle"); return 1; }
    return h->impl.step(y, noise_level, pe, pe_frames, c1, c2, sigma, z, B, T, workspace, workspace_bytes,
                        (cudaStream_t)stream);
}

B200_HANDLE_API(pwgan, b200tts_pwgan, b200tts_pwgan_config)

int b200tts_pwgan_min_frames(const b200tts_pwgan* h) { return h ? h->impl.min_frames : 0; }
int b200tts_pwgan_forward(const b200tts_pwgan* h, const float* mel, const float* noise, int B, int T, int pad, float* out,
                          void* workspace, size_t workspace_bytes, void* stream) {
    if (!h) { set_error("pwgan_forward: null handle"); return 1; }
    return h->impl.forward(mel, noise, B, T, pad, out, workspace, workspace_bytes, (cudaStream_t)stream);
}
int b200tts_pwgan_layer(const b200tts_pwgan* h, int layer, const float* mel, int B, int T, int pad, const float* x,
                        float* skip, float* x_new, int pitch, void* workspace, size_t workspace_bytes, void* stream) {
    if (!h) { set_error("pwgan_layer: null handle"); return 1; }
    return h->impl.layer(layer, mel, B, T, pad, x, skip, x_new, pitch, workspace, workspace_bytes, (cudaStream_t)stream);
}
int b200tts_pwgan_upsample(const b200tts_pwgan* h, const float* a, int rows, int Tf, float* out, void* stream) {
    if (!h) { set_error("pwgan_upsample: null handle"); return 1; }
    return h->impl.upsample(a, rows, Tf, out, (cudaStream_t)stream);
}

B200_HANDLE_API(univnet, b200tts_univnet, b200tts_univnet_config)

int b200tts_univnet_forward(const b200tts_univnet* h, const float* mel, const float* noise, int B, int T, float* out,
                            void* workspace, size_t workspace_bytes, void* stream) {
    if (!h) { set_error("univnet_forward: null handle"); return 1; }
    return h->impl.forward(mel, noise, B, T, out, workspace, workspace_bytes, (cudaStream_t)stream);
}
int b200tts_univnet_predict(const b200tts_univnet* h, int block, const float* mel, int B, int T, float* pred,
                            void* workspace, size_t workspace_bytes, void* stream) {
    if (!h) { set_error("univnet_predict: null handle"); return 1; }
    return h->impl.predict(block, mel, B, T, pred, workspace, workspace_bytes, (cudaStream_t)stream);
}
int b200tts_univnet_lvc_layer(const b200tts_univnet* h, int block, int layer, const float* x, const float* pred, int B,
                              int T, float* x_new, int pitch, void* stream) {
    if (!h) { set_error("univnet_lvc_layer: null handle"); return 1; }
    return h->impl.lvc_layer(block, layer, x, pred, B, T, x_new, pitch, (cudaStream_t)stream);
}

int b200tts_overflow_create(const b200tts_overflow_config* cfg, const float* const* weights, int num_weights,
                            b200tts_overflow** out) {
    if (!cfg || !weights || !out) { set_error("overflow_create: null argument"); return 1; }
    *out = nullptr;
    b200tts_overflow* h = new (std::nothrow) b200tts_overflow();
    if (!h) { set_error("overflow_create: out of host memory"); return 1; }
    int rc = h->impl.init(*cfg, weights, num_weights);
    if (rc) { delete h; return rc; }
    *out = h;
    return 0;
}
void b200tts_overflow_destroy(b200tts_overflow* h) { delete h; }
size_t b200tts_overflow_workspace_bytes(const b200tts_overflow* h, int B, int Tt, int F) {
    return h ? h->impl.workspace_bytes(B, Tt, F) : 0;
}
int b200tts_overflow_encode(const b200tts_overflow* h, const int64_t* tokens, const int64_t* lengths, int B, int Tt,
                            float* states, void* workspace, size_t workspace_bytes, void* stream) {
    if (!h) { set_error("overflow_encode: null handle"); return 1; }
    return h->impl.encode((const long long*)tokens, (const long long*)lengths, B, Tt, states, workspace, workspace_bytes,
                          (cudaStream_t)stream);
}
int b200tts_overflow_sample(const b200tts_overflow* h, const int64_t* lengths, int B, int Tt, float temp, int max_frames,
                            float threshold, const float* noise, const uint8_t* drop, int chunk_frames, float* hmm_out,
                            int32_t* states_travelled, int32_t* frames, void* workspace, size_t workspace_bytes,
                            void* stream) {
    if (!h) { set_error("overflow_sample: null handle"); return 1; }
    return h->impl.sample((const long long*)lengths, B, Tt, temp, max_frames, threshold, noise, drop, chunk_frames,
                          hmm_out, states_travelled, frames, workspace, workspace_bytes, (cudaStream_t)stream);
}
int b200tts_overflow_decode(const b200tts_overflow* h, const float* hmm_out, const int32_t* frames, int B, int F,
                            int Fpitch, float* mel, void* workspace, size_t workspace_bytes, void* stream) {
    if (!h) { set_error("overflow_decode: null handle"); return 1; }
    return h->impl.decode(hmm_out, frames, B, F, Fpitch, mel, workspace, workspace_bytes, (cudaStream_t)stream);
}

int b200tts_tacotron2_create(const b200tts_tacotron2_config* cfg, const float* const* weights, int num_weights,
                             b200tts_tacotron2** out) {
    if (!cfg || !weights || !out) { set_error("tacotron2_create: null argument"); return 1; }
    *out = nullptr;
    b200tts_tacotron2* h = new (std::nothrow) b200tts_tacotron2();
    if (!h) { set_error("tacotron2_create: out of host memory"); return 1; }
    int rc = h->impl.init(*cfg, weights, num_weights);
    if (rc) { delete h; return rc; }
    *out = h;
    return 0;
}
void b200tts_tacotron2_destroy(b200tts_tacotron2* h) { delete h; }
size_t b200tts_tacotron2_workspace_bytes(const b200tts_tacotron2* h, int B, int Tt, int F) {
    return h ? h->impl.workspace_bytes(B, Tt, F) : 0;
}
int b200tts_tacotron2_encode(const b200tts_tacotron2* h, const int64_t* tokens, const int64_t* lengths, int B, int Tt,
                             float* enc_out, void* workspace, size_t workspace_bytes, void* stream) {
    if (!h) { set_error("tacotron2_encode: null handle"); return 1; }
    return h->impl.encode((const long long*)tokens, (const long long*)lengths, B, Tt, enc_out, workspace,
                          workspace_bytes, (cudaStream_t)stream);
}
int b200tts_tacotron2_decode_loop(const b200tts_tacotron2* h, const int64_t* lengths, const float* enc_out, int B,
                                  int Tt, int r, int max_steps, const uint8_t* drop, int chunk_steps, float* dec_out,
                                  float* stop_tokens, float* alignments, int32_t* steps, void* workspace,
                                  size_t workspace_bytes, void* stream) {
    if (!h) { set_error("tacotron2_decode_loop: null handle"); return 1; }
    return h->impl.decode_loop((const long long*)lengths, enc_out, B, Tt, r, max_steps, drop, chunk_steps, dec_out,
                               stop_tokens, alignments, steps, workspace, workspace_bytes, (cudaStream_t)stream);
}
int b200tts_tacotron2_postnet(const b200tts_tacotron2* h, const float* dec_out, const int32_t* frames, int B, int F,
                              int Fpitch, float* mel, void* workspace, size_t workspace_bytes, void* stream) {
    if (!h) { set_error("tacotron2_postnet: null handle"); return 1; }
    return h->impl.postnet(dec_out, frames, B, F, Fpitch, mel, workspace, workspace_bytes, (cudaStream_t)stream);
}

int b200tts_tacotron_create(const b200tts_tacotron_config* cfg, const float* const* weights, int num_weights,
                            b200tts_tacotron** out) {
    if (!cfg || !weights || !out) { set_error("tacotron_create: null argument"); return 1; }
    *out = nullptr;
    b200tts_tacotron* h = new (std::nothrow) b200tts_tacotron();
    if (!h) { set_error("tacotron_create: out of host memory"); return 1; }
    int rc = h->impl.init(*cfg, weights, num_weights);
    if (rc) { delete h; return rc; }
    *out = h;
    return 0;
}
void b200tts_tacotron_destroy(b200tts_tacotron* h) { delete h; }
size_t b200tts_tacotron_workspace_bytes(const b200tts_tacotron* h, int B, int Tt, int F) {
    return h ? h->impl.workspace_bytes(B, Tt, F) : 0;
}
int b200tts_tacotron_encode(const b200tts_tacotron* h, const int64_t* tokens, const int64_t* lengths, int B, int Tt,
                            float* enc_out, void* workspace, size_t workspace_bytes, void* stream) {
    if (!h) { set_error("tacotron_encode: null handle"); return 1; }
    return h->impl.encode((const long long*)tokens, (const long long*)lengths, B, Tt, enc_out, workspace,
                          workspace_bytes, (cudaStream_t)stream);
}
int b200tts_tacotron_decode_loop(const b200tts_tacotron* h, const int64_t* lengths, const float* enc_out, int B, int Tt,
                                 int r, int max_steps, const uint8_t* drop, int chunk_steps, float* dec_out,
                                 float* stop_tokens, float* alignments, int32_t* steps, void* workspace,
                                 size_t workspace_bytes, void* stream) {
    if (!h) { set_error("tacotron_decode_loop: null handle"); return 1; }
    return h->impl.decode_loop((const long long*)lengths, enc_out, B, Tt, r, max_steps, drop, chunk_steps, dec_out,
                               stop_tokens, alignments, steps, workspace, workspace_bytes, (cudaStream_t)stream);
}
int b200tts_tacotron_postnet(const b200tts_tacotron* h, const float* dec_out, const int32_t* frames, int B, int F,
                             int Fpitch, float* out, void* workspace, size_t workspace_bytes, void* stream) {
    if (!h) { set_error("tacotron_postnet: null handle"); return 1; }
    return h->impl.postnet(dec_out, frames, B, F, Fpitch, out, workspace, workspace_bytes, (cudaStream_t)stream);
}

}  // extern "C"

