// Engine handles behind the C ABI (include/tts_b200.h).  Immutable after init(): safe to share
// across streams/threads; all scratch comes from the caller's workspace.
#pragma once
#include <algorithm>
#include <string.h>

#include "../../include/tts_b200.h"
#include "common.cuh"

namespace b200tts {

struct Hifigan {
    b200tts_hifigan_config c;
    ConvLayer conv_pre, cond, conv_post;
    std::vector<ConvLayer> ups;
    std::vector<std::vector<ConvLayer>> rb_c1, rb_c2;
    int prec = B200TTS_PRECISION_FP32;   // tensor-core operand type of the conv_pre / ups / resblock convs
    ~Hifigan();
    int init(const b200tts_hifigan_config& cfg, const float* const* w, int nw, int precision = B200TTS_PRECISION_FP32);
    void stage_dims(int T, std::vector<int>& C, std::vector<int>& L) const;
    size_t workspace_bytes(int B, int T) const;
    int out_len(int T) const;
    // peak_bits (nullable): device word that conv_post's store folds max|wav| into (atomicMax on the float's bits; the
    // caller zeroes it) -- the first half of save_wav's peak normalisation without another pass over the waveform
    // lens (nullable, device int32 [B]): valid frames per row.  With it, padded frames are neither computed nor read:
    // every launch stops `need` samples past a row's end, where `need` is the receptive field of the layers that still
    // follow (worked out in init()), so all samples below lens[b] * prod(upsample_factors) are bit-identical to the dense
    // call; the rest of the row is zero.
    // [frame_begin, frame_end) (default: all T frames): a window of input frames.  Only wav[b, :, frame_begin * hop,
    // frame_end * hop) is written, bit-identical to the full call; every launch produces its columns of the window plus
    // the same margin `need` on both sides (the margins are symmetric bounds on each conv's reach), on the full call's
    // tile grid.  Nothing is carried between windows: each one recomputes its halo from x.
    int forward(const float* x, const float* g, int B, int T, float* wav, void* ws, size_t ws_bytes,
                cudaStream_t st, unsigned* peak_bits = nullptr, const int* lens = nullptr, int frame_begin = 0,
                int frame_end = -1) const;
    // per-launch exactness margins (samples at the tensor's own rate), see init()
    int need_P = 0;
    std::vector<int> need_OUT, need_U, need_q_ups, rate;
    std::vector<std::vector<int>> need_T1, need_X;
    void plan_margins();
};

struct WaveNet {
    int H = 0, K = 0, L = 0, cond_ch = 0;
    ConvLayer cond;
    std::vector<ConvLayer> in_layers, res_skip;
    ~WaveNet();
    int init(int hidden, int kernel_size, int dilation_rate, int num_layers, int cond_channels,
             const float* const* w, int* consumed);
    size_t scratch_floats(int B, int T) const;
    int forward(float* h, float* out, const float* mask, const float* g, int B, int T, float* acts, float* condv,
                cudaStream_t st, const int* lens = nullptr) const;
};

struct Flow {
    struct Block { ConvLayer pre, post; WaveNet wn; bool odd = false; };
    b200tts_flow_config c;
    bool fwd = false;
    std::vector<Block*> blocks;
    ~Flow();
    int init(const b200tts_flow_config& cfg, const float* const* w, int nw, int forward_direction = 0);
    size_t workspace_bytes(int B, int T) const;
    // lens (nullable, device int32 [B]): frames per row; rows are neither computed nor read past their length (every
    // tensor in the flow is re-masked, so the frames below lens[b] are bit-identical to the dense call; z keeps its
    // input values beyond a row's end instead of the zeros the masking would write -- callers mask z afterwards)
    int reverse(float* z, const float* mask, const float* g, int B, int T, void* ws, size_t ws_bytes,
                cudaStream_t st, const int* lens = nullptr) const;
};

struct PosteriorEnc {
    b200tts_posterior_config c;
    ConvLayer pre, proj;
    WaveNet wn;
    ~PosteriorEnc();
    int init(const b200tts_posterior_config& cfg, const float* const* w, int nw);
    size_t workspace_bytes(int B, int T) const;
    int forward(const float* x, const float* mask, const float* g, const float* noise, int B, int T, float* z,
                float* stats, void* ws, size_t ws_bytes, cudaStream_t st) const;
};

struct DurPred {
    b200tts_duration_predictor_config c;
    ConvLayer conv1, conv2, proj, cond, cond_lang;
    float *g1 = nullptr, *b1 = nullptr, *g2 = nullptr, *b2 = nullptr;
    ~DurPred();
    int init(const b200tts_duration_predictor_config& cfg, const float* const* w, int nw);
    size_t workspace_bytes(int B, int T) const;
    int forward(const float* x, const float* mask, const float* g, const float* lang_emb, int B, int T, float* logw,
                void* ws, size_t ws_bytes, cudaStream_t st) const;
};

int launch_upsample_linear(const float* x, int rows, int Tin, float scale_factor, float* y, int Tout, cudaStream_t st);
int launch_add_layernorm(const float* x, const float* y, const float* gamma, const float* beta, const float* mask,
                         float* out, int B, int C, int T, float eps, cudaStream_t st);
// text_encoder.cu's embedding (x = emb[tok] * sqrt(hidden) * mask, plus the x_mask; without the sqrt(hidden) scale when
// scale_sqrt_hidden is false) and multi-head attention over a fused [B, 3C, T] q|k|v tensor; window < 0: no
// relative-position terms (rel_k / rel_v unused).  Heads up to 384 channels.
int launch_embed(const long long* tokens, const long long* lengths, const float* emb, const float* lang_emb, int B,
                 int T, int hidden, int C, float* x, float* x_mask, cudaStream_t st, bool scale_sqrt_hidden = true);
int launch_attention(const float* qkv, const float* x_mask, const float* rel_k, const float* rel_v, float* out, int B,
                     int C, int T, int num_heads, int window, cudaStream_t st);

struct TextEncoder {
    struct Layer {
        ConvLayer qkv, o, ffn1, ffn2;
        float *rel_k = nullptr, *rel_v = nullptr, *ln1_g = nullptr, *ln1_b = nullptr, *ln2_g = nullptr, *ln2_b = nullptr;
    };
    b200tts_text_encoder_config c;
    int C = 0, d = 0;
    float* emb = nullptr;
    std::vector<Layer*> layers;
    ConvLayer proj;
    ~TextEncoder();
    int init(const b200tts_text_encoder_config& cfg, const float* const* w, int nw);
    size_t workspace_bytes(int B, int T) const;
    int forward(const long long* tokens, const long long* lengths, const float* lang_emb, int B, int T, float* x,
                float* stats, float* x_mask, void* ws, size_t ws_bytes, cudaStream_t st) const;
};

struct DDSConv {
    int C = 0, K = 0, L = 0;
    std::vector<ConvLayer> conv1x1;
    std::vector<float*> sep_w, sep_b, g1, b1, g2, b2, dev;
    ~DDSConv();
    int init(int channels, int kernel_size, int num_layers, const float* const* w, int* consumed);
    int forward(float* x, const float* mask, int B, int T, float* y1, float* y2, cudaStream_t st) const;
};

struct SDP {
    struct CFlow { float *pre_w = nullptr, *pre_b = nullptr; DDSConv convs; ConvLayer proj; };
    b200tts_sdp_config c;
    ConvLayer pre, cond, cond_lang, proj;
    DDSConv convs;
    float *ea_t = nullptr, *ea_ls = nullptr;
    std::vector<CFlow*> flows;
    ~SDP();
    int init(const b200tts_sdp_config& cfg, const float* const* w, int nw);
    size_t workspace_bytes(int B, int T) const;
    int reverse(const float* x, const float* mask, const float* noise, const float* g, const float* lang_emb,
                float noise_scale, int B, int T, float* logw, int* err_flag, void* ws, size_t ws_bytes,
                cudaStream_t st) const;
};

struct Stft {
    int n_fft = 0, hop = 0, log2n = 0, n_mels = 0;
    float *window = nullptr, *twiddle = nullptr;
    ConvLayer mel;
    ~Stft();
    int init(int n_fft, int hop, const float* window_host, const float* mel_basis_host, int n_mels);
    int magnitude(const float* wav, int B, int T, int pad1, int pad2, int mode, float power, float* spec, int n_frames,
                  cudaStream_t st) const;
    int mel_project(const float* spec, int B, int n_frames, float log_clamp, float* out, cudaStream_t st) const;
};

// H/ASP ResNet speaker encoder (speaker_encoder.cu).  Activations are freq-major with one zero row above and below,
// [H + 2][C][L]: the B windows sit side by side on the time axis, window b in columns [b*P, b*P + T) of its stage, with
// zero columns up to (b+1)*P; a 3x3 conv is then a 1D conv over the 3C channel rows of three adjacent freq rows.
struct SpeakerEncoder {
    struct Block {
        ConvLayer c1, c2, ds;                  // c2 and ds carry their BatchNorm folded in; c1's bn1 follows the ReLU
        float *s1 = nullptr, *t1 = nullptr;    // bn1 as a per-channel affine after the ReLU
        float *fc1w = nullptr, *fc1b = nullptr, *fc2w = nullptr, *fc2b = nullptr;   // SE MLP
        int C = 0, Cin = 0, Cr = 0;
        bool down = false;                     // first block of stages 2..4: stride 2 + downsample
    };
    b200tts_speaker_encoder_config c;
    Stft stft;
    float pre0 = 0.f, pre1 = 1.f;              // pre-emphasis taps: y[t] = pre0 * x[t-1] + pre1 * x[t]
    ConvLayer conv1, att1, att2, fc;
    float *s0 = nullptr, *t0 = nullptr;        // stem bn1 (after the ReLU)
    std::vector<Block> blocks;
    int stage_first[5] = {0, 0, 0, 0, 0};      // index of each stage's first block (stage_first[4] = blocks.size())
    ~SpeakerEncoder();
    int init(const b200tts_speaker_encoder_config& cfg, const float* const* w, int nw);
    size_t workspace_bytes(int B, int T) const;
    // stop < 0: full forward into emb [groups, proj_dim]; stop = 0..4: dense features of that stage into feat
    int run(const float* x, const int* starts, int B, int T, int groups, int l2_norm, float* emb, int stop, float* feat,
            void* ws, size_t ws_bytes, cudaStream_t st) const;
};

// Glow-TTS inference (glow_tts.cu): encoder (optional prenet, transformer without relative terms, LayerNorm type "1"),
// duration predictor on cat(x, g), then -- after the caller's one host read of max(y_lengths) -- the expanded prior and
// the Glow decoder in reverse.  The decoder works on the squeezed latent [B, C*num_squeeze, Tq] (Tq = frames /
// num_squeeze, padded to a multiple of 4 for the tensor-core convs, masked zero beyond); each block is start 1x1 ->
// WaveNet -> end 1x1, then one elementwise pass for the inverse affine coupling, InvConvNear^-1 and ActNorm^-1.
struct GlowTTS {
    struct Prenet { ConvLayer conv; float *g = nullptr, *b = nullptr; };
    struct Block {
        ConvLayer start, end;
        WaveNet wn;
        float *mix = nullptr, *an_bias = nullptr, *an_logs = nullptr;   // inverse InvConvNear weight [ns][ns], ActNorm
    };
    b200tts_glow_tts_config c;
    int Cs = 0;                        // squeezed channels out_channels * num_squeeze
    float* emb = nullptr;
    std::vector<Prenet> prenet;
    ConvLayer prenet_proj, proj;       // proj: [proj_m | proj_s] rows (proj_s all zero when mean_only)
    std::vector<TextEncoder::Layer*> layers;
    DurPred dp;
    std::vector<Block*> blocks;
    ~GlowTTS();
    int init(const b200tts_glow_tts_config& cfg, const float* const* w, int nw);
    int tq(int Ty) const { return (Ty / c.num_squeeze + 3) / 4 * 4; }
    size_t encode_bytes(int B, int Tt) const;
    size_t decode_bytes(int B, int Ty) const;
    int encode(const long long* tokens, const long long* lengths, const float* g, float length_scale, int B, int Tt,
               float* o_stats, float* logw, float* x_mask, float* w_ceil, float* cum, float* dur_log,
               long long* y_lengths, long long* meta, void* ws, size_t ws_bytes, cudaStream_t st) const;
    int decode(const float* o_stats, const float* x_mask, const float* cum, const long long* y_lengths, const float* g,
               const float* noise, float noise_scale, int B, int Tt, int Ty, float* attn, float* y_mean,
               float* y_log_scale, float* mel, void* ws, size_t ws_bytes, cudaStream_t st) const;
};

// ForwardTTS inference (forward_tts.cu): FastPitch / FastSpeech / FastSpeech2 with FFTransformer encoder and decoder.
// encode runs the text side on the exact FP32 FMA conv (embedding, encoder, speaker add, duration / pitch / energy
// predictors and embeddings, durations); after the caller's one host read of max(y_lengths), decode expands the encoder
// output with the positional encoding and runs the decoder on the 3xTF32 tensor-core convs and attention_tc3.cu.
// Decoder tensors are [B, C, Tp] with Tp = frames rounded up to 4 (16-byte rows); every row stops at its y_length.
struct ForwardTTS {
    struct Layer {   // FFTransformer (TTS/tts/layers/generic/transformer.py:6-35)
        ConvLayer qkv, o, ffn1, ffn2;
        float *ln1_g = nullptr, *ln1_b = nullptr, *ln2_g = nullptr, *ln2_b = nullptr;
    };
    b200tts_forward_tts_config c;
    float* emb = nullptr;
    float* pe = nullptr;               // pos_encoder.pe [C][pe_len] (null without positional encoding)
    std::vector<Layer*> enc, dec;
    ConvLayer proj_g, pitch_emb, energy_emb, postnet;
    DurPred dp, pitch_dp, energy_dp;
    ~ForwardTTS();
    int init(const b200tts_forward_tts_config& cfg, const float* const* w, int nw);
    static int tp(int Ty) { return (Ty + 3) / 4 * 4; }
    size_t encode_bytes(int B, int Tt) const;
    size_t decode_bytes(int B, int Ty) const;
    int encode(const long long* tokens, const long long* lengths, const float* g, float length_scale, int B, int Tt,
               float* o_en, float* logw, float* pitch, float* energy, float* x_mask, float* dur, float* cum,
               long long* y_lengths, long long* meta, void* ws, size_t ws_bytes, cudaStream_t st) const;
    int decode(const float* o_en, const float* x_mask, const float* cum, const long long* y_lengths, int B, int Tt,
               int Ty, float* attn, float* mel, void* ws, size_t ws_bytes, cudaStream_t st) const;
};
// attention_tc3.cu: self-attention over a [B, 3C, pitch] q|k|v tensor (batch stride qkv_bs) into out [B, C, pitch] (batch
// stride out_bs), per row over the first lens[b] frames only (queries and keys; the other columns of out are zeroed)
bool attention_tc3_takes(int head_dim);
int launch_attention_tc3(const float* qkv, long long qkv_bs, int pitch, const int* lens, float* out, long long out_bs,
                         int B, int C, int num_heads, int T, cudaStream_t st);

// MelGAN generators (melgan.cu): conv_pre -> per stage [lrelu 0.2 -> ConvTranspose1d -> residual stack] -> lrelu 0.2 ->
// conv_post -> tanh, every k > 1 conv reflect-padded; optional PQMF synthesis of the band signals.  Stage tensors use a row
// pitch rounded up to 4 floats (16-byte aligned rows for the tensor-core producers).
struct Melgan {
    struct Block { ConvLayer dil, c1x1, shortcut; };
    b200tts_melgan_config c;
    ConvLayer conv_pre, conv_post;
    std::vector<ConvLayer> ups;
    std::vector<std::vector<Block>> blocks;   // [stage][block]
    float* G = nullptr;                       // device [bands][taps + 1] PQMF synthesis filter (pqmf_bands > 0)
    ~Melgan();
    int init(const b200tts_melgan_config& cfg, const float* const* w, int nw);
    void stage_dims(int T, std::vector<int>& C, std::vector<int>& L) const;
    size_t workspace_bytes(int B, int T) const;
    int out_len(int T) const;
    int check_len(int T) const;               // 0, or 1 with the error set when a reflect pad would exceed its input
    int forward(const float* x, int B, int T, int synthesize, float* out, unsigned* peak_bits, void* ws, size_t ws_bytes,
                cudaStream_t st) const;
};
// PQMF synthesis (melgan.cu): x [B, N, Tb] (row pitch x_cs, batch stride x_bs) -> y [B, 1, N * Tb]; G [N][taps + 1]
int launch_pqmf_synthesis(const float* x, long long x_bs, int x_cs, int B, int N, int Tb, const float* G, int taps, float* y,
                          unsigned* peak_bits, cudaStream_t st);

// durations -> path -> expanded prior (path.cu)
int launch_durations(const float* logw, const float* x_mask, float length_scale, int B, int T, float* w_ceil,
                     float* cum, long long* y_lengths, const int* err_flag, long long* meta, cudaStream_t st);
// ForwardTTS rule (forward_tts.py:369-371): dur = round_half_even(max(1, (exp(logw) - 1) * x_mask * length_scale)) for a
// valid token, 0 for a padded one; y_lengths = sum(dur)
int launch_durations_forward(const float* logw, const float* x_mask, float length_scale, int B, int T, float* dur,
                             float* cum, long long* y_lengths, long long* meta, cudaStream_t st);
// Glow-TTS rule: w_ceil = max(1, ceil((exp(logw) - 1) * x_mask * length_scale)); dur_log = log(1 + w_ceil * x_mask) * x_mask
int launch_durations_glow(const float* logw, const float* x_mask, float length_scale, int B, int T, float* w_ceil,
                          float* cum, long long* y_lengths, float* dur_log, long long* meta, cudaStream_t st);
// z_p may be NULL (then noise may be too): attn / m_p / logs_p / y_mask only
int launch_expand_prior(const float* cum, const float* x_mask, const long long* y_lengths, const float* stats,
                        const float* noise, float noise_scale, int B, int Tx, int Ty, int C, float* attn, float* m_p,
                        float* logs_p, float* z_p, float* y_mask, cudaStream_t st);

// vocoder hand-off (vocoder_io.cu)
int vocoder_input_len(int T, float scale_factor, int pad);
int launch_vocoder_input(const float* x, long long x_bs, int x_cs, int x_ts, int B, int C, int T,
                         const b200tts_audio_norm* denorm, const b200tts_audio_norm* norm, float scale_factor, int pad,
                         float* y, int y_pitch, cudaStream_t st);
int launch_absmax(const float* x, long long n, unsigned* peak_bits, cudaStream_t st);
int launch_absmax_window(const float* x, int rows, long long pitch, int lo, int hi, unsigned* peak_bits, cudaStream_t st);
int launch_to_int16(const float* x, long long n, const unsigned* peak_bits, short* out, cudaStream_t st);

// monotonic alignment search (mas.cu)
size_t mas_workspace_bytes(int B, int Tx, int Ty);
int mas_forward(const float* value, const float* mask, const int* t_x, const int* t_y, int B, int Tx, int Ty,
                void* path, int path_is_f32, void* ws, size_t ws_bytes, cudaStream_t st);
size_t mas_from_stats_workspace_bytes(int B, int Tx, int Ty);
int mas_from_stats(const float* z_p, const float* m_p, const float* logs_p, const int* t_x, const int* t_y, int B, int C,
                   int Tx, int Ty, void* path, int path_is_f32, float* logp_out, void* ws, size_t ws_bytes, cudaStream_t st);

}  // namespace b200tts
