// Engine handles behind the C ABI (include/tts_b200.h).  Immutable after init(): safe to share
// across streams/threads; all scratch comes from the caller's workspace.
#pragma once
#include <algorithm>
#include <functional>
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
    int init(int hidden, int kernel_size, int dilation_rate, int num_layers, int cond_channels,
             WeightList& wl);
    int forward(float* h, float* out, const float* mask, const float* g, int B, int T, float* acts, float* condv,
                cudaStream_t st, const int* lens = nullptr) const;
};

struct Flow {
    struct Block { ConvLayer pre, post; WaveNet wn; bool odd = false; };
    b200tts_flow_config c;
    bool fwd = false;
    std::vector<Block> blocks;
    // no other member makes Flow move-only, and std::vector's copy constructor is declared whatever the element type
    Flow() = default;
    Flow(const Flow&) = delete;
    Flow& operator=(const Flow&) = delete;
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
    int init(const b200tts_posterior_config& cfg, const float* const* w, int nw);
    size_t workspace_bytes(int B, int T) const;
    int forward(const float* x, const float* mask, const float* g, const float* noise, int B, int T, float* z,
                float* stats, void* ws, size_t ws_bytes, cudaStream_t st) const;
};

struct DurPred {
    b200tts_duration_predictor_config c;
    ConvLayer conv1, conv2, proj, cond, cond_lang;
    DevBuf<float> g1, b1, g2, b2;
    int init(const b200tts_duration_predictor_config& cfg, const float* const* w, int nw);
    int init(const b200tts_duration_predictor_config& cfg, WeightList& wl);   // as a component of a larger model
    size_t workspace_bytes(int B, int T) const;
    int forward(const float* x, const float* mask, const float* g, const float* lang_emb, int B, int T, float* logw,
                void* ws, size_t ws_bytes, cudaStream_t st) const;
};

int launch_upsample_linear(const float* x, int rows, int Tin, float scale_factor, float* y, int Tout, cudaStream_t st);
int launch_add_layernorm(const float* x, const float* y, const float* gamma, const float* beta, const float* mask,
                         float* out, int B, int C, int T, float eps, cudaStream_t st);
// forward_tts.cu's FFTransformer norm: LayerNorm_c(twice ? (x + y) + y : x + y) (eps 1e-5) where mask[b, t] != 0, an
// exact 0 elsewhere (a select: NaN in masked columns does not leak); y and mask are required
int launch_add_norm(const float* x, const float* y, bool twice, const float* g, const float* bta, const float* mask,
                    float* out, int B, int C, int T, cudaStream_t st);
// text_encoder.cu's embedding (x = emb[tok] * sqrt(hidden) * mask, plus the x_mask; without the sqrt(hidden) scale when
// scale_sqrt_hidden is false) and multi-head attention over a fused [B, 3C, T] q|k|v tensor; window < 0: no
// relative-position terms (rel_k / rel_v unused).  Heads up to 384 channels.
int launch_embed(const long long* tokens, const long long* lengths, const float* emb, const float* lang_emb, int B,
                 int T, int hidden, int C, float* x, float* x_mask, cudaStream_t st, bool scale_sqrt_hidden = true);
int launch_attention(const float* qkv, const float* x_mask, const float* rel_k, const float* rel_v, float* out, int B,
                     int C, int T, int num_heads, int window, cudaStream_t st);

// RelativePositionTransformer (text_encoder.cu; TTS/tts/layers/glow_tts/transformer.py:322-432) on the exact FP32 FMA
// conv, shared by the VITS text encoder (window 4, LayerNorm type "2": eps 1e-5) and Glow-TTS (no window, type "1":
// eps 1e-4).  Per layer: fused q|k|v 1x1, attention, conv_o, add+LayerNorm, k-tap FFN with same padding, add+LayerNorm
// with the mask folded in.  Layer is also ForwardTTS's FFTransformer layer (without rel_k / rel_v).
struct RelPosTransformer {
    struct Layer {
        ConvLayer qkv, o, ffn1, ffn2;
        DevBuf<float> rel_k, rel_v, ln1_g, ln1_b, ln2_g, ln2_b;
    };
    int C = 0, F = 0, heads = 0, window = -1;   // window < 0: no relative-position terms
    float eps = 0.f;
    std::vector<Layer> layers;
    // wl per layer: emb_rel_k [1,2w+1,d], emb_rel_v (window >= 0 only), conv_q.w/.b, conv_k.w/.b, conv_v.w/.b,
    // conv_o.w/.b, norm_1.gamma/.beta, ffn.conv_1.w/.b, ffn.conv_2.w/.b, norm_2.gamma/.beta
    int init(int channels, int ffn_channels, int kernel_size, int num_heads, int window, float eps, int num_layers,
             WeightList& wl);
    size_t workspace_bytes(int B, int T) const;   // q|k|v, attention output, y, FFN hidden
    // x [B, C, T], already masked: every layer in place; x is left masked
    int forward(float* x, const float* x_mask, int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) const;
};

struct TextEncoder {
    b200tts_text_encoder_config c;
    int C = 0;
    DevBuf<float> emb;
    RelPosTransformer tf;
    ConvLayer proj;
    int init(const b200tts_text_encoder_config& cfg, const float* const* w, int nw);
    size_t workspace_bytes(int B, int T) const;
    int forward(const long long* tokens, const long long* lengths, const float* lang_emb, int B, int T, float* x,
                float* stats, float* x_mask, void* ws, size_t ws_bytes, cudaStream_t st) const;
};

struct DDSConv {
    int C = 0, K = 0, L = 0;
    std::vector<ConvLayer> conv1x1;
    std::vector<DevBuf<float>> sep_w, sep_b, g1, b1, g2, b2;
    int init(int channels, int kernel_size, int num_layers, WeightList& wl);
    int forward(float* x, const float* mask, int B, int T, float* y1, float* y2, cudaStream_t st) const;
};

struct SDP {
    struct CFlow { DevBuf<float> pre_w, pre_b; DDSConv convs; ConvLayer proj; };
    b200tts_sdp_config c;
    ConvLayer pre, cond, cond_lang, proj;
    DDSConv convs;
    DevBuf<float> ea_t, ea_ls;
    std::vector<CFlow> flows;
    int init(const b200tts_sdp_config& cfg, const float* const* w, int nw);
    size_t workspace_bytes(int B, int T) const;
    int reverse(const float* x, const float* mask, const float* noise, const float* g, const float* lang_emb,
                float noise_scale, int B, int T, float* logw, int* err_flag, void* ws, size_t ws_bytes,
                cudaStream_t st) const;
};

struct Stft {
    int n_fft = 0, hop = 0, log2n = 0, n_mels = 0;
    DevBuf<float> window;
    DevBuf<float2> twiddle;            // n_fft / 2 (cos, sin) pairs
    ConvLayer mel;
    int init(int n_fft, int hop, const float* window_host, const float* mel_basis_host, int n_mels);
    int magnitude(const float* wav, int B, int T, int pad1, int pad2, int mode, float power, float* spec, int n_frames,
                  cudaStream_t st) const;
    int mel_project(const float* spec, int B, int n_frames, float log_clamp, float* out, cudaStream_t st) const;
};

// Griffin-Lim (griffin_lim.cu): a normalised [B, C, T] linear or mel spectrogram -> waveform [B, hop (T_b - 1)].
struct GriffinLim {
    int n_fft = 0, hop = 0, log2n = 0, n_mels = 0;   // n_mels > 0: mel input through the pseudo-inverse
    int win_lo = 0, win_hi = 0;                      // the window's nonzero span in [0, n_fft)
    DevBuf<float> window;                            // [n_fft], the analysis window centred in the frame
    DevBuf<float2> twiddle;                          // n_fft / 2 (cos, sin) pairs
    ConvLayer pinv;                                  // [F, n_mels] pinv(mel_basis) as a 1x1 conv
    int init(int n_fft, int hop, const float* window_host, const float* pinv_host, int n_mels);
    size_t workspace_bytes(int B, int T) const;
    int forward(const float* x, long long x_bs, int x_cs, int x_ts, int B, int C, int T, const int* lens,
                const b200tts_audio_norm& norm, float base, float spec_gain, float power, int num_iter, float preemphasis,
                const float* u, float* wav, long long wav_pitch, int* wav_lengths, void* ws, size_t ws_bytes,
                cudaStream_t st) const;
};

// H/ASP ResNet speaker encoder (speaker_encoder.cu).  Activations are freq-major with one zero row above and below,
// [H + 2][C][L]: the B windows sit side by side on the time axis, window b in columns [b*P, b*P + T) of its stage, with
// zero columns up to (b+1)*P; a 3x3 conv is then a 1D conv over the 3C channel rows of three adjacent freq rows.
struct SpeakerEncoder {
    struct Block {
        ConvLayer c1, c2, ds;                  // c2 and ds carry their BatchNorm folded in; c1's bn1 follows the ReLU
        DevBuf<float> s1, t1;                  // bn1 as a per-channel affine after the ReLU
        DevBuf<float> fc1w, fc1b, fc2w, fc2b;  // SE MLP
        int C = 0, Cin = 0, Cr = 0;
        bool down = false;                     // first block of stages 2..4: stride 2 + downsample
    };
    b200tts_speaker_encoder_config c;
    Stft stft;
    float pre0 = 0.f, pre1 = 1.f;              // pre-emphasis taps: y[t] = pre0 * x[t-1] + pre1 * x[t]
    ConvLayer conv1, att1, att2, fc;
    DevBuf<float> s0, t0;                      // stem bn1 (after the ReLU)
    std::vector<Block> blocks;
    int stage_first[5] = {0, 0, 0, 0, 0};      // index of each stage's first block (stage_first[4] = blocks.size())
    int init(const b200tts_speaker_encoder_config& cfg, const float* const* w, int nw);
    size_t workspace_bytes(int B, int T) const;
    // stop < 0: full forward into emb [groups, proj_dim]; stop = 0..4: dense features of that stage into feat
    int run(const float* x, const int* starts, int B, int T, int groups, int l2_norm, float* emb, int stop, float* feat,
            void* ws, size_t ws_bytes, cudaStream_t st) const;
};

// The Glow decoder in reverse (glow_tts.cu; TTS/tts/layers/glow_tts/decoder.py:113-137), shared by Glow-TTS and
// Overflow.  It works on the squeezed latent [B, C*num_squeeze, Tq] (Tq: squeezed frames padded to a multiple of 4 for
// the tensor-core convs, masked zero beyond); each block is start 1x1 -> WaveNet -> end 1x1, then one elementwise pass
// for the inverse affine coupling, InvConvNear^-1 and ActNorm^-1.  The last block writes the unsqueezed mel
// [B, C, Tv * num_squeeze].
struct GlowDecoder {
    struct Block {
        ConvLayer start, end;
        WaveNet wn;
        DevBuf<float> mix, an_bias, an_logs;   // inverse InvConvNear weight [ns][ns], ActNorm
    };
    int Cs = 0, Hd = 0, ns = 0, nsq = 0, sigmoid_scale = 0;   // Cs: squeezed channels out_channels * num_squeeze
    std::vector<Block> blocks;
    // wl: per block ActNorm logs, bias, InvConvNear^-1, start.w, .b, WaveNet, end.w, .b (see b200tts_glow_tts_config)
    int init(int out_channels, int hidden, int kernel_size, int dilation_rate, int num_blocks, int num_layers,
             int cond_channels, int num_splits, int num_squeeze, int sigmoid_scale, WeightList& wl);
    size_t workspace_bytes(int B, int Tq) const;
    // z [B, Cs, Tq] (overwritten), msk [B, Tq] -> mel [B, C, Tv * num_squeeze]
    int reverse(float* z, const float* msk, const float* g, int B, int Tq, int Tv, float* mel, void* ws, size_t ws_bytes,
                cudaStream_t st) const;
};

// Glow-TTS inference (glow_tts.cu): encoder (optional prenet, RelPosTransformer without a window, LayerNorm type "1"),
// duration predictor on cat(x, g), then -- after the caller's one host read of max(y_lengths) -- the expanded prior and
// the Glow decoder in reverse.  Squeeze is folded into the kernel that builds the latent, unsqueeze into the last
// block's elementwise pass.
struct GlowTTS {
    struct Prenet { ConvLayer conv; DevBuf<float> g, b; };
    b200tts_glow_tts_config c;
    int Cs = 0;                        // squeezed channels out_channels * num_squeeze
    DevBuf<float> emb;
    std::vector<Prenet> prenet;
    ConvLayer prenet_proj, proj;       // proj: [proj_m | proj_s] rows (proj_s all zero when mean_only)
    RelPosTransformer tf;
    DurPred dp;
    GlowDecoder dec;
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

// ---- recurrent building blocks of the autoregressive text-to-mel models (recurrent.cu), exact FP32 on the FMA pipe
// One LSTM input segment: columns [0, K) of W (row stride ldw) times x[b, 0:K] (batch stride x_bs); w_ds / x_ds: the
// offsets of direction blockIdx.y (BiLSTM).
struct LstmSeg {
    const float* W = nullptr; int ldw = 0; long long w_ds = 0;
    const float* x = nullptr; int x_bs = 0; long long x_ds = 0;
    int K = 0;
};
// One LSTM time step (launch_lstm): gates = sum over the segments W_s x_s, plus
//   pre[b, d*4H + row, t]   (BiLSTM: pre = W_ih x + b_ih + b_hh for every token; direction d; forward t = step, backward
//                            t = len_b - 1 - step; rows with step >= len_b skip), or
//   bias                    (LSTMCell: bias = b_ih + b_hh; rows with done[b] set skip)
// c = f c + i g, h = o tanh(c) -> c (in place, [dirs][B][H]), h_out[d * st_ds + b * h_bs + j], out[b, t, d*H + j]
struct LstmArgs {
    LstmSeg seg[3]; int nseg = 0;
    int H = 0;
    float* h_out = nullptr; int h_bs = 0; float* c = nullptr; long long st_ds = 0;
    const float* bias = nullptr;
    const float* pre = nullptr; long long pre_bs = 0; int pre_cs = 0;
    float* out = nullptr; long long out_bs = 0; int out_ts = 0;
    const long long* lens = nullptr; int step = 0;
    const int* done = nullptr;
    int B = 0;
};
// rows_per_block (8 or 32): batch rows served by one weight read; a row's result does not depend on it.
int launch_lstm(const LstmArgs& a, int dirs, int rows_per_block, int dispatch_id, cudaStream_t st, bool note);
// y[b, r] = act(W[r] . [x[b, 0:K] | x2[b, 0:K2]] + bias[r] + add[b, r, state[b]]), then the prenet dropout
// (drop[b, ctl[1], drop_layer, r] ? 2v : 0, drop [B, drop_F, drop_L, R]); rows with done[b] set skip.
struct LinArgs {
    const float* W = nullptr; const float* bias = nullptr; int K = 0, R = 0;
    const float* x = nullptr; int x_bs = 0;
    const float* x2 = nullptr; int x2_bs = 0, K2 = 0;
    float* y = nullptr; int y_bs = 0;
    const float* add = nullptr; long long add_bs = 0; int add_rs = 0; const int* state = nullptr;
    int relu = 0;
    const unsigned char* drop = nullptr; int drop_layer = 0, drop_L = 0, drop_F = 0; const int* ctl = nullptr;
    const int* done = nullptr;
    int B = 0;
};
int launch_linear(const LinArgs& a, cudaStream_t st, bool note);
// One GRUCell step (launch_gru): segments [0, nin) are the input x, [nin, nseg) the hidden state (torch rows r, z, n of
// W_ih / W_hh, H each); bias [4][H] = (b_ir + b_hr, b_iz + b_hz, b_in, b_hn); h_in [b * hin_bs + j] is the previous h.
// h_out[b * h_bs + j] = h'; with x_out also x_out[b * xo_bs + j] = h' + res[b * res_bs + j].  Rows with done[b] skip.
struct GruArgs {
    LstmSeg seg[3]; int nseg = 0, nin = 0;
    int H = 0;
    const float* bias = nullptr;
    const float* h_in = nullptr; int hin_bs = 0;
    float* h_out = nullptr; int h_bs = 0;
    const float* res = nullptr; int res_bs = 0;
    float* x_out = nullptr; int xo_bs = 0;
    const int* done = nullptr;
    int B = 0;
};
// rows_per_block (8 or 32): batch rows served by one weight read; a row's result does not depend on it.
int launch_gru(const GruArgs& a, int rows_per_block, cudaStream_t st, bool note);
// A bidirectional GRU layer of hidden size GRU_H over whole sequences, one launch (launch_bigru, B x 2 CTAs):
// pre[b * pre_bs + (d * 3H + row) * pre_cs + t] = W_ih x + b_ih, plus b_hr / b_hz on the r / z rows (direction d);
// whh: both directions' W_hh as pack_bigru_whh lays them out; bhn [2][H].  out[b * out_bs + t * out_ts + (d * H + j) *
// out_cs] = h_t of direction d for t < len_b (lens32 or lens64), zero for len_b <= t < T.
constexpr int GRU_H = 128, BIGRU_THREADS = 4 * GRU_H;
struct BiGruArgs {
    const float* pre = nullptr; long long pre_bs = 0; int pre_cs = 0;
    const float* whh = nullptr; const float* bhn = nullptr;
    float* out = nullptr; long long out_bs = 0; int out_ts = 0, out_cs = 0;
    const int* lens32 = nullptr; const long long* lens64 = nullptr;
    int T = 0;
};
// one direction's W_hh [3H][H] (torch layout) -> dst [3 * 32][BIGRU_THREADS], the kernel's shared-memory image
int pack_bigru_whh(const float* whh, float* dst);
int launch_bigru(const BiGruArgs& a, int B, cudaStream_t st);
// y[b, c, n] = x[b, n, c] for x [B, N, E]
int launch_transpose(const float* x, float* y, int B, int N, int E, cudaStream_t st);
// An autoregressive loop as CUDA-graph chunks: step(stream, parity, note) enqueues one step (parity = step index within
// the chunk, even chunk); `chunk` steps are captured once and replayed until ctl[0] (rows still running) reads 0 or
// max_steps steps have run, with one read of ctl [2 + B] words into host after each chunk.
int run_step_graph(const char* who, int chunk, int max_steps, int launches_per_step,
                   const std::function<int(cudaStream_t, int, bool)>& step, const int* ctl, int B, std::vector<int>& host,
                   cudaStream_t st);

// An eval-mode BatchNorm folded into the layer before it (recurrent.cu), taking from wl: w [Cout][row] (row = Cin * K),
// bias [Cout] when has_bias, then gamma, beta, running_mean, running_var [Cout].  wf = w * s, bf = beta - mean * s (no
// bias) or (bias - mean) * s + beta, s = gamma / sqrt(var + eps), in double.
int fold_bn(WeightList& wl, bool has_bias, double eps, int Cout, size_t row, std::vector<float>& wf,
            std::vector<float>& bf);

// The Tacotron2 text encoder (TTS/tts/layers/tacotron/tacotron2.py:73-112, also Overflow's encoder): embedding,
// n_convs x (conv k5 with BatchNorm folded -> ReLU), the LSTM input projection of both directions as one 1x1 conv, then
// one BiLSTM launch per time step (lstm_bi), each row at its own length.
struct SeqEncoder {
    int n_vocab = 0, E = 0, H = 0, n_convs = 0;   // H: LSTM hidden size per direction
    DevBuf<float> emb;
    ConvLayer convs[8], lstm_in;
    DevBuf<float> whh;                            // [2][4H][H]
    // wl: emb [n_vocab, E]; per conv: weight [E, E, 5], bias, BN weight, bias, running_mean, running_var;
    // lstm weight_ih, weight_hh, bias_ih, bias_hh, then the same four _reverse
    int init(int n_vocab, int E, int H, int n_convs, WeightList& wl);
    // encode's scratch, carved by the parent model: the conv stack's two tensors and mask, the LSTM input projection,
    // h (double-buffered) and c
    struct Scratch { float *x, *y, *xmask, *pre, *hb, *cb; };
    Scratch carve(Arena& ar, int B, int Tt) const;
    // out [B, Tt, 2H], zero past each row's length
    int encode(const long long* tokens, const long long* lengths, int B, int Tt, float* out, const Scratch& s,
               cudaStream_t st) const;
};

// Overflow / Neural-HMM inference (overflow.cu).  encode: the SeqEncoder (hidden E / 2 * spp per direction) into the
// encoder states [B, Tt*spp, E] and the hoisted encoder-state part of the output net's first layer (W_z z + b for every
// state).  sample: the autoregressive loop, chunk_frames frames per CUDA graph replay, one host read per chunk.  decode
// (Overflow only): the Glow decoder in reverse and x * std + mean.
struct Overflow {
    b200tts_overflow_config c;
    int H = 0;                         // LSTM hidden size per direction: E / 2 * state_per_phone
    int O1 = 0;                        // output-net first-layer width
    SeqEncoder enc;
    ConvLayer zproj;
    std::vector<DevBuf<float>> prenet_w;        // [P][in] (no bias)
    DevBuf<float> mem_wih, mem_whh, mem_b;      // [4M][P], [4M][M], b_ih + b_hh
    // out_w / out_b layer 0: the h part [O1][M]; layers 1..: [O_l][O_{l-1}]; last [2C+1][O_last]
    std::vector<DevBuf<float>> out_w, out_b;
    DevBuf<float> go, mean, std_;               // go_tokens [ar_order], mean / std [C]
    GlowDecoder dec;
    int init(const b200tts_overflow_config& cfg, const float* const* w, int nw);
    int tq(int F) const { return (F / c.num_squeeze + 3) / 4 * 4; }
    size_t workspace_bytes(int B, int Tt, int F) const;
    int encode(const long long* tokens, const long long* lengths, int B, int Tt, float* states, void* ws,
               size_t ws_bytes, cudaStream_t st) const;
    int sample(const long long* lengths, int B, int Tt, float temp, int max_frames, float threshold, const float* noise,
               const unsigned char* drop, int chunk_frames, float* hmm_out, int* states_travelled, int* frames,
               void* ws, size_t ws_bytes, cudaStream_t st) const;
    int decode(const float* hmm_out, const int* frames, int B, int F, int Fpitch, float* mel, void* ws, size_t ws_bytes,
               cudaStream_t st) const;
};

// ---- the decoder plumbing of the Tacotron models (taco_decoder.cu)
// The loop state both models keep at the start of the workspace from encode to the end of the loop: inputs_layer of
// the encoder outputs pin [B, 128, Tt], the loop control ctl [2 + B] ({rows running, step, steps per row}), done [B],
// the attention weights alpha and their running sum cum [B, Tt], the projection proj [B, RC], the stop logit [B], then
// nzero floats zeroed at the start of the loop, out of which each model slices its RNN states, context and go frame.
struct TacoLoop {
    float *pin, *alpha, *cum, *proj, *logit, *zero;
    int *ctl, *done;
    size_t nzero;
};
// lays the state out from the arena's current offset
void taco_loop_layout(Arena& ar, int B, int Tt, int RC, size_t nzero, TacoLoop& p);
// the loop's start: zeroes dec_out [B, S, rC], stop [B, S], align [B, S, Tt], cum and the zeroed region; alpha zero
// (original attention) or one-hot at token 0 (one_hot: DCA); no row done, step 0
int taco_loop_start(const TacoLoop& p, int B, int Tt, int S, int rC, int one_hot, float* dec_out, float* stop,
                    float* align, cudaStream_t st);
// The attention step (OriginalAttention, optionally location-sensitive, or MonotonicDynamicConvolutionAttention, with
// mask None), one CTA per running row over its len_b tokens: the weights, the context and the alignment row of step
// ctl[1].  Query / encoder widths 1024 / 512 (Tacotron2) or 256 / 256 (Tacotron); attention dim 128.
struct TacoAttention {
    int Q = 0, E = 0, type = 0, location = 0, softmax = 0;   // type 0: original, 1: dynamic convolution
    ConvLayer inproj;                          // inputs_layer as a 1x1 conv (original attention)
    DevBuf<float> wq, bq, v, wc, wd;           // query_layer, its bias (DCA), v, location conv and dense
    DevBuf<float> prior, wk, ws, wsl, wdl, bdl;   // DCA: prior, key_layer, static conv / layer, dynamic layer
    float vb = 0.f;                            // v's bias (original attention)
    // wl, original: query_layer, inputs_layer, v.weight, v.bias[, location_conv1d, location_dense]; DCA: prior,
    // query_layer.weight, .bias, key_layer, static_filter_conv, static_filter_layer, dynamic_filter_layer.weight, .bias, v
    int init(int Q, int E, int type, int location, int softmax, WeightList& wl);
    // the step-invariant keys pin [B, 128, Tt] = inputs_layer(enc) for every token (original attention; DCA: nothing),
    // through encT [B, E, Tt]
    int keys(const float* enc, float* encT, float* pin, int B, int Tt, cudaStream_t st) const;
    // the dynamic shared memory of the step for Tt tokens (set as the kernel's limit on the current device; fails past
    // the opt-in maximum)
    int prepare(int Tt, size_t* smem) const;
    // one step from q [B, Q] and enc [B, Tt, E] into ctx [B, E], p's alpha / cum and align [B, S, Tt]
    int launch(const TacoLoop& p, const float* q, float* ctx, const float* enc, float* align, int S,
               const long long* lens, int B, int Tt, size_t smem, cudaStream_t st, bool note) const;
};
// the postnet input: x [B, C, Tp] = dec [B, Fpitch, C] transposed below frames[b], else 0; mask [B, Tp] likewise
int launch_frames_in(const float* dec, int Fpitch, const int* frames, float* x, float* mask, int B, int C, int Tp,
                     cudaStream_t st);
// out [B, F, C] = y [B, C, Tp] transposed, t < F
int launch_frames_out(const float* y, int Tp, float* out, int B, int F, int C, cudaStream_t st);

// Tacotron2 inference (tacotron2.cu, on the plumbing above).  encode: the SeqEncoder (hidden 256 per direction) into the encoder outputs
// [B, Tt, 512] and, for the original attention, inputs_layer of them for every token as one 1x1 conv.  decode_loop: the
// attention decoder, chunk_steps steps per CUDA graph replay, one host read per chunk.  postnet: the 5 ConvBNBlocks
// (BatchNorm folded) on the conv engine, masked past each row's frames, plus the decoder output.
struct Tacotron2 {
    b200tts_tacotron2_config c;
    SeqEncoder enc;
    TacoAttention att;
    ConvLayer post[5];
    DevBuf<float> prenet_w[2], prenet_b[2];     // bias: the folded "bn" prenet only
    DevBuf<float> arnn_wih, arnn_whh, arnn_b;   // [4096][768], [4096][1024], b_ih + b_hh
    DevBuf<float> drnn_wih, drnn_whh, drnn_b;   // [4096][1536], [4096][1024], b_ih + b_hh
    DevBuf<float> proj_w, proj_b, stop_w, stop_b;
    int init(const b200tts_tacotron2_config& cfg, const float* const* w, int nw);
    size_t workspace_bytes(int B, int Tt, int F) const;
    int encode(const long long* tokens, const long long* lengths, int B, int Tt, float* enc_out, void* ws,
               size_t ws_bytes, cudaStream_t st) const;
    int decode_loop(const long long* lengths, const float* enc_out, int B, int Tt, int r, int max_steps,
                    const unsigned char* drop, int chunk_steps, float* dec_out, float* stop_tokens, float* alignments,
                    int* steps, void* ws, size_t ws_bytes, cudaStream_t st) const;
    int postnet(const float* dec_out, const int* frames, int B, int F, int Fpitch, float* mel, void* ws,
                size_t ws_bytes, cudaStream_t st) const;
};

// Tacotron (1) inference (tacotron.cu, on the plumbing above).  encode: embedding, the encoder prenet and CBHG (K = 16) into the encoder
// outputs [B, Tt, 256] and, for the original attention, inputs_layer of them.  decode_loop: the GRU attention decoder,
// chunk_steps steps per CUDA graph replay.  postnet: the postnet CBHG (K = 8) and last_linear.  A CBHG is the conv bank
// as one conv over the union tap window, the two projections (BatchNorm, eps 1e-3, folded; ReLU in the epilogue; masked
// past each row), the fused highway stack, the biGRU input projection as a 1x1 conv and the persistent biGRU.
struct Tacotron {
    struct Cbhg {
        int Cin = 0, K = 0, P1 = 0;
        ConvLayer bank, proj1, proj2, gru_in;
        DevBuf<float> pre_w;                   // pre_highway transposed [Cin][128] (empty: none)
        DevBuf<float> hw_w, hw_b;              // per highway [H | T] transposed [128][256], bias [256]
        DevBuf<float> whh, bhn;                // pack_bigru_whh images of both directions, b_hn [2][128]
        int init(int Cin, int K, int P1, WeightList& wl);
        // run's scratch, carved by the model: the bank and projection outputs, the highway output, the biGRU input
        struct Scratch { float *bank, *y2, *y3, *hx, *pre; };
        Scratch carve(Arena& ar, int B, int T) const;
        // x [B, Cin, T] (zero past each row) -> out as BiGruArgs describes it
        int run(const float* x, const float* mask, const int* lens32, const long long* lens64, int B, int T, float* out,
                long long out_bs, int out_ts, int out_cs, const Scratch& s, cudaStream_t st) const;
    };
    b200tts_tacotron_config c;
    int Cm = 0;                                // prenet input width: C * memory_size (memory queue) or C
    DevBuf<float> emb;
    ConvLayer eprenet[2];
    Cbhg ecbhg, pcbhg;
    ConvLayer last;
    TacoAttention att;
    DevBuf<float> prenet_w[2], prenet_b[2];
    DevBuf<float> arnn_wih, arnn_whh, arnn_b;   // [768][384], [768][256], bias as GruArgs
    DevBuf<float> pdi_w, pdi_b;                 // project_to_decoder_in [256][512]
    DevBuf<float> drnn_wih[2], drnn_whh[2], drnn_b[2];
    DevBuf<float> proj_w, proj_b, stop_w, stop_b;
    int init(const b200tts_tacotron_config& cfg, const float* const* w, int nw);
    size_t workspace_bytes(int B, int Tt, int F) const;
    int encode(const long long* tokens, const long long* lengths, int B, int Tt, float* enc_out, void* ws,
               size_t ws_bytes, cudaStream_t st) const;
    int decode_loop(const long long* lengths, const float* enc_out, int B, int Tt, int r, int max_steps,
                    const unsigned char* drop, int chunk_steps, float* dec_out, float* stop_tokens, float* alignments,
                    int* steps, void* ws, size_t ws_bytes, cudaStream_t st) const;
    int postnet(const float* dec_out, const int* frames, int B, int F, int Fpitch, float* mel, void* ws,
                size_t ws_bytes, cudaStream_t st) const;
};

// ForwardTTS inference (forward_tts.cu): FastPitch / FastSpeech / FastSpeech2 with FFTransformer encoder and decoder.
// encode runs the text side on the exact FP32 FMA conv (embedding, encoder, speaker add, duration / pitch / energy
// predictors and embeddings, durations); after the caller's one host read of max(y_lengths), decode expands the encoder
// output with the positional encoding and runs the decoder on the 3xTF32 tensor-core convs and attention_tc3.cu.
// Decoder tensors are [B, C, Tp] with Tp = frames rounded up to 4 (16-byte rows); every row stops at its y_length.
// SpeedySpeech (init_conv_bn) swaps the FFTransformer stacks for residual conv-BatchNorm ones (feed_forward/encoder.py:41-73,
// decoder.py:125-160): its encoder runs on the FP32 FMA conv like the rest of the text side, its decoder on 3xTF32 from
// Tp >= 128 frames, as the FFTransformer decoder's convs do.
struct ForwardTTS {
    using Layer = RelPosTransformer::Layer;   // FFTransformer (TTS/tts/layers/generic/transformer.py:6-35)
    // Conv1dBN (res_conv_bn.py:18-46): unpadded conv, zero-padded output (edges lo / hi), ReLU, then eval BatchNorm as the
    // per-channel affine s, h
    struct ConvBN { ConvLayer conv; DevBuf<float> s, h; int lo = 0, hi = 0; };
    using ResStack = std::vector<std::vector<ConvBN>>;   // ResidualConv1dBNBlock: [block][conv]
    b200tts_forward_tts_config c;
    bool conv_bn = false;              // SpeedySpeech: the members below replace enc / dec
    DevBuf<float> emb;
    DevBuf<float> pe;                  // pos_encoder.pe [C][pe_len] (empty without positional encoding)
    std::vector<Layer> enc, dec;
    ConvLayer proj_g, pitch_emb, energy_emb, postnet;   // SpeedySpeech: postnet = decoder.postnet.1
    ResStack enc_res, dec_res;
    ConvLayer enc_prenet, enc_out, dec_post_conv;       // encoder prenet.0 / postnet.3, decoder post_conv
    ConvBN enc_post;                                    // encoder postnet.0-2: 1x1 conv, ReLU, BatchNorm
    std::vector<ConvBN> dec_post;                       // decoder postnet.0: Conv1dBNBlock (dilation 1)
    DurPred dp, pitch_dp, energy_dp;
    int init(const b200tts_forward_tts_config& cfg, const float* const* w, int nw);
    int init_conv_bn(const b200tts_speedy_speech_config& cfg, const float* const* w, int nw);
    int init_shared(WeightList& wl);   // proj_g, the predictors and embeddings, pe: between the encoder and the decoder
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
    DevBuf<float> G;                          // device [bands][taps + 1] PQMF synthesis filter (pqmf_bands > 0)
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

// Parallel WaveGAN generator (pwgan.cu): the folded conditioning conv A = [W_aux,l W_in]_l c (replicate pad as clamped
// reads), first_conv, one fused split-fp16 tensor-core launch per residual layer (gate conv + U(A_l) + gate + out|skip
// 1x1), then ReLU -> 1x1 -> ReLU -> 1x1 on the conv engine.  64 residual / 128 gate / 64 skip channels, kernel 3.
struct UTab;
struct Pwgan {
    b200tts_pwgan_config c;
    int P = 1;                                    // samples per frame, prod(upsample_factors)
    DevBuf<float> first_w, first_b;               // [64]
    DevBuf<float> aux_w;                          // [L * 128][80]: W_aux,l W_in, gate row order
    DevBuf<float> b1, b2;                         // [L][128]: gate bias (gate row order), out | skip bias
    std::vector<DevBuf<unsigned char>> w1, w2;    // per layer: gate conv / out|skip images (pack_tc, PREC_F16X3)
    std::vector<DevBuf<float>> rs1, rs2;          // their row scales
    ConvLayer tail1, tail2;                       // last_conv_layers.1 (64 -> 64) and .3 (64 -> 1)
    // U: coefficient rows [uE0 left edge | P interior phases | uE1 right edge][uTW frames]; interior sample n reads
    // frames n / P - uoff ..; exact for inputs of at least min_frames frames
    DevBuf<float> ucoef;
    int uE0 = 0, uE1 = 0, uTW = 0, uoff = 0, min_frames = 0;
    int init(const b200tts_pwgan_config& cfg, const float* const* w, int nw);
    int dilation(int l) const;
    size_t workspace_bytes(int B, int Tf) const;  // Tf: frames after the pad
    // mel [B, 80, T], replicate-padded by `pad` frames each side; noise [B, 1, (T + 2 pad) P] -> out [B, 1, (T + 2 pad) P]
    int forward(const float* mel, const float* noise, int B, int T, int pad, float* out, void* ws, size_t ws_bytes,
                cudaStream_t st) const;
    // residual layer l of forward() on its own: the conditioning of layer l from mel (as forward), then x [B, 64, pitch]
    // -> x_new [B, 64, pitch] and skip [B, 64, pitch] updated as that layer of forward() updates it (stored by layer 0,
    // scaled by sqrt(1 / L) after the sum by the last layer); only columns [0, (T + 2 pad) P) are read or written
    int layer(int l, const float* mel, int B, int T, int pad, const float* x, float* skip, float* x_new, int pitch, void* ws,
              size_t ws_bytes, cudaStream_t st) const;
    // U alone: a [rows, Tf] -> out [rows, Tf * P]
    int upsample(const float* a, int rows, int Tf, float* out, cudaStream_t st) const;
  private:
    int build_u(const std::vector<std::vector<double>>& fir);
    UTab utab() const;
    int check_call(const char* who, int B, int T, int pad, int* Tf) const;
    int launch_aux(const float* mel, int B, int T, int pad, int l0, int nl, float* A, cudaStream_t st) const;
    int launch_layer(int l, const float* x, float* xn, float* skip, int B, int pitch, int Tf, const float* A, long long A_bs,
                     int* err, int num_sms, cudaStream_t st) const;
};

// UnivNet generator (univnet.cu): first_conv, per block the kernel predictor on the conv engine (frame rate) feeding one
// split-fp16 tensor-core GEMM that writes the predicted kernels frame-major, the transposed upsampler on the conv engine
// and one fused launch per LVC layer (conv_i + location-variable conv + gate + residual), then last_conv + tanh.
// hidden_channels 32, lvc_kernel_size 3.
struct Univnet {
    struct Block {
        ConvLayer up, kin;                        // upsample (ConvTranspose1d), kernel_predictor.input_conv
        std::vector<ConvLayer> kres;              // the six residual_conv convs
        DevBuf<float> pw, pb;                     // kernel_conv | bias_conv, rows permuted: [MP][Kp * Ch] (tap-major), [MP]
        DevBuf<float> cw, cb;                     // conv_i: [L][32][3 * 32] (tap-major), [L][32]
        int hop = 1;                              // cumulative hop of this block
    };
    b200tts_univnet_config c;
    ConvLayer first, last;
    std::vector<Block> blocks;
    int hop_total = 1;                            // prod(upsample_factors)
    int MP = 0;                                   // floats of one frame's predicted kernels and biases: L * (6144 + 64)
    int init(const b200tts_univnet_config& cfg, const float* const* w, int nw);
    size_t workspace_bytes(int B, int T) const;
    // mel [B, cond, T], noise [B, in, T] -> out [B, out, T * hop_total]
    int forward(const float* mel, const float* noise, int B, int T, float* out, void* ws, size_t ws_bytes,
                cudaStream_t st) const;
    // block blk's predicted kernels and biases alone: P [B * T][MP] (frame-major, layout in univnet.cu)
    int predict(int blk, const float* mel, int B, int T, float* P, void* ws, size_t ws_bytes, cudaStream_t st) const;
    // LVC layer l of block blk alone: x [B, 32, pitch] -> x_new, P as predict() writes it
    int lvc_layer(int blk, int l, const float* x, const float* P, int B, int T, float* x_new, int pitch,
                  cudaStream_t st) const;
  private:
    int check_call(const char* who, int B, int T) const;
    int launch_predict(int blk, const float* mel, int B, int T, float* P, float* H0, float* H1, float* H2, int* err,
                       cudaStream_t st) const;
    int launch_lvc(int blk, int l, const float* x, float* xn, int B, int T, int pitch, const float* P, int* err,
                   cudaStream_t st) const;
};

// WaveGrad (wavegrad.cu): the refinement network on the shared conv engine.  Down path y_conv -> FiLM[0] -> per DBlock
// [res (1x1), three lrelu -> k3 convs, dilations 1 / 2 / 4, on the decimated input] -> FiLM[i+1]; up path x_conv ->
// per UBlock [res (1x1) and main0 on the nearest-upsampled input, main1, out0, out1 with the FiLM pair of its rate] ->
// out_conv.  The resampling is an input addressing mode (ConvIO::near_src) and FiLM / the FiLM input epilogue are the
// conv engine's WaveGrad epilogue, so no resampled or FiLM-ed tensor is written on its own.  x_conv(spectrogram) runs
// once per inference (condition); each refinement step runs the network with out_conv fused into the update
//   y = clamp(c1 * (y - c2 * eps) + sigma * z, -1, 1)
// so eps never reaches memory.  Tensors use row pitches rounded up to 4 floats (16-byte rows).
struct Wavegrad {
    struct DBlock { ConvLayer res, m0, m1, m2; int f = 1; };
    struct Film { ConvLayer in, out; };
    struct UBlock { ConvLayer res, m0, m1, o0, o1; int f = 1; };
    b200tts_wavegrad_config c;
    ConvLayer y_conv, x_conv;
    DevBuf<float> out_w, out_b;                 // out_conv [Clast][3] and its bias (own single-row kernel)
    std::vector<DBlock> db;
    std::vector<Film> film;
    std::vector<UBlock> ub;
    int init(const b200tts_wavegrad_config& cfg, const float* const* w, int nw);
    int hop() const;
    // down-path lengths: L[0] = hop * T, L[i + 1] = L[i] / f_i; FiLM i runs at L[i]
    void lengths(int T, std::vector<int>& L) const;
    size_t workspace_bytes(int B, int T) const;
    // x_conv(x) into the workspace; step() reads it from there (same B, T and workspace)
    int condition(const float* x, int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) const;
    // Wavegrad.forward: eps [B, 1, hop T] from y [B, 1, hop T], x [B, in, T] and noise_scale (device [B]); pe[i]: device
    // [film_in_i][Lp[i]] tables pe / 5000 of FiLM i built for pe_frames >= T frames (Lp = lengths(pe_frames): the row
    // pitch; only the first L[i] columns are read)
    int forward(const float* y, const float* x, const float* noise_scale, const float* const* pe, int pe_frames, int B, int T,
                float* eps, void* ws, size_t ws_bytes, cudaStream_t st) const;
    // one refinement step in place on y (z nullable: no noise term); noise_level device [B]
    int step(float* y, const float* noise_level, const float* const* pe, int pe_frames, float c1, float c2, float sigma,
             const float* z, int B, int T, void* ws, size_t ws_bytes, cudaStream_t st) const;
  private:
    int network(const float* y, const float* noise_level, const float* const* pe, int pe_frames, int B, int T, float* out,
                float c1, float c2, float sigma, const float* z, int update, void* ws, size_t ws_bytes,
                cudaStream_t st) const;
};

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
