/* tts_b200 -- C ABI of the H100-native (sm_90a) VITS + HiFiGAN inference hot path.
 *
 * The reference (coqui-ai/TTS v0.22.0) has no FFI for this path: its "operator API" is Python
 * classes + state_dict (SURVEY.md section 8b).  Each entry point below replaces the body of one
 * reference call; the Python mirror in tts_b200/ binds them with ctypes and keeps the reference's
 * class / function signatures.  INTEGRATION.md shows the binding a maintainer would add.
 *
 * Conventions
 *   - every function returns 0 on success, non-zero on error (1 = bad argument, 2 = CUDA error);
 *     b200tts_last_error() returns a thread-local message.  Nothing throws across the ABI.
 *   - tensors are raw DEVICE pointers, fp32 unless stated, in the reference's layouts
 *     ([B, C, T] with T contiguous); the caller owns every buffer.
 *   - *_create() takes HOST pointers to fp32 weights in PyTorch layout (weight-norm already
 *     folded: w = g * v / ||v||), packs them for the kernels and uploads them once.
 *   - scratch comes from a caller workspace sized by *_workspace_bytes(); handles are immutable
 *     after creation and may be shared by concurrent streams (each with its own workspace).
 *   - `stream` is a cudaStream_t passed as void*.
 */
#ifndef TTS_B200_H
#define TTS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

const char* b200tts_last_error(void);
/* number of kernels launched by this library in this process (bench.py "gpu_launches") */
unsigned long long b200tts_launch_count(void);
int b200tts_version(void);
/* Bit 0 (value 1): a tensor-core conv launch (on any device of this process) ever hit a pipeline timeout.  Bit 1
 * (value 2): a split-fp16 launch (B200TTS_PRECISION_F16X3, the HiFiGAN default) read an activation with |x| >= 65504,
 * which fp16 cannot hold, so its output is invalid.  The flags live in mapped host memory: no synchronisation here
 * (call after a stream sync to cover the launches before it).  Every later conv launch on that device also checks them
 * and returns status 1, so neither can pass silently: a timeout for good, a range error once (that launch then clears
 * it -- the data was out of range, the device is fine). */
int b200tts_debug_tc_error(void);
/* Debug / test aid: the number of device buffers the library's handles hold right now, over all handles and devices of
 * this process.  Creating a handle raises it; destroying the handle returns it to where it was. */
long long b200tts_debug_device_buffers(void);

/* Debug / test aids: record, on the calling thread, which kernel family every conv launch dispatched to.
 * ids: 0 FP32-FMA tile kernel, 3 tensor-core kernel (M = rows), 5 tensor-core kernel grouped (narrow layers), 6 single-row streaming kernel (conv_post), 7 fused ResBlock kernel,
 *      8 / 9 the tensor-core kernels 3 / 5 with 16-bit (bf16 / fp16) operands; the WaveGrad variants (the WaveGrad
 *      epilogue or a nearest-resampled input): 12 / 14 tensor cores with 3xTF32 / split-fp16 operands, 16 the FMA tile
 *      kernel, each + 1 with a resampled input. */
void b200tts_debug_dispatch_begin(void);
int b200tts_debug_dispatch_end(int32_t* ids, int cap); /* returns the number of launches recorded */

/* Operand precision of the tensor-core convs (FP32 is the default everywhere).
 *   FP32: fp32-class accuracy, the arithmetic chosen per engine: F16X3 for the HiFiGAN decoder's conv_pre, upsamplers
 *     and resblock convs, TF32X3 for every other layer and for b200tts_conv1d.
 *   TF32X3: 3xTF32 split operands (hi + lo, 3 tf32 MMAs per product), fp32-class accuracy over fp32's whole range.
 *   F16X3: the same split in fp16 (same 11-bit significand, twice the MMA rate): weights rows scaled by a power of two
 *     into fp16's range at pack time, activations split as hi = fp16(x), lo = fp16((x - hi) * 2^11); fp32-class accuracy
 *     (operands to 2^-22 relative) for |x| < 65504.  A larger activation sets bit 1 of b200tts_debug_tc_error and
 *     fails the next conv launch; TF32X3 takes such models.  Dispatch ids stay 3 / 5.
 *   BF16 / FP16: activations (after the leaky ReLU) and weights (after the weight-norm fold) are rounded to the 16-bit type
 *     and multiplied with fp32 accumulation; epilogues, residuals and every tensor in memory stay fp32.  bf16 keeps fp32's
 *     range with an 8-bit significand; fp16 has an 11-bit significand but overflows past +-65504 (such values become
 *     +-inf).  Only layers with in_channels % 16 == 0 take the 16-bit kernels (dispatch ids 8 / 9); others stay FP32. */
enum { B200TTS_PRECISION_FP32 = 0, B200TTS_PRECISION_BF16 = 1, B200TTS_PRECISION_FP16 = 2, B200TTS_PRECISION_TF32X3 = 3,
       B200TTS_PRECISION_F16X3 = 4 };

/* ---- one conv layer with the fused prologue / epilogue the engines use -------------------------
 * The building block every dense contraction of the path runs on; replaces one
 * F.conv1d / F.conv_transpose1d call together with the element-wise ops around it, e.g. the ResBlock1 step
 * `xt = F.leaky_relu(x, 0.1); xt = c1(xt)` ... `x = xt + x` (TTS/vocoder/models/hifigan_generator.py:93-99) or
 * `o = self.ups[i](F.leaky_relu(o, 0.1))` (:248-249):
 *   y = ((conv(leaky_relu(x, in_slope)) + bias) + residual) * scale [+ y_old if accumulate] / post_div
 * weight: host, PyTorch layout ([Cout,Cin,K], or [Cin,Cout,K] when transposed); bias host or NULL; x [B,Cin,T],
 * residual / y [B,Cout,Tout] device.  in_slope = 1 disables the prologue.  allow_tensor_cores != 0 opts the layer into
 * the wgmma 3xTF32 kernels (the decoder / flow setting); 0 keeps it on the exact FP32-FMA kernel (text encoder).
 */
typedef struct {
    int in_channels, out_channels, kernel_size, dilation, padding;
    int transposed; /* 1: ConvTranspose1d with `stride` (dilation must be 1) */
    int stride;
} b200tts_conv1d_config;
typedef struct b200tts_conv1d b200tts_conv1d;
int b200tts_conv1d_create(const b200tts_conv1d_config* cfg, const float* weight, const float* bias,
                          int allow_tensor_cores, b200tts_conv1d** out);
/* the same layer on the tensor-core kernels with a chosen operand precision (B200TTS_PRECISION_*; FP32 is
 * b200tts_conv1d_create with allow_tensor_cores = 1) */
int b200tts_conv1d_create_ex(const b200tts_conv1d_config* cfg, const float* weight, const float* bias, int precision,
                             b200tts_conv1d** out);
void b200tts_conv1d_destroy(b200tts_conv1d* h);
int b200tts_conv1d_out_len(const b200tts_conv1d* h, int T);
int b200tts_conv1d_forward(const b200tts_conv1d* h, const float* x, int B, int T, float in_slope, const float* residual,
                           float scale, int accumulate, float post_div, float* y, void* stream);
/* Padding modes of b200tts_conv1d_create_padded (nn.Conv1d's padding_mode).  REFLECT reads input column t < 0 as x[-t]
 * and t >= T as x[2T - 2 - t] (nn.ReflectionPad1d(padding) followed by an unpadded conv); it needs padding <= T - 1 and
 * is not available for transposed convs. */
enum { B200TTS_PAD_ZEROS = 0, B200TTS_PAD_REFLECT = 1 };
/* b200tts_conv1d_create / _create_ex with a padding mode (allow_tensor_cores = 0: the FP32-FMA kernel only) */
int b200tts_conv1d_create_padded(const b200tts_conv1d_config* cfg, const float* weight, const float* bias,
                                 int allow_tensor_cores, int precision, int padding_mode, b200tts_conv1d** out);
/* b200tts_conv1d_forward on an input with arbitrary batch / channel strides (floats; time contiguous), with an optional
 * tanh epilogue (tanh = 1: y = tanh(conv(leaky_relu(x)) + bias), no residual / accumulate) and an optional peak word
 * (tanh only) that max|y| is folded into, as in b200tts_hifigan_forward_ex. */
int b200tts_conv1d_forward_strided(const b200tts_conv1d* h, const float* x, long long x_batch_stride, int x_channel_stride,
                                   int B, int T, float in_slope, const float* residual, float scale, int accumulate,
                                   float post_div, int tanh, float* y, uint32_t* peak_bits, void* stream);

/* one conv with the WaveGrad variants (the layers of b200tts_wavegrad_*, one at a time): the input is read through
 * nearest resampling when near_src > 0 (x holds near_src columns, the conv sees T; 0: x holds T columns), then
 *   v = acc + bias; [lrelu(v, 0.2)] (lrelu != 0); [+ act_add[b]] (device [B], nullable); [+ residual[b, c, t]] (nullable,
 *   any strides, batch stride 0 broadcasts); [y2 <- v] (nullable, y's strides); [v = film[b, c, t] + film[b, film_half + c,
 *   t] * v] (film nullable); y <- v.
 * y [B, out, out_len(T)] with the given strides.  A zero-padded, non-transposed conv only. */
int b200tts_conv1d_forward_wavegrad(const b200tts_conv1d* h, const float* x, long long x_batch_stride, int x_channel_stride,
                                    int B, int T, int near_src, float in_slope, int lrelu, const float* act_add,
                                    const float* residual, long long res_batch_stride, int res_channel_stride,
                                    const float* film, long long film_batch_stride, int film_channel_stride, int film_half,
                                    float* y, long long y_batch_stride, int y_channel_stride, float* y2, void* stream);

/* Debug / test aids: one conv layer with every prologue / epilogue option the engines use internally (the WaveNet gate
 * and res/skip split, masks, per-row conditioning, ReLU / log-clamp, ragged rows, column windows), so that each option
 * can be checked on its own against a float64 reference.  Not a stable interface.
 *   create: b200tts_conv1d_create_padded plus the packing options of the engines: gate_half > 0 (= out_channels / 2)
 *     interleaves rows (p, p + gate_half) into one (tanh, sigmoid) GEMM row pair; in_perm / out_perm (host int32,
 *     nullable, in_channels / out_channels entries) put logical channel c at physical channel perm[c] (the flow's channel
 *     flips).  Not for transposed convs.  The handle is a b200tts_conv1d (destroy, out_len and the forward calls apply).
 *   launch: y[b, r, t] (t < out_len(T)) in the documented order
 *     prologue  x *= xmask[b, t] (xmask nullable); x = leaky_relu(x, in_slope)
 *     v = conv + bias[r] + cond[b, r]   (cond nullable, indexed by GEMM row: gate layers take it interleaved)
 *     gate      (EPI_GATE 1): v = tanh(v[2p]) * sigmoid(v[2p + 1]) -> output row p; takes no other epilogue option
 *     act       0 none, 1 relu, 2 tanh, 3 log(max(v, act_param))
 *     mask_pre  (EPI_MASK_PRE 2): v *= ymask[b, t]
 *     v += res[b, r, t] (nullable); v *= scale; accumulate (EPI_ACCUM 8): v += y_old; v /= post_div
 *     mask_post (EPI_MASK_POST 4): v *= ymask[b, t]
 *     split     (EPI_SPLIT 16, WaveNet res/skip): rows r < split go to y[b, r] with accumulate and mask_post forced on,
 *               rows r >= split to y2[b, r - split], accumulating only with EPI_ACCUM2 (32), never masked
 *   Conv1dBN (SpeedySpeech's layers, b200tts_debug_conv1d_launch_bn; no gate, split, conditioning or column window):
 *     window    (EPI_WINDOW 128): v = 0 instead of conv + bias outside columns [bn->edge_lo, len_b - bn->edge_hi) of
 *               row b, len_b = min(lens[b], out_len) with lens, else out_len
 *     affine    (bn->aff_s, aff_h: device [out_channels], both or neither): v = v * aff_s[r] + aff_h[r] right after act
 *               (relu or none)
 *   ymask needs EPI_MASK_PRE, EPI_MASK_POST or EPI_SPLIT (status 1 otherwise).  lens (device int32 [B], nullable): row b
 *   is computed below lens[b] * rate_out + need_out and reads its input as zero from lens[b] * rate_in + need_in on (the
 *   FP32-FMA kernel computes every column).  [q_lo, q_hi): the output columns to produce (the tensor-core kernels may
 *   write other columns of their tiles too); [in_lo, in_hi): the input columns that hold data.  Returns the engine's
 *   status. */
enum { B200TTS_DEBUG_EPI_GATE = 1, B200TTS_DEBUG_EPI_MASK_PRE = 2, B200TTS_DEBUG_EPI_MASK_POST = 4,
       B200TTS_DEBUG_EPI_ACCUM = 8, B200TTS_DEBUG_EPI_SPLIT = 16, B200TTS_DEBUG_EPI_ACCUM2 = 32,
       B200TTS_DEBUG_EPI_WINDOW = 128 };
enum { B200TTS_DEBUG_ACT_NONE = 0, B200TTS_DEBUG_ACT_RELU = 1, B200TTS_DEBUG_ACT_TANH = 2, B200TTS_DEBUG_ACT_LOGCLAMP = 3 };
typedef struct {
    const float* x; long long x_batch_stride; int x_channel_stride; int T;
    const float* xmask; long long xmask_batch_stride;
    float in_slope;
    const float* cond; long long cond_batch_stride;
    float* y; long long y_batch_stride; int y_channel_stride;
    const float* res; long long res_batch_stride; int res_channel_stride;
    const float* ymask; long long ymask_batch_stride;
    float* y2; long long y2_batch_stride; int y2_channel_stride;
    int split;
    float scale, post_div;
    int act; float act_param;
    int flags;
    int B;
    const int32_t* lens; int rate_out, need_out, rate_in, need_in;
    int q_lo, q_hi, in_lo, in_hi;
} b200tts_debug_conv_io;
int b200tts_debug_conv1d_create(const b200tts_conv1d_config* cfg, const float* weight, const float* bias,
                                int allow_tensor_cores, int precision, int padding_mode, int gate_half,
                                const int32_t* in_perm, const int32_t* out_perm, b200tts_conv1d** out);
int b200tts_debug_conv1d_launch(const b200tts_conv1d* h, const b200tts_debug_conv_io* io, void* stream);
typedef struct {
    int edge_lo, edge_hi;
    const float* aff_s; const float* aff_h;
} b200tts_debug_conv_bn;
int b200tts_debug_conv1d_launch_bn(const b200tts_conv1d* h, const b200tts_debug_conv_io* io, const b200tts_debug_conv_bn* bn,
                                   void* stream);

/* Debug / test aids: the transformer layers' attention and add + LayerNorm kernels, one launch at a time, as the engines
 * call them (device pointers, [B, C, T] layouts, time contiguous).  Not a stable interface.
 *   attention: the FP32-FMA multi-head attention of the VITS / Glow-TTS text encoders, ForwardTTS's text encoder and
 *     the ForwardTTS decoder's fallback.  qkv [B, 3C, T] (rows q | k | v, head h owns channels [h d, (h + 1) d), d =
 *     C / num_heads <= 384), mask [B, T] (1 valid, 0 padded), out [B, C, T]:
 *       s_ij = (q_i . k_j + [|j - i| <= window] q_i . rel_k[j - i + window]) / sqrt(d);  s_ij = -1e4 where
 *       mask_i mask_j == 0;  p = softmax_j(s);  out_i = sum_j p_ij v_j + sum_{|j - i| <= window} p_ij rel_v[j - i + window]
 *     rel_k / rel_v [2 window + 1, d] (shared by the heads); window = -1: no relative terms and rel_k / rel_v unused
 *     (NULL); window <= 15.  Every column below T is read, padded ones included: they must be finite.  A padded query
 *     row is the uniform softmax over all T keys.  Status 1 (no launch) for d > 384, window > 15, or T past the
 *     kernel's shared memory (8 (d + Tp) + 33 (d + 1) + 2 nrel d floats <= 200 KiB, Tp = T rounded up to 32, nrel =
 *     2 window + 1, or 0 without a window).
 *   add_layernorm: out[b, :, t] = LayerNorm over the C channels of v = x + y (y NULL: v = x), biased variance,
 *     (v - mean) / sqrt(var + eps) * gamma + beta, then
 *       kind 0 (VITS / Glow-TTS layers, Glow-TTS prenet, duration predictor): times mask[b, t] (mask NULL: 1); twice = 0;
 *       kind 1 (ForwardTTS FFTransformer): v = (x + y) + y when twice != 0; y and mask required; an exact 0 where
 *         mask[b, t] == 0, whatever x and y hold there (a select, so NaN does not leak); eps must be 1e-5.
 *     out may be x (the layers run in place).  Status 1 (no launch) for anything else. */
int b200tts_debug_attention(const float* qkv, const float* mask, const float* rel_k, const float* rel_v, float* out,
                            int B, int C, int T, int num_heads, int window, void* stream);
int b200tts_debug_add_layernorm(int kind, const float* x, const float* y, int twice, const float* gamma,
                                const float* beta, const float* mask, float* out, int B, int C, int T, float eps,
                                void* stream);

/* ---- monotonic alignment search ------------------------------------------------------------
 * Replaces maximum_path_c / maximum_path_each, TTS/tts/utils/monotonic_align/core.pyx:11-47
 * (called through TTS/tts/utils/helpers.py:172-194 from Vits.forward_mas, vits.py:919).
 * value [B,Tx,Ty] f32 (NOT modified, unlike the reference's in-place DP); mask [B,Tx,Ty] f32 or
 * NULL (when given, value*mask is formed on load exactly like helpers.py:184); t_x,t_y int32 [B]
 * device pointers; path [B,Tx,Ty] written in full (zeros and ones) as int32 (path_is_f32 = 0,
 * the reference dtype, core.pyx:11) or float32 (path_is_f32 = 1, the dtype helpers.py:194 casts to).
 */
size_t b200tts_mas_workspace_bytes(int B, int Tx, int Ty);
int b200tts_mas(const float* value, const float* mask, const int32_t* t_x, const int32_t* t_y, int B, int Tx,
                int Ty, void* path, int path_is_f32, void* workspace, size_t workspace_bytes, void* stream);

/* Alignment straight from the prior statistics: replaces the body of Vits.forward_mas up to `attn`
 * (TTS/tts/models/vits.py:909-919): logp[b,x,y] = sum_c exp(-2 logs_p)(-0.5 z_p^2) + sum_c (m_p exp(-2 logs_p)) z_p
 * + sum_c(-0.5 log 2pi - logs_p) + sum_c(-0.5 m_p^2 exp(-2 logs_p)), then maximum_path(logp, mask) with
 * t_x / t_y = the lengths the masks encode.  z_p [B,C,Ty], m_p / logs_p [B,C,Tx]; path as b200tts_mas; logp_out
 * (nullable) [B,Tx,Ty] receives the log-likelihoods (otherwise they live in the workspace only). */
size_t b200tts_mas_from_stats_workspace_bytes(int B, int Tx, int Ty);
int b200tts_mas_from_stats(const float* z_p, const float* m_p, const float* logs_p, const int32_t* t_x, const int32_t* t_y,
                           int B, int C, int Tx, int Ty, void* path, int path_is_f32, float* logp_out, void* workspace,
                           size_t workspace_bytes, void* stream);

/* ---- HiFiGAN generator -----------------------------------------------------------------------
 * Replaces HifiganGenerator.forward, TTS/vocoder/models/hifigan_generator.py:236-265
 * (ctor arguments :163-178).
 * weights (host pointers, PyTorch layouts), in this order:
 *   conv_pre.w [C0,Cin,7], conv_pre.b [C0]
 *   cond_layer.w [C0,cond,1], cond_layer.b [C0]                      (only if cond_channels > 0)
 *   for each upsample stage s:
 *     ups[s].w [Cs_in, Cs_in/2, k] (ConvTranspose1d layout), ups[s].b
 *     for each resblock kernel j, for each dilation n:
 *       type "1": convs1[n].w, convs1[n].b, convs2[n].w, convs2[n].b
 *       type "2": convs[n].w,  convs[n].b
 *   conv_post.w [Cout, Clast, 7], conv_post.b (NULL pointer when conv_post_bias=False)
 */
typedef struct {
    int in_channels;
    int out_channels;
    int upsample_initial_channel;
    int cond_channels;
    int resblock_type; /* 1 or 2 */
    int num_upsamples;
    int upsample_factors[8];
    int upsample_kernel_sizes[8];
    int num_kernels;
    int resblock_kernel_sizes[8];
    int num_dilations;
    int resblock_dilations[8][8];
} b200tts_hifigan_config;

typedef struct b200tts_hifigan b200tts_hifigan;
int b200tts_hifigan_create(const b200tts_hifigan_config* cfg, const float* const* weights, int num_weights,
                           b200tts_hifigan** out);
/* the same with the operand precision (B200TTS_PRECISION_*) of conv_pre, the upsamplers and the resblock convs;
 * cond_layer and conv_post stay fp32.  Every forward entry point below takes either kind of handle. */
int b200tts_hifigan_create_ex(const b200tts_hifigan_config* cfg, const float* const* weights, int num_weights, int precision,
                              b200tts_hifigan** out);
int b200tts_hifigan_precision(const b200tts_hifigan* h); /* the handle's B200TTS_PRECISION_*, -1 for NULL */
void b200tts_hifigan_destroy(b200tts_hifigan* h);
size_t b200tts_hifigan_workspace_bytes(const b200tts_hifigan* h, int B, int T);
int b200tts_hifigan_out_len(const b200tts_hifigan* h, int T);
/* x [B,Cin,T]; g [B,cond,1] or NULL; wav [B,Cout,out_len(T)] */
int b200tts_hifigan_forward(const b200tts_hifigan* h, const float* x, const float* g, int B, int T, float* wav,
                            void* workspace, size_t workspace_bytes, void* stream);

/* b200tts_hifigan_forward with two optional extras (either may be NULL):
 *  - frame_lengths, device int32 [B]: valid frames per row of a padded batch.  Padded frames are then neither computed nor
 *    read: every launch stops a layer-specific margin past a row's end (the receptive field of the layers that still
 *    follow; b200tts_hifigan_margin_frames() is the largest, at the input rate), so every sample below
 *    frame_lengths[b] * prod(upsample_factors) is BIT-IDENTICAL to the dense call and the rest of the row is zero
 *    (the dense call, like the reference, fills it with the network's response to zero input, which no caller keeps).
 *  - peak_bits: conv_post's store folds max|wav| over everything it writes into *peak_bits (atomicMax on the float's
 *    bit pattern; the caller zeroes the word first, several calls may share it): the first half of save_wav's peak
 *    normalisation, TTS/utils/audio/numpy_transforms.py:439, without another pass. */
int b200tts_hifigan_forward_ex(const b200tts_hifigan* h, const float* x, const float* g, int B, int T, float* wav,
                               const int32_t* frame_lengths, uint32_t* peak_bits, void* workspace, size_t workspace_bytes,
                               void* stream);
int b200tts_hifigan_margin_frames(const b200tts_hifigan* h);
/* Streaming decode: writes wav[b, :, frame_begin*hop : frame_end*hop) of a [B, Cout, out_len(T)] buffer (hop =
 * prod(upsample_factors)), bit-identical to what b200tts_hifigan_forward_ex(same x, g, frame_lengths) writes there; every
 * other sample is untouched.  x holds all T frames (the halo reads up to b200tts_hifigan_margin_frames() frames either side
 * of the window).  Windows carry no state: any sequence of calls, e.g. consecutive chunks, may share one workspace of
 * b200tts_hifigan_workspace_bytes(B, T) bytes.  peak_bits (nullable) folds max|wav| over the window's samples.
 * Status 1 unless 0 <= frame_begin < frame_end <= T and out_len(T) == T * hop (every upsampler with k - u even). */
int b200tts_hifigan_forward_window(const b200tts_hifigan* h, const float* x, const float* g, int B, int T,
                                   int frame_begin, int frame_end, float* wav, const int32_t* frame_lengths,
                                   uint32_t* peak_bits, void* workspace, size_t workspace_bytes, void* stream);

/* ---- hand-off around a standalone vocoder ---------------------------------------------------------
 * b200tts_vocoder_input replaces, in one pass on the device, what Synthesizer.tts does on the host between the TTS
 * model and the vocoder (TTS/utils/synthesizer.py:412-429):
 *   tts_ap.denormalize (TTS/utils/audio/processor.py:303-337)  ->  vocoder_ap.normalize (:259-301)
 *   -> interpolate_vocoder_input (TTS/vocoder/utils/generic_utils.py:11-29; bilinear, align_corners=False,
 *      recompute_scale_factor=True, scale [1, scale_factor])   -> replicate padding of HifiganGenerator.inference
 *      (TTS/vocoder/models/hifigan_generator.py:281)
 * x is addressed as x[b*x_batch_stride + c*x_channel_stride + t*x_time_stride] (the TTS model's [B,T,C] output or a
 * [B,C,T] spectrogram alike); y is [B, C, y_pitch] with b200tts_vocoder_input_len(T, scale_factor, padding) valid
 * columns per row (give y_pitch a multiple of 4 for the tensor-core kernels).  scaler_mean / scaler_scale: DEVICE
 * pointers to the [C] statistics of a mean-var AudioProcessor (stats_path), NULL otherwise.
 * b200tts_absmax / b200tts_to_int16: save_wav's `wav * (32767 / max(0.01, max|wav|))` -> int16
 * (TTS/utils/audio/numpy_transforms.py:439-441); *peak_bits as above.
 */
typedef struct {
    int signal_norm, symmetric_norm, clip_norm;
    float max_norm, min_level_db, ref_level_db;
    const float* scaler_mean;
    const float* scaler_scale;
} b200tts_audio_norm;
int b200tts_vocoder_input_len(int T, float scale_factor, int padding);
int b200tts_vocoder_input(const float* x, long long x_batch_stride, int x_channel_stride, int x_time_stride, int B, int C,
                          int T, const b200tts_audio_norm* denormalize, const b200tts_audio_norm* normalize,
                          float scale_factor, int padding, float* y, int y_pitch, void* stream);
int b200tts_absmax(const float* x, long long n, uint32_t* peak_bits, void* stream);
int b200tts_to_int16(const float* x, long long n, const uint32_t* peak_bits, int16_t* out, void* stream);

/* ---- residual-coupling flow, reverse direction ------------------------------------------------
 * Replaces ResidualCouplingBlocks.forward(reverse=True), TTS/tts/layers/vits/networks.py:214-232
 * (blocks :138-166, WaveNet TTS/tts/layers/generic/wavenet.py:94-115) as called at vits.py:1156.
 * weights per flow n = 0..num_flows-1 (host, PyTorch layouts, weight norm folded):
 *   pre.w [H, C/2, 1], pre.b
 *   enc.cond_layer.w [2*H*L, cond, 1], enc.cond_layer.b            (only if cond_channels > 0)
 *   for each WN layer i: enc.in_layers[i].w [2H,H,k], .b, enc.res_skip_layers[i].w [2H or H,H,1], .b
 *   post.w [C/2, H, 1], post.b
 * z [B,C,T] is transformed IN PLACE; mask [B,T] (1/0 floats, the reference's y_mask); g [B,cond] or NULL.
 */
typedef struct {
    int channels;
    int hidden_channels;
    int kernel_size;
    int dilation_rate;
    int num_layers;
    int num_flows;
    int cond_channels;
} b200tts_flow_config;

typedef struct b200tts_flow b200tts_flow;
int b200tts_flow_create(const b200tts_flow_config* cfg, const float* const* weights, int num_weights,
                        b200tts_flow** out);
/* same weights, packed for the forward direction (networks.py:223-227; voice conversion, vits.py:1226):
 * run it with b200tts_flow_reverse() -- the handle remembers its direction */
int b200tts_flow_create_forward(const b200tts_flow_config* cfg, const float* const* weights, int num_weights,
                                b200tts_flow** out);
void b200tts_flow_destroy(b200tts_flow* h);
size_t b200tts_flow_workspace_bytes(const b200tts_flow* h, int B, int T);
int b200tts_flow_reverse(const b200tts_flow* h, float* z, const float* mask, const float* g, int B, int T,
                         void* workspace, size_t workspace_bytes, void* stream);
/* Same with frame_lengths (device int32 [B], = the row sums of mask): rows are neither computed nor read past their
 * length.  Everything in the flow is re-masked, so frames below frame_lengths[b] are bit-identical to the dense call;
 * beyond a row's end z keeps its input values (the dense call writes zeros there): mask z afterwards. */
int b200tts_flow_reverse_ragged(const b200tts_flow* h, float* z, const float* mask, const float* g,
                                const int32_t* frame_lengths, int B, int T, void* workspace, size_t workspace_bytes,
                                void* stream);

/* ---- latent upsampling (VitsArgs.encoder_sample_rate) -----------------------------------------
 * Replaces torch.nn.functional.interpolate(z, scale_factor=[f], mode="linear") in Vits.upsampling_z,
 * TTS/tts/models/vits.py:944-959.  x [rows, Tin] -> y [rows, Tout], Tout = floor(Tin * f) chosen by the caller.
 */
int b200tts_upsample_linear(const float* x, int rows, int Tin, float scale_factor, float* y, int Tout, void* stream);

/* ---- posterior encoder (training / voice conversion) ----------------------------------------
 * Replaces PosteriorEncoder.forward, TTS/tts/layers/vits/networks.py:275-288.
 * weights: pre.w [H,Cin,1], pre.b, [enc.cond_layer.w, .b], per WN layer enc.in_layers[i].w,.b, enc.res_skip_layers[i].w,.b,
 *          proj.w [2*out,H,1], proj.b.
 * x [B,Cin,T] (linear spectrogram); mask [B,T]; g [B,cond] or NULL; noise [B,out,T] = the randn_like(mean) draw of :287.
 * outputs: z [B,out,T] = (mean + noise*exp(log_scale))*mask; stats [B,2*out,T] = [mean | log_scale] (masked).
 */
typedef struct {
    int in_channels;
    int out_channels;
    int hidden_channels;
    int kernel_size;
    int dilation_rate;
    int num_layers;
    int cond_channels;
} b200tts_posterior_config;
typedef struct b200tts_posterior b200tts_posterior;
int b200tts_posterior_create(const b200tts_posterior_config* cfg, const float* const* weights, int num_weights,
                             b200tts_posterior** out);
void b200tts_posterior_destroy(b200tts_posterior* h);
size_t b200tts_posterior_workspace_bytes(const b200tts_posterior* h, int B, int T);
int b200tts_posterior_forward(const b200tts_posterior* h, const float* x, const float* mask, const float* g,
                              const float* noise, int B, int T, float* z, float* stats, void* workspace,
                              size_t workspace_bytes, void* stream);

/* ---- deterministic duration predictor (VitsArgs.use_sdp = False) ----------------------------
 * Replaces DurationPredictor.forward, TTS/tts/layers/glow_tts/duration_predictor.py:44-69.
 * weights: conv_1.w [F,Cin,k], .b, norm_1.gamma [F], .beta, conv_2.w [F,F,k], .b, norm_2.gamma, .beta, proj.w [1,F,1], .b,
 *          [cond.w [Cin,cond,1], .b], [cond_lang.w [Cin,L,1], .b]          (Cin = in_channels + language_emb_dim)
 * x [B,Cin,T]; mask [B,T]; g [B,cond] / lang_emb [B,L] or NULL -> log-durations [B,T].
 */
typedef struct {
    int in_channels;
    int hidden_channels;
    int kernel_size;
    int cond_channels;
    int language_emb_dim;
} b200tts_duration_predictor_config;
typedef struct b200tts_duration_predictor b200tts_duration_predictor;
int b200tts_duration_predictor_create(const b200tts_duration_predictor_config* cfg, const float* const* weights,
                                      int num_weights, b200tts_duration_predictor** out);
void b200tts_duration_predictor_destroy(b200tts_duration_predictor* h);
size_t b200tts_duration_predictor_workspace_bytes(const b200tts_duration_predictor* h, int B, int T);
int b200tts_duration_predictor_forward(const b200tts_duration_predictor* h, const float* x, const float* mask,
                                       const float* g, const float* lang_emb, int B, int T, float* logw,
                                       void* workspace, size_t workspace_bytes, void* stream);

/* ---- text encoder ----------------------------------------------------------------------------
 * Replaces TextEncoder.forward, TTS/tts/layers/vits/networks.py:80-100 (RelativePositionTransformer
 * TTS/tts/layers/glow_tts/transformer.py:411-432, layer_norm_type "2", heads_share=True).
 * weights (host): emb.weight [n_vocab, hidden];
 *   per layer l: attn.emb_rel_k [1,2w+1,d], attn.emb_rel_v, conv_q.w,.b, conv_k.w,.b, conv_v.w,.b, conv_o.w,.b,
 *                norm_layers_1.gamma,.beta, ffn.conv_1.w,.b, ffn.conv_2.w,.b, norm_layers_2.gamma,.beta
 *   proj.w [2*out, C, 1], proj.b                      (C = hidden_channels + language_emb_dim)
 * tokens int64 [B,T]; lengths int64 [B]; lang_emb [B, language_emb_dim] or NULL.
 * outputs: x [B,C,T]; stats [B,2*out,T] (m_p = rows [0,out), logs_p = rows [out,2*out)); x_mask [B,T].
 */
typedef struct {
    int n_vocab;
    int out_channels;
    int hidden_channels;
    int hidden_channels_ffn;
    int num_heads;
    int num_layers;
    int kernel_size;
    int rel_attn_window_size;
    int language_emb_dim;
} b200tts_text_encoder_config;

typedef struct b200tts_text_encoder b200tts_text_encoder;
int b200tts_text_encoder_create(const b200tts_text_encoder_config* cfg, const float* const* weights,
                                int num_weights, b200tts_text_encoder** out);
void b200tts_text_encoder_destroy(b200tts_text_encoder* h);
size_t b200tts_text_encoder_workspace_bytes(const b200tts_text_encoder* h, int B, int T);
int b200tts_text_encoder_forward(const b200tts_text_encoder* h, const int64_t* tokens, const int64_t* lengths,
                                 const float* lang_emb, int B, int T, float* x, float* stats, float* x_mask,
                                 void* workspace, size_t workspace_bytes, void* stream);

/* ---- stochastic duration predictor, reverse ---------------------------------------------------
 * Replaces StochasticDurationPredictor.forward(reverse=True),
 * TTS/tts/layers/vits/stochastic_duration_predictor.py:222-239,285-294 (+ transforms.py spline inverse).
 * weights (host): pre.w [H,in,1], pre.b; [cond.w, cond.b]; [cond_lang.w, cond_lang.b];
 *   convs: 3 x (convs_sep.w [H,1,k], .b, convs_1x1.w [H,H,1], .b, norms_1.gamma,.beta, norms_2.gamma,.beta);
 *   proj.w [H,H,1], proj.b; flows.0.translation [2], flows.0.log_scale [2];
 *   for f = 1..num_flows: flows.f.pre.w [H,1,1], .b, flows.f.convs (3 x 8 as above), flows.f.proj.w [3*nb-1,H,1], .b
 * x [B,in,T]; mask [B,T]; noise [B,2,T] = the standard-normal draw of :287 (made by the caller so
 * that results are reproducible against the reference); g [B,cond] / lang_emb [B,L] or NULL.
 * logw [B,T].  err_flag: device int set to 1 if the spline discriminant goes negative (the reference
 * asserts, transforms.py:168); may be NULL.
 */
typedef struct {
    int in_channels;
    int hidden_channels;
    int kernel_size;
    int num_flows;
    int cond_channels;
    int language_emb_dim;
    int num_bins;
    float tail_bound;
} b200tts_sdp_config;

typedef struct b200tts_sdp b200tts_sdp;
int b200tts_sdp_create(const b200tts_sdp_config* cfg, const float* const* weights, int num_weights,
                       b200tts_sdp** out);
void b200tts_sdp_destroy(b200tts_sdp* h);
size_t b200tts_sdp_workspace_bytes(const b200tts_sdp* h, int B, int T);
int b200tts_sdp_reverse(const b200tts_sdp* h, const float* x, const float* mask, const float* noise, const float* g,
                        const float* lang_emb, float noise_scale, int B, int T, float* logw, int32_t* err_flag,
                        void* workspace, size_t workspace_bytes, void* stream);

/* ---- durations -> path -> expanded prior ------------------------------------------------------
 * Replaces the glue at TTS/tts/models/vits.py:1140-1155 (generate_path: TTS/tts/utils/helpers.py:154-169).
 * b200tts_durations : w_ceil [B,T] = ceil(exp(logw) * x_mask * length_scale); cum [B,T] = cumsum(w_ceil);
 *                     y_lengths int64 [B] = max(1, sum(w_ceil)); meta int64 [2] (or NULL) = {max_b y_lengths,
 *                     *err_flag (the duration predictor's spline flag, may be NULL -> 0)}: the one host read of
 *                     Vits.inference (sequence_mask(y_lengths, None), helpers.py:53-54) fetches both.
 * b200tts_expand_prior (after the caller has read max(y_lengths) = Ty): attn [B,Tx,Ty] one-hot (or NULL),
 *   m_p / logs_p / z_p [B,C,Ty] with z_p = m_p + noise * exp(logs_p) * noise_scale (z_p may be NULL, and then noise
 *   too), y_mask [B,Ty] (or NULL);
 *   stats is the text encoder's [B,2C,Tx]; noise [B,C,Ty] is the randn_like(m_p) draw of vits.py:1155.
 */
int b200tts_durations(const float* logw, const float* x_mask, float length_scale, int B, int T, float* w_ceil,
                      float* cum, int64_t* y_lengths, const int32_t* err_flag, int64_t* meta, void* stream);
int b200tts_expand_prior(const float* cum, const float* x_mask, const int64_t* y_lengths, const float* stats,
                         const float* noise, float noise_scale, int B, int Tx, int Ty, int C, float* attn,
                         float* m_p, float* logs_p, float* z_p, float* y_mask, void* stream);

/* ---- STFT magnitude / mel front end ----------------------------------------------------------
 * Replaces wav_to_spec / spec_to_mel / wav_to_mel, TTS/tts/models/vits.py:96-208, and TorchSTFT.__call__,
 * TTS/utils/audio/torch_transforms.py:104-145.
 * create: window [n_fft] (host; the analysis window already zero-padded to n_fft), mel_basis [n_mels, n_fft/2+1]
 *         (host, e.g. librosa.filters.mel) or NULL.  n_fft must be a power of two.
 * magnitude: wav [B,T] -> spec [B, n_fft/2+1, n_frames].  The signal is reflect-padded by pad1 samples, then by
 *   pad2 samples (both each side; 0 = none), then framed with hop (no centering of its own):
 *     wav_to_spec  : pad1 = (n_fft-hop)/2, pad2 = 0,        mode 0: sqrt(re^2+im^2+1e-6)
 *     TorchSTFT    : pad1 = pad_wav ? (n_fft-hop)/2 : 0, pad2 = n_fft/2 (center=True), mode 1: sqrt(max(.,1e-8))
 *     MelSpectrogram (torchaudio, power 2): pad1 = 0, pad2 = n_fft/2, mode 2: re^2+im^2 (no clamp, no root)
 *   power != 1 raises the magnitude to that power (TorchSTFT.power).
 * mel_project: mel [B,n_mels,n_frames] = basis @ spec, followed by log(max(., log_clamp)) when log_clamp > 0.
 */
typedef struct b200tts_stft b200tts_stft;
int b200tts_stft_create(int n_fft, int hop_length, const float* window, const float* mel_basis, int n_mels,
                        b200tts_stft** out);
void b200tts_stft_destroy(b200tts_stft* h);
int b200tts_stft_magnitude(const b200tts_stft* h, const float* wav, int B, int T, int pad1, int pad2, int mode,
                           float power, float* spec, int n_frames, void* stream);
int b200tts_stft_mel_project(const b200tts_stft* h, const float* spec, int B, int n_frames, float log_clamp,
                             float* mel, void* stream);

/* ---- Griffin-Lim: spectrogram -> waveform ---------------------------------------------------------
 * Replaces AudioProcessor.inv_spectrogram / inv_melspectrogram, TTS/utils/audio/processor.py:444-458, with
 * numpy_transforms.griffin_lim (:220-230; librosa stft / istft, center=True, reflect padding) and the inverse
 * preemphasis (scipy.signal.lfilter([1], [1, -preemphasis])), batched; the reference runs one row at a time on the host.
 * create: window [n_fft] (host; the periodic analysis window already centred and zero-padded to n_fft), n_fft a power
 *   of two in [32, 8192], 1 <= hop_length <= n_fft.  pinv (host, [n_fft/2+1, n_mels], np.linalg.pinv(mel_basis)) makes
 *   a mel handle (C == n_mels); NULL makes a linear one (C == n_fft/2+1).
 * forward: x is addressed as x[b*x_batch_stride + c*x_channel_stride + t*x_time_stride] ([B,C,T] or [B,T,C]);
 *   lengths (DEVICE int32 [B], each in [2, T]; NULL: all T) are the rows' frame counts.  Per row:
 *     S = denormalize(x) (norm; scaler_mean / scaler_scale as for b200tts_vocoder_input)
 *     S = base ** (S / spec_gain)            (base 10 or e; base 0: x is already a magnitude, norm must be identity)
 *     S = max(1e-10, pinv @ S)               (mel handles)
 *     S = |S| ** power
 *     y = istft(S exp(2 pi i angles)), then num_iter times y = istft(S exp(i angle(stft(y))))
 *     wav = lfilter([1], [1, -preemphasis], y)   (preemphasis 0: wav = y)
 *   angles: DEVICE [B, n_fft/2+1, T] draws in [0, 1).  wav: [B, wav_pitch] with wav_pitch >= hop_length * (T - 1); row
 *   b holds wav_lengths[b] = hop_length * (lengths[b] - 1) samples and zeros after them, or, when the first istft of
 *   the row is not finite everywhere, the reference's single 0.0 sample (wav_lengths[b] = 1).  No host synchronisation.
 */
typedef struct b200tts_griffin_lim b200tts_griffin_lim;
int b200tts_griffin_lim_create(int n_fft, int hop_length, const float* window, const float* pinv, int n_mels,
                               b200tts_griffin_lim** out);
void b200tts_griffin_lim_destroy(b200tts_griffin_lim* h);
size_t b200tts_griffin_lim_workspace_bytes(const b200tts_griffin_lim* h, int B, int T);
int b200tts_griffin_lim_forward(const b200tts_griffin_lim* h, const float* x, long long x_batch_stride,
                                int x_channel_stride, int x_time_stride, int B, int C, int T, const int32_t* lengths,
                                const b200tts_audio_norm* norm, float base, float spec_gain, float power, int num_iter,
                                float preemphasis, const float* angles, float* wav, long long wav_pitch,
                                int32_t* wav_lengths, void* workspace, size_t workspace_bytes, void* stream);

/* ---- H/ASP ResNet speaker encoder (d-vectors) --------------------------------------------------
 * Replaces ResNetSpeakerEncoder.forward, TTS/encoder/models/resnet.py:153-198, with the front end of
 * BaseEncoder.get_torch_mel_spectrogram_class, TTS/encoder/models/base_encoder.py:12-61 (PreEmphasis, then
 * torchaudio MelSpectrogram: centred STFT with reflect padding, power 2, mel filterbank).
 * weights (host, PyTorch layout; every BatchNorm is 4 tensors: weight, bias, running_mean, running_var):
 *   if use_torch_spec: torch_spec.0.filter [2], torch_spec.1.spectrogram.window [win_length],
 *                      torch_spec.1.mel_scale.fb [fft_size/2+1, input_dim]
 *   conv1.weight [F0,1,3,3], conv1.bias, bn1 (4)
 *   per stage s, per block i (layerS.i): conv1.weight [F,Fin,3,3], bn1 (4), conv2.weight [F,F,3,3], bn2 (4),
 *     se.fc.0.weight [F/8,F], se.fc.0.bias, se.fc.2.weight [F,F/8], se.fc.2.bias,
 *     and for block 0 of stages 2..4: downsample.0.weight [F,Fin,1,1], downsample.1 (4)
 *   attention.0.weight [128, F3*input_dim/8, 1], attention.0.bias, attention.2 (4), attention.3.weight, .bias
 *   fc.weight [proj_dim, (ASP ? 2 : 1) * F3*input_dim/8], fc.bias
 * forward: B windows of T samples (use_torch_spec) or T frames (spectrogram input), window b starting at element
 *   starts[b] (device int32) of x.  Waveform: x is flat, each window is pre-emphasised and framed at its own edges.
 *   Spectrogram: window b is the [input_dim, T] block at x + starts[b] (channel stride T).  Consecutive runs of
 *   B / groups windows are averaged after the optional l2 norm: emb [groups, proj_dim].  B % groups must be 0.
 * features: the same pipeline stopped after stage `stage` (0: instance-normed input [B, input_dim, T'];
 *   s = 1..4: layerS output [B, F(s-1), H_s, T_s]), written densely to out.  For tests and inspection.
 * workspace_bytes covers both calls for B windows of length T.
 */
typedef struct {
    int input_dim;        /* mel bins (64) */
    int proj_dim;         /* embedding size (512) */
    int layers[4];        /* SE blocks per stage ([3, 4, 6, 3]) */
    int num_filters[4];   /* channels per stage ([32, 64, 128, 256]) */
    int encoder_type;     /* 0 = SAP, 1 = ASP */
    int log_input;        /* log(x + 1e-6) before the instance norm */
    int use_torch_spec;   /* 1: waveform input through the mel front end; 0: [input_dim, T] spectrogram input */
    int fft_size, win_length, hop_length;   /* front end (use_torch_spec only) */
} b200tts_speaker_encoder_config;
typedef struct b200tts_speaker_encoder b200tts_speaker_encoder;
int b200tts_speaker_encoder_create(const b200tts_speaker_encoder_config* cfg, const float* const* weights,
                                   int num_weights, b200tts_speaker_encoder** out);
void b200tts_speaker_encoder_destroy(b200tts_speaker_encoder* h);
size_t b200tts_speaker_encoder_workspace_bytes(const b200tts_speaker_encoder* h, int B, int T);
int b200tts_speaker_encoder_forward(const b200tts_speaker_encoder* h, const float* x, const int32_t* starts, int B,
                                    int T, int groups, int l2_norm, float* emb, void* workspace, size_t workspace_bytes,
                                    void* stream);
int b200tts_speaker_encoder_features(const b200tts_speaker_encoder* h, const float* x, const int32_t* starts, int B,
                                     int T, int stage, float* out, void* workspace, size_t workspace_bytes,
                                     void* stream);

/* ---- Glow-TTS inference (text -> mel spectrogram) ----------------------------------------------
 * Replaces GlowTTS.inference, TTS/tts/models/glow_tts.py:342-374, for encoder_type "rel_pos_transformer" (no
 * relative-position window, layer_norm_type "1": LayerNorm over channels with eps 1e-4), in two calls around the one
 * host read of the decoder length: encode (encoder + durations), then decode (path, prior, Glow decoder in reverse).
 * weights (host, PyTorch layouts, weight norm folded), state-dict order:
 *   encoder.emb.weight [n_vocab, H]
 *   if use_prenet: 3 x (prenet.conv_layers.i.w [H,H,5], .b, prenet.norm_layers.i.gamma [H], .beta), prenet.proj.w [H,H,1], .b
 *   per transformer layer: conv_q.w [H,H,1], .b, conv_k.w, .b, conv_v.w, .b, conv_o.w, .b, norm_layers_1.gamma [H],
 *     .beta, ffn.conv_1.w [F,H,k], .b, ffn.conv_2.w [H,F,k], .b, norm_layers_2.gamma, .beta
 *   proj_m.w [C,H,1], .b, (unless mean_only) proj_s.w [C,H,1], .b
 *   duration_predictor: conv_1.w [Fdp, H+c_in, 3], .b, norm_1.gamma [Fdp], .beta, conv_2.w [Fdp,Fdp,3], .b,
 *     norm_2.gamma, .beta, proj.w [1,Fdp,1], .b
 *   per decoder block n (flows 3n, 3n+1, 3n+2; Cs = C * num_squeeze, ns = num_splits):
 *     ActNorm logs [Cs], bias [Cs]; the INVERSE of InvConvNear.weight [ns, ns] (torch.inverse(weight.float()), as
 *     store_inverse computes it); start.w [Hd, Cs/2, 1], .b; WaveNet (cond_layer.w, .b if c_in_channels, then per layer
 *     in_layers.i.w [2Hd,Hd,k], .b, res_skip_layers.i.w, .b); end.w [Cs, Hd, 1], .b
 * encode: tokens int64 [B,Tt], lengths int64 [B], g [B, c_in_channels] (the l2-normalised speaker vector) or NULL ->
 *   o_stats [B, 2C, Tt] (o_mean rows [0,C), o_log_scale rows [C,2C)), logw [B,Tt] (durations_log), x_mask [B,Tt],
 *   w_ceil [B,Tt], cum [B,Tt] (cumulative w_ceil), dur_log [B,Tt] (total_durations_log), y_lengths int64 [B],
 *   meta int64 [2] = {max_b y_lengths, 0}: read it to size the decode call (Ty = meta[0]).
 * decode: noise [B,C,Ty] (the randn_like(y_mean) draw of :361) or NULL (= noise_scale 0) ->
 *   attn [B,Tt,Ty] (or NULL), y_mean / y_log_scale [B,C,Ty], mel [B, C, Ty'] with Ty' = num_squeeze * (Ty / num_squeeze)
 *   (the reference's model_outputs before its transpose to [B, Ty', C]).
 * workspace_bytes(B, Tt, Ty) covers both calls.  No float atomics: repeat calls are bit-identical.
 */
typedef struct {
    int n_vocab;
    int out_channels;          /* mel channels C */
    int hidden_channels_enc;   /* H */
    int hidden_channels_ffn;   /* F */
    int num_heads;
    int num_layers_enc;
    int kernel_size_enc;       /* transformer FFN kernel */
    int use_prenet;
    int mean_only;
    int hidden_channels_dp;    /* Fdp */
    int c_in_channels;         /* speaker vector size, 0: single speaker */
    int hidden_channels_dec;   /* Hd */
    int kernel_size_dec;
    int dilation_rate;
    int num_flow_blocks;
    int num_block_layers;
    int num_splits;
    int num_squeeze;
    int sigmoid_scale;
} b200tts_glow_tts_config;
typedef struct b200tts_glow_tts b200tts_glow_tts;
int b200tts_glow_tts_create(const b200tts_glow_tts_config* cfg, const float* const* weights, int num_weights,
                            b200tts_glow_tts** out);
void b200tts_glow_tts_destroy(b200tts_glow_tts* h);
size_t b200tts_glow_tts_workspace_bytes(const b200tts_glow_tts* h, int B, int Tt, int Ty);
int b200tts_glow_tts_encode(const b200tts_glow_tts* h, const int64_t* tokens, const int64_t* lengths, const float* g,
                            float length_scale, int B, int Tt, float* o_stats, float* logw, float* x_mask, float* w_ceil,
                            float* cum, float* dur_log, int64_t* y_lengths, int64_t* meta, void* workspace,
                            size_t workspace_bytes, void* stream);
int b200tts_glow_tts_decode(const b200tts_glow_tts* h, const float* o_stats, const float* x_mask, const float* cum,
                            const int64_t* y_lengths, const float* g, const float* noise, float noise_scale, int B, int Tt,
                            int Ty, float* attn, float* y_mean, float* y_log_scale, float* mel, void* workspace,
                            size_t workspace_bytes, void* stream);

/* ---- ForwardTTS inference (FastPitch / FastSpeech / FastSpeech2: text -> mel spectrogram) ----------------------------
 * Replaces ForwardTTS.inference, TTS/tts/models/forward_tts.py:672-714, for encoder_type and decoder_type "fftransformer"
 * (FFTransformerBlock, TTS/tts/layers/generic/transformer.py:6-69), in two calls around the one host read of the
 * decoder length: encode (:685-704: encoder, speaker add, duration / pitch / energy predictors, format_durations
 * :353-372), then decode (:417-451: generate_path, expansion, positional encoding :generic/pos_encoding.py:38-69,
 * FFTransformerDecoder :feed_forward/decoder.py:117-122).
 * Batched, unlike the reference (whose inference takes x_lengths = [T], :686): row b computes the reference's
 * inference(x[b:b+1, :lengths[b]]).  Padded tokens get 0 frames; keys, conv inputs and outputs stop at each row's length.
 * weights (host, PyTorch layouts), in this order:
 *   emb.weight [n_vocab, C]
 *   per encoder layer: self_attn.in_proj_weight [3C, C] (rows q|k|v), in_proj_bias [3C], out_proj.weight [C, C], .bias,
 *     conv1.w [Fe, C, 3], .b, conv2.w [C, Fe, 3], .b, norm1.weight [C], .bias, norm2.weight, .bias
 *   if proj_g_in > 0: proj_g.weight [C, proj_g_in], .bias [C]            (nn.Linear, :303)
 *   duration_predictor: conv_1.w [Fd, C, k], .b, norm_1.gamma, .beta, conv_2.w, .b, norm_2.gamma, .beta, proj.w, .b
 *   if use_pitch: pitch_predictor (same 10 tensors), pitch_emb.w [C, 1, kp], .b
 *   if use_energy: energy_predictor (same 10 tensors), energy_emb.w [C, 1, ke], .b
 *   if pe_len > 0: pos_encoder.pe [C, pe_len]
 *   per decoder layer: the 12 tensors of an encoder layer (Fdec channels in the FFN)
 *   decoder.postnet.w [out_channels, C, 1], .b
 * encode: tokens int64 [B,Tt], lengths int64 [B], g [B, C] (emb_g row or d-vector) or [B, proj_g_in] (d-vector to
 *   project) or NULL -> o_en [B, C, Tt] (encoder output + g, + pitch / energy embeddings), logw [B,Tt] (durations_log),
 *   pitch / energy [B,Tt] (NULL without the predictor), x_mask [B,Tt], dur [B,Tt] (frames per token), cum [B,Tt],
 *   y_lengths int64 [B], meta int64 [2] = {max_b y_lengths, min_b y_lengths}: read it to size the decode call
 *   (Ty = meta[0]).
 * decode: attn [B, Ty, Tt] (the returned alignments; or NULL), mel [B, Ty, out_channels] (model_outputs, zero past each
 *   row's y_length).  Ty > pe_len is an error, as in PositionalEncoding.forward.
 * No float atomics: repeat calls are bit-identical.
 */
typedef struct {
    int n_vocab;
    int hidden_channels;       /* C */
    int out_channels;
    int enc_heads, enc_layers, enc_ffn;
    int dec_heads, dec_layers, dec_ffn;
    int proj_g_in;             /* d-vector width projected by proj_g, 0: g (if any) is added as given */
    int dp_hidden, dp_kernel;
    int use_pitch, pitch_hidden, pitch_kernel, pitch_emb_kernel;
    int use_energy, energy_hidden, energy_kernel, energy_emb_kernel;
    int pe_len;                /* columns of pos_encoder.pe, 0: no positional encoding (and no sqrt(C) scale) */
} b200tts_forward_tts_config;
typedef struct b200tts_forward_tts b200tts_forward_tts;
int b200tts_forward_tts_create(const b200tts_forward_tts_config* cfg, const float* const* weights, int num_weights,
                               b200tts_forward_tts** out);
void b200tts_forward_tts_destroy(b200tts_forward_tts* h);
size_t b200tts_forward_tts_encode_workspace_bytes(const b200tts_forward_tts* h, int B, int Tt);
size_t b200tts_forward_tts_decode_workspace_bytes(const b200tts_forward_tts* h, int B, int Ty);
int b200tts_forward_tts_encode(const b200tts_forward_tts* h, const int64_t* tokens, const int64_t* lengths,
                               const float* g, float length_scale, int B, int Tt, float* o_en, float* logw, float* pitch,
                               float* energy, float* x_mask, float* dur, float* cum, int64_t* y_lengths, int64_t* meta,
                               void* workspace, size_t workspace_bytes, void* stream);
int b200tts_forward_tts_decode(const b200tts_forward_tts* h, const float* o_en, const float* x_mask, const float* cum,
                               const int64_t* y_lengths, int B, int Tt, int Ty, float* attn, float* mel, void* workspace,
                               size_t workspace_bytes, void* stream);

/* ---- SpeedySpeech inference (ForwardTTS with encoder_type and decoder_type "residual_conv_bn") ------------------------
 * The same inference as above, with ResidualConv1dBNEncoder (TTS/tts/layers/feed_forward/encoder.py:41-73) and
 * ResidualConv1dBNDecoder (decoder.py:125-160) in place of the FFTransformer stacks.  Their layer is Conv1dBN
 * (generic/res_conv_bn.py:18-46): an unpadded conv with kernel k and dilation d whose output is zero padded by
 * floor(d (k - 1) / 2) columns in front and the rest behind, then ReLU, then BatchNorm (eps 1e-5).  A row needs more than
 * d (k - 1) columns in every such layer, as in the reference; meta[1] of encode is the shortest row's frame count.
 * The handle is a b200tts_forward_tts: destroy, the workspace calls, encode and decode apply.  The encoder runs on the
 * exact FP32 conv, the decoder on 3xTF32 tensor-core convs from 128 frames on.
 * weights (host, PyTorch layouts; "bn" = BatchNorm1d weight, bias, running_mean, running_var [C], num_batches_tracked
 * left out), in this order:
 *   emb.weight [n_vocab, C]
 *   encoder.encoder: prenet.0.w [C, C, 1], .b; per res block, per conv: conv_bn_blocks.j.conv1d.w [C, C, enc_kernel], .b,
 *     conv_bn_blocks.j.norm (bn); postnet.0.w [C, C, 1], .b, postnet.2 (bn), postnet.3.w [C, C, 1], .b
 *   proj_g, the predictors and embeddings and pos_encoder.pe as for b200tts_forward_tts_create
 *   decoder.decoder: per res block, per conv: as in the encoder (dec_kernel); post_conv.w [C, C, 1], .b;
 *     postnet.0.conv_bn_blocks.{0,1}: conv1d.w [C, C, dec_kernel], .b, norm (bn); postnet.1.w [out_channels, C, 1], .b
 */
#define B200TTS_CONV_BN_MAX_BLOCKS 32
typedef struct {
    int n_vocab;
    int hidden_channels;       /* C */
    int out_channels;
    int enc_kernel, enc_blocks, enc_convs;              /* kernel size, residual blocks, convs per block */
    int enc_dilations[B200TTS_CONV_BN_MAX_BLOCKS];      /* one per residual block */
    int dec_kernel, dec_blocks, dec_convs;
    int dec_dilations[B200TTS_CONV_BN_MAX_BLOCKS];
    int proj_g_in;
    int dp_hidden, dp_kernel;
    int use_pitch, pitch_hidden, pitch_kernel, pitch_emb_kernel;
    int use_energy, energy_hidden, energy_kernel, energy_emb_kernel;
    int pe_len;
} b200tts_speedy_speech_config;
int b200tts_speedy_speech_create(const b200tts_speedy_speech_config* cfg, const float* const* weights, int num_weights,
                                 b200tts_forward_tts** out);

/* ---- self-attention on the tensor cores (ForwardTTS decoder) --------------------------------------------------------
 * Replaces nn.MultiheadAttention's attention core (softmax((q d^-1/2) k^T) v, torch/nn/functional.py
 * multi_head_attention_forward) over a fused [B, 3C, pitch] q|k|v tensor, per row over its first lens[b] (int32) frames.
 * out [B, C, pitch]; columns lens[b] .. pitch-1 are zeroed.  Heads need (C / num_heads) % 8 == 0 and <= 384.
 * T <= pitch bounds the rows' lengths (lens[b] <= T); columns of q|k|v at or past lens[b] are never read.
 */
int b200tts_attention_tc3(const float* qkv, const int* lens, int B, int C, int num_heads, int T, int pitch, float* out,
                          void* stream);

/* ---- MelGAN generators (plain, full-band, multi-band with PQMF synthesis) ---------------------------
 * Replaces MelganGenerator.forward (TTS/vocoder/models/melgan_generator.py:9-74, ResidualStack
 * TTS/vocoder/layers/melgan.py:6-36) and, for the multi-band generator, PQMF.synthesis (TTS/vocoder/layers/pqmf.py:50-53;
 * MultibandMelganGenerator.inference, multiband_melgan_generator.py:36-43).  Every conv with kernel > 1 reflect-pads
 * (nn.ReflectionPad1d); the leaky-ReLU slope is 0.2 everywhere, also before conv_post.  Upsampler s is
 * ConvTranspose1d(kernel 2u, stride u, padding u/2 + u%2, output_padding u%2), so every stage multiplies the length by u.
 * weights (host pointers, PyTorch layouts, weight norm folded), in this order:
 *   conv_pre.w [base, in, proj_kernel], conv_pre.b                                      (melgan_generator.py:32-35)
 *   for each upsample stage s (Cs = base / 2^(s+1)):
 *     ups[s].w [2 Cs, Cs, 2u] (ConvTranspose1d layout), ups[s].b                          (:43-57)
 *     for each residual block m: blocks[m][2].w [Cs, Cs, res_kernel] (dilation res_kernel^m), blocks[m][2].b,
 *                                blocks[m][4].w [Cs, Cs, 1], blocks[m][4].b, shortcuts[m].w [Cs, Cs, 1], shortcuts[m].b
 *                                                                                         (melgan.py:17-31)
 *   conv_post.w [out, Clast, proj_kernel], conv_post.b                                   (melgan_generator.py:66-70)
 *   G [1, pqmf_bands, pqmf_taps + 1]: the PQMF synthesis filter (pqmf.py:31), only if pqmf_bands > 0
 */
typedef struct {
    int in_channels, out_channels, base_channels, proj_kernel, res_kernel, num_res_blocks;
    int num_upsamples;
    int upsample_factors[8];
    int pqmf_bands; /* 0: no PQMF (plain / full-band); else out_channels must equal it */
    int pqmf_taps;  /* filter taps (62 in the reference; G has taps + 1) */
} b200tts_melgan_config;
typedef struct b200tts_melgan b200tts_melgan;
int b200tts_melgan_create(const b200tts_melgan_config* cfg, const float* const* weights, int num_weights,
                          b200tts_melgan** out);
void b200tts_melgan_destroy(b200tts_melgan* h);
size_t b200tts_melgan_workspace_bytes(const b200tts_melgan* h, int B, int T);
/* samples per row of the generator output (conv_post): T * prod(upsample_factors); the synthesised waveform of a
 * multi-band generator has pqmf_bands times as many */
int b200tts_melgan_out_len(const b200tts_melgan* h, int T);
/* x [B, in, T] -> out.  synthesize = 0: the generator output [B, out_channels, out_len(T)] (the band signals of a
 * multi-band generator: its forward()); synthesize = 1 (multi-band only): the PQMF-synthesised waveform
 * [B, 1, pqmf_bands * out_len(T) - pqmf_taps % 2].  peak_bits (nullable, zeroed by the caller) folds max|out| in, for
 * b200tts_to_int16.  Every reflect pad needs padding <= length - 1 at its layer (at least 28 columns at stage 0 with
 * 4 residual blocks); a shorter input returns status 1 before anything is launched. */
int b200tts_melgan_forward(const b200tts_melgan* h, const float* x, int B, int T, int synthesize, float* out,
                           uint32_t* peak_bits, void* workspace, size_t workspace_bytes, void* stream);

/* PQMF synthesis alone (TTS/vocoder/layers/pqmf.py:50-53): x [B, N, Tb] -> y [B, 1, N * Tb - taps % 2] (an odd tap
 * count loses one sample, as conv1d with padding taps / 2 does),
 *   y[n] = sum_k sum_j N G[0,k,j] x[k, (n + j - taps/2) / N]   (only integer indices inside [0, Tb): zero padding).
 * G: device [1, N, taps + 1].  peak_bits as above (nullable). */
int b200tts_pqmf_synthesis(const float* x, int B, int N, int Tb, const float* G, int taps, float* y, uint32_t* peak_bits,
                           void* stream);

/* ---- WaveGrad vocoder --------------------------------------------------------------------------------------------
 * Replaces Wavegrad.forward (TTS/vocoder/models/wavegrad.py:106-120; DBlock, FiLM, UBlock, PositionalEncoding:
 * TTS/vocoder/layers/wavegrad.py:19-154) and the body of the refinement loop of Wavegrad.inference (wavegrad.py:138-145).
 * Every conv zero-pads; F.interpolate is nearest (torch's index rule), the leaky-ReLU slope 0.2.  With n upsample
 * factors f_0 .. f_{n-1}: n - 1 DBlocks (DBlock i: factor f_{n-1-i}), n FiLMs, n UBlocks (UBlock j: factor f_j, dilations
 * upsample_dilations[j]).  hop = prod(f).  FiLM i runs at L[i], with L[0] = hop * T and L[i + 1] = L[i] / f_{n-1-i}.
 * weights (host pointers, PyTorch layouts, weight norm folded), in state-dict order:
 *   y_conv.w [yc, 1, 5], y_conv.b
 *   per DBlock i: res_block.w [oc, ic, 1], .b, main_block.{0,1,2}.w [oc, ic | oc, 3], .b
 *   per FiLM i:   input_conv.w [ic, ic, 3], .b, output_conv.w [2 oc, ic, 3], .b     (ic: yc, then dblock_out[i - 1];
 *                                                                                  oc: ublock_out[n - 1 - i])
 *   per UBlock j: res_block.w [hc, ic, 1], .b, main_block.{0,1}.w, .b, out_block.{0,1}.w, .b
 *   x_conv.w [xc, in, 3], x_conv.b, out_conv.w [1, ublock_out[n-1], 3], out_conv.b
 * pe, pe_frames (all calls): a host array of n device pointers; pe[i] = the [C_i, Lp[i]] table PositionalEncoding.pe / 5000
 * of FiLM i (built the way the reference builds it, C_i its input channels) for pe_frames >= T mel frames, Lp[i] being
 * L[i] at pe_frames: its row pitch.  So one set of tables, grown to the longest input, serves every shorter one, as the
 * reference's cache does.
 */
typedef struct {
    int in_channels, out_channels, y_conv_channels, x_conv_channels;
    int num_upsamples;                 /* n, 1 .. 8; out_channels must be 1 */
    int upsample_factors[8];
    int dblock_out_channels[8];        /* n - 1 used; dblock_out_channels[i] == ublock_out_channels[n - 1 - i] */
    int ublock_out_channels[8];        /* n used */
    int upsample_dilations[8][4];
} b200tts_wavegrad_config;
typedef struct b200tts_wavegrad b200tts_wavegrad;
int b200tts_wavegrad_create(const b200tts_wavegrad_config* cfg, const float* const* weights, int num_weights,
                            b200tts_wavegrad** out);
void b200tts_wavegrad_destroy(b200tts_wavegrad* h);
/* the true scratch size for [B, in, T] mel input: the conditioning x_conv(x), the n FiLM (shift, scale) tensors and five
 * stage tensors (each as large as the largest activation of the network) */
size_t b200tts_wavegrad_workspace_bytes(const b200tts_wavegrad* h, int B, int T);
/* Wavegrad.forward(y, x, noise_scale) (wavegrad.py:106-120): y [B, 1, hop T], x [B, in, T], noise_scale device [B]
 * -> eps [B, 1, hop T] */
int b200tts_wavegrad_forward(const b200tts_wavegrad* h, const float* y, const float* x, const float* noise_scale,
                             const float* const* pe, int pe_frames, int B, int T, float* eps, void* workspace,
                             size_t workspace_bytes, void* stream);
/* x_conv(x) (wavegrad.py:115) into the workspace, once per inference: the input is the same at every step */
int b200tts_wavegrad_condition(const b200tts_wavegrad* h, const float* x, int B, int T, void* workspace,
                               size_t workspace_bytes, void* stream);
/* one refinement step (wavegrad.py:139-145) on the conditioning condition() left in the same workspace, in place on y:
 *   y = clamp(c1 * (y - c2 * forward(y, x, noise_level)) + sigma * z, -1, 1)
 * noise_level: device [B]; z (nullable: the last step, no noise term) [B, 1, hop T].  The network output never reaches
 * memory (out_conv's epilogue applies the update); no host synchronisation. */
int b200tts_wavegrad_step(const b200tts_wavegrad* h, float* y, const float* noise_level, const float* const* pe,
                          int pe_frames, float c1, float c2, float sigma, const float* z, int B, int T, void* workspace,
                          size_t workspace_bytes, void* stream);

/* ---- Parallel WaveGAN generator ----------------------------------------------------------------------------------
 * Replaces ParallelWaveganGenerator.forward / .inference (TTS/vocoder/models/parallel_wavegan_generator.py:12-118;
 * ResidualBlock TTS/vocoder/layers/parallel_wavegan.py, ConvUpsample TTS/vocoder/layers/upsample.py) for the shapes
 * setup_generator builds: 1 noise channel in, 1 out, 64 residual / 128 gate / 64 skip channels, kernel 3, 80 mel
 * channels, no upsampler nonlinearity.  Layer l has dilation 2^(l % (num_res_blocks / stacks)).
 * The conditioning is folded: W_aux,l W_in (float64 at create) on the frame-rate mel, then the upsampler's linear map,
 * tabulated at create from unit impulses (float64), added inside each layer; the residual layers run on split-fp16
 * tensor cores (3 products, fp32 accumulation).
 * weights (host pointers, PyTorch layouts, weight norm folded), in state-dict order:
 *   first_conv.w [64, 1, 1], first_conv.b [64]
 *   upsample_net.conv_in.w [80, 80, 1]
 *   per upsample stage s: upsample_net.upsample.up_layers.(2s+1).w [1, 1, 1, 2 u_s + 1]
 *   per layer l: conv.w [128, 64, 3], conv.b [128], conv1x1_aux.w [128, 80, 1], conv1x1_out.w [64, 64, 1], .b,
 *                conv1x1_skip.w [64, 64, 1], .b
 *   last_conv_layers.1.w [64, 64, 1], .b, last_conv_layers.3.w [1, 64, 1], .b
 */
typedef struct {
    int num_res_blocks, stacks;        /* num_res_blocks % stacks == 0, at most 16 layers per stack */
    int num_upsamples;                 /* 1 .. 8 */
    int upsample_factors[8];           /* product at most 4096 */
} b200tts_pwgan_config;
typedef struct b200tts_pwgan b200tts_pwgan;
int b200tts_pwgan_create(const b200tts_pwgan_config* cfg, const float* const* weights, int num_weights,
                         b200tts_pwgan** out);
void b200tts_pwgan_destroy(b200tts_pwgan* h);
/* scratch for B rows of Tf frames (the length after the replicate pad) */
size_t b200tts_pwgan_workspace_bytes(const b200tts_pwgan* h, int B, int Tf);
/* the shortest padded input (frames) the upsampler tables are exact for; 5 or less for every factor list >= 2 */
int b200tts_pwgan_min_frames(const b200tts_pwgan* h);
/* mel [B, 80, T] (device, dense), replicate-padded by `pad` frames each side as read (0: forward(c), 2: inference(c));
 * noise [B, 1, Tf * P] (device; Tf = T + 2 pad, P = prod(upsample_factors)) -> out [B, 1, Tf * P].  Split-fp16 range:
 * a residual-layer activation with |x| >= 65504 makes the next launch on the device fail (once), as for the conv
 * engine's split-fp16 layers. */
int b200tts_pwgan_forward(const b200tts_pwgan* h, const float* mel, const float* noise, int B, int T, int pad, float* out,
                          void* workspace, size_t workspace_bytes, void* stream);
/* residual layer l alone, as b200tts_pwgan_forward runs it (0 <= l < num_res_blocks): the layer's conditioning from mel
 * [B, 80, T] (replicate-padded by `pad`), then x [B, 64, pitch] -> x_new [B, 64, pitch] (never the buffer x is) and
 * skip [B, 64, pitch] updated (layer 0 stores it; the last layer multiplies the sum by sqrt(1 / num_res_blocks)).  Only
 * columns [0, Tf * P) are read or written (Tf = T + 2 pad, pitch >= Tf * P); workspace: at least
 * b200tts_pwgan_workspace_bytes(h, B, Tf). */
int b200tts_pwgan_layer(const b200tts_pwgan* h, int layer, const float* mel, int B, int T, int pad, const float* x,
                        float* skip, float* x_new, int pitch, void* workspace, size_t workspace_bytes, void* stream);
/* the upsampler's linear map alone, as the layers apply it: a [rows, Tf] (device) -> out [rows, Tf * P] */
int b200tts_pwgan_upsample(const b200tts_pwgan* h, const float* a, int rows, int Tf, float* out, void* stream);

/* ---- UnivNet generator (vocoder) ----------------------------------------------------------------------------------
 * Replaces UnivnetGenerator.forward (TTS/vocoder/models/univnet_generator.py, LVCBlock / KernelPredictor in
 * TTS/vocoder/layers/lvc_block.py) on supplied noise.  Per block: the kernel predictor runs at frame rate on the conv
 * engine, kernel_conv | bias_conv as one split-fp16 tensor-core GEMM writing the kernels frame-major, the transposed
 * upsampler on the conv engine, and one fused split-fp16 tensor-core launch per LVC layer.  hidden_channels must be 32
 * and lvc_kernel_size 3; kpnet_hidden_channels a multiple of 16; kpnet_conv_size odd.
 * weights (host pointers, PyTorch layouts, weight norm folded):
 *   first_conv.w [32, in, 7], .b [32]
 *   per block n: upsample.w [32, 32, 2 u_n], .b [32]
 *                kernel_predictor.input_conv.0.w [Ch, cond, 5], .b
 *                kernel_predictor.residual_conv.{1,3,6,8,11,13}.w [Ch, Ch, Kp], .b   (six convs, in that order)
 *                kernel_predictor.kernel_conv.w [L * 32 * 64 * 3, Ch, Kp], .b
 *                kernel_predictor.bias_conv.w [L * 64, Ch, Kp], .b
 *                per layer i < L: convs.i.w [32, 32, 3], .b
 *   last_conv_layers.0.w [out, 32, 7], .b
 * (Ch = kpnet_hidden_channels, Kp = kpnet_conv_size, L = lvc_layers) */
typedef struct {
    int in_channels, out_channels, hidden_channels, cond_channels;
    int num_upsamples;                 /* 1 .. 8 */
    int upsample_factors[8];           /* product at most 4096 */
    int lvc_layers;                    /* lvc_layers_each_block, 1 .. 8 */
    int lvc_kernel_size;
    int kpnet_hidden_channels, kpnet_conv_size;
} b200tts_univnet_config;
typedef struct b200tts_univnet b200tts_univnet;
int b200tts_univnet_create(const b200tts_univnet_config* cfg, const float* const* weights, int num_weights,
                           b200tts_univnet** out);
void b200tts_univnet_destroy(b200tts_univnet* h);
/* scratch for B rows of T frames: one block's predicted kernels (B * T * L * 6208 floats) dominate */
size_t b200tts_univnet_workspace_bytes(const b200tts_univnet* h, int B, int T);
/* mel [B, cond, T], noise [B, in, T] (device, dense) -> out [B, out, T * prod(upsample_factors)].  Split-fp16 range: an
 * activation or predicted kernel with |v| >= 65504 makes the next launch on the device fail (once), as for the conv
 * engine's split-fp16 layers. */
int b200tts_univnet_forward(const b200tts_univnet* h, const float* mel, const float* noise, int B, int T, float* out,
                            void* workspace, size_t workspace_bytes, void* stream);
/* block `block`'s kernel predictor alone: mel [B, cond, T] -> pred [B * T][L * 6208] frame-major; per frame the kernels
 * [layer][co 64][tap * 32 + ci] (channel ((l * 32 + ci) * 64 + co) * 3 + tap of kernel_conv), then the biases
 * [layer][co 64].  Workspace: at least b200tts_univnet_workspace_bytes(h, B, T). */
int b200tts_univnet_predict(const b200tts_univnet* h, int block, const float* mel, int B, int T, float* pred,
                            void* workspace, size_t workspace_bytes, void* stream);
/* LVC layer `layer` of block `block` alone, as forward runs it: x [B, 32, pitch] (columns [0, T * hop_block) used) and
 * pred as b200tts_univnet_predict writes it -> x_new [B, 32, pitch] (never the buffer x is; only those columns are
 * written). */
int b200tts_univnet_lvc_layer(const b200tts_univnet* h, int block, int layer, const float* x, const float* pred, int B,
                              int T, float* x_new, int pitch, void* stream);

/* ---- Overflow / Neural-HMM inference (text -> mel spectrogram, autoregressive) ----------------------------------
 * Replaces Overflow.inference (TTS/tts/models/overflow.py:207-246) and NeuralhmmTTS.inference
 * (TTS/tts/models/neuralhmm_tts.py) in three calls:
 *   encode  - Encoder.inference (TTS/tts/layers/overflow/common_layers.py:70-92): embedding, 3 x ConvBNBlock
 *             (TTS/tts/layers/tacotron/tacotron2.py:11-44, eval BatchNorm folded into the conv), bidirectional nn.LSTM,
 *             the reshape to [B, Tt*spp, E]; plus the encoder-state part of the output net's first layer for every
 *             state (hoisted out of the loop: the loop only gathers the current state's column).
 *   sample  - NeuralHMM.inference / sample (TTS/tts/layers/overflow/neural_hmm.py:338-464): Prenet
 *             (tacotron/common_layers.py:63-120, prenet_type "original"), LSTMCell, Outputnet / ParameterModel
 *             (overflow/common_layers.py:95-219), EmissionModel.sample and the deterministic transition rule.  The loop
 *             runs chunk_frames frames per CUDA graph replay and reads 1 + B words after each chunk; no kernel waits on
 *             another block.
 *   decode  - Overflow only: Decoder (overflow/decoder.py:56-78, the Glow decoder in reverse) and inverse_normalize;
 *             for Neural-HMM (has_decoder 0) only inverse_normalize (neuralhmm_tts.py inference).
 * Batched, unlike the reference (whose Encoder.inference ignores x_lengths): row b computes the reference's
 * inference(text[b:b+1, :lengths[b]]).  Everything up to the decoder runs in FP32 on the FMA pipe, so the duration
 * decisions (thresholds on a running product) do not depend on tensor-core rounding.
 * weights (host, PyTorch layouts), in this order:
 *   encoder.emb.weight [n_vocab, E]
 *   per conv i < n_convs: convolution1d.weight [E, E, 5], .bias [E], batch_normalization.weight, .bias, .running_mean,
 *     .running_var [E] (eps 1e-5)
 *   encoder.lstm.weight_ih_l0 [4H, E], weight_hh_l0 [4H, H], bias_ih_l0, bias_hh_l0, then the same four _reverse
 *     (H = E / 2 * state_per_phone)
 *   neural_hmm.go_tokens [ar_order, 1]
 *   per prenet layer: linear_layer.weight [P, in] (in = C * ar_order for the first, P after; no bias)
 *   memory_rnn.weight_ih [4M, P], weight_hh [4M, M], bias_ih, bias_hh
 *   per output-net layer l: linear_layer.weight [O_l, in_l] (in_0 = M + E: columns [0, M) take h, [M, M + E) the state),
 *     .bias [O_l]; last_layer.weight [2C + 1, O_last], .bias
 *   mean [C], std [C] (a scalar buffer expanded to C)
 *   has_decoder: the Glow decoder blocks as for b200tts_glow_tts_config (no cond layer)
 */
typedef struct {
    int n_vocab;
    int encoder_dim;           /* E, even */
    int n_convs;               /* encoder conv blocks, <= 8 */
    int state_per_phone;       /* spp */
    int out_channels;          /* C (mel channels) */
    int ar_order;
    int prenet_dim;            /* P */
    int prenet_n_layers;       /* 1 .. 8 */
    int prenet_dropout;        /* 0: no dropout layer; else p = 0.5 where drop masks are given */
    int memory_rnn_dim;        /* M */
    int outputnet_n_layers;    /* 1 .. 8 */
    int outputnet_size[8];
    float std_floor;
    int has_decoder;           /* 1: Overflow (Glow decoder), 0: Neural-HMM */
    int hidden_channels_dec, kernel_size_dec, dilation_rate, num_flow_blocks, num_block_layers, num_splits, num_squeeze,
        sigmoid_scale;
} b200tts_overflow_config;
typedef struct b200tts_overflow b200tts_overflow;
int b200tts_overflow_create(const b200tts_overflow_config* cfg, const float* const* weights, int num_weights,
                            b200tts_overflow** out);
void b200tts_overflow_destroy(b200tts_overflow* h);
/* one workspace serves all three calls of an utterance batch: B rows of up to Tt tokens and up to F frames */
size_t b200tts_overflow_workspace_bytes(const b200tts_overflow* h, int B, int Tt, int F);
/* tokens int64 [B, Tt], lengths int64 [B] (1 .. Tt) -> states [B, Tt * spp, E] (zero past lengths[b] * spp); the
 * hoisted first-layer term stays in the workspace for sample() */
int b200tts_overflow_encode(const b200tts_overflow* h, const int64_t* tokens, const int64_t* lengths, int B, int Tt,
                            float* states, void* workspace, size_t workspace_bytes, void* stream);
/* the sampling loop on the state encode() left in the same workspace.  temp: sampling_temp (> 0: x = mean +
 * (std * temp) * noise); max_frames: max_sampling_time (>= 1); threshold: duration_threshold.  noise (nullable when
 * temp <= 0): device [B, max_frames, C] standard-normal draws; drop (nullable: no dropout): device uint8
 * [B, max_frames, prenet_n_layers, P], 1 keeps (x 2) and 0 drops a prenet unit.  Outputs: hmm_out [B, max_frames, C]
 * (zero past a row's frames), states_travelled int32 [B, max_frames + 1] (-1 past a row's frames + 1 entries),
 * frames (host int32 [B]): frames per row. */
int b200tts_overflow_sample(const b200tts_overflow* h, const int64_t* lengths, int B, int Tt, float temp, int max_frames,
                            float threshold, const float* noise, const uint8_t* drop, int chunk_frames, float* hmm_out,
                            int32_t* states_travelled, int32_t* frames, void* workspace, size_t workspace_bytes,
                            void* stream);
/* hmm_out [B, Fpitch, C] (as sample wrote it), frames device int32 [B], F = max frames -> mel [B, F', C]:
 * Overflow: F' = F floored to num_squeeze, each row's frames floored likewise, the decoder in reverse, x * std + mean
 * (padded frames come out as mean); Neural-HMM: F' = F, hmm_out * std + mean. */
int b200tts_overflow_decode(const b200tts_overflow* h, const float* hmm_out, const int32_t* frames, int B, int F,
                            int Fpitch, float* mel, void* workspace, size_t workspace_bytes, void* stream);

/* ---- Tacotron2 inference (text -> mel spectrogram, autoregressive attention decoder) -----------------------------
 * Replaces Tacotron2.inference (TTS/tts/models/tacotron2.py:238-300) in three calls:
 *   encode      - embedding + Encoder.inference (TTS/tts/layers/tacotron/tacotron2.py:105-112): 3 x ConvBNBlock (eval
 *                 BatchNorm folded), bidirectional nn.LSTM (256 per direction); for the original attention also
 *                 inputs_layer of every encoder output (step-invariant, hoisted out of the loop).
 *   decode_loop - Decoder.inference (tacotron2.py:329-367): Prenet (common_layers.py:63-119, no bias, "bn" folded),
 *                 attention LSTMCell (1024), OriginalAttention (location-sensitive or not, sigmoid or softmax norm) or
 *                 MonotonicDynamicConvolutionAttention (attentions.py), decoder LSTMCell (1024), linear_projection and
 *                 stopnet.  The loop runs chunk_steps steps per CUDA graph replay and reads 2 + B words after each chunk.
 *   postnet     - decoder_outputs + Postnet(decoder_outputs) (tacotron2.py:47-70), BatchNorm folded.
 * Batched, unlike the reference (which cannot batch): row b computes the reference's inference(text[b:b+1,
 * :lengths[b]]): attention, convolutions and the BiLSTM read only a row's tokens, the postnet only its frames, and the
 * stop rule is the one-row rule (a row stops after step t >= 1 once sigmoid(stop logit) > 0.5, or after max_steps
 * steps).  The loop runs in FP32 on the FMA pipe, so the stop decisions do not depend on tensor-core rounding.
 * Fixed widths (as the reference hard-codes them): embedding / encoder 512, attention RNN and decoder RNN 1024,
 * attention 128, prenet 256.
 * weights (host, PyTorch layouts), in this order:
 *   embedding.weight [n_vocab, 512]
 *   per encoder conv i < 3: convolution1d.weight [512, 512, 5], .bias, batch_normalization.weight, .bias,
 *     .running_mean, .running_var (eps 1e-5)
 *   encoder.lstm.weight_ih_l0 [1024, 512], weight_hh_l0 [1024, 256], bias_ih_l0, bias_hh_l0, then the four _reverse
 *   per prenet layer l < 2: linear_layer.weight [256, in] (in = C, then 256); prenet_bn: then batch_normalization.weight,
 *     .bias, .running_mean, .running_var
 *   attention_rnn.weight_ih [4096, 768], weight_hh [4096, 1024], bias_ih, bias_hh
 *   original attention: query_layer.linear_layer.weight [128, 1024], inputs_layer.linear_layer.weight [128, 512],
 *     v.linear_layer.weight [1, 128], .bias [1]; location_attn: location_conv1d.weight [32, 2, 31],
 *     location_dense.linear_layer.weight [128, 32]
 *   dynamic convolution: prior [11], query_layer.weight [128, 1024], .bias, key_layer.weight [168, 128],
 *     static_filter_conv.weight [8, 1, 21], static_filter_layer.weight [128, 8], dynamic_filter_layer.weight [128, 8],
 *     .bias, v.weight [1, 128]
 *   decoder_rnn.weight_ih [4096, 1536], weight_hh [4096, 1024], bias_ih, bias_hh
 *   linear_projection.linear_layer.weight [C * r_init, 1536], .bias; stopnet.1.linear_layer.weight
 *     [1, 1024 + C * r_init], .bias [1]
 *   per postnet conv i < 5: convolution1d.weight, .bias, batch_normalization.weight, .bias, .running_mean, .running_var
 */
typedef struct {
    int n_vocab;
    int out_channels;          /* C (mel channels) */
    int r_init;                /* linear_projection has C * r_init rows */
    int attention_type;        /* 0: "original", 1: "dynamic_convolution" */
    int location_attn;         /* original: location-sensitive */
    int attention_norm;        /* original: 0 sigmoid, 1 softmax */
    int prenet_bn;             /* prenet_type "bn" */
    int prenet_dropout;        /* 0: no dropout layer; else p = 0.5 where decode_loop is given masks */
} b200tts_tacotron2_config;
typedef struct b200tts_tacotron2 b200tts_tacotron2;
int b200tts_tacotron2_create(const b200tts_tacotron2_config* cfg, const float* const* weights, int num_weights,
                             b200tts_tacotron2** out);
void b200tts_tacotron2_destroy(b200tts_tacotron2* h);
/* one workspace serves all three calls of an utterance batch: B rows of up to Tt tokens and up to F mel frames */
size_t b200tts_tacotron2_workspace_bytes(const b200tts_tacotron2* h, int B, int Tt, int F);
/* tokens int64 [B, Tt], lengths int64 [B] (1 .. Tt) -> enc_out [B, Tt, 512] (zero past lengths[b]); the hoisted
 * inputs_layer term stays in the workspace for decode_loop() */
int b200tts_tacotron2_encode(const b200tts_tacotron2* h, const int64_t* tokens, const int64_t* lengths, int B, int Tt,
                             float* enc_out, void* workspace, size_t workspace_bytes, void* stream);
/* the decoder loop on encode()'s state in the same workspace.  r: reduction rate (1 .. r_init); max_steps: decoder
 * steps at most (>= 1); drop (nullable; used with prenet_dropout only): uint8 [B, max_steps, 2, 256], nonzero keeps a
 * unit (doubled), null runs the prenet without dropout;
 * chunk_steps: steps per graph replay (even).  Out (device, zero past each row): dec_out [B, max_steps * r, C],
 * stop_tokens [B, max_steps] (sigmoid values), alignments [B, max_steps, Tt]; steps (host int32 [B]): decoder steps per
 * row (frames = steps * r).  Synchronises the stream. */
int b200tts_tacotron2_decode_loop(const b200tts_tacotron2* h, const int64_t* lengths, const float* enc_out, int B,
                                  int Tt, int r, int max_steps, const uint8_t* drop, int chunk_steps, float* dec_out,
                                  float* stop_tokens, float* alignments, int32_t* steps, void* workspace,
                                  size_t workspace_bytes, void* stream);
/* dec_out [B, Fpitch, C], frames (device int32 [B]) -> mel [B, F, C] = dec_out + Postnet(dec_out) below frames[b],
 * zero past it */
int b200tts_tacotron2_postnet(const b200tts_tacotron2* h, const float* dec_out, const int32_t* frames, int B, int F,
                              int Fpitch, float* mel, void* workspace, size_t workspace_bytes, void* stream);

/* ---- Tacotron (1) inference (text -> spectrogram, autoregressive GRU attention decoder) ----------------------------
 * Replaces Tacotron.inference (TTS/tts/models/tacotron.py:218-271) in three calls:
 *   encode      - embedding (256) + Encoder (TTS/tts/layers/tacotron/tacotron.py:210-229): Prenet (Linear 256 -> 256 ->
 *                 128 with bias, ReLU, no dropout at inference) and the CBHG (K = 16, projections [128, 128]); for the
 *                 original attention also inputs_layer of every encoder output (step-invariant, hoisted out of the loop).
 *   decode_loop - Decoder.inference (tacotron.py:457-485): Prenet (256, 128, with bias, "bn" folded), attention GRUCell
 *                 (256), OriginalAttention or MonotonicDynamicConvolutionAttention, project_to_decoder_in, two residual
 *                 GRUCells (256), proj_to_mel and the stopnet.  chunk_steps steps per CUDA graph replay, 2 + B words
 *                 read after each chunk.
 *   postnet     - last_linear(PostCBHG(decoder_outputs)) (K = 8, projections [256, C], pre_highway when C != 128).
 * A CBHG's convs are BatchNormConv1d (no conv bias, eval BatchNorm with eps 1e-3 folded), padded [(k-1)/2, k/2].
 * Batched, unlike the reference: row b computes the reference's inference(text[b:b+1, :lengths[b]]): every conv sees
 * zeros past the row, the backward GRU starts at the row's last token or frame, outputs are zero past the row, and the
 * stop rule is the reference's: with n steps taken, stop once n > lengths[b] / 4 and (sigmoid(stop logit) > 0.6 or the
 * attention weight at token lengths[b] - 1 > 0.6), or once n > max_decoder_steps (so up to max_decoder_steps + 1 steps).
 * The loop runs in FP32 on the FMA pipe.
 * weights (host, PyTorch layouts), in this order (a CBHG: per bank conv k = 1..K conv1d.weight [128, Cin, k],
 * bn.weight, .bias, .running_mean, .running_var; the same five for each of the two projections; pre_highway.weight
 * [128, Cin] when Cin != 128; per highway H.weight, H.bias, T.weight, T.bias; gru weight_ih_l0 [384, 128],
 * weight_hh_l0 [384, 128], bias_ih_l0, bias_hh_l0, then the four _reverse):
 *   embedding.weight [n_vocab, 256]
 *   encoder.prenet layer l < 2: linear_layer.weight, .bias
 *   encoder CBHG (Cin 128, K 16, projections 128, 128)
 *   decoder prenet layer l < 2: linear_layer.weight [out, in] (in = frame_channels * memory_size with a memory queue,
 *     else frame_channels; then 256), .bias; prenet_bn: then batch_normalization.weight, .bias, .running_mean,
 *     .running_var (eps 1e-5)
 *   attention_rnn.weight_ih [768, 384], weight_hh [768, 256], bias_ih, bias_hh
 *   attention as b200tts_tacotron2 (query width 256, inputs_layer [128, 256])
 *   project_to_decoder_in.weight [256, 512], .bias
 *   decoder_rnns.{0,1}.weight_ih [768, 256], weight_hh [768, 256], bias_ih, bias_hh
 *   proj_to_mel.weight [C * r_init, 256], .bias; stopnet.linear.weight [1, 256 + C * r_init], .bias
 *   postnet CBHG (Cin C, K 8, projections 256, C)
 *   last_linear.weight [out_channels, 256], .bias
 */
typedef struct {
    int n_vocab;
    int frame_channels;        /* C: decoder_output_dim */
    int out_channels;          /* last_linear rows */
    int r_init;                /* proj_to_mel has C * r_init rows */
    int memory_size;           /* <= 0: the prenet reads the last frame; else a queue of memory_size frames */
    int attention_type;        /* 0: "original", 1: "dynamic_convolution" */
    int location_attn;         /* original: location-sensitive */
    int attention_norm;        /* original: 0 sigmoid, 1 softmax */
    int prenet_bn;             /* prenet_type "bn" */
    int prenet_dropout;        /* 0: no dropout layer; else p = 0.5 where decode_loop is given masks */
} b200tts_tacotron_config;
typedef struct b200tts_tacotron b200tts_tacotron;
int b200tts_tacotron_create(const b200tts_tacotron_config* cfg, const float* const* weights, int num_weights,
                            b200tts_tacotron** out);
void b200tts_tacotron_destroy(b200tts_tacotron* h);
/* one workspace serves all three calls of an utterance batch: B rows of up to Tt tokens and up to F frames */
size_t b200tts_tacotron_workspace_bytes(const b200tts_tacotron* h, int B, int Tt, int F);
/* tokens int64 [B, Tt], lengths int64 [B] (1 .. Tt) -> enc_out [B, Tt, 256] (zero past lengths[b]); the hoisted
 * inputs_layer term stays in the workspace for decode_loop() */
int b200tts_tacotron_encode(const b200tts_tacotron* h, const int64_t* tokens, const int64_t* lengths, int B, int Tt,
                            float* enc_out, void* workspace, size_t workspace_bytes, void* stream);
/* the decoder loop on encode()'s state in the same workspace.  r: reduction rate (1 .. r_init); max_steps:
 * max_decoder_steps (>= 1), so S = max_steps + 1 steps at most; drop (nullable; used with prenet_dropout only): uint8
 * [B, S, 2, 256] (layer 1 reads the first 128 of its 256), nonzero keeps a unit (doubled); chunk_steps: steps per graph
 * replay (even).  Out (device, zero past each row): dec_out [B, S * r, C], stop_tokens [B, S] (sigmoid values),
 * alignments [B, S, Tt]; steps (host int32 [B]): decoder steps per row (frames = steps * r).  Synchronises the
 * stream. */
int b200tts_tacotron_decode_loop(const b200tts_tacotron* h, const int64_t* lengths, const float* enc_out, int B, int Tt,
                                 int r, int max_steps, const uint8_t* drop, int chunk_steps, float* dec_out,
                                 float* stop_tokens, float* alignments, int32_t* steps, void* workspace,
                                 size_t workspace_bytes, void* stream);
/* dec_out [B, Fpitch, C], frames (device int32 [B]) -> out [B, F, out_channels] = last_linear(PostCBHG(dec_out)) below
 * frames[b], zero past it */
int b200tts_tacotron_postnet(const b200tts_tacotron* h, const float* dec_out, const int32_t* frames, int B, int F,
                             int Fpitch, float* out, void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TTS_B200_H */
