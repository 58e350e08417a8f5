// tts_b200 -- shared declarations for the sm_90a hot-path kernels.
// Host-side C++ here is the "engine" above the kernels; the only public surface is the
// C ABI in include/tts_b200.h (implemented in capi.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

namespace b200tts {

// ------------------------------------------------------------------ errors
void set_error(const char* fmt, ...);
const char* last_error();

#define B200_CUDA_OK(expr)                                                                  \
    do {                                                                                    \
        cudaError_t _e = (expr);                                                            \
        if (_e != cudaSuccess) {                                                            \
            ::b200tts::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr,              \
                                 cudaGetErrorString(_e));                                   \
            return 2;                                                                       \
        }                                                                                   \
    } while (0)

#define B200_REQUIRE(cond, ...)                                                             \
    do {                                                                                    \
        if (!(cond)) {                                                                      \
            ::b200tts::set_error(__VA_ARGS__);                                              \
            return 1;                                                                       \
        }                                                                                   \
    } while (0)

// ------------------------------------------------------------------ per-device one-time initialisation
// Function attributes (cudaFuncSetAttribute), device-side flags and the SM count belong to ONE device; the Python
// layer picks the device per tensor, so "done once per process" would leave a second GPU of the same process
// unconfigured.  State is keyed by cudaGetDevice() and set up under a mutex (handles may be shared across threads).
constexpr int MAX_DEVICES = 64;
struct DeviceOnce {
    std::mutex mu;
    std::atomic<bool> done[MAX_DEVICES];
    DeviceOnce() { for (auto& d : done) d.store(false); }
};
// Runs f(device) the first time it is called with a given current device; returns f's status (0 = ok) or 2.
template <class F>
inline int device_once(DeviceOnce& o, int* dev_out, F&& f) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= MAX_DEVICES) {
        set_error("device_once: cannot identify the current CUDA device");
        return 2;
    }
    if (dev_out) *dev_out = dev;
    if (o.done[dev].load(std::memory_order_acquire)) return 0;
    std::lock_guard<std::mutex> g(o.mu);
    if (o.done[dev].load(std::memory_order_relaxed)) return 0;
    if (int rc = f(dev)) return rc;
    o.done[dev].store(true, std::memory_order_release);
    return 0;
}

// launch accounting (bench.py reports "gpu_launches" from this counter)
extern unsigned long long g_launch_count;
inline void count_launch(int n = 1) { g_launch_count += (unsigned long long)n; }

// ------------------------------------------------------------------ conv1d implicit GEMM
// y[b, row, t] = epilogue( sum_ci sum_k W[row, ci, k] * prologue(x[b, ci, t + k*dil - pad]) )
//
// prologue : x *= xmask[b,t] (optional);  x = leaky_relu(x, in_slope)  (1.0 = identity)
// epilogue : v = acc + bias[row] + cond[b,row]
//            GATE      : rows come in (tanh,sigmoid) pairs -> v = tanh(v0)*sigmoid(v1), one output row per pair
//            act       : 0 none, 1 relu, 2 tanh
//            mask_pre  : v *= ymask[b,t]
//            res       : v += res[b,row,t]
//            scale     : v *= scale
//            accum     : v += y_old
//            post_div  : v /= post_div
//            mask_post : v *= ymask[b,t]
//            SPLIT (WN res/skip): rows <  split -> (y , accum=1, mask_post=1)
//                                 rows >= split -> (y2, accum=accum2, no mask), row index -= split
//            ups > 1 (polyphase transposed conv): row r -> channel r/ups, time q*ups + r%ups
//            launch_conv rejects what some kernel family would silently ignore: ymask without MASK_PRE / MASK_POST /
//            SPLIT, and GATE with ymask, another flag, a residual, an act, scale or post_div (no engine sends these)
//            WAVEGRAD (EPI_WAVEGRAD / ConvIO::near_src): v = acc + bias; [lrelu(v, act_param)]; [+ act_add[b]]; [+ res];
//                       [y2 <- v]; [v = shift + scale * v]; y <- v   (own kernel variants, see ConvIO)
enum : int { ACT_NONE = 0, ACT_RELU = 1, ACT_TANH = 2, ACT_LOGCLAMP = 3,   // LOGCLAMP: log(max(v, act_param))
             ACT_LRELU = 4 };                                             // LRELU: leaky ReLU, slope act_param (WaveGrad)
enum : int { EPI_GATE = 1, EPI_MASK_PRE = 2, EPI_MASK_POST = 4, EPI_ACCUM = 8, EPI_SPLIT = 16, EPI_ACCUM2 = 32,
             EPI_WAVEGRAD = 64 };

// ------------------------------------------------------------------ device memory
// Device buffers held by the engines, all made by upload() below.
inline std::atomic<long long> g_device_buffers{0};   // live DevBuf allocations (b200tts_debug_device_buffers)

// The owner of one device allocation: freed when the owner is destroyed or assigned over.  Move-only, so a struct
// holding DevBufs (a ConvLayer, an engine) cannot be copied and no buffer is freed twice.  Converts to T*, so kernel
// arguments take it as they would the raw pointer.
template <class T> class DevBuf {
  public:
    DevBuf() = default;
    DevBuf(DevBuf&& o) noexcept : p_(o.p_) { o.p_ = nullptr; }
    DevBuf& operator=(DevBuf&& o) noexcept {
        if (this != &o) { release(); p_ = o.p_; o.p_ = nullptr; }
        return *this;
    }
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { release(); }
    operator T*() const { return p_; }
    // replaces the buffer with n elements (n > 0); on failure the owner is left empty
    cudaError_t alloc(size_t n) {
        release();
        const cudaError_t e = cudaMalloc((void**)&p_, n * sizeof(T));
        if (e == cudaSuccess) g_device_buffers.fetch_add(1);
        else p_ = nullptr;
        return e;
    }
  private:
    void release() {
        if (!p_) return;
        cudaFree(p_);
        p_ = nullptr;
        g_device_buffers.fetch_sub(1);
    }
    T* p_ = nullptr;
};

// allocation + H2D copy (empty for n == 0)
template <class T> inline int upload(DevBuf<T>& dst, const T* src, size_t n) {
    dst = DevBuf<T>();
    if (n == 0) return 0;
    B200_REQUIRE(src, "upload: null host array of %zu elements", n);
    B200_CUDA_OK(dst.alloc(n));
    B200_CUDA_OK(cudaMemcpy(dst, src, n * sizeof(T), cudaMemcpyHostToDevice));
    return 0;
}

enum : int { TC_NONE = -1 };  // ConvLayer::tc_prec: no tensor-core images

struct ConvLayer {            // immutable after pack(); owned by an engine handle
    DevBuf<float> w;          // device, packed [row_tiles][CinPad][K][CO_T]
    DevBuf<float> bias;       // device, [RowsPad] (zeros when the layer has no bias)
    int Cin = 0, CinPad = 0;  // input channels (padded to the ci chunk)
    int Rows = 0, RowsPad = 0;  // GEMM rows (Cout, or Cout*ups for transposed conv; 2*H interleaved for gate)
    int K = 1, dil = 1, pad = 0;
    int ups = 1;              // >1: polyphase ConvTranspose1d
    int co_tile = 64;         // 32 or 64
    int tr_kernel = 0, tr_pad = 0, tr_outpad = 0;  // original transposed-conv kernel size / padding / output_padding (Tout)
    // tensor cores: set BEFORE packing to TC_NONE or the requested operand type (B200TTS_PRECISION_* other than TF32X3,
    // which is FP32 here); packing records the
    // type of the images it built (a 16-bit or split-fp16 request with Cin % 16 != 0 gets 3xTF32; no image: TC_NONE).  The text and
    // duration path requests none, so durations stay bit-stable on the exact FP32 FMA kernel.
    int tc_prec = TC_NONE;
    DevBuf<unsigned char> w_tc;   // device, plain image: [128-row tile][chunk][tap] blocks (rows >= 32), see pack_tc
    DevBuf<unsigned char> w_tcg;  // device, grouped image: [chunk][tap block] blocks (rows == 32 / 64), empty: none
    int tc_grp = 0;           // tap groups of the grouped image (128 / rows), 0: none
    DevBuf<float> tc_rscale;  // device, [Rows] 2^-e_r of the split-fp16 images (tc_prec == PREC_F16X3), else empty
};

// One [B][C][T] operand of a conv launch: element (b, c, t) is at p[b * bs + c * cs + t].  The pointer and its strides
// are set together (the only constructor that takes a pointer takes both strides), so no launch can give a tensor and
// forget a stride.  An InView is read and an OutView written; an OutView converts to an InView, not the other way.
// Views are trivially copyable: the kernels take them as arguments, inside the launch's ConvIO.
template <class T> struct View {
    T* p = nullptr; long long bs = 0; int cs = 0;
    View() = default;
    View(T* p_, long long bs_, int cs_) : p(p_), bs(bs_), cs(cs_) {}
    template <class U, std::enable_if_t<std::is_same_v<T, const U> && !std::is_const_v<U>, int> = 0>
    View(const View<U>& v) : p(v.p), bs(v.bs), cs(v.cs) {}   // InView from an OutView
    __host__ __device__ explicit operator bool() const { return p != nullptr; }
    // row c of batch b (element t of it is row(b, c)[t])
    __host__ __device__ T* row(int b, int c) const { return p + (long long)b * bs + (long long)c * cs; }
    // every row starts on a 16-byte boundary (whole float4 accesses along T)
    __host__ __device__ bool aligned16() const {
        return (cs & 3) == 0 && (bs & 3) == 0 && (reinterpret_cast<uintptr_t>(p) & 15) == 0;
    }
};
using InView = View<const float>;
using OutView = View<float>;
// the common case: a packed [B][C][pitch] tensor
inline OutView dense(float* p, int C, int pitch) { return {p, (long long)C * pitch, pitch}; }
inline InView dense(const float* p, int C, int pitch) { return {p, (long long)C * pitch, pitch}; }
// a per-batch vector, read only: a mask [B, 1, T] or a conditioning bias [B, RowsPad]; element (b, i) is at p[b * bs + i]
struct VecView {
    const float* p = nullptr; long long bs = 0;
    VecView() = default;
    VecView(const float* p_, long long bs_) : p(p_), bs(bs_) {}
    __host__ __device__ explicit operator bool() const { return p != nullptr; }
    __host__ __device__ const float* row(int b) const { return p + (long long)b * bs; }
};
static_assert(std::is_trivially_copyable_v<InView> && std::is_trivially_copyable_v<OutView> &&
              std::is_trivially_copyable_v<VecView>, "views are kernel arguments");

struct ConvIO {
    InView x; int Tin = 0;
    VecView xmask;
    float in_slope = 1.0f;
    VecView cond;   // [B, RowsPad-compatible] per-(b,row) bias
    OutView y; int Tout = 0;
    InView res;
    VecView ymask;
    OutView y2;
    int split = 0;
    float scale = 1.0f;
    float post_div = 1.0f;   // applied after accumulation (MRF mean: z_sum / num_kernels)
    int act = ACT_NONE;
    float act_param = 0.f;
    int flags = 0;
    int B = 1;
    unsigned* peak_bits = nullptr;   // single-row tanh kernel only: atomicMax of |y| (as float bits) over everything stored
    // ragged batch (null: dense).  lens[b] = valid FRAMES of row b; this launch's output is only computed below
    // lens[b] * rate_out + need_out (time steps of y; for a transposed conv `rate_out` counts GEMM columns, i.e. input
    // steps), its input is read as zero from lens[b] * rate_in + need_in on.  Honoured by the persistent tensor-core kernels
    // and the single-row kernel; the FMA tile kernel computes the full tensor (valid samples are identical either way).
    const int* lens = nullptr; int rate_out = 1, need_out = 0, rate_in = 1, need_in = 0;
    // column window (streaming decode): only GEMM columns [q_lo, q_hi) of y must be produced, and the input holds data
    // in columns [in_lo, in_hi) (outside is stale scratch, read as zero where a kernel reads past a conv's reach: the
    // grouped tensor-core mode's zero-padded taps).  Tiles stay on the full tensor's column grid, so every column inside
    // the window is computed exactly as by the unwindowed launch.  The defaults are the whole tensor.
    int q_lo = 0, q_hi = 0x7fffffff, in_lo = 0, in_hi = 0x7fffffff;
    // reflection padding (nn.ReflectionPad1d before the conv): an input column t outside [0, Tin) reads x[-t] (t < 0) or
    // x[2 Tin - 2 - t] (t >= Tin) instead of zero; no column outside [0, Tin) is ever read.  Needs pad <= Tin - 1; not
    // combined with lens, a column window or a transposed conv.
    int reflect = 0;
    // ---- WaveGrad variants (flags EPI_WAVEGRAD or near_src > 0; dense, unwindowed, ups 1, no masks).  They run on kernel
    // instantiations of their own, so every other launch compiles to the code it always did.
    // nearest resampling (F.interpolate(mode="nearest") of the input): the conv reads a virtual input of Tin columns whose
    // column t is x[nearest(t)], x holding near_src columns -- torch's rule: t when Tin == near_src, t >> 1 when
    // Tin == 2 near_src, else min(floor(t * (float)(near_src / Tin)), near_src - 1).  Covers the UBlock upsampling and the
    // DBlock decimation (t * f) without materialising the resampled tensor.  0: off.
    int near_src = 0;
    // FiLM (wavegrad.py shif_and_scale): v = shift + scale * v with shift = film[b, c, t] and scale = film[b, film_half + c,
    // t] (the two chunks of a FiLM output_conv tensor); y2 (nullable) receives v before it.  act_add (device [B], nullable):
    // added after the activation (the FiLM noise level).  With EPI_WAVEGRAD, act may be ACT_LRELU.
    InView film; int film_half = 0;
    const float* act_add = nullptr;
};

// Host weights in PyTorch layout.  conv: w[Cout][Cin][K];  transposed: w[Cin][Cout][Kt].
// gate_half > 0 interleaves rows (p, p+gate_half) for the fused WaveNet gate.
// in_perm / out_perm (nullable) remap logical->physical channels (flow channel flips).
int pack_conv(ConvLayer& L, const float* w, const float* bias, int Cout, int Cin, int K, int dil, int pad,
              int gate_half = 0, const int* in_perm = nullptr, const int* out_perm = nullptr);
int pack_conv_transpose(ConvLayer& L, const float* w, const float* bias, int Cin, int Cout, int Kt, int stride,
                        int padding, int output_padding = 0);
int launch_conv(const ConvLayer& L, const ConvIO& io, cudaStream_t stream);
// a 1x1 conv of one vector per batch row, [B, L.Cin] -> [B, L.Rows] with output rows y_pitch apart (the speaker and
// language conditioning projections); accum adds to y instead of overwriting it
inline int launch_conv_vec(const ConvLayer& L, const float* x, float* y, int y_pitch, int B, bool accum,
                           cudaStream_t stream) {
    ConvIO io;
    io.x = {x, L.Cin, 1}; io.Tin = 1;
    io.y = {y, y_pitch, 1}; io.Tout = 1; io.B = B;
    if (accum) io.flags = EPI_ACCUM;
    return launch_conv(L, io, stream);
}
int conv_tc_error_flag();
// one tensor-core weight image of logical weights Wl(r, ci, k) in the block layout of conv_tc3.cuh (see conv1d.cu);
// prec PREC_F16X3 also uploads the row scales 2^-e_r into *rscale (when it is still empty)
int pack_tc(DevBuf<unsigned char>& dst, const std::vector<float>& Wl, int rows, int Cin, int K, int prec, int G,
            DevBuf<float>* rscale = nullptr);
// the tensor-core state of the current device, set up on first use: the mapped error words ([0] pipeline timeout,
// [ERR_RANGE] split-fp16 range), the SM count and the opt-in shared memory per block.  Fails (once) when an earlier
// launch set one of the error words.
int tc_device(int** err, int* num_sms, size_t* max_smem);
// which kernel family a launch_conv call dispatched to (recorded per thread between dispatch_begin/end; tests pin it)
enum : int { DISPATCH_FMA = 0, DISPATCH_TC3 = 3, DISPATCH_TC3_GROUPED = 5, DISPATCH_ROW1 = 6,
             DISPATCH_TC16 = 8, DISPATCH_TC16_GROUPED = 9,    // TC16*: the same kernels with bf16 / fp16 operands
             // ForwardTTS decoder attention: the tensor-core kernel, or the FP32-FMA kernel for heads it does not take
             DISPATCH_ATTN_TC3 = 10, DISPATCH_ATTN_FMA = 11,
             // WaveGrad variants (EPI_WAVEGRAD / ConvIO::near_src): tensor cores by operand type, FMA tile; +1: resampled input
             DISPATCH_TC3W_TF32 = 12, DISPATCH_TC3W_F16X3 = 14, DISPATCH_FMA_WG = 16,
             // Overflow / Neural-HMM (overflow.cu): the BiLSTM time step, the LSTMCell, a GEMV layer, the frame epilogue
             DISPATCH_LSTM_BI = 18, DISPATCH_LSTM_CELL = 19, DISPATCH_HMM_LINEAR = 20, DISPATCH_HMM_STEP = 21,
             // Parallel WaveGAN (pwgan.cu): the fused residual layer, the folded conditioning conv
             DISPATCH_PWGAN_TC = 22, DISPATCH_PWGAN_AUX = 23,
             // Tacotron2 (taco_decoder.cu, tacotron2.cu): the attention step, the step epilogue; the LSTMCell with 32 rows per weight read
             DISPATCH_TACO_ATTN = 24, DISPATCH_TACO_STEP = 25, DISPATCH_LSTM_CELL32 = 26,
             // UnivNet (univnet.cu): the kernel-prediction GEMM, the fused LVC layer
             DISPATCH_UNIVNET_PREDICT = 27, DISPATCH_UNIVNET_LVC = 28,
             // Tacotron (tacotron.cu, recurrent.cu): the GRUCell (8 / 32 rows per weight read), the persistent biGRU,
             // the highway stack, the step epilogue
             DISPATCH_GRU_CELL = 29, DISPATCH_GRU_CELL32 = 30, DISPATCH_BIGRU = 31, DISPATCH_HIGHWAY = 32,
             DISPATCH_TACO1_STEP = 33,
             // Griffin-Lim (griffin_lim.cu): the magnitude preparation, one iteration, the deemphasis / output pass
             DISPATCH_GL_PREPARE = 34, DISPATCH_GL_ITER = 35, DISPATCH_GL_DEEMPHASIS = 36 };
void dispatch_begin();
int dispatch_end(int* ids, int cap);
void dispatch_note(int id);
inline int conv_transpose_out_len(const ConvLayer& L, int Tin) {
    return (Tin - 1) * L.ups - 2 * L.tr_pad + L.tr_kernel + L.tr_outpad;
}

// ------------------------------------------------------------------ bump allocator over a caller workspace
// Every engine lays its scratch out with one carve, a function of (Arena&, shape); its workspace size is arena_size over
// that same carve, so the layout is written once.  Blocks are 256-byte aligned.  ok() turns false at the first
// allocation that does not fit and stays false, so a carve is checked once, after its last allocation.
struct Arena {
    char* base; size_t cap; size_t off;
    bool good = true;
    Arena(void* p, size_t bytes) : base((char*)p), cap(bytes), off(0) {}
    // n raw bytes (a child component's workspace)
    void* bytes(size_t n) {
        const size_t b = (n + 255) & ~size_t(255);
        if (!good || off + b > cap) { good = false; return nullptr; }
        void* r = base + off;
        off += b;
        return r;
    }
    float* f32(size_t n) { return (float*)bytes(n * sizeof(float)); }
    bool ok() const { return good; }
};
// bytes an allocation sequence f(Arena&) takes from an Arena (a dry run over an unbounded one)
template <class F> size_t arena_size(F&& f) {
    Arena ar(nullptr, ~size_t(0) >> 1);
    f(ar);
    return ar.off;
}

// ------------------------------------------------------------------ cursor over an engine's weight list
// Every engine's init reads its flat weight list (order: include/tts_b200.h) front to back through one cursor, which its
// components take by reference, so the reads are the only description of the order.  Past the end take() returns null
// and keeps counting; whatever reads a taken pointer on the host refuses a null it cannot accept.  finish() then checks
// the list's length against the reads.
struct WeightList {
    const float* const* w; int n; int pos = 0;   // pos > n: the reads ran past the end
    WeightList(const float* const* list, int count) : w(list), n(count) {}
    const float* take() { const int i = pos++; return i < n ? w[i] : nullptr; }
    int finish(const char* who) const {
        B200_REQUIRE(pos <= n, "%s: the weight list ends after %d tensors; the config reads more", who, n);
        B200_REQUIRE(pos == n, "%s: expected %d weight tensors, got %d", who, pos, n);
        return 0;
    }
};

}  // namespace b200tts
