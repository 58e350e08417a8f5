// Recurrent building blocks shared by the autoregressive text-to-mel models (Overflow / Neural-HMM, Tacotron2, Tacotron):
// the Tacotron2-style text encoder (embedding, ConvBNBlocks, BiLSTM), the batch-amortised LSTM and GRU steps, the
// persistent bidirectional GRU, the GEMV layer with the prenet dropout, and the driver that runs an autoregressive loop
// as CUDA-graph chunks of steps.
// Everything is exact FP32 on the FMA pipe: the loops' stop decisions feed back through them, so they must not depend
// on tensor-core rounding.
#include <math.h>

#include <memory>
#include <type_traits>

#include "engines.cuh"

namespace b200tts {

namespace {

constexpr int UNITS = 8;          // LSTM units (4 gate rows each) or GEMV rows per 256-thread block: one per warp
constexpr int LIN_NB = 8;         // batch rows per block of the GEMV kernel
constexpr int STAGE = 12288;      // floats of staged input per block (48 KB): NB rows x STAGE / NB columns per chunk

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

template <int N>
__device__ __forceinline__ void warp_sum(float (&v)[N]) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int i = 0; i < N; ++i) v[i] += __shfl_xor_sync(0xffffffffu, v[i], o);
    }
}

// Stage O of the warp reduction of acc [NB][4]: the butterfly for O >= NB, else keep the half of the rows selected by
// lane bit O and add the partner's copy of it.
template <int O, int NB>
__device__ __forceinline__ void reduce_rows(float (&acc)[4 * NB], int lane) {
    if constexpr (O >= NB) {
#pragma unroll
        for (int i = 0; i < 4 * NB; ++i) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], O);
    } else {
        const bool up = (lane & O) != 0;
#pragma unroll
        for (int i = 0; i < 4 * O; ++i) {
            const float lo = acc[i], hi = acc[i + 4 * O];
            acc[i] = (up ? hi : lo) + __shfl_xor_sync(0xffffffffu, up ? lo : hi, O);
        }
    }
    if constexpr (O > 1) reduce_rows<O / 2, NB>(acc, lane);
}

// True when every batch row [b0, b0 + nb) of the block has finished (LSTMCell / GEMV mode): the whole block returns
// before it streams any weights, so steps after the last row stops cost no weight traffic.
__device__ __forceinline__ bool block_rows_done(const int* done, int b0, int nb) {
    if (!done) return false;
    for (int i = 0; i < nb; ++i)
        if (!done[b0 + i]) return false;
    return true;
}

// One LSTM time step for UNITS hidden units x NB batch rows per block; warp w owns unit j and its gate rows
// (i, f, g, o) = (j, H + j, 2H + j, 3H + j) of the torch layout.  The input is up to three segments read in place and
// staged through shared memory in chunks of STAGE / NB columns; lane l accumulates columns k = l (mod 32) of each
// segment in order, so a row's sums do not depend on NB.  The warp reduction is the xor butterfly, turned into a
// reduce-scatter below offset NB (the same pairs in the same order, so the same sums): lane l ends with row l % NB.
template <int NB>
__global__ void __launch_bounds__(256) lstm_kernel(LstmArgs a) {
    constexpr int KC = STAGE / NB;
    __shared__ float xs[NB * KC];
    const int H = a.H, d = blockIdx.y, b0 = blockIdx.z * NB, nb = min(NB, a.B - b0);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, j = blockIdx.x * UNITS + warp;
    if (!a.lens && block_rows_done(a.done, b0, nb)) return;
    float acc[4 * NB];   // [bb][g]
#pragma unroll
    for (int i = 0; i < 4 * NB; ++i) acc[i] = 0.f;
    for (int s = 0; s < a.nseg; ++s) {
        const LstmSeg& sg = a.seg[s];
        const float* W = sg.W + d * sg.w_ds;
        const float* x = sg.x + d * sg.x_ds;
        for (int k0 = 0; k0 < sg.K; k0 += KC) {
            const int kc = min(KC, sg.K - k0);
            __syncthreads();
            for (int i = threadIdx.x; i < nb * kc; i += blockDim.x) {
                const int bb = i / kc, k = i - bb * kc;
                xs[bb * KC + k] = x[(size_t)(b0 + bb) * sg.x_bs + k0 + k];
            }
            __syncthreads();
            if (j >= H) continue;
            for (int k = lane; k < kc; k += 32) {
                float w[4];
#pragma unroll
                for (int g = 0; g < 4; ++g) w[g] = W[(size_t)(g * H + j) * sg.ldw + k0 + k];
#pragma unroll
                for (int bb = 0; bb < NB; ++bb) {
                    const float xv = xs[(bb < nb ? bb : 0) * KC + k];
#pragma unroll
                    for (int g = 0; g < 4; ++g) acc[bb * 4 + g] = fmaf(w[g], xv, acc[bb * 4 + g]);
                }
            }
        }
    }
    if (j >= H) return;
    reduce_rows<16, NB>(acc, lane);
    if (lane >= nb) return;
    float gv[4] = {acc[0], acc[1], acc[2], acc[3]};
    const int b = b0 + lane;
    int t = 0;
    if (a.lens) {
        const int len = (int)a.lens[b];
        if (a.step >= len) return;
        t = d ? len - 1 - a.step : a.step;
#pragma unroll
        for (int g = 0; g < 4; ++g) gv[g] += a.pre[(size_t)b * a.pre_bs + (size_t)(d * 4 * H + g * H + j) * a.pre_cs + t];
    } else {
        if (a.done[b]) return;
#pragma unroll
        for (int g = 0; g < 4; ++g) gv[g] += a.bias[g * H + j];
    }
    float* cp = a.c + d * a.st_ds + (size_t)b * H + j;
    const float cn = sigmoidf_(gv[1]) * *cp + sigmoidf_(gv[0]) * tanhf(gv[2]);
    const float h = sigmoidf_(gv[3]) * tanhf(cn);
    *cp = cn;
    a.h_out[d * a.st_ds + (size_t)b * a.h_bs + j] = h;
    if (a.out) a.out[(size_t)b * a.out_bs + (size_t)t * a.out_ts + d * H + j] = h;
}

// Segment s of a GRU step: the (r, z, n) rows (j, H + j, 2H + j) of W times the staged columns, n into acc slot NS
// (2: the input part W_in x, 3: the hidden part W_hn h, which the n gate scales by r).
template <int NB, int NS>
__device__ __forceinline__ void gru_seg_fma(float (&acc)[4 * NB], const float* W, int ldw, int H, int j, int k0,
                                            const float* xs, int KC, int kc, int nb, int lane) {
    for (int k = lane; k < kc; k += 32) {
        float w[3];
#pragma unroll
        for (int g = 0; g < 3; ++g) w[g] = W[(size_t)(g * H + j) * ldw + k0 + k];
#pragma unroll
        for (int bb = 0; bb < NB; ++bb) {
            const float xv = xs[(bb < nb ? bb : 0) * KC + k];
            acc[bb * 4 + 0] = fmaf(w[0], xv, acc[bb * 4 + 0]);
            acc[bb * 4 + 1] = fmaf(w[1], xv, acc[bb * 4 + 1]);
            acc[bb * 4 + NS] = fmaf(w[2], xv, acc[bb * 4 + NS]);
        }
    }
}

// One GRUCell step for UNITS hidden units x NB batch rows per block, batch-amortised as lstm_kernel: warp w owns unit j,
// segments [0, nin) are the input x and the rest the hidden state h, lane l sums columns l (mod 32) of each segment in
// order, and the same reduction leaves lane l with row l % NB's four sums (r, z, n_x, n_h).
//   r = sig(sum_r + b_r), z = sig(sum_z + b_z), n = tanh(n_x + b_in + r (n_h + b_hn)), h' = (1 - z) n + z h
template <int NB>
__global__ void __launch_bounds__(256) gru_kernel(GruArgs a) {
    constexpr int KC = STAGE / NB;
    __shared__ float xs[NB * KC];
    const int H = a.H, b0 = blockIdx.z * NB, nb = min(NB, a.B - b0);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, j = blockIdx.x * UNITS + warp;
    if (block_rows_done(a.done, b0, nb)) return;
    float acc[4 * NB];   // [bb][r, z, n_x, n_h]
#pragma unroll
    for (int i = 0; i < 4 * NB; ++i) acc[i] = 0.f;
    for (int s = 0; s < a.nseg; ++s) {
        const LstmSeg& sg = a.seg[s];
        for (int k0 = 0; k0 < sg.K; k0 += KC) {
            const int kc = min(KC, sg.K - k0);
            __syncthreads();
            for (int i = threadIdx.x; i < nb * kc; i += blockDim.x) {
                const int bb = i / kc, k = i - bb * kc;
                xs[bb * KC + k] = sg.x[(size_t)(b0 + bb) * sg.x_bs + k0 + k];
            }
            __syncthreads();
            if (j >= H) continue;
            if (s < a.nin) gru_seg_fma<NB, 2>(acc, sg.W, sg.ldw, H, j, k0, xs, KC, kc, nb, lane);
            else gru_seg_fma<NB, 3>(acc, sg.W, sg.ldw, H, j, k0, xs, KC, kc, nb, lane);
        }
    }
    if (j >= H) return;
    reduce_rows<16, NB>(acc, lane);
    if (lane >= nb) return;
    const int b = b0 + lane;
    if (a.done[b]) return;
    const float r = sigmoidf_(acc[0] + a.bias[j]);
    const float z = sigmoidf_(acc[1] + a.bias[H + j]);
    const float n = tanhf(acc[2] + a.bias[2 * H + j] + r * (acc[3] + a.bias[3 * H + j]));
    const float h = (1.f - z) * n + z * a.h_in[(size_t)b * a.hin_bs + j];
    a.h_out[(size_t)b * a.h_bs + j] = h;
    if (a.x_out) a.x_out[(size_t)b * a.xo_bs + j] = h + a.res[(size_t)b * a.res_bs + j];
}

// A whole bidirectional GRU layer (H = 128) in one launch: CTA (b, d) runs direction d of row b over its len_b steps
// (forward t = s, backward t = len_b - 1 - s) with W_hh resident in shared memory for the whole sequence.  Thread
// tid = 4 j + q owns unit j and the columns k = 4 i + q (i < 32) of its three W_hh rows, stored at [(g * 32 + i) * 512 +
// tid] so a warp reads 32 consecutive words; h is double-buffered in shared memory, so a step has one barrier.  The
// four partial sums of a row are combined by the xor butterfly (the same two pairs in the same order for every row).
// Past len_b the row's outputs are zero.
__global__ void __launch_bounds__(BIGRU_THREADS, 1) bigru_kernel(BiGruArgs a) {
    extern __shared__ float sm[];
    float* Ws = sm;                              // [3 * 32][512]
    float* hs = sm + 3 * 32 * BIGRU_THREADS;     // [2][128]
    const int b = blockIdx.x, d = blockIdx.y, tid = threadIdx.x, j = tid >> 2, q = tid & 3;
    const int len = a.lens64 ? (int)a.lens64[b] : a.lens32[b];
    {
        const float4* src = reinterpret_cast<const float4*>(a.whh + (size_t)d * 3 * 32 * BIGRU_THREADS);
        float4* dst = reinterpret_cast<float4*>(Ws);
        for (int i = tid; i < 3 * 32 * BIGRU_THREADS / 4; i += BIGRU_THREADS) dst[i] = src[i];
    }
    if (tid < 2 * GRU_H) hs[tid] = 0.f;
    float* out = a.out + (size_t)b * a.out_bs + (size_t)(d * GRU_H) * a.out_cs;
    for (int i = tid; i < (a.T - len) * GRU_H; i += BIGRU_THREADS) {
        const int t = len + i / GRU_H, c = i % GRU_H;
        out[(size_t)t * a.out_ts + (size_t)c * a.out_cs] = 0.f;
    }
    const float bhn = a.bhn[d * GRU_H + j];
    const float* pre = a.pre + (size_t)b * a.pre_bs + (size_t)(d * 3 * GRU_H + j) * a.pre_cs;
    float pr = 0.f, pz = 0.f, pn = 0.f;
    if (q == 0 && len > 0) {
        const int t = d ? len - 1 : 0;
        pr = pre[t]; pz = pre[(size_t)GRU_H * a.pre_cs + t]; pn = pre[(size_t)2 * GRU_H * a.pre_cs + t];
    }
    __syncthreads();
    for (int s = 0; s < len; ++s) {
        const int t = d ? len - 1 - s : s;
        const float* hc = hs + (s & 1) * GRU_H;
        float* hn = hs + ((s & 1) ^ 1) * GRU_H;
        float npr = 0.f, npz = 0.f, npn = 0.f;   // the next step's input projection, loaded under this step's sums
        if (q == 0 && s + 1 < len) {
            const int tn = d ? t - 1 : t + 1;
            npr = pre[tn]; npz = pre[(size_t)GRU_H * a.pre_cs + tn]; npn = pre[(size_t)2 * GRU_H * a.pre_cs + tn];
        }
        float ar = 0.f, az = 0.f, an = 0.f;
#pragma unroll 8
        for (int i = 0; i < 32; ++i) {
            const float hv = hc[4 * i + q];
            ar = fmaf(Ws[(0 * 32 + i) * BIGRU_THREADS + tid], hv, ar);
            az = fmaf(Ws[(1 * 32 + i) * BIGRU_THREADS + tid], hv, az);
            an = fmaf(Ws[(2 * 32 + i) * BIGRU_THREADS + tid], hv, an);
        }
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
            ar += __shfl_xor_sync(0xffffffffu, ar, o);
            az += __shfl_xor_sync(0xffffffffu, az, o);
            an += __shfl_xor_sync(0xffffffffu, an, o);
        }
        if (q == 0) {
            const float r = sigmoidf_(pr + ar), z = sigmoidf_(pz + az);
            const float n = tanhf(pn + r * (an + bhn));
            const float h = (1.f - z) * n + z * hc[j];
            hn[j] = h;
            out[(size_t)t * a.out_ts + (size_t)j * a.out_cs] = h;
        }
        pr = npr; pz = npz; pn = npn;
        __syncthreads();
    }
}

// y[b, r] = act(W[r] . [x | x2][b] + bias[r] + add[b, r, state[b]]), then the prenet dropout (drop[b, f, layer, r] ?
// 2v : 0 with f the loop's step counter ctl[1]); rows that are done skip.  One warp per row r, LIN_NB batch rows per
// block; the input is staged in chunks of STAGE / LIN_NB columns (lane l sums columns l (mod 32) in order).
__global__ void __launch_bounds__(256) linear_kernel(LinArgs a) {
    constexpr int KC = STAGE / LIN_NB;
    __shared__ float xs[LIN_NB * KC];
    const int b0 = blockIdx.y * LIN_NB, nb = min(LIN_NB, a.B - b0);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, r = blockIdx.x * UNITS + warp;
    const int K = a.K + a.K2;
    if (block_rows_done(a.done, b0, nb)) return;
    float acc[LIN_NB];
#pragma unroll
    for (int i = 0; i < LIN_NB; ++i) acc[i] = 0.f;
    const float* w = a.W + (size_t)r * K;
    for (int k0 = 0; k0 < K; k0 += KC) {
        const int kc = min(KC, K - k0);
        __syncthreads();
        for (int i = threadIdx.x; i < nb * kc; i += blockDim.x) {
            const int bb = i / kc, k = k0 + i - bb * kc;
            xs[bb * KC + k - k0] = k < a.K ? a.x[(size_t)(b0 + bb) * a.x_bs + k]
                                           : a.x2[(size_t)(b0 + bb) * a.x2_bs + k - a.K];
        }
        __syncthreads();
        if (r >= a.R) continue;
        for (int k = lane; k < kc; k += 32) {
            const float wv = w[k0 + k];
#pragma unroll
            for (int bb = 0; bb < LIN_NB; ++bb) acc[bb] = fmaf(wv, xs[(bb < nb ? bb : 0) * KC + k], acc[bb]);
        }
    }
    if (r >= a.R) return;
    warp_sum(acc);
    float v = 0.f;
#pragma unroll
    for (int bb = 0; bb < LIN_NB; ++bb)
        if (lane == bb) v = acc[bb];
    if (lane >= nb) return;
    const int b = b0 + lane;
    if (a.done[b]) return;
    if (a.bias) v += a.bias[r];
    if (a.add) v += a.add[(size_t)b * a.add_bs + (size_t)r * a.add_rs + a.state[b]];
    if (a.relu) v = fmaxf(v, 0.f);
    if (a.drop) {
        const int f = a.ctl[1];
        v = a.drop[(((size_t)b * a.drop_F + f) * a.drop_L + a.drop_layer) * a.R + r] ? v * 2.f : 0.f;
    }
    a.y[(size_t)b * a.y_bs + r] = v;
}

// y[b, c, n] = x[b, n, c]
__global__ void transpose_kernel(const float* x, float* y, int N, int E) {
    __shared__ float tile[32][33];
    const int b = blockIdx.z, n0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int n = n0 + i, c = c0 + threadIdx.x;
        tile[i][threadIdx.x] = (n < N && c < E) ? x[((size_t)b * N + n) * E + c] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int c = c0 + i, n = n0 + threadIdx.x;
        if (n < N && c < E) y[((size_t)b * E + c) * N + n] = tile[threadIdx.x][i];
    }
}

}  // namespace

int launch_lstm(const LstmArgs& a, int dirs, int rows_per_block, int dispatch_id, cudaStream_t st, bool note) {
    B200_REQUIRE(a.nseg >= 1 && a.nseg <= 3 && a.H > 0 && a.B >= 1, "lstm: bad arguments");
    const int nb = rows_per_block;
    dim3 grid((a.H + UNITS - 1) / UNITS, dirs, (a.B + nb - 1) / nb);
    switch (nb) {
        case 8: lstm_kernel<8><<<grid, 256, 0, st>>>(a); break;
        case 32: lstm_kernel<32><<<grid, 256, 0, st>>>(a); break;
        default: set_error("lstm: rows_per_block must be 8 or 32, got %d", nb); return 1;
    }
    count_launch();
    if (note) dispatch_note(dispatch_id);
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

int launch_gru(const GruArgs& a, int rows_per_block, cudaStream_t st, bool note) {
    B200_REQUIRE(a.nseg >= 1 && a.nseg <= 3 && a.nin >= 1 && a.nin < a.nseg && a.H > 0 && a.B >= 1 && a.done &&
                 (!a.x_out || a.res), "gru: bad arguments");
    const int nb = rows_per_block;
    dim3 grid((a.H + UNITS - 1) / UNITS, 1, (a.B + nb - 1) / nb);
    switch (nb) {
        case 8: gru_kernel<8><<<grid, 256, 0, st>>>(a); break;
        case 32: gru_kernel<32><<<grid, 256, 0, st>>>(a); break;
        default: set_error("gru: rows_per_block must be 8 or 32, got %d", nb); return 1;
    }
    count_launch();
    if (note) dispatch_note(nb == 32 ? DISPATCH_GRU_CELL32 : DISPATCH_GRU_CELL);
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

int pack_bigru_whh(const float* whh, float* dst) {
    B200_REQUIRE(whh, "pack_bigru_whh: null W_hh");
    for (int g = 0; g < 3; ++g)
        for (int i = 0; i < 32; ++i)
            for (int t = 0; t < BIGRU_THREADS; ++t) {
                const int j = t >> 2, q = t & 3;
                dst[(size_t)(g * 32 + i) * BIGRU_THREADS + t] = whh[(size_t)(g * GRU_H + j) * GRU_H + 4 * i + q];
            }
    return 0;
}

int launch_bigru(const BiGruArgs& a, int B, cudaStream_t st) {
    B200_REQUIRE(a.pre && a.whh && a.bhn && a.out && (a.lens32 || a.lens64) && B >= 1 && a.T >= 1, "bigru: bad arguments");
    constexpr int smem = sizeof(float) * (3 * 32 * BIGRU_THREADS + 2 * GRU_H);
    static DeviceOnce once;
    if (int rc = device_once(once, nullptr, [](int) -> int {
            B200_CUDA_OK(cudaFuncSetAttribute(bigru_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
            return 0;
        }))
        return rc;
    bigru_kernel<<<dim3(B, 2), BIGRU_THREADS, smem, st>>>(a);
    count_launch();
    dispatch_note(DISPATCH_BIGRU);
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

int launch_linear(const LinArgs& a, cudaStream_t st, bool note) {
    B200_REQUIRE(a.R > 0 && a.K > 0 && a.B >= 1 && (a.K2 == 0 || a.x2), "linear: bad arguments");
    dim3 grid((a.R + UNITS - 1) / UNITS, (a.B + LIN_NB - 1) / LIN_NB);
    linear_kernel<<<grid, 256, 0, st>>>(a);
    count_launch();
    if (note) dispatch_note(DISPATCH_HMM_LINEAR);
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

int launch_transpose(const float* x, float* y, int B, int N, int E, cudaStream_t st) {
    dim3 grid((N + 31) / 32, (E + 31) / 32, B);
    transpose_kernel<<<grid, dim3(32, 8), 0, st>>>(x, y, N, E);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

// scoped owners of run_step_graph's capture stream, graph and executable graph
template <class H, cudaError_t (*destroy)(H)> struct CudaDestroy {
    void operator()(H h) const { destroy(h); }
};
template <class H, cudaError_t (*destroy)(H)>
using CudaOwned = std::unique_ptr<std::remove_pointer_t<H>, CudaDestroy<H, destroy>>;

int run_step_graph(const char* who, int chunk, int max_steps, int launches_per_step,
                   const std::function<int(cudaStream_t, int, bool)>& step, const int* ctl, int B, std::vector<int>& host,
                   cudaStream_t st) {
    cudaStream_t cs = nullptr;
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    B200_CUDA_OK(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
    const CudaOwned<cudaStream_t, cudaStreamDestroy> cs_owner(cs);
    int rc = 0;
    if (cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal) != cudaSuccess) {
        set_error("%s: cannot capture the step graph", who);
        return 2;
    }
    const unsigned long long launches = g_launch_count;   // captured launches are counted per replay below
    for (int f = 0; f < chunk && rc == 0; ++f) rc = step(cs, f & 1, f == 0);
    const cudaError_t ce = cudaStreamEndCapture(cs, &graph);
    g_launch_count = launches;
    const CudaOwned<cudaGraph_t, cudaGraphDestroy> graph_owner(graph);
    if (rc || ce != cudaSuccess) {
        if (!rc) set_error("%s: step graph capture failed: %s", who, cudaGetErrorString(ce));
        return rc ? rc : 2;
    }
    const cudaError_t ie = cudaGraphInstantiate(&exec, graph, 0);
    const CudaOwned<cudaGraphExec_t, cudaGraphExecDestroy> exec_owner(exec);
    if (ie != cudaSuccess) {
        set_error("%s: cannot instantiate the step graph: %s", who, cudaGetErrorString(ie));
        return 2;
    }
    // replay until no row runs: every row is done by step max_steps - 1, so steps past it do no work
    host.assign(2 + B, 0);
    for (int done_steps = 0; done_steps < max_steps; done_steps += chunk) {
        cudaError_t e = cudaGraphLaunch(exec, st);
        count_launch(launches_per_step * chunk);
        if (e == cudaSuccess) e = cudaMemcpyAsync(host.data(), ctl, sizeof(int) * (2 + B), cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) {
            set_error("%s: %s", who, cudaGetErrorString(e));
            return 2;
        }
        if (host[0] == 0) break;
    }
    return 0;
}

int fold_bn(WeightList& wl, bool has_bias, double eps, int Cout, size_t row, std::vector<float>& wf,
            std::vector<float>& bf) {
    const float* w = wl.take();
    const float* bias = has_bias ? wl.take() : nullptr;
    const float *gamma = wl.take(), *beta = wl.take(), *mean = wl.take(), *var = wl.take();
    B200_REQUIRE(w && (bias || !has_bias) && gamma && beta && mean && var, "fold_bn: null weight or BatchNorm tensor");
    wf.assign((size_t)Cout * row, 0.f);
    bf.assign(Cout, 0.f);
    for (int o = 0; o < Cout; ++o) {
        const double s = (double)gamma[o] / sqrt((double)var[o] + eps);
        for (size_t k = 0; k < row; ++k) wf[(size_t)o * row + k] = (float)(w[(size_t)o * row + k] * s);
        bf[o] = bias ? (float)(((double)bias[o] - mean[o]) * s + beta[o]) : (float)((double)beta[o] - mean[o] * s);
    }
    return 0;
}

// ------------------------------------------------------------------ the text encoder
int SeqEncoder::init(int vocab, int dim, int hidden, int convs_n, WeightList& wl) {
    n_vocab = vocab; E = dim; H = hidden; n_convs = convs_n;
    B200_REQUIRE(n_vocab > 0 && E > 0 && H > 0 && n_convs >= 1 && n_convs <= 8, "encoder: unsupported config");
    int rc;
    if ((rc = upload(emb, wl.take(), (size_t)n_vocab * E))) return rc;
    std::vector<float> wf, bf;
    for (int l = 0; l < n_convs; ++l) {   // ConvBNBlock: BatchNorm1d (eps 1e-5) folded into the conv
        if ((rc = fold_bn(wl, true, 1e-5, E, (size_t)E * 5, wf, bf))) return rc;
        if ((rc = pack_conv(convs[l], wf.data(), bf.data(), E, E, 5, 1, 2))) return rc;
    }
    {   // LSTM: both directions' input projections as one 1x1 conv (rows [fwd 4H | bwd 4H]), bias b_ih + b_hh
        std::vector<float> wi((size_t)8 * H * E), bi((size_t)8 * H), wh((size_t)8 * H * H);
        for (int d = 0; d < 2; ++d) {
            const float *w_ih = wl.take(), *w_hh = wl.take(), *b_ih = wl.take(), *b_hh = wl.take();
            B200_REQUIRE(w_ih && w_hh && b_ih && b_hh, "encoder: null LSTM weight or bias");
            memcpy(wi.data() + (size_t)d * 4 * H * E, w_ih, sizeof(float) * 4 * H * E);
            memcpy(wh.data() + (size_t)d * 4 * H * H, w_hh, sizeof(float) * 4 * H * H);
            for (int r = 0; r < 4 * H; ++r) bi[(size_t)d * 4 * H + r] = b_ih[r] + b_hh[r];
        }
        if ((rc = pack_conv(lstm_in, wi.data(), bi.data(), 8 * H, E, 1, 1, 0))) return rc;
        if ((rc = upload(whh, wh.data(), wh.size()))) return rc;
    }
    return 0;
}

SeqEncoder::Scratch SeqEncoder::carve(Arena& ar, int B, int Tt) const {
    Scratch s;
    s.x = ar.f32((size_t)B * E * Tt);
    s.y = ar.f32((size_t)B * E * Tt);
    s.xmask = ar.f32((size_t)B * Tt);
    s.pre = ar.f32((size_t)B * 8 * H * Tt);
    s.hb = ar.f32((size_t)4 * B * H);
    s.cb = ar.f32((size_t)2 * B * H);
    return s;
}

int SeqEncoder::encode(const long long* tokens, const long long* lengths, int B, int Tt, float* out, const Scratch& s,
                       cudaStream_t st) const {
    float *x = s.x, *y = s.y, *xmask = s.xmask, *pre = s.pre, *hb = s.hb, *cb = s.cb;
    int rc;
    // emb(x) without a scale, zero past each row's length (the reference runs each row at its own length)
    if ((rc = launch_embed(tokens, lengths, emb, nullptr, B, Tt, E, E, x, xmask, st, false))) return rc;
    for (int l = 0; l < n_convs; ++l) {   // conv -> BN (folded) -> ReLU -> Dropout (eval: identity), masked
        ConvIO io;
        io.x = dense(x, E, Tt); io.Tin = Tt;
        io.y = dense(y, E, Tt); io.Tout = Tt; io.B = B;
        io.act = ACT_RELU; io.ymask = {xmask, Tt}; io.flags = EPI_MASK_POST;
        if ((rc = launch_conv(convs[l], io, st))) return rc;
        std::swap(x, y);
    }
    {   // pre[b, d*4H + row, t] = W_ih x + b_ih + b_hh, both directions
        ConvIO io;
        io.x = dense(x, E, Tt); io.Tin = Tt;
        io.y = dense(pre, 8 * H, Tt); io.Tout = Tt; io.B = B;
        if ((rc = launch_conv(lstm_in, io, st))) return rc;
    }
    B200_CUDA_OK(cudaMemsetAsync(hb, 0, sizeof(float) * 2 * B * H, st));
    B200_CUDA_OK(cudaMemsetAsync(cb, 0, sizeof(float) * 2 * B * H, st));
    B200_CUDA_OK(cudaMemsetAsync(out, 0, sizeof(float) * (size_t)B * Tt * 2 * H, st));
    for (int s = 0; s < Tt; ++s) {   // out [B, Tt, 2H]: forward | backward
        LstmArgs a;
        a.seg[0].W = whh; a.seg[0].ldw = H; a.seg[0].w_ds = (long long)4 * H * H; a.seg[0].K = H;
        a.seg[0].x = hb + (size_t)(s & 1) * 2 * B * H; a.seg[0].x_bs = H; a.seg[0].x_ds = (long long)B * H;
        a.nseg = 1;
        a.H = H; a.h_out = hb + (size_t)((s + 1) & 1) * 2 * B * H; a.h_bs = H;
        a.c = cb; a.st_ds = (long long)B * H;
        a.pre = pre; a.pre_bs = (long long)8 * H * Tt; a.pre_cs = Tt;
        a.out = out; a.out_bs = (long long)Tt * 2 * H; a.out_ts = 2 * H;
        a.lens = lengths; a.step = s; a.B = B;
        if ((rc = launch_lstm(a, 2, 8, DISPATCH_LSTM_BI, st, true))) return rc;
    }
    return 0;
}

}  // namespace b200tts
