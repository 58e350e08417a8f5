// Generic fused conv1d as an FP32 implicit GEMM on the sm_90a FMA pipe.
//
// This one kernel carries >99% of the VITS+HiFiGAN inference FLOPs: the HiFiGAN MRF convs
// (reference: TTS/vocoder/models/hifigan_generator.py:84-99,236-265), the polyphase form of its
// ConvTranspose1d upsamplers (:207-218), the WaveNet k5 / 1x1 convs of the flow
// (TTS/tts/layers/generic/wavenet.py:94-115) and the 1x1 / k3 convs of the text encoder
// (TTS/tts/layers/glow_tts/transformer.py:109-121,290-295).
//
// Layout: activations stay in the reference's [B, C, T] layout (T contiguous).  A CTA owns a
// [CO_T rows] x [T_T time] output tile.  Input channels are streamed in chunks of 8 through a
// double-buffered shared-memory window [8][T_T + (K-1)*dil] (coalesced loads along T, prologue
// -- mask, leaky-relu -- applied once on the way in) next to the chunk's weights
// [8][K][CO_T] (cp.async).  Each lane owns TJ time steps strided by 32 (conflict-free LDS.32,
// tap shifts are plain address offsets) and CJ=16 consecutive rows (warp-uniform weight LDS.128
// broadcasts), accumulating row pairs (x as broadcast scalar).
// Bias / conditioning / gate / residual / mask / MRF-accumulate epilogues are fused.
#include "common.cuh"
#include "engines.cuh"
#include "conv_tc.cuh"
#include "conv_tc3.cuh"

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdarg.h>
#include <string.h>

#include <algorithm>
#include <cmath>

namespace b200tts {

// ------------------------------------------------------------------ error plumbing / counters
static thread_local char g_err[1024] = "";
unsigned long long g_launch_count = 0;

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
const char* last_error() { return g_err; }

// ------------------------------------------------------------------ device helpers
constexpr int CI_MAX = 16;  // CinPad granularity (largest input-channel chunk of any instantiation)

typedef unsigned long long u64;

__device__ __forceinline__ void unpack2(u64 v, float& lo, float& hi) {
    asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ u64 pack2(float lo, float hi) {
    u64 v;
    asm("mov.b64 %0, {%1, %2};" : "=l"(v) : "f"(lo), "f"(hi));
    return v;
}
// row pair += w pair * x: two rounded FMAs (sm_90 has no packed FP32 FMA; the register moves compile away)
__device__ __forceinline__ void ffma2(u64& d, u64 a, float x) {
    float d0, d1, a0, a1;
    unpack2(d, d0, d1);
    unpack2(a, a0, a1);
    d = pack2(fmaf(a0, x, d0), fmaf(a1, x, d1));
}
__device__ __forceinline__ void cp_async16(float* smem_dst, const float* gsrc) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gsrc));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// KEPI_BN: the generic epilogue plus the Conv1dBN options (ConvIO::edge_lo / aff_s), compiled only into its own
// instantiations so that the generic ones keep their code
enum : int { KEPI_GENERIC = 0, KEPI_GATE = 1, KEPI_TANH = 2, KEPI_PLAIN = 3, KEPI_WAVEGRAD = 4, KEPI_BN = 5 };

// CJ rows x TJ time steps per lane, WCO x WT warps, CIC input channels per stage, EPI epilogue family.
// KG > 1: intra-CTA split-K for launch-starved shapes (text encoder / duration predictor: 64 frames x 32 utterances
// give only 96 CTAs of 4 warps) -- KG warp groups each own a double-buffered stage and every KG-th channel chunk of
// the SAME output tile; their accumulators are summed through shared memory in a fixed order (deterministic).
template <int CJ, int TJ, int WCO, int WT, int CIC, int EPI, int KG = 1>
__global__ void __launch_bounds__(32 * WCO * WT * KG, (KG > 1) ? 1 : ((WCO * WT >= 8) ? 2 : 3)) conv1d_kernel(const ConvKArgs a) {
    constexpr int CO_T = CJ * WCO, T_T = 32 * TJ * WT, NT = 32 * WCO * WT;
    extern __shared__ __align__(16) float smem[];
    const int XS = a.XS;
    const int wchunk = CIC * a.K * CO_T;
    const int kg = (KG > 1) ? (int)(threadIdx.x / NT) : 0;              // split-K group of this warp
    const int stage_floats = 2 * CIC * XS + 2 * wchunk;
    float* xs0 = smem + (size_t)kg * stage_floats;
    float* ws0 = xs0 + 2 * CIC * XS;
    const int tid = threadIdx.x % NT, lane = tid & 31, warp = tid >> 5;   // group-local thread / warp index
    const int wco = warp % WCO, wt = warp / WCO;
    auto group_sync = [&]() {
        if constexpr (KG > 1) asm volatile("bar.sync %0, %1;" ::"r"(kg + 1), "r"(NT) : "memory");
        else __syncthreads();
    };
    const int b = blockIdx.z, tile_co = blockIdx.y;
    const int q0 = blockIdx.x * T_T;
    if (q0 >= a.io.q_hi || q0 + T_T <= a.io.q_lo) return;     // tile outside the column window: nothing to produce
    const int tin0 = q0 - a.pad;
    const float* xb = a.io.x.p + b * a.io.x.bs;
    const float* mb = a.io.xmask ? a.io.xmask.row(b) : nullptr;
    const float* wg = a.w + (size_t)tile_co * a.CinPad * a.K * CO_T;
    const int nchunks = (a.Cin + CIC - 1) / CIC;   // CinPad is a multiple of CI_MAX >= CIC; skip all-zero chunks
    const float slope = a.io.in_slope;

    auto load_chunk = [&](int chunk, int buf) {
        const float* src = wg + (size_t)chunk * wchunk;
        float* dst = ws0 + buf * wchunk;
        for (int i = tid * 4; i < wchunk; i += NT * 4) cp_async16(dst + i, src + i);
        cp_async_commit();
        float* xd = xs0 + buf * CIC * XS;
        const int c0 = chunk * CIC;
        for (int i = tid; i < XS; i += NT) {
            int t = tin0 + i;
            if (a.io.reflect) t = t < 0 ? -t : (t >= a.io.Tin ? 2 * a.io.Tin - 2 - t : t);   // mirrored; columns past the reach stay out
            const bool tok = (t >= a.io.in_lo) && (t < a.io.Tin);   // below in_lo: stale scratch of a windowed producer
            float m = 1.f;
            if (tok && mb) m = __ldg(mb + t);
            int ts = t;                                        // source column
            if constexpr (EPI == KEPI_WAVEGRAD) {
                if (a.io.near_src && tok) ts = tc3::near_col(t, a.io.near_src, a.io.Tin, a.near_scale);
            }
#pragma unroll
            for (int h = 0; h < CIC; h += 8) {
                float v[8];
#pragma unroll
                for (int ci = 0; ci < 8; ++ci) {
                    v[ci] = 0.f;
                    if (tok && (c0 + h + ci) < a.Cin) v[ci] = __ldg(xb + (long long)(c0 + h + ci) * a.io.x.cs + ts);
                }
#pragma unroll
                for (int ci = 0; ci < 8; ++ci) {
                    float u = v[ci] * m;
                    u = u > 0.f ? u : u * slope;
                    xd[(h + ci) * XS + i] = u;
                }
            }
        }
    };

    u64 acc[CJ / 2][TJ];
#pragma unroll
    for (int p = 0; p < CJ / 2; ++p)
#pragma unroll
        for (int j = 0; j < TJ; ++j) acc[p][j] = 0ull;

    if (kg < nchunks) load_chunk(kg, 0);
    cp_async_wait_all();
    group_sync();

    const int K = a.K, dil = a.dil;
    for (int ch = kg, it = 0; ch < nchunks; ch += KG, ++it) {
        const int buf = it & 1;
        if (ch + KG < nchunks) load_chunk(ch + KG, buf ^ 1);
        const float* xr = xs0 + buf * CIC * XS + wt * 32 * TJ + lane;
        const float* wr = ws0 + buf * wchunk + wco * CJ;
#pragma unroll 1
        for (int ci = 0; ci < CIC; ++ci) {
            const float* xp = xr + ci * XS;
            const ulonglong2* wp = reinterpret_cast<const ulonglong2*>(wr + ci * K * CO_T);
#pragma unroll 1
            for (int k = 0; k < K; ++k) {
                float xv[TJ];
#pragma unroll
                for (int j = 0; j < TJ; ++j) xv[j] = xp[32 * j];
                u64 wv[CJ / 2];
#pragma unroll
                for (int p = 0; p < CJ / 4; ++p) {
                    const ulonglong2 t2 = wp[p];
                    wv[2 * p] = t2.x;
                    wv[2 * p + 1] = t2.y;
                }
#pragma unroll
                for (int j = 0; j < TJ; ++j)
#pragma unroll
                    for (int p = 0; p < CJ / 2; ++p) ffma2(acc[p][j], wv[p], xv[j]);
                xp += dil;
                wp += CO_T / 4;
            }
        }
        cp_async_wait_all();
        group_sync();
    }

    if constexpr (KG > 1) {
        // fixed-order sum of the groups' partial accumulators (group 0 += group 1 += ...), through the stage memory
        __syncthreads();
        u64* red = reinterpret_cast<u64*>(smem);
        if (kg > 0) {
#pragma unroll
            for (int p = 0; p < CJ / 2; ++p)
#pragma unroll
                for (int j = 0; j < TJ; ++j) red[(((size_t)(kg - 1) * (CJ / 2) + p) * TJ + j) * NT + tid] = acc[p][j];
        }
        __syncthreads();
        if (kg > 0) return;
#pragma unroll
        for (int g2 = 1; g2 < KG; ++g2)
#pragma unroll
            for (int p = 0; p < CJ / 2; ++p)
#pragma unroll
                for (int j = 0; j < TJ; ++j) {
                    float v0, v1, w0, w1;
                    unpack2(acc[p][j], v0, v1);
                    unpack2(red[(((size_t)(g2 - 1) * (CJ / 2) + p) * TJ + j) * NT + tid], w0, w1);
                    acc[p][j] = pack2(v0 + w0, v1 + w1);
                }
    }

    // ---------------------------------------------------------------- epilogue
    const int row_base = tile_co * CO_T + wco * CJ;
    const int qb = q0 + wt * 32 * TJ + lane;
    auto inw = [&](int q) { return q < a.io.Tout && q >= a.io.q_lo && q < a.io.q_hi; };   // stored columns: the window only
    if (EPI == KEPI_GATE) {
        // rows (2p, 2p+1) = (tanh half, sigmoid half) of output row row_base/2 + p   (wavenet.py:6-13)
#pragma unroll
        for (int p = 0; p < CJ / 2; ++p) {
            const int r0 = row_base + 2 * p;
            if (r0 + 1 < a.Rows) {
                float b0 = a.bias[r0], b1 = a.bias[r0 + 1];
                if (a.io.cond) { b0 += __ldg(a.io.cond.row(b) + r0); b1 += __ldg(a.io.cond.row(b) + r0 + 1); }
                float* yrow = a.io.y.row(b, r0 >> 1);
#pragma unroll
                for (int j = 0; j < TJ; ++j) {
                    const int q = qb + 32 * j;
                    float v0, v1;
                    unpack2(acc[p][j], v0, v1);
                    v0 += b0; v1 += b1;
                    if (inw(q)) yrow[q] = tanhf(v0) * (1.f / (1.f + expf(-v1)));
                }
            }
        }
        return;
    }
    if (EPI == KEPI_TANH) {   // conv_post: y = tanh(acc + bias)   (hifigan_generator.py:263-264)
#pragma unroll
        for (int p = 0; p < CJ / 2; ++p) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = row_base + 2 * p + h;
                if (r < a.Rows) {
                    const float bb = a.bias[r];
                    float* yrow = a.io.y.row(b, r);
#pragma unroll
                    for (int j = 0; j < TJ; ++j) {
                        const int q = qb + 32 * j;
                        float v0, v1;
                        unpack2(acc[p][j], v0, v1);
                        if (inw(q)) yrow[q] = tanhf((h ? v1 : v0) + bb);
                    }
                }
            }
        }
        return;
    }
    if (EPI == KEPI_WAVEGRAD) {
        // v = acc + bias; [lrelu]; [+ act_add[b]]; [+ res]; [y2 <- v]; [v = shift + scale * v]; y <- v, each operation
        // rounded on its own (the reference's order); res / y2 may alias element for element (load before store)
        const bool lrelu = a.io.act == ACT_LRELU;
        const float add = a.io.act_add ? __ldg(a.io.act_add + b) : 0.f;
#pragma unroll
        for (int p = 0; p < CJ / 2; ++p) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = row_base + 2 * p + h;
                if (r >= a.Rows) continue;
                const float bb = a.bias[r];
                float* yrow = a.io.y.row(b, r);
                float* y2row = a.io.y2 ? a.io.y2.row(b, r) : nullptr;
                const float* rrow = a.io.res ? a.io.res.row(b, r) : nullptr;
                const float* srow = a.io.film ? a.io.film.row(b, r) : nullptr;
#pragma unroll
                for (int j = 0; j < TJ; ++j) {
                    const int q = qb + 32 * j;
                    if (!inw(q)) continue;
                    float v0, v1;
                    unpack2(acc[p][j], v0, v1);
                    float u = __fadd_rn(h ? v1 : v0, bb);
                    if (lrelu) u = u > 0.f ? u : __fmul_rn(u, a.io.act_param);
                    if (a.io.act_add) u = __fadd_rn(u, add);
                    if (rrow) u = __fadd_rn(u, rrow[q]);
                    if (y2row) y2row[q] = u;
                    if (srow) u = __fadd_rn(srow[q], __fmul_rn(srow[(long long)a.io.film_half * a.io.film.cs + q], u));
                    yrow[q] = u;
                }
            }
        }
        return;
    }
    if (EPI == KEPI_PLAIN) {   // y = act(acc + bias + cond) [* mask]   -- no residual / accumulate / upsampling
        const bool relu_p = a.io.act == ACT_RELU;
        const bool logc_p = a.io.act == ACT_LOGCLAMP;
        float mkp[TJ];
#pragma unroll
        for (int j = 0; j < TJ; ++j) {
            const int q = qb + 32 * j;
            mkp[j] = (a.io.ymask && q < a.io.Tout) ? __ldg(a.io.ymask.row(b) + q) : 1.f;
        }
#pragma unroll
        for (int p = 0; p < CJ / 2; ++p) {
            const int r0 = row_base + 2 * p;
            float b0 = 0.f, b1 = 0.f;
            if (r0 < a.Rows) { b0 = a.bias[r0]; if (a.io.cond) b0 += __ldg(a.io.cond.row(b) + r0); }
            if (r0 + 1 < a.Rows) { b1 = a.bias[r0 + 1]; if (a.io.cond) b1 += __ldg(a.io.cond.row(b) + r0 + 1); }
            float* y0 = a.io.y.row(b, r0);
            float* y1 = y0 + a.io.y.cs;
#pragma unroll
            for (int j = 0; j < TJ; ++j) {
                const int q = qb + 32 * j;
                float v0, v1;
                unpack2(acc[p][j], v0, v1);
                v0 += b0; v1 += b1;
                if (relu_p) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                if (logc_p) { v0 = logf(fmaxf(v0, a.io.act_param)); v1 = logf(fmaxf(v1, a.io.act_param)); }
                v0 *= mkp[j]; v1 *= mkp[j];
                if (inw(q)) {
                    if (r0 < a.Rows) y0[q] = v0;
                    if (r0 + 1 < a.Rows) y1[q] = v1;
                }
            }
        }
        return;
    }
    // generic: v = act(acc + bias + cond) [*m] [+res] *scale [+y_old] [/div] [*m]; all loads are issued before
    // any store (res / y_old may alias y only element-for-element, never across threads)
    const int ups = a.ups;
    const bool relu = a.io.act == ACT_RELU;
    const bool split = (a.io.flags & EPI_SPLIT) != 0;
    float mk[TJ];
    int tq[TJ];
#pragma unroll
    for (int j = 0; j < TJ; ++j) {
        const int q = qb + 32 * j;
        tq[j] = (q >= a.io.q_lo && q < a.io.q_hi) ? q * ups : 0x7fffffff;   // outside the window: fails every bound below
        mk[j] = 1.f;
        if (a.io.ymask && ups == 1 && tq[j] < a.io.Tout) mk[j] = __ldg(a.io.ymask.row(b) + tq[j]);
    }
    // per-row destination: recomputed per phase instead of kept in registers (16 rows x 2 pointers would spill)
    auto rowinfo = [&](int i, float*& yp, const float*& rp, bool& accum, bool& mpost, int& tlim) -> bool {
        const int r = row_base + i;
        int chn = r, ph = 0;
        if (ups > 1) { chn = r / ups; ph = r - chn * ups; }
        accum = (a.io.flags & EPI_ACCUM) != 0;
        mpost = (a.io.flags & EPI_MASK_POST) != 0;
        yp = a.io.y.row(b, chn) + ph;
        if (split) {
            if (chn < a.io.split) { accum = true; mpost = true; }
            else { yp = a.io.y2.row(b, chn - a.io.split); accum = (a.io.flags & EPI_ACCUM2) != 0; mpost = false; }
        }
        rp = a.io.res ? a.io.res.row(b, chn) + ph : nullptr;
        tlim = a.io.Tout - ph;   // element (q*ups + ph) exists iff q*ups < Tout - ph
        return r < a.Rows;
    };
    const bool mpre = (a.io.flags & EPI_MASK_PRE) != 0;
    // Conv1dBN: the valid window [edge_lo, len_b - edge_hi) of this row, per column of this lane (a select: columns
    // outside it read data past the row), and the per-row affine
    bool vw[TJ];
    const bool aff = EPI == KEPI_BN && a.io.aff_s != nullptr;
    if constexpr (EPI == KEPI_BN) {
        const bool win = (a.io.flags & EPI_WINDOW) != 0;
        const int hi = (a.io.lens ? min(a.io.lens[b], a.io.Tout) : a.io.Tout) - a.io.edge_hi;
#pragma unroll
        for (int j = 0; j < TJ; ++j) {
            const int q = qb + 32 * j;
            vw[j] = !win || (q >= a.io.edge_lo && q < hi);
        }
    }
    // phase 1: bias / cond / activation / pre-mask (registers only)
#pragma unroll
    for (int p = 0; p < CJ / 2; ++p) {
        const int r0 = row_base + 2 * p;
        float b0 = 0.f, b1 = 0.f;
        if (r0 < a.Rows) { b0 = a.bias[r0]; if (a.io.cond) b0 += __ldg(a.io.cond.row(b) + r0); }
        if (r0 + 1 < a.Rows) { b1 = a.bias[r0 + 1]; if (a.io.cond) b1 += __ldg(a.io.cond.row(b) + r0 + 1); }
        float s0 = 1.f, s1 = 1.f, h0 = 0.f, h1 = 0.f;
        if (aff) {
            if (r0 < a.Rows) { s0 = a.io.aff_s[r0]; h0 = a.io.aff_h[r0]; }
            if (r0 + 1 < a.Rows) { s1 = a.io.aff_s[r0 + 1]; h1 = a.io.aff_h[r0 + 1]; }
        }
#pragma unroll
        for (int j = 0; j < TJ; ++j) {
            float v0, v1;
            unpack2(acc[p][j], v0, v1);
            v0 += b0; v1 += b1;
            if constexpr (EPI == KEPI_BN) {
                if (!vw[j]) { v0 = 0.f; v1 = 0.f; }
            }
            if (relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
            if (aff) { v0 = fmaf(v0, s0, h0); v1 = fmaf(v1, s1, h1); }
            if (mpre) { v0 *= mk[j]; v1 *= mk[j]; }
            acc[p][j] = pack2(v0, v1);
        }
    }
    // phase 2: residual (all loads first)
    if (a.io.res) {
#pragma unroll
        for (int p = 0; p < CJ / 2; ++p) {
            float *yp0, *yp1; const float *rp0, *rp1; bool ac0, ac1, mp0, mp1; int tl0, tl1;
            const bool ok0 = rowinfo(2 * p, yp0, rp0, ac0, mp0, tl0), ok1 = rowinfo(2 * p + 1, yp1, rp1, ac1, mp1, tl1);
#pragma unroll
            for (int j = 0; j < TJ; ++j) {
                float v0, v1, r0v = 0.f, r1v = 0.f;
                if (ok0 && tq[j] < tl0) r0v = rp0[tq[j]];
                if (ok1 && tq[j] < tl1) r1v = rp1[tq[j]];
                unpack2(acc[p][j], v0, v1);
                acc[p][j] = pack2(v0 + r0v, v1 + r1v);
            }
        }
    }
    // phase 3: scale, accumulate into the destination (all loads first)
    const float scale = a.io.scale;
    if (split || (a.io.flags & EPI_ACCUM)) {
#pragma unroll
        for (int p = 0; p < CJ / 2; ++p) {
            float *yp0, *yp1; const float *rp0, *rp1; bool ac0, ac1, mp0, mp1; int tl0, tl1;
            const bool ok0 = rowinfo(2 * p, yp0, rp0, ac0, mp0, tl0), ok1 = rowinfo(2 * p + 1, yp1, rp1, ac1, mp1, tl1);
#pragma unroll
            for (int j = 0; j < TJ; ++j) {
                float v0, v1, o0 = 0.f, o1 = 0.f;
                if (ac0 && ok0 && tq[j] < tl0) o0 = yp0[tq[j]];
                if (ac1 && ok1 && tq[j] < tl1) o1 = yp1[tq[j]];
                unpack2(acc[p][j], v0, v1);
                acc[p][j] = pack2(v0 * scale + o0, v1 * scale + o1);
            }
        }
    } else if (scale != 1.f) {
#pragma unroll
        for (int p = 0; p < CJ / 2; ++p)
#pragma unroll
            for (int j = 0; j < TJ; ++j) {
                float v0, v1;
                unpack2(acc[p][j], v0, v1);
                acc[p][j] = pack2(v0 * scale, v1 * scale);
            }
    }
    // phase 4: mean / post-mask / store
    const float div = a.io.post_div;
#pragma unroll
    for (int p = 0; p < CJ / 2; ++p) {
        float *yp0, *yp1; const float *rp0, *rp1; bool ac0, ac1, mp0, mp1; int tl0, tl1;
        const bool ok0 = rowinfo(2 * p, yp0, rp0, ac0, mp0, tl0), ok1 = rowinfo(2 * p + 1, yp1, rp1, ac1, mp1, tl1);
#pragma unroll
        for (int j = 0; j < TJ; ++j) {
            float v0, v1;
            unpack2(acc[p][j], v0, v1);
            if (div != 1.f) { v0 = v0 / div; v1 = v1 / div; }
            if (mp0) v0 *= mk[j];
            if (mp1) v1 *= mk[j];
            if (ok0 && tq[j] < tl0) yp0[tq[j]] = v0;
            if (ok1 && tq[j] < tl1) yp1[tq[j]] = v1;
        }
    }
}

// ------------------------------------------------------------------ host: packing
static inline int round_up(int v, int m) { return (v + m - 1) / m * m; }

// PREC_F16X3 row scaling 2^e_r of row r (n weights): e_r puts the row's max |w| * 2^e_r in [2^14, 2^15); all-zero rows: 1
static float f16x3_row_up(const std::vector<float>& Wl, int r, size_t n) {
    float m = 0.f;
    for (size_t i = (size_t)r * n; i < (size_t)(r + 1) * n; ++i) m = std::max(m, std::fabs(Wl[i]));
    if (m == 0.f) return 1.f;
    int E;
    std::frexp(m, &E);                                     // m in [2^(E-1), 2^E)
    return std::ldexp(1.f, std::min(126, std::max(-126, 15 - E)));
}

// One tensor-core weight image (conv_tc3.cuh): per (128-row tile, input-channel chunk, tap block) the block the weight
// loader copies with one cp.async.bulk, [slabs][128 MMA rows][16 B], slab s holding the chunk's channels s*SLC .. +SLC-1:
//   3xTF32 (PREC_FP32): 8-channel chunks, {hi, lo}[2 slabs] of 4 floats, hi = v & 0xFFFFE000 (exact in TF32), lo = v - hi
//   bf16 / fp16:        16-channel chunks, [2 slabs] of 8 values rounded to nearest even (as cvt.rn rounds the activations)
//   PREC_F16X3:         16-channel chunks, {hi, lo}[2 slabs] of 8 fp16 values of the scaled row w' = w * 2^e_r (e_r puts
//                       the row's max |w'| in [2^14, 2^15); all-zero rows: e_r = 0): hi = fp16(w'), lo = fp16(w' - hi);
//                       the kernel makes the third operand, fp16(hi * 2^-11), from hi in registers, and its epilogue
//                       multiplies by rscale[r] = 2^-e_r, which the first call returns in *rscale
// With G tap groups (1: plain; 128 / rows: grouped), MMA row m = g * (128 / G) + co of tile t carries weight row
// t * 128 + co and, in tap block j, tap G * j + g.  Rows >= `rows`, taps >= K and channels >= Cin are zero.  The weight
// norm is already folded (in fp32) into Wl; each weight is rounded once, here.
int pack_tc(DevBuf<unsigned char>& dst, const std::vector<float>& Wl, int rows, int Cin, int K, int prec, int G,
            DevBuf<float>* rscale) {
    const bool tf32 = prec == tc::PREC_FP32, x3 = prec == tc::PREC_F16X3;
    const int kc = tf32 ? tc3::KC2 : tc3::KC16, slc = kc / 2, ch = tc3::MROWS / G;
    const int ntiles = (rows + tc3::MROWS - 1) / tc3::MROWS, nchunks = (Cin + kc - 1) / kc, J = (K + G - 1) / G;
    const size_t slab = (size_t)tc3::MROWS * 16, blk = (tf32 || x3 ? 4 : 2) * slab;
    std::vector<unsigned char> img((size_t)ntiles * nchunks * J * blk, 0);
    std::vector<float> up(x3 ? rows : 0, 1.f), down(x3 ? rows : 0, 1.f);   // 2^e_r, 2^-e_r
    for (int r = 0; r < (x3 ? rows : 0); ++r) {
        up[r] = f16x3_row_up(Wl, r, (size_t)Cin * K);
        down[r] = 1.f / up[r];
    }
    for (int t = 0; t < ntiles; ++t)
        for (int c = 0; c < nchunks; ++c)
            for (int j = 0; j < J; ++j)
                for (int m = 0; m < tc3::MROWS; ++m) {
                    const int r = t * tc3::MROWS + m % ch, k = G * j + m / ch;
                    if (r >= rows || k >= K) continue;
                    unsigned char* row = img.data() + (((size_t)t * nchunks + c) * J + j) * blk + (size_t)m * 16;
                    for (int i = 0; i < kc && c * kc + i < Cin; ++i) {
                        const float v = Wl[((size_t)r * Cin + c * kc + i) * K + k];
                        unsigned char* p = row + (i / slc) * slab;
                        const int e = i % slc;
                        if (tf32) {
                            uint32_t u;
                            memcpy(&u, &v, 4);
                            u &= 0xFFFFE000u;
                            float hi;
                            memcpy(&hi, &u, 4);
                            const float lo = v - hi;
                            memcpy(p + 4 * e, &hi, 4);
                            memcpy(p + 2 * slab + 4 * e, &lo, 4);
                        } else if (x3) {
                            const float ws = v * up[r];
                            const __half hi = __float2half_rn(ws);
                            const __half lo = __float2half_rn(ws - __half2float(hi));
                            memcpy(p + 2 * e, &hi, 2);
                            memcpy(p + 2 * slab + 2 * e, &lo, 2);
                        } else if (prec == tc::PREC_BF16) {
                            const __nv_bfloat16 h = __float2bfloat16_rn(v);
                            memcpy(p + 2 * e, &h, 2);
                        } else {
                            const __half h = __float2half_rn(v);
                            memcpy(p + 2 * e, &h, 2);
                        }
                    }
                }
    const int rc = upload(dst, img.data(), img.size());
    if (rc == 0 && x3 && rscale && !*rscale) return upload(*rscale, down.data(), down.size());
    return rc;
}

// The time-major kernel's PREC_F16X3 image for exactly 32 / 64 rows (the B operand, conv_tc3.cuh tm_consumers): per
// (16-channel chunk, tap) one block {W_hs, W_lo, W_hi}[2 slabs][rows][16 B], slab s holding channels 8 s .. 8 s + 7.  The
// row scaling and W_hi / W_lo are pack_tc's; W_hs = fp16(W_hi * 2^-11) is stored (a B operand cannot come from registers).
static int pack_tc_tm(DevBuf<unsigned char>& dst, const std::vector<float>& Wl, int rows, int Cin, int K) {
    const int nchunks = (Cin + tc3::KC16 - 1) / tc3::KC16;
    const size_t slab = (size_t)rows * 16, plane = 2 * slab, blk = tc3::tm_block_bytes(rows);
    std::vector<unsigned char> img((size_t)nchunks * K * blk, 0);
    for (int r = 0; r < rows; ++r) {
        const float up = f16x3_row_up(Wl, r, (size_t)Cin * K);
        for (int c = 0; c < nchunks; ++c)
            for (int k = 0; k < K; ++k)
                for (int i = 0; i < tc3::KC16 && c * tc3::KC16 + i < Cin; ++i) {
                    const float ws = Wl[((size_t)r * Cin + c * tc3::KC16 + i) * K + k] * up;
                    const __half hi = __float2half_rn(ws);
                    const __half lo = __float2half_rn(ws - __half2float(hi));
                    const __half hs = __float2half_rn(__half2float(hi) / 2048.f);
                    unsigned char* p = img.data() + ((size_t)c * K + k) * blk + (i / 8) * slab + (size_t)r * 16 + 2 * (i % 8);
                    memcpy(p, &hs, 2);
                    memcpy(p + plane, &lo, 2);
                    memcpy(p + 2 * plane, &hi, 2);
                }
    }
    return upload(dst, img.data(), img.size());
}

// Wl(r, ci, k): logical weights already expressed as a correlation-form conv with `rows` GEMM rows
static int pack_rows(ConvLayer& L, const std::vector<float>& Wl, const std::vector<float>& bl, int rows, int Cin,
                     int K) {
    L.Rows = rows;
    L.co_tile = rows >= 64 ? 64 : 32;
    L.RowsPad = round_up(rows, L.co_tile);
    L.Cin = Cin;
    L.CinPad = round_up(Cin, CI_MAX);
    L.K = K;
    const int T = L.co_tile, ntile = L.RowsPad / T;
    std::vector<float> P((size_t)ntile * L.CinPad * K * T, 0.f);
    for (int r = 0; r < rows; ++r) {
        const int tile = r / T, col = r % T;
        for (int ci = 0; ci < Cin; ++ci)
            for (int k = 0; k < K; ++k)
                P[(((size_t)tile * L.CinPad + ci) * K + k) * T + col] = Wl[((size_t)r * Cin + ci) * K + k];
    }
    std::vector<float> bp(L.RowsPad, 0.f);
    for (int r = 0; r < rows; ++r) bp[r] = bl[r];
    if (upload(L.w, P.data(), P.size())) return 2;
    if (upload(L.bias, bp.data(), bp.size())) return 2;
    // tensor-core images for a layer that requests them: rows >= 32 get the plain image (M = 128: two m64 warpgroups);
    // exactly 32 / 64 rows also get the grouped one (no padding), which the dispatcher prefers.  3xTF32 needs Cin >= 8, and
    // a 16-bit request packs 3xTF32 unless Cin % 16 == 0, so such a layer shows up as tc3 / tc3_grouped in the dispatch log
    if (L.tc_prec != TC_NONE && Cin % tc3::KC16 != 0) L.tc_prec = tc::PREC_FP32;
    if (rows < 32 || Cin < tc3::KC2) L.tc_prec = TC_NONE;
    if (L.tc_prec == TC_NONE) return 0;
    if (pack_tc(L.w_tc, Wl, rows, Cin, K, L.tc_prec, 1, &L.tc_rscale)) return 2;
    if (L.ups == 1 && (rows == 32 || rows == 64)) {
        const int rc = L.tc_prec == tc::PREC_F16X3 ? pack_tc_tm(L.w_tcg, Wl, rows, Cin, K)
                                                    : pack_tc(L.w_tcg, Wl, rows, Cin, K, L.tc_prec, tc3::MROWS / rows, &L.tc_rscale);
        if (rc) return 2;
        L.tc_grp = tc3::MROWS / rows;
    }
    return 0;
}

int pack_conv(ConvLayer& L, const float* w, const float* bias, int Cout, int Cin, int K, int dil, int pad,
              int gate_half, const int* in_perm, const int* out_perm) {
    B200_REQUIRE(w != nullptr && Cout > 0 && Cin > 0 && K > 0, "pack_conv: bad arguments");
    B200_REQUIRE(gate_half == 0 || 2 * gate_half == Cout, "pack_conv: gate_half must be Cout/2");
    std::vector<float> Wl((size_t)Cout * Cin * K), bl(Cout, 0.f);
    for (int r = 0; r < Cout; ++r) {
        int rn = r;
        if (gate_half > 0) rn = (r < gate_half) ? 2 * r : 2 * (r - gate_half) + 1;
        if (out_perm) rn = out_perm[r];
        for (int ci = 0; ci < Cin; ++ci) {
            const int cn = in_perm ? in_perm[ci] : ci;
            for (int k = 0; k < K; ++k) Wl[((size_t)rn * Cin + cn) * K + k] = w[((size_t)r * Cin + ci) * K + k];
        }
        if (bias) bl[rn] = bias[r];
    }
    L.dil = dil;
    L.pad = pad;
    L.ups = 1;
    return pack_rows(L, Wl, bl, Cout, Cin, K);
}

int pack_conv_transpose(ConvLayer& L, const float* w, const float* bias, int Cin, int Cout, int Kt, int s, int p, int op) {
    // y[co, q*s+ph] = sum_ci sum_m x[ci, q-m] * w[ci, co, ph + p + m*s]   (0 <= ph+p+m*s < Kt); output_padding `op` only
    // lengthens the output (the extra samples follow the same formula, as in torch)
    B200_REQUIRE(w != nullptr && s >= 1 && Kt >= 1, "pack_conv_transpose: bad arguments");
    B200_REQUIRE(op >= 0 && op < s, "pack_conv_transpose: output_padding %d must be in [0, stride %d)", op, s);
    auto floordiv = [](int a, int b) { return (a >= 0) ? a / b : -((-a + b - 1) / b); };
    const int m_lo = -floordiv(s - 1 + p, s);  // ceil(-(s-1+p)/s)
    const int m_hi = floordiv(Kt - 1 - p, s);
    const int K = m_hi - m_lo + 1;
    B200_REQUIRE(K >= 1, "pack_conv_transpose: empty tap range");
    const int rows = Cout * s;
    std::vector<float> Wl((size_t)rows * Cin * K, 0.f), bl(rows, 0.f);
    for (int co = 0; co < Cout; ++co)
        for (int ph = 0; ph < s; ++ph) {
            const int r = co * s + ph;
            if (bias) bl[r] = bias[co];
            for (int kk = 0; kk < K; ++kk) {
                const int m = m_hi - kk;
                const int kt = ph + p + m * s;
                if (kt < 0 || kt >= Kt) continue;
                for (int ci = 0; ci < Cin; ++ci)
                    Wl[((size_t)r * Cin + ci) * K + kk] = w[((size_t)ci * Cout + co) * Kt + kt];
            }
        }
    L.dil = 1;
    L.pad = m_hi;
    L.ups = s;
    L.tr_kernel = Kt;
    L.tr_pad = p;
    L.tr_outpad = op;
    return pack_rows(L, Wl, bl, rows, Cin, K);
}

// ------------------------------------------------------------------ single-output-row conv (HiFiGAN conv_post)
// y[b, 0, t] = act(bias + sum_ci sum_k w[ci, k] * lrelu(x[b, ci, t + k - pad])), K taps, dilation 1.  One output row has
// no reuse across rows, so this is a pure streaming kernel: each thread owns four consecutive samples and reads its
// window as aligned float4 (neighbouring threads' overlaps are L1 hits), 4*K FMAs per channel.  HBM-bound by the x read
// (Cin * 4 B per output sample).  Reference: hifigan_generator.py:262-264.  Eight CTAs per SM (32 registers): a full
// SM of warps to keep the loads in flight.
// REFLECT: reflection padding (ConvIO::reflect, K = 7 only), a compile-time switch: the edge threads mirror their own
// register window, no extra loads; 40 registers (six CTAs per SM), which the two edge fix-ups need to stay unspilled.
// w_stride: the distance of row 0's consecutive weights in the FMA image (the layer's co_tile); blk_lo: the grid's first
// block (the column window's)
template <int K, bool REFLECT>
__global__ void __launch_bounds__(256, REFLECT ? 6 : 8) conv1d_row1_kernel(const ConvKArgs a, int w_stride, int blk_lo) {
    constexpr int PAD = (K - 1) / 2, NL = (4 + 4 + (K - 1 - PAD) + 3) / 4;   // float4 loads covering [t0 - 4, t0 + 4 + K-1-PAD)
    static_assert(!REFLECT || K == 7, "the in-window mirror below is laid out for K = 7");
    const int Cin = a.Cin, T = a.io.Tout, q_lo = a.io.q_lo, q_hi = a.io.q_hi;
    unsigned* const peak_bits = a.io.peak_bits;
    extern __shared__ float ws[];
    for (int i = threadIdx.x; i < Cin * K; i += blockDim.x) ws[i] = a.w[(size_t)i * w_stride];
    __syncthreads();
    const int b = blockIdx.y;
    // ragged batch: row b is computed below Tb only (a multiple of 4) and samples from Tb on are written as zeros, so the
    // padded tail of the waveform is clean; the input holds data below Ti (its producer's extent) and reads as zero beyond
    int Tb = T, Ti = T;
    if (a.io.lens) {
        const long long base = (long long)a.io.lens[b] * a.io.rate_out;
        const long long e = (base + a.io.need_out + 3) / 4 * 4, ei = (base + a.io.need_in + 3) / 4 * 4;
        Tb = (int)(e < (long long)T ? (e > 0 ? e : 0) : (long long)T);
        Ti = (int)(ei < (long long)T ? (ei > 0 ? ei : 0) : (long long)T);
    }
    // column window [q_lo, hi): the grid starts at block blk_lo, only samples inside the window are stored (and folded
    // into the peak), and the input holds data from in_lo on (whole float4s below it read as zero)
    const int hi = min(q_hi, T), in_lo4 = a.io.in_lo & ~3;
    const int blk0 = (int)((blockIdx.x + blk_lo) * blockDim.x) * 4;
    const int t0 = blk0 + (int)threadIdx.x * 4;
    const bool inside = t0 >= q_lo && t0 + 4 <= hi;              // all four samples in the window: one float4 store
    const bool any = t0 < hi && t0 + 4 > q_lo;
    float* yp = a.io.y.row(b, 0) + t0;
    auto store = [&](const float4& v) {
        if (inside) {
            *reinterpret_cast<float4*>(yp) = v;
        } else if (any) {
            const float* pv = &v.x;
#pragma unroll
            for (int j = 0; j < 4; ++j) if (t0 + j >= q_lo && t0 + j < hi) yp[j] = pv[j];
        }
    };
    if (blk0 >= Tb && !peak_bits) {        // whole block beyond the row: zero fill and leave
        store(make_float4(0.f, 0.f, 0.f, 0.f));
        return;
    }
    const bool valid = t0 < Tb && any;
    if (!valid) store(make_float4(0.f, 0.f, 0.f, 0.f));
    if (!valid && !peak_bits) return;
    float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
    if (valid) {
        const float* xb = a.io.x.p + b * a.io.x.bs + t0;
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
        for (int ci = 0; ci < Cin; ++ci) {
            const float* xr = xb + (long long)ci * a.io.x.cs;
            float win[4 * NL];
#pragma unroll
            for (int l = 0; l < NL; ++l) {
                const int t = t0 - 4 + 4 * l;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (t >= in_lo4 && t < Ti) v = __ldg(reinterpret_cast<const float4*>(xr - 4 + 4 * l));   // Ti % 4 == 0: all in or all out
                win[4 * l] = v.x; win[4 * l + 1] = v.y; win[4 * l + 2] = v.z; win[4 * l + 3] = v.w;
            }
            if constexpr (REFLECT) {
                // the mirrored columns of the two edge threads lie in their own window (T % 4 == 0, K = 7): win[i] holds
                // column t0 - 4 + i, so at the row end (t0 = T - 4) column T + j reads T - 2 - j = win[14 - i], and at the
                // start (t0 = 0) column -j reads j = win[8 - i] (end first: for T = 4 the start's source win[8] is past the end)
                if (t0 + 4 == T) { win[8] = win[6]; win[9] = win[5]; win[10] = win[4]; win[11] = win[3]; }
                if (t0 == 0) { win[0] = win[8]; win[1] = win[7]; win[2] = win[6]; win[3] = win[5]; }
            }
#pragma unroll
            for (int i = 0; i < 4 * NL; ++i) win[i] = win[i] > 0.f ? win[i] : win[i] * a.io.in_slope;
#pragma unroll
            for (int k = 0; k < K; ++k) {
                const float wk = ws[ci * K + k];
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[j] = fmaf(wk, win[4 - PAD + j + k], acc[j]);
            }
        }
        const float bv = a.bias[0];
        float* po = &o.x;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float u = acc[j] + bv;
            if (a.io.act == ACT_TANH) u = tanhf(u);
            po[j] = u;
        }
        store(o);
        if (!inside) {
#pragma unroll
            for (int j = 0; j < 4; ++j) if (t0 + j < q_lo || t0 + j >= hi) po[j] = 0.f;   // not stored: not in the peak
        }
    }
    if (peak_bits) {   // save_wav's max|wav| (numpy_transforms.py:439) folded into the store: one atomic per warp
        float m = fmaxf(fmaxf(fabsf(o.x), fabsf(o.y)), fmaxf(fabsf(o.z), fabsf(o.w)));
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
        if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(peak_bits, __float_as_uint(m));
    }
}

// ------------------------------------------------------------------ host: launch
template <int CJ, int TJ, int WCO, int WT, int CIC, int EPI, int KG = 1>
static int launch_variant(const ConvKArgs& ka, int B, int RowsPad, cudaStream_t st) {
    constexpr int CO_T = CJ * WCO, T_T = 32 * TJ * WT, NT = 32 * WCO * WT * KG;
    ConvKArgs a = ka;
    a.XS = round_up(T_T + (a.K - 1) * a.dil, 4);
    size_t smem = (size_t)KG * (2 * CIC * a.XS + 2 * CIC * a.K * CO_T) * sizeof(float);
    if (KG > 1) smem = std::max(smem, (size_t)(KG - 1) * (CJ / 2) * TJ * (NT / KG) * sizeof(u64));
    B200_REQUIRE(smem <= 227 * 1024, "conv1d: K=%d dil=%d needs %zu B of shared memory", a.K, a.dil, smem);
    static DeviceOnce attr_once;   // one per template instantiation
    if (int rc = device_once(attr_once, nullptr, [](int) -> int {
            B200_CUDA_OK(cudaFuncSetAttribute(conv1d_kernel<CJ, TJ, WCO, WT, CIC, EPI, KG>,
                                              cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
            return 0;
        })) return rc;
    dim3 grid((a.Tq + T_T - 1) / T_T, RowsPad / CO_T, B);
    B200_REQUIRE(grid.y <= 65535 && grid.z <= 65535, "conv1d: grid too large");
    conv1d_kernel<CJ, TJ, WCO, WT, CIC, EPI, KG><<<grid, NT, smem, st>>>(a);
    count_launch();
    dispatch_note(EPI == KEPI_WAVEGRAD ? DISPATCH_FMA_WG + (a.io.near_src > 0 ? 1 : 0) : DISPATCH_FMA);
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

template <int CIC, int EPI>
static int launch_tiles(const ConvKArgs& a, int co_tile, int B, int RowsPad, cudaStream_t st) {
    const bool small_t = a.Tq <= 128;
    if (co_tile == 64) {
        if constexpr (EPI == KEPI_PLAIN) {
            // launch-starved shape (fewer CTAs than SMs, long channel loop): split the channel chunks over 4 warp groups
            const long long ctas = (long long)((a.Tq + 63) / 64) * (RowsPad / 64) * B;
            const int nchunks = (a.Cin + CIC - 1) / CIC;
            const size_t smem4 = (size_t)4 * (2 * CIC * round_up(64 + (a.K - 1) * a.dil, 4) + 2 * CIC * a.K * 64) * sizeof(float);
            if (small_t && ctas <= 160 && nchunks >= 8 && smem4 <= 200 * 1024)
                return launch_variant<16, 2, 4, 1, CIC, EPI, 4>(a, B, RowsPad, st);
        }
        if (small_t) return launch_variant<16, 2, 4, 1, CIC, EPI>(a, B, RowsPad, st);
        return launch_variant<16, 4, 4, 2, CIC, EPI>(a, B, RowsPad, st);
    }
    if (small_t) return launch_variant<16, 2, 2, 2, CIC, EPI>(a, B, RowsPad, st);
    return launch_variant<16, 4, 2, 4, CIC, EPI>(a, B, RowsPad, st);
}

template <int EPI>
static int launch_cic(const ConvKArgs& a, int co_tile, int B, int RowsPad, cudaStream_t st) {
    // keep the work per pipeline stage roughly constant: CIC * K ~ 48..112 tap-steps
    if (a.K >= 9) return launch_tiles<8, EPI>(a, co_tile, B, RowsPad, st);
    return launch_tiles<16, EPI>(a, co_tile, B, RowsPad, st);
}

// ------------------------------------------------------------------ dispatch log (debug / tests)
static thread_local std::vector<int> t_dispatch;
static thread_local bool t_dispatch_on = false;
void dispatch_begin() { t_dispatch.clear(); t_dispatch_on = true; }
int dispatch_end(int* ids, int cap) {
    if (!t_dispatch_on) return 0;
    const int n = (int)t_dispatch.size();
    for (int i = 0; i < n && i < cap; ++i) ids[i] = t_dispatch[i];
    t_dispatch.clear();
    t_dispatch_on = false;
    return n;
}
void dispatch_note(int id) { if (t_dispatch_on) t_dispatch.push_back(id); }

// tensor-core path: returns -1 when the layer / shape / epilogue is not eligible (caller falls through to the FMA kernel)
// Per-device state of the tensor-core path: the pipeline-timeout flag lives in mapped pinned host memory (the kernels
// write it with a system-scope store), so every later launch on that device reads it WITHOUT a synchronisation and
// fails loudly instead of returning garbage audio.
struct TcDevice { int* err = nullptr; int num_sms = 0; int max_smem = 0; };
static TcDevice g_tc_dev[MAX_DEVICES];
static DeviceOnce g_tc_once;

// launch with programmatic stream serialization: the kernel may be scheduled while its predecessor drains (the kernel
// itself waits with griddepcontrol.wait before touching activations).
static cudaError_t launch_tc3(tc3::Tc3Kernel k, int grid, size_t smem, cudaStream_t st, const tc3::Tc3Args& t) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(tc3::NTHREADS2);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, k, t);
}
// ragged batches: the prefix table lives behind everything else in dynamic shared memory (when it still fits)
static void set_ragged(tc3::Tc3Args& t, size_t& smem, size_t max_smem) {
    if (!t.io.lens) return;
    const size_t off = (smem + 15) / 16 * 16, extra = tc3::ragged_table_bytes(t.io.B);
    if (off + extra > max_smem) {                   // enormous batch: fall back to the dense schedule (still correct)
        t.io.lens = nullptr;
        return;
    }
    t.pref_off = (int)off;
    smem = off + extra;
}
// column window: the window's tiles per row on the full call's tile grid (the whole tensor by default)
static void set_window(tc3::Tc3Args& t) {
    // the grouped mode's zero-padded taps (K not a multiple of GRP) read past the conv's reach: 0 * stale scratch must
    // not reach the window (NaN), so the input extent also stops where its producer's window ends
    t.io.Tin = std::min(t.io.Tin, t.io.in_hi);
    t.t_lo = t.io.q_lo / t.tstep;
    const int hi = std::min(t.Tq, t.io.q_hi);
    t.n_ttiles = std::max(0, (hi + t.tstep - 1) / t.tstep - t.t_lo);
}

static int tc_device_init(int d) {
    int smem_optin = 0;
    B200_CUDA_OK(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, d));
    for (int p : {tc::PREC_FP32, tc::PREC_BF16, tc::PREC_FP16, tc::PREC_F16X3}) {
        for (bool lean : {true, false})
            B200_CUDA_OK(cudaFuncSetAttribute(tc3::plain_kernel(p, lean), cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin));
        B200_CUDA_OK(cudaFuncSetAttribute(tc3::plain_kernel(p, true, true), cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin));
        for (int g : {2, 4})
            for (bool refl : {false, true}) {
                if (p != tc::PREC_F16X3)
                    B200_CUDA_OK(cudaFuncSetAttribute(tc3::grouped_kernel(g, p, refl), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                      smem_optin));
                else
                    for (int tms : {1, 2})
                        B200_CUDA_OK(cudaFuncSetAttribute(tc3::timemajor_kernel(tc3::MROWS / g, tms, refl),
                                                          cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin));
            }
        for (bool near : {false, true})
            if (tc3::wavegrad_kernel(p, near))
                B200_CUDA_OK(cudaFuncSetAttribute(tc3::wavegrad_kernel(p, near), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                  smem_optin));
    }
    B200_CUDA_OK(cudaFuncSetAttribute(tc3::bn_kernel(), cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin));
    int* flag = nullptr;   // [0] pipeline timeout, [tc::ERR_RANGE] fp16 range (PREC_F16X3)
    B200_CUDA_OK(cudaHostAlloc((void**)&flag, 2 * sizeof(int), cudaHostAllocMapped | cudaHostAllocPortable));
    flag[0] = flag[tc::ERR_RANGE] = 0;
    g_tc_dev[d].err = flag;    // unified addressing: the host pointer is valid on the device
    g_tc_dev[d].max_smem = smem_optin;
    B200_CUDA_OK(cudaDeviceGetAttribute(&g_tc_dev[d].num_sms, cudaDevAttrMultiProcessorCount, d));
    return 0;
}

int tc_device(int** err, int* num_sms, size_t* max_smem) {
    int dev = 0;
    if (int rc = device_once(g_tc_once, &dev, tc_device_init)) return rc;
    int* const g_tc_err = g_tc_dev[dev].err;
    B200_REQUIRE(*reinterpret_cast<volatile int*>(g_tc_err) == 0,
                 "tensor-core conv: an earlier launch on device %d hit a pipeline timeout (its output is invalid)", dev);
    // a range error is reported once, by the next launch: the data was out of range, the device state is fine
    volatile int* const range_err = reinterpret_cast<volatile int*>(g_tc_err + tc::ERR_RANGE);
    if (*range_err) {
        *range_err = 0;
        B200_REQUIRE(false, "tensor-core conv: an earlier split-fp16 launch on device %d read an activation with |x| >= 65504, "
                            "outside fp16's range (its output is invalid; B200TTS_PRECISION_TF32X3 takes such models)", dev);
    }
    *err = g_tc_err;
    if (num_sms) *num_sms = g_tc_dev[dev].num_sms;
    if (max_smem) *max_smem = (size_t)g_tc_dev[dev].max_smem;
    return 0;
}

static int try_launch_tc(const ConvLayer& L, const ConvKArgs& a, cudaStream_t st) {
    const ConvIO& io = a.io;
    if (L.tc_prec == TC_NONE || a.Tq < 128) return -1;
    if (io.act == ACT_LOGCLAMP || io.act == ACT_TANH) return -1;
    if (!(io.in_slope >= 0.f && io.in_slope <= 1.f)) return -1;   // the producers' leaky ReLU is max(x, slope * x)
    const bool needs_v3 = (io.flags & (EPI_MASK_PRE | EPI_SPLIT | EPI_ACCUM2 | EPI_GATE)) != 0;
    int* g_tc_err = nullptr;
    int num_sms = 0;
    size_t max_smem = 0;
    if (int rc = tc_device(&g_tc_err, &num_sms, &max_smem)) return rc;
    // persistent kernels: 16-byte aligned activation rows for the cp.async staging, no input mask
    const bool persistent_ok = io.x.aligned16() && !io.xmask &&
                               (L.ups == 1 || (!io.res && !(io.flags & EPI_ACCUM) && !io.ymask && !io.cond));
    auto fits = [&](int rp) { return rp <= 320 && tc3::smem_bytes3(rp, L.tc_prec) <= max_smem; };
    // grouped mode for the layers with a grouped image: M = tap groups x channels, N = 256 time steps, 240 per tile
    const int G = L.tc_grp, J = G ? (L.K + G - 1) / G : 0;
    const int rp_grouped = (tc3::TT2 + (J - 1) * G * L.dil + 7) / 8 * 8;
    const bool wg = (io.flags & EPI_WAVEGRAD) != 0;   // WaveGrad epilogue / resampled input: conv1d_tc3w_kernel
    if (wg && !tc3::wavegrad_kernel(L.tc_prec, false)) return -1;
    const bool bn = (io.flags & EPI_WINDOW) || io.aff_s;   // Conv1dBN: conv1d_tc3bn_kernel, plain mode, 3xTF32 only
    if (bn && L.tc_prec != tc::PREC_FP32) return -1;
    const bool grouped = G && !wg && !bn && !needs_v3 && !io.ymask && (G - 1) * L.dil <= 15 && a.Tq >= 256 && fits(rp_grouped);
    // plain mode otherwise: M = rows (128 per tile, zero padded), N = 256 time steps.  Everything neither mode takes
    // (unaligned or masked inputs, shared-memory budget) runs on the exact FP32-FMA kernel.
    // At PREC_F16X3 the grouped layers run on the time-major kernel (M = time, N = the 32 / 64 channels): 256-column tiles,
    // or 128 where a 256-column window (tile + reach) would not fit the 320 staging rows or, with room for a ragged
    // prefix table of 255 rows, shared memory.  The width is fixed per layer, so every column takes the same sum whatever
    // its tile origin (ragged / windowed calls match the dense one bit for bit).
    const bool tm = grouped && L.tc_prec == tc::PREC_F16X3;
    const int reach = (L.K - 1) * L.dil, rp256 = (tc3::TT2 + reach + 7) / 8 * 8;
    const int tm_slices = rp256 <= 320 && tc3::smem_bytes_tm(rp256, L.Rows, 2) + 1024 <= max_smem ? 2 : 1;   // per warpgroup
    const int rows_pad = tm ? (128 * tm_slices + reach + 7) / 8 * 8
                            : grouped ? rp_grouped : rp256;
    if (!persistent_ok || !fits(rows_pad)) return -1;
    tc3::Tc3Args t{a};
    t.w_tc = grouped ? L.w_tcg : L.w_tc; t.rscale = L.tc_rscale;
    t.KJ = grouped && !tm ? J : L.K; t.dil_blk = grouped && !tm ? G * L.dil : L.dil;
    t.tstep = tm ? 128 * tm_slices : grouped ? tc3::TSTEP_GROUPED : tc3::TT2;
    t.rows_pad = rows_pad; t.raw_w = rows_pad + 4;
    t.n_rtiles = (L.Rows + tc3::MROWS - 1) / tc3::MROWS;   // 1 in grouped mode (32 / 64 rows)
    set_window(t);
    t.err = g_tc_err;
    size_t smem = tm ? tc3::smem_bytes_tm(rows_pad, L.Rows, tm_slices) : tc3::smem_bytes3(rows_pad, L.tc_prec);
    set_ragged(t, smem, max_smem);
    // plain layers (bias, residual, accumulate): the kernel with the lean epilogue; everything else (WaveNet gate / split,
    // masks, ReLU, scale, final divide, transposed convs) the one with the general epilogue inline
    const bool plain_epi = L.ups == 1 && !(io.flags & EPI_GATE) && io.split == 0 && io.act != ACT_RELU && !io.ymask &&
                           io.scale == 1.f && io.post_div == 1.f && !bn;
    const bool reflect = io.reflect != 0;   // reflection padding: the lean kernels' reflect variants only
    if (reflect && !grouped && !plain_epi) return -1;
    const tc3::Tc3Kernel k = wg ? tc3::wavegrad_kernel(L.tc_prec, io.near_src > 0)
                                : bn      ? tc3::bn_kernel()
                                : tm      ? tc3::timemajor_kernel(L.Rows, tm_slices, reflect)
                                : grouped ? tc3::grouped_kernel(G, L.tc_prec, reflect)
                                          : tc3::plain_kernel(L.tc_prec, plain_epi, reflect);
    const long long tiles = (long long)io.B * t.n_ttiles * t.n_rtiles;
    const int grid = (int)std::max(1LL, tiles < num_sms ? tiles : num_sms);
    B200_CUDA_OK(launch_tc3(k, grid, smem, st, t));
    count_launch();
    const bool b16 = L.tc_prec == tc::PREC_BF16 || L.tc_prec == tc::PREC_FP16;   // PREC_F16X3 logs as tc3
    if (wg)
        dispatch_note((L.tc_prec == tc::PREC_F16X3 ? DISPATCH_TC3W_F16X3 : DISPATCH_TC3W_TF32) + (io.near_src > 0 ? 1 : 0));
    else
        dispatch_note(grouped ? (b16 ? DISPATCH_TC16_GROUPED : DISPATCH_TC3_GROUPED) : (b16 ? DISPATCH_TC16 : DISPATCH_TC3));
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

// 1 if any tensor-core launch (on any device) hit a pipeline timeout, 2 if one read an activation outside fp16's range
// (PREC_F16X3), 3 for both; call after a sync
int conv_tc_error_flag() {
    int f = 0;
    for (int d = 0; d < MAX_DEVICES; ++d) {
        if (!g_tc_dev[d].err) continue;
        const volatile int* e = g_tc_dev[d].err;
        if (e[0]) f |= 1;
        if (e[tc::ERR_RANGE]) f |= 2;
    }
    return f;
}

int launch_conv(const ConvLayer& L, const ConvIO& call, cudaStream_t st) {
    B200_REQUIRE(L.w && call.x && call.y, "launch_conv: null tensor");
    ConvKArgs a{call};
    ConvIO& io = a.io;   // normalised here, so that every kernel family reads the same options
    io.q_lo = std::max(0, io.q_lo);
    io.in_lo = std::max(0, io.in_lo);
    if (io.near_src > 0) io.flags |= EPI_WAVEGRAD;
    if (!(io.flags & EPI_SPLIT)) io.split = 0;   // the tensor-core epilogues test split > 0, the FMA kernel the flag
    a.w = L.w; a.bias = L.bias;
    a.Cin = L.Cin; a.CinPad = L.CinPad; a.K = L.K; a.dil = L.dil; a.pad = L.pad; a.Rows = L.Rows; a.ups = L.ups;
    a.Tq = (L.ups > 1) ? (io.Tout + L.ups - 1) / L.ups : io.Tout;
    a.near_scale = io.near_src > 0 ? (float)io.near_src / (float)io.Tin : 1.f;
    const bool windowed = io.q_lo > 0 || io.q_hi < a.Tq;
    if (io.reflect) {   // torch's ReflectionPad1d limit; nothing needs reflection together with the options below
        B200_REQUIRE(L.pad <= io.Tin - 1, "launch_conv: reflection padding %d needs at least %d input columns, got %d", L.pad,
                     L.pad + 1, io.Tin);
        B200_REQUIRE(!io.lens && !windowed && io.in_lo == 0 && io.in_hi == 0x7fffffff && L.ups == 1 && !io.xmask,
                     "launch_conv: reflection padding takes no lens, column window, input mask or upsampling");
    }
    if (io.flags & EPI_WAVEGRAD) {   // WaveGrad layers: their own kernel variants (tensor cores, else the FMA tile kernel)
        B200_REQUIRE(L.ups == 1 && !io.lens && !windowed && io.in_lo == 0 && io.in_hi == 0x7fffffff && !io.xmask && !io.ymask &&
                         !io.cond && !io.reflect && io.flags == EPI_WAVEGRAD && io.scale == 1.f && io.post_div == 1.f &&
                         (io.act == ACT_NONE || io.act == ACT_LRELU) && (!io.film || (io.film_half > 0 && io.film.cs > 0)) &&
                         io.near_src >= 0 && !io.aff_s && !io.aff_h,
                     "launch_conv: the WaveGrad epilogue takes only lrelu / act_add / res / y2 / film, on a dense launch");
        if (a.Tq <= 0 || io.B <= 0) return 0;
        if (int rc = try_launch_tc(L, a, st); rc != -1) return rc;
        return launch_cic<KEPI_WAVEGRAD>(a, L.co_tile, io.B, L.RowsPad, st);
    }
    B200_REQUIRE(io.act != ACT_LRELU, "launch_conv: the leaky-ReLU epilogue needs EPI_WAVEGRAD");
    if (a.Tq <= 0 || io.B <= 0) return 0;
    B200_REQUIRE(!(io.flags & (EPI_MASK_PRE | EPI_MASK_POST | EPI_SPLIT)) || io.ymask,
                 "launch_conv: masked/split epilogue needs ymask");
    B200_REQUIRE(!(io.flags & EPI_SPLIT) || io.y2, "launch_conv: split epilogue needs y2");
    B200_REQUIRE(!(io.ymask && L.ups > 1), "launch_conv: output mask with an upsampling layer is not supported");
    // a mask without a flag saying where it applies: the FMA plain epilogue would apply it, the others would not
    B200_REQUIRE(!io.ymask || (io.flags & (EPI_MASK_PRE | EPI_MASK_POST | EPI_SPLIT)),
                 "launch_conv: ymask needs EPI_MASK_PRE, EPI_MASK_POST or EPI_SPLIT");
    if ((io.flags & EPI_WINDOW) || io.aff_s || io.aff_h) {   // Conv1dBN layers: their own kernel variants
        B200_REQUIRE(L.ups == 1 && !io.reflect && !windowed && !io.cond && !(io.flags & (EPI_GATE | EPI_SPLIT | EPI_ACCUM2)) &&
                         (io.act == ACT_NONE || io.act == ACT_RELU) && io.scale == 1.f && io.post_div == 1.f &&
                         !io.aff_s == !io.aff_h && io.edge_lo >= 0 && io.edge_hi >= 0,
                     "launch_conv: the Conv1dBN epilogue takes a window, relu, an affine, masks, res and accumulate, on an "
                     "unwindowed launch without conditioning");
        if (int rc = try_launch_tc(L, a, st); rc != -1) return rc;
        return launch_cic<KEPI_BN>(a, L.co_tile, io.B, L.RowsPad, st);
    }
    if (io.flags & EPI_GATE) {
        B200_REQUIRE(L.ups == 1 && !io.res && !io.ymask && io.act == ACT_NONE && io.flags == EPI_GATE && io.scale == 1.f &&
                         io.post_div == 1.f,
                     "launch_conv: gate epilogue takes no other options");
        if (int rc = try_launch_tc(L, a, st); rc != -1) return rc;
        return launch_cic<KEPI_GATE>(a, L.co_tile, io.B, L.RowsPad, st);
    }
    if (io.act == ACT_TANH) {
        B200_REQUIRE(L.ups == 1 && !io.res && !io.cond && io.flags == 0 && io.scale == 1.f && io.post_div == 1.f,
                     "launch_conv: tanh epilogue takes no other options");
        // conv_post (one output row, 7 taps): streaming kernel when rows are 16-byte aligned
        if (L.Rows == 1 && L.K == 7 && L.dil == 1 && L.pad == 3 && !io.xmask && io.Tin == io.Tout && (io.Tout % 4) == 0 &&
            io.x.aligned16() && (io.y.bs % 4) == 0 && (reinterpret_cast<uintptr_t>(io.y.p) & 15) == 0 &&
            (size_t)L.Cin * L.K * 4 <= 48 * 1024) {
            const int blk_lo = io.q_lo / 1024, blk_hi = (std::min(io.q_hi, io.Tout) + 1023) / 1024;   // 1024 samples per CTA
            dim3 grid(std::max(1, blk_hi - blk_lo), io.B);
            if (grid.y <= 65535) {
                auto kern = io.reflect ? conv1d_row1_kernel<7, true> : conv1d_row1_kernel<7, false>;
                kern<<<grid, 256, (size_t)L.Cin * L.K * 4, st>>>(a, L.co_tile, blk_lo);
                count_launch();
                dispatch_note(DISPATCH_ROW1);
                B200_CUDA_OK(cudaGetLastError());
                return 0;
            }
        }
        if (int rc = launch_cic<KEPI_TANH>(a, L.co_tile, io.B, L.RowsPad, st)) return rc;
        if (io.peak_bits) {   // the streaming kernel was not eligible: fold the peak in a pass of its own
            B200_REQUIRE(io.y.cs == io.Tout && io.y.bs == (long long)L.Rows * io.Tout, "launch_conv: peak needs a dense output");
            if (windowed)   // only the samples this launch stored
                return launch_absmax_window(io.y.p, io.B * L.Rows, io.Tout, io.q_lo, std::min(io.q_hi, io.Tout), io.peak_bits, st);
            return launch_absmax(io.y.p, (long long)io.B * L.Rows * io.Tout, io.peak_bits, st);
        }
        return 0;
    }
    if (int rc = try_launch_tc(L, a, st); rc != -1) return rc;
    const bool plain = L.ups == 1 && !io.res && io.scale == 1.f && io.post_div == 1.f &&
                       (io.flags & ~(EPI_MASK_POST | EPI_MASK_PRE)) == 0;
    if (plain) return launch_cic<KEPI_PLAIN>(a, L.co_tile, io.B, L.RowsPad, st);
    B200_REQUIRE(io.act != ACT_LOGCLAMP, "launch_conv: log-clamp activation only with the plain epilogue");
    return launch_cic<KEPI_GENERIC>(a, L.co_tile, io.B, L.RowsPad, st);
}

}  // namespace b200tts
