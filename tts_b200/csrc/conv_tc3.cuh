// Persistent Hopper wgmma 3xTF32 conv1d: M = output rows (weights are the A operand), N = 256 time steps (the activation
// window is the B operand).  Tap k of a chunk is the same staged activation tile with its descriptor start address
// advanced by k*dil rows (16 B each), see conv_tc.cuh.
//
//   warps 0-7   consumers : two warpgroups, each D[64 rows x 256 time steps] in registers (wgmma m64n256k8, 3 MMAs per tap
//                           and chunk: lo*hi, hi*lo, hi*hi; one tap's group in flight while the next is issued).  After the last chunk of a tile both warpgroups store their
//                           accumulators to a shared [128][ACC_LD] tile and all eight warps run the epilogue from it
//                           (warp w: rows 32 (w & 3) .. + 31, columns 128 (w >> 2) .. + 127).  A warpgroup starts the next
//                           tile's MMAs as soon as its own epilogue is done; the tile is only rewritten after both are.
//   warps 8-10  producers : cp.async raw [8 ch][time] windows (NRAW-deep ring) -> leaky-ReLU + hi/lo split -> K-major slabs
//                           (NA2 stages)
//   warp  11    loader    : per-tap weight blocks {hi,lo}[2 slabs][128 rows][4] by cp.async.bulk, one lane per ring slot
//
// PREC (compile time) = PREC_BF16 / PREC_FP16: 16-bit operands with fp32 accumulation.  A chunk is 16 input channels: the
// producers stage them as two 8-channel cp.async slots of one raw ring stage, apply the leaky ReLU and round to the
// 16-bit type into two slabs [rows][8] (no hi/lo split); the loader streams tap blocks [2 slabs][128 rows][8] (4 KB); the
// consumers issue one m64n256k16 MMA per tap and chunk.  Epilogues, residuals and every tensor in global memory stay
// fp32.  Shared memory: the raw ring doubles (+31 KB), the activation stages and weight slots halve (-20 KB, -12 KB).
//
// Grouped mode (GRP = 2 / 4) for narrow layers (exactly 64 / 32 output rows, the last two HiFiGAN stages): the 128
// MMA rows are GRP tap-groups x (128/GRP) channels -- row g * (128/GRP) + c carries the weights of channel c for taps
// g, g+GRP, g+2*GRP, ... so one instruction stream of ceil(K/GRP) "tap blocks" (B shifted by GRP*dil rows per block)
// replaces K of them and no MMA row is zero padding.  D_g[c, col] then still misses its own g*dil shift: the epilogue
// reads row g * (128/GRP) + c at column col + g*dil and sums the GRP partials.  Tiles advance by 240 columns so every
// shifted read stays inside the 256-column accumulator.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "conv_tc.cuh"   // descriptor / barrier / wgmma helpers

namespace b200tts {
namespace tc3 {

using namespace tc;       // smem_u32, mbar_*, make_desc, wgmma_*

constexpr int TT2 = 256;          // time steps per tile = MMA N
constexpr int MROWS = 128;        // output rows per tile (weight rows are zero padded up to it): two m64 warpgroups
constexpr int KC2 = 8;            // input channels per chunk (2 slabs, one MMA k-step)
constexpr int KC16 = 16;          // input channels per chunk with 16-bit operands (2 slabs, one k16 step)
constexpr int RAWS = 324;         // raw (cp.async) row stride in floats: the widest window (320 slab rows + 4), a constant so
                                  // that the transform's shared loads use immediate offsets
constexpr int NRAW = 3;           // raw (cp.async) ring depth
constexpr int NA2 = 2;            // transformed activation stages
constexpr int NB2 = 3;            // weight ring depth (one 8 KB tap block per slot)
constexpr int ACC_LD = 260;       // row stride (floats) of the shared accumulator tile: float4 reads of 8 rows are conflict free
constexpr int ACC_BYTES = MROWS * ACC_LD * 4;
constexpr int NPW = 3;            // producer warps
constexpr int NPROD = 32 * NPW;
constexpr int NCONS = 256;        // consumer threads (two warpgroups)
constexpr int W_PROD = 8, W_LOAD = 8 + NPW;
constexpr int NTHREADS2 = 32 * (W_LOAD + 1);

struct Tc3Args {
    const float* x; long long x_bs; int x_cs; int Tin;
    float in_slope;
    const void* w;             // packed [row_tile][chunk][tap]{hi[2][128][4], lo[2][128][4]} fp32 (16-bit: [2][128][8])
    const float* bias;
    const float* cond; long long cond_bs;
    int Cin, K, dil, pad, Rows, N;
    float* y; long long y_bs; int y_cs; int Tout;
    int ups;                   // 1, or the polyphase factor of a transposed conv (row r -> channel r/ups, phase r%ups)
    int Tq;                    // GEMM columns in time (= Tout for ups == 1)
    const float* res; long long res_bs; int res_cs;
    const float* ymask; long long ymask_bs;
    float scale; float post_div; int relu; int accum; int mask_post;
    int mask_pre;              // multiply by ymask before the residual / accumulate (coupling `post`)
    int gate;                  // rows are (tanh, sigmoid) pairs: out[r/2] = tanh(v[2p]) * sigmoid(v[2p+1])  (WaveNet)
    int split;                 // > 0: rows < split -> y (accumulate, mask); rows >= split -> y2 (accumulate iff accum2)
    float* y2; long long y2_bs; int y2_cs; int accum2;
    int KJ;                    // tap blocks per chunk (= K, or ceil(K / GRP) in grouped mode)
    int dil_blk;               // B-row shift between tap blocks (= dil, or GRP * dil)
    int tstep;                 // time steps a tile advances (= TT2, or 240 in grouped mode)
    int rows_pad;              // slab rows  (TT2 + halo, multiple of 8)
    int raw_w;                 // raw row width in floats (rows_pad + 4, multiple of 4)
    int B, n_ttiles, n_rtiles;
    int* err;
    // ---- ragged batches (null lens: every row spans the full tensor).  Row b only has tiles for GEMM columns below
    // min(Tq, lens[b] * rate_q + need_q) and its input is read as zero from min(Tin, lens[b] * rate_in + need_in) on:
    // padded frames cost nothing, and `need` keeps every sample below lens[b] bit-identical to the full computation
    // (it is the receptive field of the layers that still follow, worked out per launch by the engine).
    const int* lens; int rate_q, need_q, rate_in, need_in;
    int pref_off;               // byte offset in dynamic shared memory of the (B + 1)-entry tile prefix table
    // ---- column window (default [0, INT_MAX), in_lo 0: the whole tensor).  A row's tiles run from floor(q_lo / tstep) to
    // ceil(min(extent, q_hi) / tstep); tile origins stay multiples of tstep counted from column 0, so every column is
    // computed (and takes the same epilogue) as in the unwindowed launch.  Input columns below in_lo are stale scratch
    // and read as zero (whole 16-byte vectors: the ones below in_lo rounded down to a multiple of 4); the host stops Tin
    // where the producer's window ends, so the grouped mode's zero-padded taps never multiply stale data.  n_ttiles counts
    // the window's tiles per row (dense schedule), t_lo = floor(q_lo / tstep) is the first one.
    int q_lo, q_hi, in_lo, t_lo;
};

// prec: PREC_FP32 (8-channel chunks, hi/lo slab pairs) or a 16-bit type (16-channel chunks, two slabs)
static inline size_t smem_bytes3(int rows_pad, int prec = PREC_FP32) {
    const size_t kch = prec ? KC16 : KC2, nsl = prec ? 2 : 4;
    return (size_t)NRAW * kch * RAWS * 4 + (size_t)NA2 * (nsl * rows_pad * 16) + (size_t)NB2 * (nsl * MROWS * 16) + ACC_BYTES + 512;
}
static inline size_t ragged_table_bytes(int B) { return ((size_t)(B + 1) * sizeof(int) + 15) / 16 * 16; }

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async16_zfill(uint32_t dst, const void* src, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async4_zfill(uint32_t dst, const void* src, uint32_t src_bytes) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
// 16 consecutive accumulator columns of one row of the shared accumulator tile
__device__ __forceinline__ void acc_ld16(const float* p, float* v) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float4 t = *reinterpret_cast<const float4*>(p + 4 * j);
        v[4 * j] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w;
    }
}

constexpr int TSTEP_GROUPED = 240;   // 15 chunks of 16 columns: leaves room for the (GRP-1)*dil <= 15 column shift

// Lean epilogue of one interior tile half (plain layers: bias, optional residual HR / accumulate HA).  Lane (r8 = lane & 7,
// p4 = lane >> 3) owns float4 p4 of rows 8 i + r8 of the warp's 32 rows, so every global instruction covers 8 rows x 64
// contiguous bytes; padding rows (>= Rows) have their loads clamped to the last real row and their stores switched off.
// HR / HA are compile-time so that every load is an unconditional definition; the residual of the next 16-column group
// is in flight while the current one is finished.  ((acc + bias) + res) + old, as in the general code.
template <bool HR, bool HA>
__device__ __forceinline__ void lean_tile(const float* at, const float* bias, const float* cond, int lane, const float* rq,
                                          float* yq, long long rcs, long long ycs, int row0, int Rows, bool do_st) {
    const int r8 = lane & 7, p4 = lane >> 3;
    const float* rrow[4];
    float* yrow[4];
    bool st_ok[4];
    float bv[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int ri = row0 + 8 * i + r8, rci = ri < Rows ? ri : Rows - 1;
        rrow[i] = rq + (long long)rci * rcs + 4 * p4;
        yrow[i] = yq + (long long)rci * ycs + 4 * p4;
        st_ok[i] = do_st && ri < Rows;
        bv[i] = bias[rci];
        if (cond) bv[i] += __ldg(cond + rci);
    }
    const float* ap = at + r8 * ACC_LD + 4 * p4;
    float r0[16], r1[16];
    auto pf = [&](int cg, float* r_) {
        if constexpr (HR) {
#pragma unroll
            for (int i = 0; i < 4; ++i)
                asm volatile("ld.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r_[4 * i]), "=f"(r_[4 * i + 1]), "=f"(r_[4 * i + 2]), "=f"(r_[4 * i + 3]) : "l"(rrow[i] + cg));
        }
    };
    auto group = [&](int cg, const float* rv, float* rn) {
        float o[16];
        if (cg + 16 < 128) pf(cg + 16, rn);
        if constexpr (HA) {
#pragma unroll
            for (int i = 0; i < 4; ++i)
                asm volatile("ld.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(o[4 * i]), "=f"(o[4 * i + 1]), "=f"(o[4 * i + 2]), "=f"(o[4 * i + 3]) : "l"(yrow[i] + cg));
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            float4 t = *reinterpret_cast<const float4*>(ap + 8 * i * ACC_LD + cg);
            t.x += bv[i]; t.y += bv[i]; t.z += bv[i]; t.w += bv[i];
            if constexpr (HR) { t.x += rv[4 * i]; t.y += rv[4 * i + 1]; t.z += rv[4 * i + 2]; t.w += rv[4 * i + 3]; }
            if constexpr (HA) { t.x += o[4 * i]; t.y += o[4 * i + 1]; t.z += o[4 * i + 2]; t.w += o[4 * i + 3]; }
            if (st_ok[i]) *reinterpret_cast<float4*>(yrow[i] + cg) = t;
        }
    };
    pf(0, r0);
#pragma unroll 1
    for (int cg = 0; cg < 128; cg += 32) {
        group(cg, r0, r1);
        group(cg + 16, r1, r0);
    }
}

// Everything the lean epilogue does not cover (WaveNet gate / res-skip split, masks, ReLU, scale, final divide, polyphase
// stores of the transposed convs, edge tiles): one tile half per call, lane = one output row, `arow` = its accumulators.
__device__ __forceinline__ void general_tile_body(const Tc3Args& a, const float* arow, int b, int rt, int q0, int lq, int half,
                                                  int lane) {
    const int ups = a.ups;
    const int r = rt * MROWS + lq * 32 + lane;             // GEMM row of this lane
    const bool rok = r < a.Rows;
    const int rc = rok ? r : a.Rows - 1;
    const int qb = q0 + half * 128;
    float bias = a.bias[rc];
    if (a.cond) bias += __ldg(a.cond + (long long)b * a.cond_bs + rc);
    if (a.gate) {
        // WaveNet gate (wavenet.py:6-13): even lane = tanh argument, odd lane = sigmoid argument of row r/2
        float* yrow = a.y + (long long)b * a.y_bs + (long long)(rc >> 1) * a.y_cs;
        const bool vec_ok = ((a.y_cs & 3) == 0) && ((reinterpret_cast<uintptr_t>(yrow) & 15) == 0);
        const bool even = (lane & 1) == 0;
        for (int cg = 0; cg < 128; cg += 16) {
            float v[16];
            acc_ld16(arow + cg, v);
            const int q = qb + cg;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const float u = v[i] + bias;
                const float act = even ? tanhf(u) : 1.f / (1.f + expf(-u));
                const float other = __shfl_xor_sync(0xffffffffu, act, 1);
                v[i] = act * other;
            }
            if (rok && even) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int qq = q + 4 * j;
                    if (vec_ok && qq + 3 < a.Tout) *reinterpret_cast<float4*>(yrow + qq) = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
                    else {
#pragma unroll
                        for (int e = 0; e < 4; ++e) if (qq + e < a.Tout) yrow[qq + e] = v[4 * j + e];
                    }
                }
            }
        }
    } else if (ups == 1) {
        float* yrow = a.y + (long long)b * a.y_bs + (long long)rc * a.y_cs;
        bool acc_r = a.accum != 0, mpost_r = a.mask_post != 0;
        if (a.split > 0) {          // WaveNet res/skip rows (wavenet.py:108-113)
            if (rc < a.split) { acc_r = true; mpost_r = true; }
            else { yrow = a.y2 + (long long)b * a.y2_bs + (long long)(rc - a.split) * a.y2_cs; acc_r = a.accum2 != 0; mpost_r = false; }
        }
        const float* rrow = a.res ? a.res + (long long)b * a.res_bs + (long long)rc * a.res_cs : nullptr;
        const float* mrow = a.ymask ? a.ymask + (long long)b * a.ymask_bs : nullptr;
        const int ycs_eff = (a.split > 0 && rc >= a.split) ? a.y2_cs : a.y_cs;
        const bool vec_ok = ((ycs_eff & 3) == 0) && (!a.res || (a.res_cs & 3) == 0) &&
                            ((reinterpret_cast<uintptr_t>(yrow) & 15) == 0) &&
                            (!rrow || (reinterpret_cast<uintptr_t>(rrow) & 15) == 0);
        // software pipeline: the (volatile) loads of group j+1 are issued before group j is finished, into the OTHER of
        // two register sets -- never copied (a move of a pending load's result waits for the load).
        float rA[16], oA[16], rB[16], oB[16];
        auto prefetch = [&](int cg, float* r_, float* o_) {
            const int q = qb + cg;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int qq = q + 4 * j;
                if (vec_ok && qq + 3 < a.Tout) {
                    if (rrow) asm volatile("ld.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r_[4 * j]), "=f"(r_[4 * j + 1]), "=f"(r_[4 * j + 2]), "=f"(r_[4 * j + 3]) : "l"(rrow + qq));
                    if (acc_r) asm volatile("ld.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(o_[4 * j]), "=f"(o_[4 * j + 1]), "=f"(o_[4 * j + 2]), "=f"(o_[4 * j + 3]) : "l"(yrow + qq));
                } else {
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const int qe = min(qq + e, a.Tout - 1);
                        if (rrow) asm volatile("ld.global.f32 %0, [%1];" : "=f"(r_[4 * j + e]) : "l"(rrow + qe));
                        if (acc_r) asm volatile("ld.global.f32 %0, [%1];" : "=f"(o_[4 * j + e]) : "l"(yrow + qe));
                    }
                }
            }
        };
        auto group = [&](int cg, const float* rv, const float* ov, float* rn, float* on) {
            float v[16];
            if (rok && cg + 16 < 128) prefetch(cg + 16, rn, on);
            acc_ld16(arow + cg, v);
            const int q = qb + cg;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                float u = v[i] + bias;
                if (a.relu) u = fmaxf(u, 0.f);
                const float mk = mrow ? __ldg(mrow + min(q + i, a.Tout - 1)) : 1.f;
                if (a.mask_pre) u *= mk;
                if (a.res) u += rv[i];
                u *= a.scale;
                if (acc_r) u += ov[i];
                if (a.post_div != 1.f) u = u / a.post_div;
                if (mpost_r) u *= mk;
                v[i] = u;
            }
            if (rok) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int qq = q + 4 * j;
                    if (vec_ok && qq + 3 < a.Tout) {
                        *reinterpret_cast<float4*>(yrow + qq) = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
                    } else {
#pragma unroll
                        for (int e = 0; e < 4; ++e) if (qq + e < a.Tout) yrow[qq + e] = v[4 * j + e];
                    }
                }
            }
        };
        if (rok) prefetch(0, rA, oA);
#pragma unroll 1
        for (int cg = 0; cg < 128; cg += 32) {
            group(cg, rA, oA, rB, oB);
            group(cg + 16, rB, oB, rA, oA);
        }
    } else {
        // polyphase store: row r = co*ups + ph, column q -> y[co][q*ups + ph]; a warp's 32 lanes cover whole
        // groups of `ups` phases, i.e. contiguous runs of `ups` output samples per channel
        if (!rok) return;
        const int co = rc / ups, ph = rc - co * ups;
        float* yrow = a.y + (long long)b * a.y_bs + (long long)co * a.y_cs + ph;
        for (int cg = 0; cg < 128; cg += 16) {
            float v[16];
            acc_ld16(arow + cg, v);
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const int q = qb + cg + i;
                float u = v[i] + bias;
                if (a.relu) u = fmaxf(u, 0.f);
                const long long t = (long long)q * ups;
                if (q < a.Tq && t + ph < a.Tout) yrow[t] = u;
            }
        }
    }
}

// Out-of-line call of the general epilogue for the kernel whose hot path is the lean one (edge tiles only): inlined into
// its tile loop the general code's loop invariants were hoisted across the lean path.  One copy of the arguments per
// call: through the reference every field use would be a generic load.
__device__ __noinline__ void general_tile_call(const Tc3Args& a_ref, const float* arow, int b, int rt, int q0, int lq, int half,
                                               int lane) {
    const Tc3Args a = a_ref;
    general_tile_body(a, arow, b, rt, q0, lq, half, lane);
}

// Grouped epilogue, one tile half: out[c, t] = sum_g D_g[c, t + g*dil] with MMA row m = g * CH + c (CH = 128 / GRP
// channels).  Thread tq of the half's 128 finishes channel co = tq * NQ / 4, float4s j0 .. j0 + NQ - 1 of every
// 16-column group (4 / NQ lanes = 64 contiguous bytes of a channel).
template <int GRP>
__device__ __forceinline__ void grouped_tile(const Tc3Args& a, const float* accs, int b, int q0, int lq, int half, int lane) {
    constexpr int CH = 128 / GRP;              // output channels
    constexpr int NQ = CH / 32;                // float4 per thread and 16-column group (1 or 2)
    constexpr int NV = 4 * NQ;
    const int tq = lq * 32 + lane;
    const int co = (tq * NQ) >> 2;
    const int coff = 4 * ((tq & (4 / NQ - 1)) * NQ);
    const int cbeg = half ? 128 : 0;
    const int cend = half ? a.tstep : min(128, a.tstep);
    const bool has_res = a.res != nullptr, acc_r = a.accum != 0;
    const bool vec_ok = ((a.y_cs & 3) == 0) && ((a.y_bs & 3) == 0) && ((reinterpret_cast<uintptr_t>(a.y) & 15) == 0) &&
                        (!a.res || (((a.res_cs & 3) == 0) && ((a.res_bs & 3) == 0) && ((reinterpret_cast<uintptr_t>(a.res) & 15) == 0)));
    const bool fast = vec_ok && (q0 + a.tstep <= a.Tout);   // interior tile: no bounds checks
    const float* rrow = has_res ? a.res + (long long)b * a.res_bs + (long long)co * a.res_cs : nullptr;
    float* yrow = a.y + (long long)b * a.y_bs + (long long)co * a.y_cs;
    float bias = a.bias[co];
    if (a.cond) bias += __ldg(a.cond + (long long)b * a.cond_bs + co);
    auto load = [&](const float* rr, int q, float* dst) {     // one thread's values of a column group of a row
#pragma unroll
        for (int j = 0; j < NQ; ++j) {
            const int qq = q + 4 * j;
            if (fast || (vec_ok && qq + 3 < a.Tout)) {
                const float4 t = *reinterpret_cast<const float4*>(rr + qq);
                dst[4 * j] = t.x; dst[4 * j + 1] = t.y; dst[4 * j + 2] = t.z; dst[4 * j + 3] = t.w;
            } else {
#pragma unroll
                for (int e = 0; e < 4; ++e) dst[4 * j + e] = rr[min(qq + e, a.Tout - 1)];
            }
        }
    };
#pragma unroll 1
    for (int cg = cbeg; cg < cend; cg += 16) {
        float R[NV], rv[NV], ov[NV];
        if (has_res) load(rrow, q0 + cg + coff, rv);
        if (acc_r) load(yrow, q0 + cg + coff, ov);
        const float* p = accs + co * ACC_LD + cg + coff;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const float p0 = p[i], p1 = p[CH * ACC_LD + a.dil + i];
            float s = p0 + p1;
            if constexpr (GRP == 4) s += p[2 * CH * ACC_LD + 2 * a.dil + i] + p[3 * CH * ACC_LD + 3 * a.dil + i];
            R[i] = s;
        }
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            float u = R[i] + bias;
            if (a.relu) u = fmaxf(u, 0.f);
            if (has_res) u += rv[i];
            u *= a.scale;
            if (acc_r) u += ov[i];
            if (a.post_div != 1.f) u = u / a.post_div;
            R[i] = u;
        }
        const int q = q0 + cg + coff;
#pragma unroll
        for (int j = 0; j < NQ; ++j) {
            const int qq = q + 4 * j;
            if (fast || (vec_ok && qq + 3 < a.Tout)) {
                *reinterpret_cast<float4*>(yrow + qq) = make_float4(R[4 * j], R[4 * j + 1], R[4 * j + 2], R[4 * j + 3]);
            } else {
#pragma unroll
                for (int e = 0; e < 4; ++e) if (qq + e < a.Tout) yrow[qq + e] = R[4 * j + e];
            }
        }
    }
}

template <int GRP, bool LEAN = true, int PREC = PREC_FP32, bool REFL = false>
                                       // GRP: tap groups stacked in the 128 MMA rows (1 = plain); LEAN:
                                       // plain-layer kernel (lean epilogue inline, general one out of line) -- false for the
                                       // WaveNet / masked / transposed layers (general epilogue inline); PREC: operand type;
                                       // REFL: reflection padding (ConvIO::reflect; dense, unwindowed launches only): input
                                       // column t < 0 reads x[-t], t >= Tin reads x[2 Tin - 2 - t].  A compile-time switch so
                                       // that the zero-padding kernels keep their register allocation.
__device__ __forceinline__ void tc3_body(const Tc3Args& a) {
    extern __shared__ __align__(128) unsigned char smem[];
    constexpr int KCH = PREC ? KC16 : KC2;       // input channels per chunk
    constexpr int NSL = PREC ? 2 : 4;            // 16-byte slabs per operand stage: two 16-bit slabs, or hi[2] + lo[2]
    constexpr int SLC = PREC ? 8 : 4;            // channels per slab row
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int ROWS = a.rows_pad, RAWW = a.raw_w, K = a.KJ;
    const uint32_t rawStage = (uint32_t)KCH * RAWS * 4;
    const uint32_t slabA = (uint32_t)ROWS * 16, stageA = NSL * slabA;
    const uint32_t slabB = (uint32_t)MROWS * 16, stageB = NSL * slabB;   // one tap block: [NSL slabs][128 rows][16 B]
    unsigned char* smRaw = smem;
    unsigned char* smA = smRaw + NRAW * rawStage;
    unsigned char* smB = smA + NA2 * stageA;
    float* accs = reinterpret_cast<float*>(smB + NB2 * stageB);
    uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<unsigned char*>(accs) + ACC_BYTES);
    const int A_FULL = 0, A_EMPTY = NA2, B_FULL = 2 * NA2, B_EMPTY = 2 * NA2 + NB2;
    const uint32_t bar0 = smem_u32(bars);
    auto BAR = [&](int i) { return bar0 + 8u * (uint32_t)i; };

    const int nchunks = (a.Cin + KCH - 1) / KCH;
    const bool ragged = a.lens != nullptr;
    int* pref = reinterpret_cast<int*>(smem + a.pref_off);    // pref[b] = first tile of row b (ragged only)
    if (ragged) {
        // tiles per row from its own length; exclusive prefix by warp 0 (rows in lane-contiguous chunks).  `lens` was
        // written several launches ago (durations kernel), so reading it before griddepcontrol.wait is safe.
        for (int b = tid; b < a.B; b += NTHREADS2) {
            const long long e = (long long)a.lens[b] * a.rate_q + a.need_q;
            const int ext = (int)(e < (long long)a.Tq ? (e > 0 ? e : 0) : (long long)a.Tq);
            const int t_hi = (min(ext, a.q_hi) + a.tstep - 1) / a.tstep;
            pref[b + 1] = max(0, t_hi - a.t_lo) * a.n_rtiles;
        }
        __syncthreads();
        if (warp == 0) {
            const int per = (a.B + 31) / 32, lo = lane * per, hi = min(a.B, lo + per);
            int sum = 0;
            for (int b = lo; b < hi; ++b) sum += pref[b + 1];
            int incl = sum;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int n = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += n; }
            int run = incl - sum;
            for (int b = lo; b < hi; ++b) { const int c = pref[b + 1]; pref[b + 1] = run + c; run += c; }
            if (lane == 0) pref[0] = 0;
        }
        __syncthreads();
    }
    const int tiles_total = ragged ? pref[a.B] : a.B * a.n_rtiles * a.n_ttiles;
    const int my_tiles = (tiles_total > (int)blockIdx.x) ? (tiles_total - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;

    if (tid == 0) {
        for (int i = 0; i < NA2; ++i) { mbar_init(BAR(A_FULL + i), NPW); mbar_init(BAR(A_EMPTY + i), NCONS / 32); }
        for (int i = 0; i < NB2; ++i) { mbar_init(BAR(B_FULL + i), 1); mbar_init(BAR(B_EMPTY + i), NCONS / 32); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    // Programmatic dependent launch: the next layer's CTAs may take SMs as this grid drains (they park in their own
    // griddepcontrol.wait); every role that touches activations waits for the previous layer here.  The weight loader
    // (warp W_LOAD) reads only constants and starts filling its ring at once.
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    if (warp != W_LOAD) asm volatile("griddepcontrol.wait;" ::: "memory");

    auto decode = [&](int it, int& b, int& rt, int& q0) {
        const int tile = (int)blockIdx.x + it * (int)gridDim.x;
        if (ragged) {
            int lo = 0, hi = a.B;                   // largest b with pref[b] <= tile (rows without tiles are skipped)
            while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (pref[mid] <= tile) lo = mid; else hi = mid; }
            b = lo;
            const int local = tile - pref[b], nt = (pref[b + 1] - pref[b]) / a.n_rtiles;
            rt = local / nt;
            q0 = (a.t_lo + local - rt * nt) * a.tstep;
            return;
        }
        const int tt = tile % a.n_ttiles, rest = tile / a.n_ttiles;
        rt = rest % a.n_rtiles;
        b = rest / a.n_rtiles;
        q0 = (a.t_lo + tt) * a.tstep;
    };
    auto input_extent = [&](int b) -> int {       // columns of x[b] that hold data; beyond it the operand is zero
        if (!ragged) return a.Tin;
        const long long e = (long long)a.lens[b] * a.rate_in + a.need_in;
        return (int)(e < (long long)a.Tin ? (e > 0 ? e : 0) : (long long)a.Tin);
    };

    if (warp >= W_PROD && warp < W_PROD + NPW) {
        // ============================================================ producers
        const int ptid = tid - 32 * W_PROD;
        const int total = my_tiles * nchunks;
        const int vec_per_row = RAWW / 4;
        const int nvec = KC2 * vec_per_row;
        const float slope = a.in_slope;
        const float* const xg = a.x;
        const long long x_bs = a.x_bs;
        const int x_cs = a.x_cs, Cin = a.Cin, pad = a.pad;
        bool ok = true;
        // Per-thread work items are decoded ONCE (no divisions in the loop), the raw row stride is a compile-time constant
        // (shared loads take immediate offsets), interior windows take a copy path without any bounds logic, and leaky
        // ReLU is max(x, slope * x).
        constexpr int MAXV = (8 * 81 + NPROD - 1) / NPROD, MAXI = (2 * 320 + NPROD - 1) / NPROD;   // raw vectors / slab rows per thread
        int v_ch[MAXV], v_t[MAXV], v_src[MAXV];    // channel in chunk (-1: none), time offset from `tal`, global float offset
        uint32_t v_dst[MAXV];                      // byte offset in a raw stage
#pragma unroll
        for (int e = 0; e < MAXV; ++e) {
            const int v = ptid + e * NPROD;
            const int ch = v / vec_per_row, j = v - ch * vec_per_row;
            v_ch[e] = (v < nvec) ? ch : -1;
            v_t[e] = 4 * j;
            v_src[e] = ch * x_cs + 4 * j;
            v_dst[e] = (uint32_t)(ch * RAWS + 4 * j) * 4u;
        }
        int i_raw[MAXI], i_dst[MAXI];              // raw float offset of channel 0 of the slab row (-1: none), slab byte offset
#pragma unroll
        for (int e = 0; e < MAXI; ++e) {
            const int idx = ptid + e * NPROD;
            const int sl = idx / ROWS, r = idx - sl * ROWS;
            i_raw[e] = (idx < 2 * ROWS) ? (SLC * sl) * RAWS + r : -1;
            i_dst[e] = (int)(sl * slabA) + r * 16;
        }
        // running positions instead of divisions / modulos per chunk
        int iss_it = 0, iss_c = 0, iss_ring = 0, iss_tal = 0, iss_Tin = 0;             // cp.async front: tile, chunk, raw slot
        const float* iss_row = xg;
        bool iss_new = true, iss_int = false;
        int tr_it = 0, tr_c = 0, tr_ring = 0, tr_q0 = 0, as = 0;                       // transform: tile, chunk, raw slot, A stage
        uint32_t pa_empty = 1;                                    // parity to wait for on A_EMPTY[as]: round 1 -> 0, round 2 -> 1, ...
        bool tr_new = true;
        const uint32_t raw_u32 = smem_u32(smRaw);
        auto issue = [&](int g) {
            if (g < total) {
                if (iss_new) {
                    int b_, rt_, q0_;
                    decode(iss_it, b_, rt_, q0_);
                    iss_Tin = input_extent(b_);
                    iss_tal = (q0_ - pad) & ~3;                            // 16-byte aligned window start (may be < 0)
                    iss_row = xg + (long long)b_ * x_bs;
                    iss_int = iss_tal >= (a.in_lo & ~3) && iss_tal + RAWW <= iss_Tin && (Cin & (KCH - 1)) == 0;
                    iss_new = false;
                }
                // a chunk is KCH / 8 slots of 8 channels (one for FP32): the per-thread work items cover one slot
#pragma unroll
                for (int h = 0; h < KCH / KC2; ++h) {
                    const uint32_t dst0 = raw_u32 + (uint32_t)iss_ring * rawStage + (uint32_t)(h * KC2 * RAWS * 4);
                    if (iss_int) {                                             // whole window inside the row: plain 16-byte copies
                        const float* src = iss_row + (long long)(iss_c * KCH + h * KC2) * x_cs + iss_tal;
#pragma unroll
                        for (int e = 0; e < MAXV; ++e)
                            if (v_ch[e] >= 0) cp_async16(dst0 + v_dst[e], src + v_src[e]);
                    } else {
#pragma unroll
                        for (int e = 0; e < MAXV; ++e) {
                            if (v_ch[e] < 0) continue;
                            const int t = iss_tal + v_t[e];
                            const int cg = iss_c * KCH + h * KC2 + v_ch[e];
                            if (REFL && (t < 0 || t + 4 > iss_Tin)) {
                                // edge vector of a reflect-padded conv (vectors inside the row keep the 16-byte copy): four
                                // mirrored 4-byte copies, each from inside the row or zero-filled where the mirror leaves
                                // it (past the conv's reach) -- never a read outside [0, Tin)
                                const float* rowp = iss_row + (long long)(cg < Cin ? cg : 0) * x_cs;
#pragma unroll
                                for (int q = 0; q < 4; ++q) {
                                    int tt = t + q;
                                    tt = tt < 0 ? -tt : (tt >= iss_Tin ? 2 * iss_Tin - 2 - tt : tt);
                                    const bool in = cg < Cin && tt >= 0 && tt < iss_Tin;
                                    cp_async4_zfill(dst0 + v_dst[e] + 4u * q, rowp + (in ? tt : 0), in ? 4u : 0u);
                                }
                                continue;
                            }
                            // t is a multiple of 4, so a vector is either wholly before the data start (zero fill),
                            // wholly inside, or cut by its end (partial source size, rest zero-filled by the hardware)
                            int nb = 0;
                            if (cg < Cin && t >= (a.in_lo & ~3)) nb = 4 * max(0, min(4, iss_Tin - t));
                            const int tsafe = (t >= 0 && t < iss_Tin) ? t : 0;
                            const float* src = iss_row + (long long)(cg < Cin ? cg : 0) * x_cs + tsafe;
                            cp_async16_zfill(dst0 + v_dst[e], src, (uint32_t)nb);
                        }
                    }
                }
                if (++iss_c == nchunks) { iss_c = 0; ++iss_it; iss_new = true; }
            }
            if (++iss_ring == NRAW) iss_ring = 0;
            asm volatile("cp.async.commit_group;" ::: "memory");
        };
        for (int g = 0; g < NRAW - 1; ++g) issue(g);
        for (int g = 0; g < total && ok; ++g) {
            asm volatile("cp.async.wait_group %0;" ::"n"(NRAW - 2) : "memory");
            named_bar_sync(1, NPROD);                                     // everyone's copies of chunk g have landed
            issue(g + NRAW - 1);                                          // refills the stage transformed last iteration
            if (g >= NA2) ok = mbar_wait(BAR(A_EMPTY + as), pa_empty, a.err);
            if (!ok) break;
            if (tr_new) {
                int b_, rt_;
                decode(tr_it, b_, rt_, tr_q0);
                tr_new = false;
            }
            const int tin0 = tr_q0 - pad, off = tin0 - (tin0 & ~3);
            const float* raw = reinterpret_cast<const float*>(smRaw + tr_ring * rawStage) + off;
            unsigned char* base = smA + as * stageA;
            float u[MAXI][SLC];
#pragma unroll
            for (int e = 0; e < MAXI; ++e) {           // all shared loads first ...
                const float* rp = raw + (i_raw[e] < 0 ? 0 : i_raw[e]);
#pragma unroll
                for (int i = 0; i < SLC; ++i) u[e][i] = rp[i * RAWS];
            }
            if constexpr (PREC != PREC_FP32) {
#pragma unroll
                for (int e = 0; e < MAXI; ++e) {       // ... then prologue, rounding to 8 x 16 bits and one 16-byte store
                    if (i_raw[e] < 0) continue;
                    uint32_t p[4];
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const float w0 = fmaxf(u[e][2 * i], u[e][2 * i] * slope);
                        const float w1 = fmaxf(u[e][2 * i + 1], u[e][2 * i + 1] * slope);
                        p[i] = PREC == PREC_BF16 ? cvt_bf16x2(w0, w1) : cvt_f16x2(w0, w1);
                    }
                    *reinterpret_cast<uint4*>(base + i_dst[e]) = make_uint4(p[0], p[1], p[2], p[3]);
                }
            } else {
#pragma unroll
                for (int e = 0; e < MAXI; ++e) {           // ... then prologue, hi/lo split and the two 16-byte stores
                    if (i_raw[e] < 0) continue;
                    float4 hi, lo;
                    float* ph = &hi.x; float* pl = &lo.x;
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const float w_ = fmaxf(u[e][i], u[e][i] * slope);        // leaky ReLU for 0 <= slope <= 1 (1: identity)
                        const float h = __uint_as_float(__float_as_uint(w_) & 0xFFFFE000u);
                        ph[i] = h;
                        pl[i] = w_ - h;
                    }
                    *reinterpret_cast<float4*>(base + i_dst[e]) = hi;
                    *reinterpret_cast<float4*>(base + 2 * slabA + i_dst[e]) = lo;
                }
            }
            fence_async_smem();                                  // generic-proxy stores -> visible to wgmma (async proxy)
            __syncwarp();
            if (lane == 0) mbar_arrive(BAR(A_FULL + as));       // one arrival per producer warp
            if (++tr_c == nchunks) { tr_c = 0; ++tr_it; tr_new = true; }
            if (++tr_ring == NRAW) tr_ring = 0;
            if (++as == NA2) { as = 0; pa_empty ^= 1u; }
        }
        asm volatile("cp.async.wait_group 0;" ::: "memory");
    } else if (warp == W_LOAD) {
        // ============================================================ weight loader
        // One lane per ring slot: lane s owns slot s and feeds it with tap blocks s, s + NB2, s + 2*NB2, ... of this CTA's
        // block sequence, so NB2 independent wait -> expect_tx -> bulk-copy chains are in flight.
        if (lane < NB2) {
            const int total = nchunks * K;                                 // tap blocks per tile (contiguous in memory)
            const long long all = (long long)my_tiles * total;
            const uint32_t full = BAR(B_FULL + lane), empty = BAR(B_EMPTY + lane);
            const uint32_t dst = smem_u32(smB + lane * stageB);
            int it = 0, j = lane;                                          // block gi = it * total + j
            while (j >= total && it < my_tiles) { j -= total; ++it; }
            int cur_it = -1;
            const unsigned char* wsrc = nullptr;
            uint32_t par = 1;                                              // parity of B_EMPTY to wait for: round 1 -> 0, 2 -> 1
            bool ok = true, first = true;
            for (long long gi = lane; gi < all && ok; gi += NB2) {
                if (it != cur_it) {
                    int b_, rt, q0_;
                    decode(it, b_, rt, q0_);
                    wsrc = reinterpret_cast<const unsigned char*>(a.w) + (size_t)rt * total * stageB;
                    cur_it = it;
                }
                if (!first) { ok = mbar_wait(empty, par, a.err); if (!ok) break; }
                mbar_expect_tx(full, stageB);
                bulk_g2s(dst, wsrc + (size_t)j * stageB, stageB, full);
                first = false;
                par ^= 1u;
                j += NB2;
                while (j >= total) { j -= total; ++it; }
            }
        }
        __syncwarp();
    } else if (warp < W_PROD) {
        // ============================================================ consumers: MMA, then epilogue
        // Every lane runs the same loop (wgmma is warpgroup-collective); after a failed wait (`ok` false, the error flag
        // is set) the remaining waits and MMAs are skipped but the named barriers are still met.
        const int wg = warp >> 2, lq = warp & 3, half = warp >> 2;
        const uint64_t wdesc0 = make_desc(smem_u32(smB) + (uint32_t)wg * 64 * 16, slabB);   // this warpgroup's 64 weight rows
        const uint64_t wlo_off = (uint64_t)((2 * slabB) >> 4), wslot = (uint64_t)(stageB >> 4);
        const uint64_t xstep = (uint64_t)a.dil_blk;                                          // B rows per tap block (16 B each)
        bool ok = true;
        int sa = 0; uint32_t pa = 0;                                                         // activation stage / its parity
        int sb = 0; uint32_t pb = 0;                                                         // weight slot / its parity
        float* const st_row = accs + (wg * 64 + lq * 16 + (lane >> 2)) * ACC_LD + 2 * (lane & 3);
#pragma unroll 1
        for (int it = 0; it < my_tiles; ++it) {
            float d[128];                              // per tile: not live across the epilogue
#pragma unroll
            for (int i = 0; i < 128; ++i) d[i] = 0.f;
            uint32_t acc = 0u;
            // One MMA group stays in flight: after committing tap k the warp waits only for tap k-1's group, then releases
            // the weight slot (and, after a chunk's last tap, the activation stage) that group read.
            int rel_b = -1, rel_a = -1;                                                  // operands of the group in flight
            auto release = [&]() {
                __syncwarp();
                if (lane == 0) {                                                         // one arrival per consumer warp
                    if (rel_b >= 0) mbar_arrive(BAR(B_EMPTY + rel_b));
                    if (rel_a >= 0) mbar_arrive(BAR(A_EMPTY + rel_a));
                }
            };
#pragma unroll 1
            for (int c = 0; c < nchunks; ++c) {
                if (ok) ok = mbar_wait(BAR(A_FULL + sa), pa, a.err);
                const uint32_t abase = smem_u32(smA + sa * stageA);
                // descriptors differ only in the start-address field: build once, then add rows (16 B each)
                uint64_t xh = make_desc(abase, slabA), xl = make_desc(abase + 2 * slabA, slabA);
#pragma unroll 1
                for (int k = 0; k < K; ++k) {
                    if (ok) ok = mbar_wait(BAR(B_FULL + sb), pb, a.err);
                    if (ok) {
                        const uint64_t w_hi = wdesc0 + (uint64_t)sb * wslot, w_lo = w_hi + wlo_off;
                        wgmma_fence();
                        if constexpr (PREC == PREC_BF16) {
                            wgmma_bf16_m64n256(d, w_hi, xh, acc);
                        } else if constexpr (PREC == PREC_FP16) {
                            wgmma_f16_m64n256(d, w_hi, xh, acc);
                        } else {
                            wgmma_tf32_m64n256(d, w_hi, xl, acc);               // small terms first
                            wgmma_tf32_m64n256(d, w_lo, xh, 1u);
                            wgmma_tf32_m64n256(d, w_hi, xh, 1u);
                        }
                        wgmma_commit();
                    }
                    wgmma_wait<1>();                                             // the previous tap's group is done
                    release();
                    rel_b = sb;
                    rel_a = (k == K - 1) ? sa : -1;
                    acc = 1u;
                    xh += xstep; xl += xstep;
                    if (++sb == NB2) { sb = 0; pb ^= 1u; }
                }
                if (++sa == NA2) { sa = 0; pa ^= 1u; }
            }
            wgmma_wait<0>();
            release();
            named_bar_sync(4, NCONS);                  // every warp is done reading the previous tile's accumulators
#pragma unroll
            for (int j = 0; j < 32; ++j) {
                *reinterpret_cast<float2*>(st_row + 8 * j) = make_float2(d[4 * j], d[4 * j + 1]);
                *reinterpret_cast<float2*>(st_row + 8 * ACC_LD + 8 * j) = make_float2(d[4 * j + 2], d[4 * j + 3]);
            }
            named_bar_sync(4, NCONS);
            if (!ok) continue;
            int b, rt, q0;
            decode(it, b, rt, q0);
            if constexpr (GRP > 1) {
                grouped_tile<GRP>(a, accs, b, q0, lq, half, lane);
            } else {
                const int qb = q0 + half * 128;
                const float* at = accs + lq * 32 * ACC_LD + half * 128;            // this warp's 32 rows x 128 columns
                const bool lean = LEAN && a.ups == 1 && !a.gate && a.split == 0 && !a.relu && !a.ymask && a.scale == 1.f &&
                                  a.post_div == 1.f && qb + 128 <= a.Tout &&
                                  ((a.y_cs & 3) == 0) && ((a.y_bs & 3) == 0) && ((reinterpret_cast<uintptr_t>(a.y) & 15) == 0) &&
                                  (!a.res || (((a.res_cs & 3) == 0) && ((a.res_bs & 3) == 0) && ((reinterpret_cast<uintptr_t>(a.res) & 15) == 0)));
                if (lean) {
                    // every interior tile half of the plain layers: coalesced global accesses, no per-option branches
                    const int row0 = rt * MROWS + lq * 32;
                    const float* cond = a.cond ? a.cond + (long long)b * a.cond_bs : nullptr;
                    float* yq = a.y + (long long)b * a.y_bs + qb;
                    const bool hres = a.res != nullptr, hacc = a.accum != 0;
                    const float* rq = hres ? a.res + (long long)b * a.res_bs + qb : yq;
                    if (hres) { if (hacc) lean_tile<true, true>(at, a.bias, cond, lane, rq, yq, a.res_cs, a.y_cs, row0, a.Rows, true);
                                else lean_tile<true, false>(at, a.bias, cond, lane, rq, yq, a.res_cs, a.y_cs, row0, a.Rows, true); }
                    else { if (hacc) lean_tile<false, true>(at, a.bias, cond, lane, rq, yq, 0, a.y_cs, row0, a.Rows, true);
                           else lean_tile<false, false>(at, a.bias, cond, lane, rq, yq, 0, a.y_cs, row0, a.Rows, true); }
                } else if constexpr (LEAN) {
                    general_tile_call(a, at + lane * ACC_LD, b, rt, q0, lq, half, lane);
                } else {
                    general_tile_body(a, at + lane * ACC_LD, b, rt, q0, lq, half, lane);
                }
            }
        }
    }
}

// PREC: PREC_FP32 (3xTF32), PREC_BF16 or PREC_FP16
template <int PREC, bool REFL = false>
__global__ void __launch_bounds__(NTHREADS2, 1) conv1d_tc3_kernel(const __grid_constant__ Tc3Args a) { tc3_body<1, true, PREC, REFL>(a); }
template <int PREC>   // gate / split / mask / polyphase
__global__ void __launch_bounds__(NTHREADS2, 1) conv1d_tc3x_kernel(const __grid_constant__ Tc3Args a) { tc3_body<1, false, PREC>(a); }
template <int GRP, int PREC, bool REFL = false>
__global__ void __launch_bounds__(NTHREADS2, 1) conv1d_tc3g_kernel(const __grid_constant__ Tc3Args a) { tc3_body<GRP, true, PREC, REFL>(a); }

typedef void (*Tc3Kernel)(const Tc3Args);
// reflect: the reflection-padding variant (lean epilogue only; the host sends reflect-padded layers that need the general
// epilogue to the FMA kernel)
static inline Tc3Kernel plain_kernel(int prec, bool lean, bool reflect = false) {
    if (reflect) {
        if (prec == PREC_BF16) return conv1d_tc3_kernel<PREC_BF16, true>;
        if (prec == PREC_FP16) return conv1d_tc3_kernel<PREC_FP16, true>;
        return conv1d_tc3_kernel<PREC_FP32, true>;
    }
    if (prec == PREC_BF16) return lean ? conv1d_tc3_kernel<PREC_BF16> : conv1d_tc3x_kernel<PREC_BF16>;
    if (prec == PREC_FP16) return lean ? conv1d_tc3_kernel<PREC_FP16> : conv1d_tc3x_kernel<PREC_FP16>;
    return lean ? conv1d_tc3_kernel<PREC_FP32> : conv1d_tc3x_kernel<PREC_FP32>;
}
// grouped kernel for 2 / 4 tap groups (any dilation with (GRP - 1) * dil <= 15)
template <bool REFL>
static inline Tc3Kernel grouped_kernel_t(int grp, int prec) {
    if (prec == PREC_BF16) return grp == 2 ? conv1d_tc3g_kernel<2, PREC_BF16, REFL> : conv1d_tc3g_kernel<4, PREC_BF16, REFL>;
    if (prec == PREC_FP16) return grp == 2 ? conv1d_tc3g_kernel<2, PREC_FP16, REFL> : conv1d_tc3g_kernel<4, PREC_FP16, REFL>;
    return grp == 2 ? conv1d_tc3g_kernel<2, PREC_FP32, REFL> : conv1d_tc3g_kernel<4, PREC_FP32, REFL>;
}
static inline Tc3Kernel grouped_kernel(int grp, int prec = PREC_FP32, bool reflect = false) {
    return reflect ? grouped_kernel_t<true>(grp, prec) : grouped_kernel_t<false>(grp, prec);
}

}  // namespace tc3
}  // namespace b200tts
