// Persistent Hopper wgmma 3xTF32 conv1d: M = output rows (weights are the A operand), N = 256 time steps (the activation
// window is the B operand).  Tap k of a chunk is the same staged activation tile with its descriptor start address
// advanced by k*dil rows (16 B each), see conv_tc.cuh.
//
//   warps 0-7   consumers : two warpgroups, each D[64 rows x 256 time steps] in registers (wgmma m64n256k8, 3 MMAs per tap
//                           and chunk: lo*hi, hi*lo, hi*hi; one tap's group in flight while the next is issued).  After the last chunk of a tile both warpgroups store their
//                           accumulators to a shared [128][ACC_LD] tile and all eight warps run the epilogue from it
//                           (warp w: rows 32 (w & 3) .. + 31, columns 128 (w >> 2) .. + 127).  A warpgroup starts the next
//                           tile's MMAs as soon as its own epilogue is done; the tile is only rewritten after both are.
//                           Whole interior tiles of plain layers without an accumulate operand skip that shared step:
//                           each warp finishes its own 16 rows in place, with the residual prefetched into them by
//                           cp.async.bulk during the MMAs, and writes them out with bulk stores (the bulk epilogue).
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
// PREC = PREC_F16X3: the 3-product fp16 split (conv_tc.cuh).  A chunk is 16 input channels, but the raw ring keeps the
// FP32 kernel's 8-channel stages: the producers fill one activation stage {X_hi[2 slabs], X_lo[2 slabs]} from two raw
// stages, one slab of each per raw stage, and arrive on it after the second; they also report any |x| >= 65504
// (err[ERR_RANGE]).  A weight tap block is two planes {W_hi, W_lo}[2 slabs][128 rows][8] (8 KB, as in 3xTF32) in the
// same NB2-deep ring, so shared memory is exactly the FP32 kernel's.  The consumers issue W_hs*X_lo, W_lo*X_hi, W_hi*X_hi
// (m64n256k16 each) per tap and chunk, W_hs = W_hi * 2^-11 built in registers: each warp loads its 16 rows of W_hi with
// one ldmatrix.x4, scales them and issues that MMA with A from registers as a commit group of its own, so the wait that
// retires the previous tap also frees the fragment registers for the next one (a second fragment set does not fit the
// 168 registers).  Every epilogue multiplies its rows by `rscale` (2^-e_r) before the bias.
//
// Grouped mode (GRP = 2 / 4) for narrow layers (exactly 64 / 32 output rows, the last two HiFiGAN stages): the 128
// MMA rows are GRP tap-groups x (128/GRP) channels -- row g * (128/GRP) + c carries the weights of channel c for taps
// g, g+GRP, g+2*GRP, ... so one instruction stream of ceil(K/GRP) "tap blocks" (B shifted by GRP*dil rows per block)
// replaces K of them and no MMA row is zero padding.  D_g[c, col] then still misses its own g*dil shift: the epilogue
// reads row g * (128/GRP) + c at column col + g*dil and sums the GRP partials.  Tiles advance by 240 columns so every
// shifted read stays inside the 256-column accumulator.  3xTF32 and 16-bit operands only: at PREC_F16X3 the same layers
// take the time-major kernel (conv1d_tc3t_kernel, tm_consumers), which swaps the GEMM's roles -- M = time, N = the 32 / 64
// channels -- so every tap is summed in the accumulator and no MMA multiplies a padded tap.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "conv_tc.cuh"   // descriptor / barrier / wgmma helpers

namespace b200tts {

// One conv launch as every conv kernel reads it (the FMA tile and single-row kernels of conv1d.cu, and Tc3Args below):
// the call's operands and options, the layer, and what launch_conv derives from them.  launch_conv normalises `io`:
// q_lo / in_lo >= 0, near_src > 0 sets EPI_WAVEGRAD, and split is 0 unless EPI_SPLIT is set.
struct ConvKArgs {
    ConvIO io;
    const float* w; const float* bias;   // the FMA kernels' weight image [row_tiles][CinPad][K][co_tile], bias [RowsPad]
    int Cin, CinPad, K, dil, pad, Rows, ups;
    int Tq;                              // GEMM columns in time (= Tout for ups == 1)
    int XS;                              // FMA tile kernel: staged window row length (launch_variant)
    float near_scale;                    // (float)near_src / Tin (WaveGrad nearest resampling)
};
static_assert(std::is_trivially_copyable_v<ConvKArgs>, "ConvKArgs is a kernel argument");

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
constexpr int NB2 = 3;            // weight ring depth (one tap block per slot: 8 KB, 16-bit operands 4 KB)
constexpr int ACC_LD = 260;       // row stride (floats) of the shared accumulator tile: float4 reads of 8 rows are conflict free
constexpr int ACC_BYTES = MROWS * ACC_LD * 4;
constexpr int NPW = 3;            // producer warps
constexpr int NPROD = 32 * NPW;
constexpr int NCONS = 256;        // consumer threads (two warpgroups)
constexpr int W_PROD = 8, W_LOAD = 8 + NPW;
constexpr int NTHREADS2 = 32 * (W_LOAD + 1);

// The launch (ConvKArgs) plus the tensor-core schedule.  Ragged batches (io.lens; null: every row spans the full tensor):
// row b only has tiles for GEMM columns below min(Tq, lens[b] * rate_out + need_out) and its input is read as zero from
// min(Tin, lens[b] * rate_in + need_in) on, so padded frames cost nothing and `need` keeps every sample below lens[b]
// bit-identical to the full computation (it is the receptive field of the layers that still follow, worked out per
// launch by the engine).  Column window (io.q_lo / q_hi / in_lo): a row's tiles run from floor(q_lo / tstep) to
// ceil(min(extent, q_hi) / tstep); tile origins stay multiples of tstep counted from column 0, so every column is computed
// (and takes the same epilogue) as in the unwindowed launch.  Input columns below in_lo are stale scratch and read as
// zero (whole 16-byte vectors: the ones below in_lo rounded down to a multiple of 4); the host stops io.Tin where the
// producer's window ends, so the grouped mode's zero-padded taps never multiply stale data.
struct Tc3Args : ConvKArgs {
    const void* w_tc;          // the plain or grouped image: [row_tile][chunk][tap]{hi[2][128][4], lo[2][128][4]} fp32
                               // (16-bit: [2][128][8]; PREC_F16X3: {hi, lo}[2][128][8] fp16), see pack_tc / pack_tc_tm
    const float* rscale;       // PREC_F16X3: [Rows] 2^-e_r, the inverse of the pack-time row scaling (see pack_tc)
    int KJ;                    // tap blocks per chunk (= K, or ceil(K / GRP) in grouped mode)
    int dil_blk;               // B-row shift between tap blocks (= dil, or GRP * dil)
    int tstep;                 // time steps a tile advances (= TT2, or 240 in grouped mode)
    int rows_pad;              // slab rows  (TT2 + halo, multiple of 8)
    int raw_w;                 // raw row width in floats (rows_pad + 4, multiple of 4)
    int n_ttiles, n_rtiles;    // the window's tiles per row (dense schedule), row tiles
    int t_lo;                  // floor(q_lo / tstep): the window's first tile
    int pref_off;              // byte offset in dynamic shared memory of the (B + 1)-entry tile prefix table (ragged)
    int* err;
};
static_assert(std::is_trivially_copyable_v<Tc3Args>, "Tc3Args is a kernel argument");

// torch's nearest source index (upsample_nearest1d's nearest_idx): identity, the exact-2x shortcut, else
// min(floor(dst * scale), src - 1) with the float scale src / dst
__device__ __forceinline__ int near_col(int t, int src, int dst, float scale) {
    if (dst == src) return t;
    if (dst == 2 * src) return t >> 1;
    return min((int)floorf(__fmul_rn((float)t, scale)), src - 1);
}

// prec: PREC_FP32 (8-channel chunks, hi/lo slab pairs), a 16-bit type (16-channel chunks, two slabs) or PREC_F16X3
// (16-channel chunks over 8-channel raw stages, hi/lo slab pairs: the FP32 kernel's total)
static inline size_t smem_bytes3(int rows_pad, int prec = PREC_FP32) {
    const bool b16 = prec == PREC_BF16 || prec == PREC_FP16;
    const size_t raw_ch = b16 ? KC16 : KC2, nsl = b16 ? 2 : 4;
    return (size_t)NRAW * raw_ch * RAWS * 4 + (size_t)NA2 * (nsl * rows_pad * 16) + NB2 * (nsl * MROWS * 16) + ACC_BYTES + 512;
}
// Time-major kernel (tm_consumers): a weight tap block is {W_hs, W_lo, W_hi}[2 slabs][C rows][16 B]; each warpgroup's
// epilogue has two [C][64 * tms + 4] fp32 tiles (residual / output, accumulate operand), rows padded by 4 floats so that
// the fragment stores of 8 time steps x 4 channels hit 32 banks
__host__ __device__ constexpr uint32_t tm_block_bytes(int C) { return 3u * 2u * (uint32_t)C * 16u; }
// Its weight ring is deeper than NB2: a tap block feeds only 3 * TMS m64nC MMAs per warpgroup, and a slot is refilled
// one tap after its MMAs retire, so NB - 2 blocks must cover the L2 -> shared copy latency.  64 channels: what shared
// memory leaves beside the 64-channel epilogue tiles.
__host__ __device__ constexpr int tm_ring(int C) { return C == 64 ? 4 : 12; }
__host__ __device__ constexpr uint32_t tm_epi_bytes(int C, int tms) { return 2u * 2u * (uint32_t)C * (64u * tms + 4u) * 4u; }
static inline size_t smem_bytes_tm(int rows_pad, int C, int tms) {
    return (size_t)NRAW * KC2 * RAWS * 4 + (size_t)NA2 * (4 * rows_pad * 16) + tm_ring(C) * tm_block_bytes(C) + tm_epi_bytes(C, tms) + 512;
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
// SC (PREC_F16X3): acc is first multiplied by the row's rscale (a power of two: exact).
template <bool HR, bool HA, bool SC>
__device__ __forceinline__ void lean_tile(const float* at, const float* bias, const float* rscale, const float* cond, int lane,
                                          const float* rq, float* yq, long long rcs, long long ycs, int row0, int Rows,
                                          bool do_st) {
    const int r8 = lane & 7, p4 = lane >> 3;
    const float* rrow[4];
    float* yrow[4];
    bool st_ok[4];
    float bv[4], sv[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int ri = row0 + 8 * i + r8, rci = ri < Rows ? ri : Rows - 1;
        rrow[i] = rq + (long long)rci * rcs + 4 * p4;
        yrow[i] = yq + (long long)rci * ycs + 4 * p4;
        st_ok[i] = do_st && ri < Rows;
        bv[i] = bias[rci];
        if (cond) bv[i] += __ldg(cond + rci);
        sv[i] = SC ? rscale[rci] : 1.f;
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
            if constexpr (SC) { t.x *= sv[i]; t.y *= sv[i]; t.z *= sv[i]; t.w *= sv[i]; }
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

// Bulk epilogue of one consumer warp (whole interior tiles of the plain layers without an accumulate operand): the
// warp's 16 MMA rows are finished in place in the shared accumulator tile, where its accumulator fragment would be stored
// (st_row, see the consumers), each element as lean_tile computes it: ((acc * rscale) + (bias + cond)) + res.  HR: the
// rows already hold the tile's residual (prefetched by cp.async.bulk during the MMAs).  bv / sv: rows lane / 4 and + 8.
template <bool HR, bool SC>
__device__ __forceinline__ void bulk_combine(const float* d, float* st_row, const float (&bv)[2], const float (&sv)[2]) {
#pragma unroll
    for (int j = 0; j < 32; ++j) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float2* p = reinterpret_cast<float2*>(st_row + h * 8 * ACC_LD + 8 * j);
            float2 t = make_float2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
            if constexpr (SC) { t.x *= sv[h]; t.y *= sv[h]; }
            t.x += bv[h]; t.y += bv[h];
            if constexpr (HR) { const float2 r = *p; t.x += r.x; t.y += r.y; }
            *p = t;
        }
    }
}

// Everything the lean epilogue does not cover (WaveNet gate / res-skip split, masks, ReLU, scale, final divide, polyphase
// stores of the transposed convs, edge tiles): one tile half per call, lane = one output row, `arow` = its accumulators.
// SC: the accumulators are scaled by the row's rscale first (PREC_F16X3).
// WG: the WaveGrad epilogue instead (conv1d_tc3w_kernel):
//   v = acc + bias; [lrelu]; [+ act_add[b]]; [+ res]; [y2 <- v]; [v = shift + scale * v]; y <- v
// with every product and sum rounded on its own (no FMA contraction), in the reference's order.
template <bool SC, bool WG = false>
__device__ __forceinline__ void general_tile_body(const ConvKArgs& a, const float* rscale, const float* arow, int b, int rt,
                                                  int q0, int lq, int half, int lane) {
    const ConvIO& io = a.io;
    const int ups = a.ups;
    const int r = rt * MROWS + lq * 32 + lane;             // GEMM row of this lane
    const bool rok = r < a.Rows;
    const int rc = rok ? r : a.Rows - 1;
    const int qb = q0 + half * 128;
    float bias = a.bias[rc];
    if (io.cond) bias += __ldg(io.cond.row(b) + rc);
    const float rs = SC ? rscale[rc] : 1.f;
    auto acc_ld = [&](const float* p, float* v) {
        acc_ld16(p, v);
        if constexpr (SC) {
#pragma unroll
            for (int i = 0; i < 16; ++i) v[i] *= rs;
        }
    };
    if constexpr (WG) {
        if (!rok) return;
        float* yrow = io.y.row(b, rc);
        float* y2row = io.y2 ? io.y2.row(b, rc) : nullptr;
        const float* rrow = io.res ? io.res.row(b, rc) : nullptr;
        const float* srow = io.film ? io.film.row(b, rc) : nullptr;
        const float* crow = srow ? srow + (long long)io.film_half * io.film.cs : nullptr;
        const float add = io.act_add ? __ldg(io.act_add + b) : 0.f;
        const bool has_add = io.act_add != nullptr, lrelu = io.act == ACT_LRELU;
        const float slope = io.act_param;
        // float4 accesses when every row pointer is 16-byte aligned (all pitches multiples of 4 floats)
        const bool vec_ok = ((reinterpret_cast<uintptr_t>(yrow) | reinterpret_cast<uintptr_t>(y2row) |
                              reinterpret_cast<uintptr_t>(rrow) | reinterpret_cast<uintptr_t>(srow) |
                              reinterpret_cast<uintptr_t>(crow)) & 15) == 0;
        for (int cg = 0; cg < 128; cg += 16) {
            float v[16];
            acc_ld(arow + cg, v);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int qq = qb + cg + 4 * j;
                if (qq >= io.Tout) break;
                const bool vec = vec_ok && qq + 3 < io.Tout;
                float r4[4] = {0.f, 0.f, 0.f, 0.f}, s4[4] = {0.f, 0.f, 0.f, 0.f}, c4[4] = {1.f, 1.f, 1.f, 1.f};
                if (vec) {
                    if (rrow) { const float4 t = *reinterpret_cast<const float4*>(rrow + qq); r4[0] = t.x; r4[1] = t.y; r4[2] = t.z; r4[3] = t.w; }
                    if (srow) {
                        const float4 t = *reinterpret_cast<const float4*>(srow + qq); s4[0] = t.x; s4[1] = t.y; s4[2] = t.z; s4[3] = t.w;
                        const float4 u = *reinterpret_cast<const float4*>(crow + qq); c4[0] = u.x; c4[1] = u.y; c4[2] = u.z; c4[3] = u.w;
                    }
                } else {
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const int qe = min(qq + e, io.Tout - 1);
                        if (rrow) r4[e] = rrow[qe];
                        if (srow) { s4[e] = srow[qe]; c4[e] = crow[qe]; }
                    }
                }
                float o[4], p[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    float u = __fadd_rn(v[4 * j + e], bias);
                    if (lrelu) u = u > 0.f ? u : __fmul_rn(u, slope);
                    if (has_add) u = __fadd_rn(u, add);
                    if (rrow) u = __fadd_rn(u, r4[e]);
                    p[e] = u;
                    o[e] = srow ? __fadd_rn(s4[e], __fmul_rn(c4[e], u)) : u;
                }
                if (vec) {
                    if (y2row) *reinterpret_cast<float4*>(y2row + qq) = make_float4(p[0], p[1], p[2], p[3]);
                    *reinterpret_cast<float4*>(yrow + qq) = make_float4(o[0], o[1], o[2], o[3]);
                } else {
#pragma unroll
                    for (int e = 0; e < 4; ++e)
                        if (qq + e < io.Tout) {
                            if (y2row) y2row[qq + e] = p[e];
                            yrow[qq + e] = o[e];
                        }
                }
            }
        }
        return;
    }
    if (io.flags & EPI_GATE) {
        // WaveNet gate (wavenet.py:6-13): even lane = tanh argument, odd lane = sigmoid argument of row r/2
        float* yrow = io.y.row(b, rc >> 1);
        const bool vec_ok = ((io.y.cs & 3) == 0) && ((reinterpret_cast<uintptr_t>(yrow) & 15) == 0);
        const bool even = (lane & 1) == 0;
        for (int cg = 0; cg < 128; cg += 16) {
            float v[16];
            acc_ld(arow + cg, v);
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
                    if (vec_ok && qq + 3 < io.Tout) *reinterpret_cast<float4*>(yrow + qq) = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
                    else {
#pragma unroll
                        for (int e = 0; e < 4; ++e) if (qq + e < io.Tout) yrow[qq + e] = v[4 * j + e];
                    }
                }
            }
        }
    } else if (ups == 1) {
        float* yrow = io.y.row(b, rc);
        bool acc_r = (io.flags & EPI_ACCUM) != 0, mpost_r = (io.flags & EPI_MASK_POST) != 0;
        if (io.split > 0) {         // WaveNet res/skip rows (wavenet.py:108-113)
            if (rc < io.split) { acc_r = true; mpost_r = true; }
            else { yrow = io.y2.row(b, rc - io.split); acc_r = (io.flags & EPI_ACCUM2) != 0; mpost_r = false; }
        }
        const float* rrow = io.res ? io.res.row(b, rc) : nullptr;
        const float* mrow = io.ymask ? io.ymask.row(b) : nullptr;
        const int ycs_eff = (io.split > 0 && rc >= io.split) ? io.y2.cs : io.y.cs;
        const bool vec_ok = ((ycs_eff & 3) == 0) && (!io.res || (io.res.cs & 3) == 0) &&
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
                if (vec_ok && qq + 3 < io.Tout) {
                    if (rrow) asm volatile("ld.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r_[4 * j]), "=f"(r_[4 * j + 1]), "=f"(r_[4 * j + 2]), "=f"(r_[4 * j + 3]) : "l"(rrow + qq));
                    if (acc_r) asm volatile("ld.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(o_[4 * j]), "=f"(o_[4 * j + 1]), "=f"(o_[4 * j + 2]), "=f"(o_[4 * j + 3]) : "l"(yrow + qq));
                } else {
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const int qe = min(qq + e, io.Tout - 1);
                        if (rrow) asm volatile("ld.global.f32 %0, [%1];" : "=f"(r_[4 * j + e]) : "l"(rrow + qe));
                        if (acc_r) asm volatile("ld.global.f32 %0, [%1];" : "=f"(o_[4 * j + e]) : "l"(yrow + qe));
                    }
                }
            }
        };
        auto group = [&](int cg, const float* rv, const float* ov, float* rn, float* on) {
            float v[16];
            if (rok && cg + 16 < 128) prefetch(cg + 16, rn, on);
            acc_ld(arow + cg, v);
            const int q = qb + cg;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                float u = v[i] + bias;
                if (io.act == ACT_RELU) u = fmaxf(u, 0.f);
                const float mk = mrow ? __ldg(mrow + min(q + i, io.Tout - 1)) : 1.f;
                if (io.flags & EPI_MASK_PRE) u *= mk;
                if (io.res) u += rv[i];
                u *= io.scale;
                if (acc_r) u += ov[i];
                if (io.post_div != 1.f) u = u / io.post_div;
                if (mpost_r) u *= mk;
                v[i] = u;
            }
            if (rok) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int qq = q + 4 * j;
                    if (vec_ok && qq + 3 < io.Tout) {
                        *reinterpret_cast<float4*>(yrow + qq) = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
                    } else {
#pragma unroll
                        for (int e = 0; e < 4; ++e) if (qq + e < io.Tout) yrow[qq + e] = v[4 * j + e];
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
        float* yrow = io.y.row(b, co) + ph;
        for (int cg = 0; cg < 128; cg += 16) {
            float v[16];
            acc_ld(arow + cg, v);
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const int q = qb + cg + i;
                float u = v[i] + bias;
                if (io.act == ACT_RELU) u = fmaxf(u, 0.f);
                const long long t = (long long)q * ups;
                if (q < a.Tq && t + ph < io.Tout) yrow[t] = u;
            }
        }
    }
}

// Out-of-line call of the general epilogue for the kernel whose hot path is the lean one (edge tiles only): inlined into
// its tile loop the general code's loop invariants were hoisted across the lean path.  One copy of the launch per call:
// through the reference every field use would be a generic load.
template <bool SC>
__device__ __noinline__ void general_tile_call(const Tc3Args& a_ref, const float* arow, int b, int rt, int q0, int lq, int half,
                                               int lane) {
    const ConvKArgs a = a_ref;
    general_tile_body<SC>(a, a_ref.rscale, arow, b, rt, q0, lq, half, lane);
}

// Grouped epilogue, one tile half: out[c, t] = sum_g D_g[c, t + g*dil] with MMA row m = g * CH + c (CH = 128 / GRP
// channels).  Thread tq of the half's 128 finishes channel co = tq * NQ / 4, float4s j0 .. j0 + NQ - 1 of every
// 16-column group (4 / NQ lanes = 64 contiguous bytes of a channel).  SC: the GRP partials of a channel share its rscale,
// applied to their sum (PREC_F16X3).
template <int GRP, bool SC>
__device__ __forceinline__ void grouped_tile(const Tc3Args& a, const float* accs, int b, int q0, int lq, int half, int lane) {
    constexpr int CH = 128 / GRP;              // output channels
    constexpr int NQ = CH / 32;                // float4 per thread and 16-column group (1 or 2)
    constexpr int NV = 4 * NQ;
    const int tq = lq * 32 + lane;
    const int co = (tq * NQ) >> 2;
    const int coff = 4 * ((tq & (4 / NQ - 1)) * NQ);
    const int cbeg = half ? 128 : 0;
    const int cend = half ? a.tstep : min(128, a.tstep);
    const ConvIO& io = a.io;
    const bool has_res = io.res.p != nullptr, acc_r = (io.flags & EPI_ACCUM) != 0;
    const bool vec_ok = io.y.aligned16() && (!has_res || io.res.aligned16());
    const bool fast = vec_ok && (q0 + a.tstep <= io.Tout);   // interior tile: no bounds checks
    const float* rrow = has_res ? io.res.row(b, co) : nullptr;
    float* yrow = io.y.row(b, co);
    float bias = a.bias[co];
    if (io.cond) bias += __ldg(io.cond.row(b) + co);
    const float rs = SC ? a.rscale[co] : 1.f;
    auto load = [&](const float* rr, int q, float* dst) {     // one thread's values of a column group of a row
#pragma unroll
        for (int j = 0; j < NQ; ++j) {
            const int qq = q + 4 * j;
            if (fast || (vec_ok && qq + 3 < io.Tout)) {
                const float4 t = *reinterpret_cast<const float4*>(rr + qq);
                dst[4 * j] = t.x; dst[4 * j + 1] = t.y; dst[4 * j + 2] = t.z; dst[4 * j + 3] = t.w;
            } else {
#pragma unroll
                for (int e = 0; e < 4; ++e) dst[4 * j + e] = rr[min(qq + e, io.Tout - 1)];
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
            if constexpr (SC) s *= rs;
            R[i] = s;
        }
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            float u = R[i] + bias;
            if (io.act == ACT_RELU) u = fmaxf(u, 0.f);
            if (has_res) u += rv[i];
            u *= io.scale;
            if (acc_r) u += ov[i];
            if (io.post_div != 1.f) u = u / io.post_div;
            R[i] = u;
        }
        const int q = q0 + cg + coff;
#pragma unroll
        for (int j = 0; j < NQ; ++j) {
            const int qq = q + 4 * j;
            if (fast || (vec_ok && qq + 3 < io.Tout)) {
                *reinterpret_cast<float4*>(yrow + qq) = make_float4(R[4 * j], R[4 * j + 1], R[4 * j + 2], R[4 * j + 3]);
            } else {
#pragma unroll
                for (int e = 0; e < 4; ++e) if (qq + e < io.Tout) yrow[qq + e] = R[4 * j + e];
            }
        }
    }
}

// Consumers of the time-major kernel (PREC_F16X3, exactly C = 32 / 64 output channels).  The GEMM is transposed: M = time,
// N = the C channels, K = input channels x taps, all summed in the accumulator.  The staged activation window is the A
// operand (its K-major slabs are a valid m64k16 A image; tap k and slice s start k * dil + 64 s rows further) and the
// weight block the B operand.  Warpgroup wg owns time steps wg * HW .. + HW - 1 of the tile (HW = 64 * TMS) for all C
// channels: TMS m64nC accumulators, W_hs*X_lo + W_lo*X_hi + W_hi*X_hi per tap and chunk (small terms first), one tap's
// group in flight while the next is issued.  Every output column takes the same sum in the same order wherever its
// tile starts.
// Epilogue, per warpgroup and without cross-warpgroup hand-off: on whole interior tiles of aligned layers, warp lq's
// lane 0 prefetches channel rows lq * C/4 .. + C/4 - 1 of the residual (and the accumulate operand) into the warpgroup's
// [C][HW] tiles by cp.async.bulk before the MMAs (RES_FULL[warp]); after them every thread finishes its fragment in
// the grouped epilogue's order, ((acc * rscale) + (bias + cond)), ReLU, + res, * scale, + old, / post_div, writes it
// transposed into the residual tile, and after a warpgroup barrier the same lanes store their rows with bulk copies.
// Edge tiles and unaligned layers finish the fragment straight to global memory with bounds checks.
template <int C, int TMS, typename Decode>
__device__ __forceinline__ void tm_consumers(const Tc3Args& a, const unsigned char* smA, const unsigned char* smB, float* epi,
                                             uint32_t bar0, const Decode& decode, int my_tiles, int nchunks, uint32_t slabA,
                                             int warp, int lane) {
    constexpr int HW = 64 * TMS, P = HW + 4, NA = C / 2;      // time steps per warpgroup, tile row pitch, accumulators per slice
    constexpr int CW = C / 4;                                   // channel rows each warp prefetches and stores
    constexpr uint32_t PLANE = 2u * C * 16u;                    // one of W_hs / W_lo / W_hi: [2 slabs][C rows][16 B]
    constexpr int NB = tm_ring(C);
    constexpr int A_FULL = 0, A_EMPTY = NA2, B_FULL = 2 * NA2, B_EMPTY = 2 * NA2 + NB, RES_FULL = 2 * NA2 + 2 * NB;
    auto BAR = [&](int i) { return bar0 + 8u * (uint32_t)i; };
    const uint32_t stageA = 4u * slabA;
    const int wg = warp >> 2, lq = warp & 3, K = a.KJ;
    float* const rbuf = epi + (size_t)wg * 2 * C * P;           // residual in, output out
    float* const obuf = rbuf + C * P;                           // accumulate operand
    const uint64_t wdesc0 = make_desc(smem_u32(smB), C * 16);
    const ConvIO& io = a.io;
    const bool has_res = io.res.p != nullptr, acc_r = (io.flags & EPI_ACCUM) != 0, relu = io.act == ACT_RELU;
    const bool bulk_layer = io.y.aligned16() && (!has_res || io.res.aligned16());
    const int c0 = 2 * (lane & 3), t0 = 16 * lq + (lane >> 2);  // fragment: channels 8j + c0 + {0,1}, time steps t0 (+8) + 64 s
    bool ok = true;
    int sa = 0; uint32_t pa = 0;                                // activation stage / its parity
    int sb = 0; uint32_t pb = 0;                                // weight slot / its parity
    uint32_t pr = 0;                                            // parity of RES_FULL
#pragma unroll 1
    for (int it = 0; it < my_tiles; ++it) {
        int b, rt, q0;
        decode(it, b, rt, q0);
        const int qw = q0 + wg * HW;                            // this warpgroup's first column
        const bool bulk = bulk_layer && q0 + 2 * HW <= io.Tout;
        const bool pre = bulk && (has_res || acc_r);
        if (bulk && lane == 0) {
            bulk_wait_read();                                   // this warp's previous bulk stores are done reading its rows
            if (pre) {
                const uint32_t rf = BAR(RES_FULL + warp);
                mbar_expect_tx(rf, (uint32_t)((has_res ? 1 : 0) + (acc_r ? 1 : 0)) * CW * HW * 4);
                for (int c = lq * CW; c < (lq + 1) * CW; ++c) {
                    if (has_res)
                        bulk_g2s(smem_u32(rbuf + c * P), io.res.row(b, c) + qw, HW * 4, rf);
                    if (acc_r)
                        bulk_g2s(smem_u32(obuf + c * P), io.y.row(b, c) + qw, HW * 4, rf);
                }
            }
        }
        float d[TMS][NA];
#pragma unroll
        for (int s = 0; s < TMS; ++s)
#pragma unroll
            for (int i = 0; i < NA; ++i) d[s][i] = 0.f;
        uint32_t acc = 0u;
        int rel_b = -1, rel_a = -1;                             // operands of the group in flight
        auto release = [&]() {
            __syncwarp();
            if (lane == 0) {                                    // one arrival per consumer warp
                if (rel_b >= 0) mbar_arrive(BAR(B_EMPTY + rel_b));
                if (rel_a >= 0) mbar_arrive(BAR(A_EMPTY + rel_a));
            }
        };
#pragma unroll 1
        for (int c = 0; c < nchunks; ++c) {
            if (ok) ok = mbar_wait(BAR(A_FULL + sa), pa, a.err);
            const uint32_t abase = smem_u32(smA + sa * stageA) + (uint32_t)(wg * HW) * 16u;
            uint64_t xh = make_desc(abase, slabA), xl = make_desc(abase + 2 * slabA, slabA);
#pragma unroll 1
            for (int k = 0; k < K; ++k) {
                if (ok) ok = mbar_wait(BAR(B_FULL + sb), pb, a.err);
                if (ok) {
                    const uint64_t whs = wdesc0 + (uint64_t)sb * (tm_block_bytes(C) >> 4);
                    const uint64_t wlo = whs + (PLANE >> 4), whi = whs + 2 * (PLANE >> 4);
                    wgmma_fence();
#pragma unroll
                    for (int s = 0; s < TMS; ++s) {                 // slice s: 64 rows = 64 descriptor units further
                        if constexpr (C == 64) {
                            wgmma_f16_m64n64(d[s], xl + 64 * s, whs, acc);
                            wgmma_f16_m64n64(d[s], xh + 64 * s, wlo, 1u);
                            wgmma_f16_m64n64(d[s], xh + 64 * s, whi, 1u);
                        } else {
                            wgmma_f16_m64n32(d[s], xl + 64 * s, whs, acc);
                            wgmma_f16_m64n32(d[s], xh + 64 * s, wlo, 1u);
                            wgmma_f16_m64n32(d[s], xh + 64 * s, whi, 1u);
                        }
                    }
                    wgmma_commit();
                }
                wgmma_wait<1>();                                // the previous tap's group is done
                release();
                rel_b = sb;
                rel_a = (k == K - 1) ? sa : -1;
                acc = 1u;
                xh += (uint64_t)a.dil; xl += (uint64_t)a.dil;
                if (++sb == NB) { sb = 0; pb ^= 1u; }
            }
            if (++sa == NA2) { sa = 0; pa ^= 1u; }
        }
        wgmma_wait<0>();
        release();

        // per-channel constants of this thread's fragment columns
        float bv[C / 8][2], sv[C / 8][2];
#pragma unroll
        for (int j = 0; j < C / 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int ch = 8 * j + c0 + e;
                bv[j][e] = a.bias[ch];
                if (io.cond) bv[j][e] += __ldg(io.cond.row(b) + ch);
                sv[j][e] = a.rscale[ch];
            }
        auto finish = [&](float v, int j, int e, float r, float o) {
            float u = v * sv[j][e] + bv[j][e];
            if (relu) u = fmaxf(u, 0.f);
            if (has_res) u += r;
            u *= io.scale;
            if (acc_r) u += o;
            if (io.post_div != 1.f) u = u / io.post_div;
            return u;
        };
        if (bulk) {
            if (pre) {                                          // waited for even after a failed wait: the copies always land
#pragma unroll 1
                for (int w = 0; w < 4; ++w) {
                    const bool landed = mbar_wait(BAR(RES_FULL + 4 * wg + w), pr, a.err);
                    ok = ok && landed;
                }
                pr ^= 1u;
            } else {
                named_bar_sync(5 + wg, 128);                    // every warp's previous bulk stores are done reading
            }
            if (ok) {
#pragma unroll
                for (int s = 0; s < TMS; ++s)
#pragma unroll
                    for (int j = 0; j < C / 8; ++j)
#pragma unroll
                        for (int h = 0; h < 2; ++h)
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                float* p = rbuf + (8 * j + c0 + e) * P + 64 * s + t0 + 8 * h;
                                const float r = has_res ? *p : 0.f;
                                const float o = acc_r ? p[C * P] : 0.f;
                                *p = finish(d[s][4 * j + 2 * h + e], j, e, r, o);
                            }
            }
            fence_async_smem();                                 // the finished rows -> visible to the bulk copies (async proxy)
            named_bar_sync(5 + wg, 128);
            if (ok && lane == 0) {
                for (int c = lq * CW; c < (lq + 1) * CW; ++c)
                    bulk_s2g(io.y.row(b, c) + qw, smem_u32(rbuf + c * P), HW * 4);
                bulk_commit();
            }
        } else if (ok) {
#pragma unroll
            for (int s = 0; s < TMS; ++s)
#pragma unroll
                for (int j = 0; j < C / 8; ++j)
#pragma unroll
                    for (int h = 0; h < 2; ++h)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int ch = 8 * j + c0 + e, q = qw + 64 * s + t0 + 8 * h;
                            if (q >= io.Tout) continue;
                            float* yp = io.y.row(b, ch) + q;
                            const float r = has_res ? io.res.p[(long long)b * io.res.bs + (long long)ch * io.res.cs + q] : 0.f;
                            const float o = acc_r ? *yp : 0.f;
                            *yp = finish(d[s][4 * j + 2 * h + e], j, e, r, o);
                        }
        }
    }
    if (lane == 0) bulk_wait_all();                             // the bulk stores are complete before the dependent grid may read
    __syncwarp();
}

template <int GRP, bool LEAN = true, int PREC = PREC_FP32, bool REFL = false, bool NEAR = false, bool WG = false,
          int TMC = 0, int TMS = 2>
                                       // TMC: the time-major kernel's output channels (32 / 64; 0: off), TMS: its m64
                                       // slices per warpgroup (tile width 128 * TMS), see tm_consumers;
                                       // GRP: tap groups stacked in the 128 MMA rows (1 = plain); LEAN:
                                       // plain-layer kernel (lean epilogue inline, general one out of line) -- false for the
                                       // WaveNet / masked / transposed layers (general epilogue inline); PREC: operand type;
                                       // REFL: reflection padding (ConvIO::reflect; dense, unwindowed launches only): input
                                       // column t < 0 reads x[-t], t >= Tin reads x[2 Tin - 2 - t].  A compile-time switch so
                                       // that the zero-padding kernels keep their register allocation.
                                       // NEAR: nearest-resampled input (ConvIO::near_src): column t in [0, Tin) reads
                                       // x[near_col(t)], staged by 4-byte copies; WG: the WaveGrad epilogue (general_tile_body).
__device__ __forceinline__ void tc3_body(const Tc3Args& a) {
    extern __shared__ __align__(128) unsigned char smem[];
    constexpr bool X3 = PREC == PREC_F16X3;      // 3-product fp16 split
    constexpr bool B16 = PREC == PREC_BF16 || PREC == PREC_FP16;
    constexpr int KCH = PREC != PREC_FP32 ? KC16 : KC2;   // input channels per chunk
    constexpr int RCH = B16 ? KC16 : KC2;        // input channels per raw ring stage
    constexpr int SPC = KCH / RCH;               // raw stages per chunk (2 for X3)
    constexpr int NSL = B16 ? 2 : 4;             // 16-byte slabs per activation stage: two 16-bit slabs, or hi[2] + lo[2]
    constexpr int SLC = PREC != PREC_FP32 ? 8 : 4;   // channels per slab row
    constexpr int NB = TMC ? tm_ring(TMC) : NB2; // weight ring depth
    constexpr bool SC = X3;                      // epilogues scale rows by rscale
    constexpr bool TM = TMC != 0;                // time-major kernel (PREC_F16X3, 32 / 64 output channels)
    constexpr bool BULK = GRP == 1 && LEAN && !TM;   // plain-layer kernel: whole interior tiles may take the bulk epilogue
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int ROWS = a.rows_pad, RAWW = a.raw_w, K = a.KJ;
    const uint32_t rawStage = (uint32_t)RCH * RAWS * 4;
    const uint32_t slabA = (uint32_t)ROWS * 16, stageA = NSL * slabA;
    // one tap block: [NSL slabs][128 rows][16 B]; time-major: {W_hs, W_lo, W_hi}[2 slabs][TMC rows][16 B]
    const uint32_t slabB = (uint32_t)MROWS * 16, stageB = TM ? tm_block_bytes(TMC) : NSL * slabB;
    unsigned char* smRaw = smem;
    unsigned char* smA = smRaw + NRAW * rawStage;
    unsigned char* smB = smA + NA2 * stageA;
    float* accs = reinterpret_cast<float*>(smB + NB * stageB);
    uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<unsigned char*>(accs) + (TM ? tm_epi_bytes(TMC, TMS) : ACC_BYTES));
    const int A_FULL = 0, A_EMPTY = NA2, B_FULL = 2 * NA2, B_EMPTY = 2 * NA2 + NB, RES_FULL = 2 * NA2 + 2 * NB;
    const uint32_t bar0 = smem_u32(bars);
    auto BAR = [&](int i) { return bar0 + 8u * (uint32_t)i; };

    const int nchunks = (a.Cin + KCH - 1) / KCH;
    const bool ragged = a.io.lens != nullptr;
    int* pref = reinterpret_cast<int*>(smem + a.pref_off);    // pref[b] = first tile of row b (ragged only)
    if (ragged) {
        // tiles per row from its own length; exclusive prefix by warp 0 (rows in lane-contiguous chunks).  `lens` was
        // written several launches ago (durations kernel), so reading it before griddepcontrol.wait is safe.
        for (int b = tid; b < a.io.B; b += NTHREADS2) {
            const long long e = (long long)a.io.lens[b] * a.io.rate_out + a.io.need_out;
            const int ext = (int)(e < (long long)a.Tq ? (e > 0 ? e : 0) : (long long)a.Tq);
            const int t_hi = (min(ext, a.io.q_hi) + a.tstep - 1) / a.tstep;
            pref[b + 1] = max(0, t_hi - a.t_lo) * a.n_rtiles;
        }
        __syncthreads();
        if (warp == 0) {
            const int per = (a.io.B + 31) / 32, lo = lane * per, hi = min(a.io.B, lo + per);
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
    const int tiles_total = ragged ? pref[a.io.B] : a.io.B * a.n_rtiles * a.n_ttiles;
    const int my_tiles = (tiles_total > (int)blockIdx.x) ? (tiles_total - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;

    if (tid == 0) {
        for (int i = 0; i < NA2; ++i) { mbar_init(BAR(A_FULL + i), NPW); mbar_init(BAR(A_EMPTY + i), NCONS / 32); }
        for (int i = 0; i < NB; ++i) { mbar_init(BAR(B_FULL + i), 1); mbar_init(BAR(B_EMPTY + i), NCONS / 32); }
        for (int i = 0; i < NCONS / 32; ++i) mbar_init(BAR(RES_FULL + i), 1);
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
            int lo = 0, hi = a.io.B;                   // largest b with pref[b] <= tile (rows without tiles are skipped)
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
        if (!ragged) return a.io.Tin;
        const long long e = (long long)a.io.lens[b] * a.io.rate_in + a.io.need_in;
        return (int)(e < (long long)a.io.Tin ? (e > 0 ? e : 0) : (long long)a.io.Tin);
    };

    if (warp >= W_PROD && warp < W_PROD + NPW) {
        // ============================================================ producers
        const int ptid = tid - 32 * W_PROD;
        const int total = my_tiles * nchunks * SPC;                      // raw stages to fill and transform
        const int vec_per_row = RAWW / 4;
        const int nvec = KC2 * vec_per_row;
        const float slope = a.io.in_slope;
        const float* const xg = a.io.x.p;
        const long long x_bs = a.io.x.bs;
        const int x_cs = a.io.x.cs, Cin = a.Cin, pad = a.pad;
        bool ok = true;
        // Per-thread work items are decoded ONCE (no divisions in the loop), the raw row stride is a compile-time constant
        // (shared loads take immediate offsets), interior windows take a copy path without any bounds logic, and leaky
        // ReLU is max(x, slope * x).
        constexpr int NIT = X3 ? 1 : 2;                 // slabs written per raw stage (X3: X_hi and X_lo of one slab)
        constexpr int MAXV = (8 * 81 + NPROD - 1) / NPROD, MAXI = (NIT * 320 + NPROD - 1) / NPROD;   // raw vectors / slab rows per thread
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
            i_raw[e] = (idx < NIT * ROWS) ? (SLC * sl) * RAWS + r : -1;
            i_dst[e] = (int)(sl * slabA) + r * 16;
        }
        // running positions instead of divisions / modulos per chunk
        int iss_it = 0, iss_c = 0, iss_h = 0, iss_ring = 0, iss_tal = 0, iss_Tin = 0;  // cp.async front: tile, chunk, raw stage of
                                                                                        // the chunk, raw slot
        const float* iss_row = xg;
        bool iss_new = true, iss_int = false;
        int tr_it = 0, tr_c = 0, tr_h = 0, tr_ring = 0, tr_q0 = 0, as = 0;             // transform: the same, A stage
        uint32_t pa_empty = 1;                                    // parity to wait for on A_EMPTY[as]: round 1 -> 0, round 2 -> 1, ...
        bool tr_new = true;
        const uint32_t raw_u32 = smem_u32(smRaw);
        float amax = 0.f;                                         // X3: largest |activation| this thread split
        auto issue = [&](int g) {
            if (g < total) {
                if (iss_new) {
                    int b_, rt_, q0_;
                    decode(iss_it, b_, rt_, q0_);
                    iss_Tin = input_extent(b_);
                    iss_tal = (q0_ - pad) & ~3;                            // 16-byte aligned window start (may be < 0)
                    iss_row = xg + (long long)b_ * x_bs;
                    iss_int = !NEAR && iss_tal >= (a.io.in_lo & ~3) && iss_tal + RAWW <= iss_Tin && (Cin & (KCH - 1)) == 0;
                    iss_new = false;
                }
                // a raw stage is RCH / 8 slots of 8 channels (two for BF16 / FP16): the per-thread work items cover one slot
                const int ch0 = iss_c * KCH + iss_h * RCH;
#pragma unroll
                for (int h = 0; h < RCH / KC2; ++h) {
                    const uint32_t dst0 = raw_u32 + (uint32_t)iss_ring * rawStage + (uint32_t)(h * KC2 * RAWS * 4);
                    if (iss_int) {                                             // whole window inside the row: plain 16-byte copies
                        const float* src = iss_row + (long long)(ch0 + h * KC2) * x_cs + iss_tal;
#pragma unroll
                        for (int e = 0; e < MAXV; ++e)
                            if (v_ch[e] >= 0) cp_async16(dst0 + v_dst[e], src + v_src[e]);
                    } else {
#pragma unroll
                        for (int e = 0; e < MAXV; ++e) {
                            if (v_ch[e] < 0) continue;
                            const int t = iss_tal + v_t[e];
                            const int cg = ch0 + h * KC2 + v_ch[e];
                            if constexpr (NEAR) {
                                // nearest-resampled input: four 4-byte copies from the source columns of t .. t + 3 (a
                                // gather, so no vector copy); columns outside the virtual row [0, Tin) are the zero padding
                                const float* rowp = iss_row + (long long)(cg < Cin ? cg : 0) * x_cs;
#pragma unroll
                                for (int q = 0; q < 4; ++q) {
                                    const int tt = t + q;
                                    const bool in = cg < Cin && tt >= 0 && tt < iss_Tin;
                                    const int src = in ? near_col(tt, a.io.near_src, iss_Tin, a.near_scale) : 0;
                                    cp_async4_zfill(dst0 + v_dst[e] + 4u * q, rowp + src, in ? 4u : 0u);
                                }
                                continue;
                            }
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
                            if (cg < Cin && t >= (a.io.in_lo & ~3)) nb = 4 * max(0, min(4, iss_Tin - t));
                            const int tsafe = (t >= 0 && t < iss_Tin) ? t : 0;
                            const float* src = iss_row + (long long)(cg < Cin ? cg : 0) * x_cs + tsafe;
                            cp_async16_zfill(dst0 + v_dst[e], src, (uint32_t)nb);
                        }
                    }
                }
                if (++iss_h == SPC) { iss_h = 0; if (++iss_c == nchunks) { iss_c = 0; ++iss_it; iss_new = true; } }
            }
            if (++iss_ring == NRAW) iss_ring = 0;
            asm volatile("cp.async.commit_group;" ::: "memory");
        };
        for (int g = 0; g < NRAW - 1; ++g) issue(g);
        for (int g = 0; g < total && ok; ++g) {
            asm volatile("cp.async.wait_group %0;" ::"n"(NRAW - 2) : "memory");
            named_bar_sync(1, NPROD);                                     // everyone's copies of chunk g have landed
            issue(g + NRAW - 1);                                          // refills the stage transformed last iteration
            if (tr_h == 0 && g >= NA2 * SPC) ok = mbar_wait(BAR(A_EMPTY + as), pa_empty, a.err);
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
            if constexpr (X3) {
#pragma unroll
                for (int e = 0; e < MAXI; ++e) {       // ... then prologue, fp16 hi/lo split of 8 channels, two 16-byte stores
                    if (i_raw[e] < 0) continue;
                    uint32_t ph[4], pl[4];
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const float w0 = fmaxf(u[e][2 * i], u[e][2 * i] * slope);
                        const float w1 = fmaxf(u[e][2 * i + 1], u[e][2 * i + 1] * slope);
                        amax = fmaxf(amax, fmaxf(fabsf(w0), fabsf(w1)));
                        split_f16x2(w0, w1, ph[i], pl[i]);
                    }
                    *reinterpret_cast<uint4*>(base + tr_h * slabA + i_dst[e]) = make_uint4(ph[0], ph[1], ph[2], ph[3]);
                    *reinterpret_cast<uint4*>(base + (2 + tr_h) * slabA + i_dst[e]) = make_uint4(pl[0], pl[1], pl[2], pl[3]);
                }
            } else if constexpr (B16) {
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
            if (++tr_ring == NRAW) tr_ring = 0;
            if (++tr_h < SPC) continue;                          // X3: the stage's second half comes from the next raw stage
            tr_h = 0;
            fence_async_smem();                                  // generic-proxy stores -> visible to wgmma (async proxy)
            __syncwarp();
            if (lane == 0) mbar_arrive(BAR(A_FULL + as));       // one arrival per producer warp
            if (++tr_c == nchunks) { tr_c = 0; ++tr_it; tr_new = true; }
            if (++as == NA2) { as = 0; pa_empty ^= 1u; }
        }
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        // X3: an activation fp16 cannot hold (|x| >= 65504) was split into an inf -- the launch's output is invalid
        if (X3 && amax >= F16X3_MAX && a.err) { *reinterpret_cast<volatile int*>(a.err + ERR_RANGE) = 1; __threadfence_system(); }
    } else if (warp == W_LOAD) {
        // ============================================================ weight loader
        // One lane per ring slot: lane s owns slot s and feeds it with tap blocks s, s + NB, s + 2*NB, ... of this CTA's
        // block sequence, so NB independent wait -> expect_tx -> bulk-copy chains are in flight.
        if (lane < NB) {
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
            for (long long gi = lane; gi < all && ok; gi += NB) {
                if (it != cur_it) {
                    int b_, rt, q0_;
                    decode(it, b_, rt, q0_);
                    wsrc = reinterpret_cast<const unsigned char*>(a.w_tc) + (size_t)rt * total * stageB;
                    cur_it = it;
                }
                if (!first) { ok = mbar_wait(empty, par, a.err); if (!ok) break; }
                mbar_expect_tx(full, stageB);
                bulk_g2s(dst, wsrc + (size_t)j * stageB, stageB, full);
                first = false;
                par ^= 1u;
                j += NB;
                while (j >= total) { j -= total; ++it; }
            }
        }
        __syncwarp();
    } else if (TM && warp < W_PROD) {
        if constexpr (TM)
            tm_consumers<TMC, TMS>(a, smA, smB, accs, bar0, decode, my_tiles, nchunks, slabA, warp, lane);
    } else if (warp < W_PROD) {
        // ============================================================ consumers: MMA, then epilogue
        // Every lane runs the same loop (wgmma is warpgroup-collective); after a failed wait (`ok` false, the error flag
        // is set) the remaining waits and MMAs are skipped but the named barriers are still met.
        const int wg = warp >> 2, lq = warp & 3, half = warp >> 2;
        const uint64_t wdesc0 = make_desc(smem_u32(smB) + (uint32_t)wg * 64 * 16, slabB);   // this warpgroup's 64 weight rows
        const uint64_t wlo_off = (uint64_t)((2 * slabB) >> 4), wslot = (uint64_t)(stageB >> 4);
        // X3: this lane's ldmatrix row of W_hi in slot 0: matrix lane / 8 is rows {0-7, 8-15} x slab {0, 1} of the warp's
        // 16 MMA rows (16 warp ..), so the x4 load is the m16k16 A fragment; each 8-lane phase reads 128 contiguous bytes
        const uint32_t whi_lds = smem_u32(smB) + (uint32_t)(lane >> 4) * slabB + (uint32_t)(warp * 16 + (lane & 15)) * 16;
        const uint64_t xstep = (uint64_t)a.dil_blk;                                          // B rows per tap block (16 B each)
        bool ok = true;
        int sa = 0; uint32_t pa = 0;                                                         // activation stage / its parity
        int sb = 0; uint32_t pb = 0;                                                         // weight slot / its parity
        float* const st_row = accs + (wg * 64 + lq * 16 + (lane >> 2)) * ACC_LD + 2 * (lane & 3);
        // Bulk epilogue: in a plain layer without an accumulate operand, a whole interior tile (q0 + 256 <= Tout) is
        // finished by each warp on its own 16 rows, which hold all 256 columns of the warp's accumulator fragment.  Before
        // the tile's MMAs lane 0 prefetches those rows of the residual into the warp's rows of `accs` (cp.async.bulk, 1 KB
        // per row, completing on RES_FULL[warp]); after them the warp adds bias and residual in place and lane 0 writes
        // the rows out with bulk stores.  No consumer-wide barrier is needed: no other warp touches these rows, except
        // in the shared-tile epilogue of the other tiles (edge tiles, accumulate and general-epilogue layers), which
        // is fenced off by a barrier when a bulk tile follows it and by the warp's bulk_wait_read when it follows one.
        // The residual may alias y: a tile reads and writes only its own columns, and only the next tile is prefetched.
        const int row_w = wg * 64 + lq * 16;            // this warp's first tile row
        const ConvIO& io = a.io;
        const bool bulk_layer = BULK && a.ups == 1 && !(io.flags & (EPI_GATE | EPI_ACCUM)) && io.split == 0 &&
                                io.act != ACT_RELU && !io.ymask && io.scale == 1.f && io.post_div == 1.f &&
                                io.y.aligned16() && (!io.res || io.res.aligned16());
        uint32_t pr = 0;                                // parity of RES_FULL[warp]
        bool shared_epi = false;                        // the previous tile's epilogue read other warps' rows of `accs`
#pragma unroll 1
        for (int it = 0; it < my_tiles; ++it) {
            bool bulk, pre;                             // bulk epilogue; residual prefetched (rows of this warp < Rows)
            {
                int b, rt, q0;
                decode(it, b, rt, q0);
                const int nrows = min(16, a.Rows - (rt * MROWS + row_w));
                bulk = bulk_layer && q0 + TT2 <= io.Tout;
                pre = bulk && io.res && nrows > 0;
                if (bulk) {
                    if (shared_epi) { fence_async_smem(); named_bar_sync(4, NCONS); }
                    if (lane == 0) bulk_wait_read();    // this warp's previous bulk stores are done reading its rows
                    __syncwarp();
                }
                if (pre && lane == 0) {
                    const uint32_t rf = BAR(RES_FULL + warp);
                    const float* src = io.res.row(b, rt * MROWS + row_w) + q0;
                    mbar_expect_tx(rf, (uint32_t)nrows * TT2 * 4);
                    for (int r = 0; r < nrows; ++r)
                        bulk_g2s(smem_u32(accs + (row_w + r) * ACC_LD), src + (long long)r * io.res.cs, TT2 * 4, rf);
                }
            }
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
                        uint32_t whs[4];                                         // X3: W_hs = W_hi * 2^-11
                        if constexpr (X3) {
                            ldsm_x4(whs, whi_lds + (uint32_t)sb * stageB);
#pragma unroll
                            for (int i = 0; i < 4; ++i) whs[i] = f16x2_times_2m11(whs[i]);
                        }
                        wgmma_fence();
                        if constexpr (PREC == PREC_BF16) {
                            wgmma_bf16_m64n256(d, w_hi, xh, acc);
                        } else if constexpr (PREC == PREC_FP16) {
                            wgmma_f16_m64n256(d, w_hi, xh, acc);
                        } else if constexpr (X3) {
                            wgmma_f16_m64n256_rs(d, whs, xl, acc);              // small terms first
                            // a group of its own, retired by the wait below: the next tap rewrites whs while only
                            // this tap's two descriptor MMAs are in flight
                            wgmma_commit();
                            wgmma_f16_m64n256(d, w_lo, xh, 1u);
                            wgmma_f16_m64n256(d, w_hi, xh, 1u);
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
                    if (++sb == NB) { sb = 0; pb ^= 1u; }
                }
                if (++sa == NA2) { sa = 0; pa ^= 1u; }
            }
            wgmma_wait<0>();
            release();
            int b, rt, q0;
            decode(it, b, rt, q0);
            if (bulk) {
                if (pre) {                             // waited for even after a failed wait: the copies always land
                    const bool landed = mbar_wait(BAR(RES_FULL + warp), pr, a.err);
                    ok = ok && landed;
                    pr ^= 1u;
                }
                shared_epi = false;
                if (!ok) continue;
                const int r0 = rt * MROWS + row_w, rl = r0 + (lane >> 2);
                float bv[2], sv[2];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int rc = min(rl + 8 * h, a.Rows - 1);
                    bv[h] = a.bias[rc];
                    if (io.cond) bv[h] += __ldg(io.cond.row(b) + rc);
                    sv[h] = SC ? a.rscale[rc] : 1.f;
                }
                if (pre) bulk_combine<true, SC>(d, st_row, bv, sv);
                else bulk_combine<false, SC>(d, st_row, bv, sv);
                fence_async_smem();                    // the combined rows -> visible to the bulk copies (async proxy)
                __syncwarp();
                if (lane == 0) {
                    const int nrows = min(16, a.Rows - r0);
                    float* dst = io.y.row(b, r0) + q0;
                    for (int r = 0; r < nrows; ++r)
                        bulk_s2g(dst + (long long)r * io.y.cs, smem_u32(accs + (row_w + r) * ACC_LD), TT2 * 4);
                    bulk_commit();
                }
                continue;
            }
            if constexpr (BULK) {
                if (lane == 0) bulk_wait_read();       // this warp's last bulk stores are done reading its rows
                __syncwarp();
            }
            named_bar_sync(4, NCONS);                  // every warp is done reading the previous tile's accumulators
#pragma unroll
            for (int j = 0; j < 32; ++j) {
                *reinterpret_cast<float2*>(st_row + 8 * j) = make_float2(d[4 * j], d[4 * j + 1]);
                *reinterpret_cast<float2*>(st_row + 8 * ACC_LD + 8 * j) = make_float2(d[4 * j + 2], d[4 * j + 3]);
            }
            named_bar_sync(4, NCONS);
            shared_epi = true;
            if (!ok) continue;
            if constexpr (GRP > 1) {
                grouped_tile<GRP, SC>(a, accs, b, q0, lq, half, lane);
            } else {
                const int qb = q0 + half * 128;
                const float* at = accs + lq * 32 * ACC_LD + half * 128;            // this warp's 32 rows x 128 columns
                const bool lean = LEAN && a.ups == 1 && !(io.flags & EPI_GATE) && io.split == 0 && io.act != ACT_RELU &&
                                  !io.ymask && io.scale == 1.f && io.post_div == 1.f && qb + 128 <= io.Tout &&
                                  io.y.aligned16() && (!io.res || io.res.aligned16());
                if (lean) {
                    // every interior tile half of the plain layers: coalesced global accesses, no per-option branches
                    const int row0 = rt * MROWS + lq * 32;
                    const float* cond = io.cond ? io.cond.row(b) : nullptr;
                    float* yq = io.y.row(b, 0) + qb;
                    const bool hres = io.res.p != nullptr, hacc = (io.flags & EPI_ACCUM) != 0;
                    const float* rq = hres ? io.res.row(b, 0) + qb : yq;
                    if (hres) { if (hacc) lean_tile<true, true, SC>(at, a.bias, a.rscale, cond, lane, rq, yq, io.res.cs, io.y.cs, row0, a.Rows, true);
                                else lean_tile<true, false, SC>(at, a.bias, a.rscale, cond, lane, rq, yq, io.res.cs, io.y.cs, row0, a.Rows, true); }
                    else { if (hacc) lean_tile<false, true, SC>(at, a.bias, a.rscale, cond, lane, rq, yq, 0, io.y.cs, row0, a.Rows, true);
                           else lean_tile<false, false, SC>(at, a.bias, a.rscale, cond, lane, rq, yq, 0, io.y.cs, row0, a.Rows, true); }
                } else if constexpr (LEAN) {
                    general_tile_call<SC>(a, at + lane * ACC_LD, b, rt, q0, lq, half, lane);
                } else {
                    general_tile_body<SC, WG>(a, a.rscale, at + lane * ACC_LD, b, rt, q0, lq, half, lane);
                }
            }
        }
        if constexpr (BULK) {
            if (lane == 0) bulk_wait_all();            // the bulk stores are complete before the dependent grid may read
            __syncwarp();
        }
    }
}

// PREC: PREC_FP32 (3xTF32), PREC_BF16, PREC_FP16 or PREC_F16X3
template <int PREC, bool REFL = false>
__global__ void __launch_bounds__(NTHREADS2, 1) conv1d_tc3_kernel(const __grid_constant__ Tc3Args a) { tc3_body<1, true, PREC, REFL>(a); }
template <int PREC>   // gate / split / mask / polyphase
__global__ void __launch_bounds__(NTHREADS2, 1) conv1d_tc3x_kernel(const __grid_constant__ Tc3Args a) { tc3_body<1, false, PREC>(a); }
template <int GRP, int PREC, bool REFL = false>
__global__ void __launch_bounds__(NTHREADS2, 1) conv1d_tc3g_kernel(const __grid_constant__ Tc3Args a) { tc3_body<GRP, true, PREC, REFL>(a); }

// WaveGrad layers (EPI_WAVEGRAD / nearest-resampled input): the WaveGrad epilogue inline, NEAR for a resampled input
template <int PREC, bool NEAR>
__global__ void __launch_bounds__(NTHREADS2, 1) conv1d_tc3w_kernel(const __grid_constant__ Tc3Args a) {
    tc3_body<1, false, PREC, false, NEAR, true>(a);
}

typedef void (*Tc3Kernel)(const Tc3Args);
// the WaveGrad kernels exist for 3xTF32 and the split-fp16 operands (the precisions WaveGrad packs)
static inline Tc3Kernel wavegrad_kernel(int prec, bool near) {
    if (prec == PREC_F16X3) return near ? conv1d_tc3w_kernel<PREC_F16X3, true> : conv1d_tc3w_kernel<PREC_F16X3, false>;
    if (prec == PREC_FP32) return near ? conv1d_tc3w_kernel<PREC_FP32, true> : conv1d_tc3w_kernel<PREC_FP32, false>;
    return nullptr;
}
// reflect: the reflection-padding variant (lean epilogue only; the host sends reflect-padded layers that need the general
// epilogue to the FMA kernel)
static inline Tc3Kernel plain_kernel(int prec, bool lean, bool reflect = false) {
    if (reflect) {
        if (prec == PREC_BF16) return conv1d_tc3_kernel<PREC_BF16, true>;
        if (prec == PREC_FP16) return conv1d_tc3_kernel<PREC_FP16, true>;
        if (prec == PREC_F16X3) return conv1d_tc3_kernel<PREC_F16X3, true>;
        return conv1d_tc3_kernel<PREC_FP32, true>;
    }
    if (prec == PREC_BF16) return lean ? conv1d_tc3_kernel<PREC_BF16> : conv1d_tc3x_kernel<PREC_BF16>;
    if (prec == PREC_FP16) return lean ? conv1d_tc3_kernel<PREC_FP16> : conv1d_tc3x_kernel<PREC_FP16>;
    if (prec == PREC_F16X3) return lean ? conv1d_tc3_kernel<PREC_F16X3> : conv1d_tc3x_kernel<PREC_F16X3>;
    return lean ? conv1d_tc3_kernel<PREC_FP32> : conv1d_tc3x_kernel<PREC_FP32>;
}
// grouped kernel for 2 / 4 tap groups (any dilation with (GRP - 1) * dil <= 15); 3xTF32 and 16-bit operands only
// (PREC_F16X3 takes the time-major kernel)
template <bool REFL>
static inline Tc3Kernel grouped_kernel_t(int grp, int prec) {
    if (prec == PREC_BF16) return grp == 2 ? conv1d_tc3g_kernel<2, PREC_BF16, REFL> : conv1d_tc3g_kernel<4, PREC_BF16, REFL>;
    if (prec == PREC_FP16) return grp == 2 ? conv1d_tc3g_kernel<2, PREC_FP16, REFL> : conv1d_tc3g_kernel<4, PREC_FP16, REFL>;
    return grp == 2 ? conv1d_tc3g_kernel<2, PREC_FP32, REFL> : conv1d_tc3g_kernel<4, PREC_FP32, REFL>;
}
static inline Tc3Kernel grouped_kernel(int grp, int prec = PREC_FP32, bool reflect = false) {
    return reflect ? grouped_kernel_t<true>(grp, prec) : grouped_kernel_t<false>(grp, prec);
}

// Time-major split-fp16 kernel for exactly C = 32 / 64 output rows, TMS m64 slices per warpgroup (tile width 128 * TMS)
template <int C, int TMS, bool REFL>
__global__ void __launch_bounds__(NTHREADS2, 1) conv1d_tc3t_kernel(const __grid_constant__ Tc3Args a) {
    tc3_body<1, true, PREC_F16X3, REFL, false, false, C, TMS>(a);
}
template <int C, bool REFL>
static inline Tc3Kernel timemajor_kernel_t(int tms) {
    return tms == 2 ? conv1d_tc3t_kernel<C, 2, REFL> : conv1d_tc3t_kernel<C, 1, REFL>;
}
static inline Tc3Kernel timemajor_kernel(int C, int tms, bool reflect) {
    if (C == 64) return reflect ? timemajor_kernel_t<64, true>(tms) : timemajor_kernel_t<64, false>(tms);
    return reflect ? timemajor_kernel_t<32, true>(tms) : timemajor_kernel_t<32, false>(tms);
}

}  // namespace tc3
}  // namespace b200tts
