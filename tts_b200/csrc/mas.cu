// Monotonic alignment search on sm_90a.
//
// Reference: TTS/tts/utils/monotonic_align/core.pyx:11-37 (maximum_path_each: in-place DP over a
// band, then a backtrack reading the DP values) and :42-47 (batch loop); caller
// TTS/tts/utils/helpers.py:178-194 (value*mask, t_x/t_y from mask sums, int32 path).
//
// HBM-bound integer/compare work (8 B per cell: value in, path out) -- no tensor cores.
// One CTA per batch item.  The y-contiguous value rows are staged through shared memory in
// [Tx][YT] tiles with 4-byte cp.async (128 B coalesced per warp, double buffered), so the
// column-serial DP reads shared memory conflict-free.  The "stored column" (the reference's
// in-place value[:, y-1]) lives in a 2-deep shared array; the comparison the backtrack will need
// (value[x,y-1] < value[x-1,y-1]) is the same pair the DP step already holds, so each step emits
// one ballot word of direction bits per warp instead of writing DP values back to HBM.
// The backtrack runs on one warp over those bit rows (prefetched 16 deep), then the whole CTA
// writes the [Tx][Ty] 0/1 path with coalesced vector stores (no separate memset pass).
//
// Exactness: only max, one add and compares touch the data (__fadd_rn/__fmul_rn, no FMA
// contraction), evaluated in the reference's order, so paths are bit-identical.  Cells outside
// the band keep value*mask exactly like the reference's untouched entries, which also makes the
// degenerate t_x > t_y case follow core.pyx (minus its unused out-of-row read at y == 0).
#include <stdlib.h>

#include "engines.cuh"

namespace b200tts {

namespace {

constexpr int MAS_NT = 256;
constexpr int MAS_DEPTH = 16;

__device__ __forceinline__ void cp_async4(float* smem_dst, const float* gsrc) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(s), "l"(gsrc));
}

__device__ __forceinline__ float lds_f32(unsigned addr) { float v; asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr)); return v; }
__device__ __forceinline__ void sts_f32(unsigned addr, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory"); }
__device__ __forceinline__ void sts_u32(unsigned addr, unsigned v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }

struct MasArgs {
    const float* value; const float* mask; const int* t_x; const int* t_y;
    int B, Tx, Ty, YT, W;     // W = ceil(Tx/32) words per direction row
    void* path; int path_is_f32;
    unsigned* dirs_global;    // [B][Ty][W] when the bit rows do not fit in shared memory
    int dirs_in_smem;
    float max_neg;
};

__global__ void __launch_bounds__(MAS_NT) mas_kernel(const MasArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int Tx = a.Tx, Ty = a.Ty, YT = a.YT, YS = YT + 1, W = a.W;
    int tx = a.t_x[b], ty = a.t_y[b];
    tx = min(max(tx, 0), Tx);
    ty = min(max(ty, 0), Ty);
    const bool has_mask = a.mask != nullptr;

    float* tileV = reinterpret_cast<float*>(smem_raw);               // [2][Tx*YS]
    float* tileM = tileV + 2 * Tx * YS;                              // [2][Tx*YS] (mask) or empty
    float* col = tileM + (has_mask ? 2 * Tx * YS : 0);               // [2][Tx+1], col[.][0] unused pad
    int* idxs = reinterpret_cast<int*>(col + 2 * (Tx + 1));          // [Ty]
    unsigned* dirs = a.dirs_in_smem ? reinterpret_cast<unsigned*>(idxs + Ty)
                                    : a.dirs_global + (size_t)b * Ty * W;  // [Ty][W]

    const float* vb = a.value + (size_t)b * Tx * Ty;
    const float* mbp = has_mask ? a.mask + (size_t)b * Tx * Ty : nullptr;
    const int ytshift = 31 - __clz(YT);

    auto load_tile = [&](int tile, int buf) {
        const int y0 = tile * YT;
        float* dv = tileV + buf * Tx * YS;
        float* dm = tileM + buf * Tx * YS;
        const int n = Tx << ytshift;
        for (int i = tid; i < n; i += MAS_NT) {
            const int x = i >> ytshift, yy = i & (YT - 1), y = y0 + yy;
            if (y < ty) {
                cp_async4(dv + x * YS + yy, vb + (size_t)x * Ty + y);
                if (has_mask) cp_async4(dm + x * YS + yy, mbp + (size_t)x * Ty + y);
            }
        }
        asm volatile("cp.async.commit_group;");
    };

    for (int x = tid; x < 2 * (Tx + 1); x += MAS_NT) col[x] = 0.f;

    const int ntiles = (ty + YT - 1) / YT;
    if (ntiles > 0) load_tile(0, 0);
    for (int tile = 0; tile < ntiles; ++tile) {
        const int buf = tile & 1;
        if (tile + 1 < ntiles) {
            load_tile(tile + 1, buf ^ 1);
            asm volatile("cp.async.wait_group 1;" ::: "memory");
        } else {
            asm volatile("cp.async.wait_group 0;" ::: "memory");
        }
        __syncthreads();
        const float* tv = tileV + buf * Tx * YS;
        const float* tm = tileM + buf * Tx * YS;
        const int y0 = tile * YT;
        const int ylim = min(YT, ty - y0);
        for (int yy = 0; yy < ylim; ++yy) {
            const int y = y0 + yy;
            const float* cp = col + (y & 1) * (Tx + 1) + 1;        // stored column y-1 (index x -> cp[x])
            float* cc = col + ((y + 1) & 1) * (Tx + 1) + 1;        // column y
            const int lo = max(0, tx + y - ty), hi = min(tx, y + 1);
            for (int x0 = 0; x0 < Tx; x0 += MAS_NT) {
                const int x = x0 + tid;
                bool dir = false;
                if (x < Tx) {
                    float raw = tv[x * YS + yy];
                    if (has_mask) raw = __fmul_rn(raw, tm[x * YS + yy]);
                    const float vc_s = cp[x];
                    const float vp_s = cp[x - 1];                   // x == 0 reads the pad slot (unused)
                    float nv = raw;
                    if (x >= lo && x < hi) {
                        const float v_cur = (x == y) ? a.max_neg : vc_s;
                        const float v_prev = (x == 0) ? (y == 0 ? 0.f : a.max_neg) : vp_s;
                        nv = __fadd_rn(fmaxf(v_cur, v_prev), raw);
                    }
                    cc[x] = nv;
                    dir = (y > 0) && (x != 0) && (x == y || vc_s < vp_s);
                }
                const unsigned word = __ballot_sync(0xffffffffu, dir);
                const int widx = (x0 >> 5) + warp;
                if (lane == 0 && widx < W) dirs[(size_t)y * W + widx] = word;
            }
            __syncthreads();
        }
    }
    __syncthreads();

    // ---------------------------------------------------------------- backtrack (warp 0)
    if (warp == 0 && tx > 0) {
        int index = tx - 1;
        for (int ytop = ty - 1; ytop >= 0; ytop -= MAS_DEPTH) {
            unsigned rows[MAS_DEPTH];
#pragma unroll
            for (int d = 0; d < MAS_DEPTH; ++d) {
                const int y = ytop - d;
                rows[d] = 0u;
                if (y >= 1 && W <= 32) rows[d] = (lane < W) ? dirs[(size_t)y * W + lane] : 0u;
            }
#pragma unroll
            for (int d = 0; d < MAS_DEPTH; ++d) {
                const int y = ytop - d;
                if (y < 0) break;
                if (lane == 0) idxs[y] = index;
                if (y >= 1) {
                    unsigned word;
                    if (W <= 32) word = __shfl_sync(0xffffffffu, rows[d], index >> 5);
                    else word = dirs[(size_t)y * W + (index >> 5)];
                    index -= (int)((word >> (index & 31)) & 1u);
                }
            }
        }
    }
    __syncthreads();

    // ---------------------------------------------------------------- path write: [Tx][Ty], ones at (idxs[y], y)
    const bool valid = tx > 0;
    if (a.path_is_f32) {
        float* pb = reinterpret_cast<float*>(a.path) + (size_t)b * Tx * Ty;
        for (size_t i = tid; i < (size_t)Tx * Ty; i += MAS_NT) {
            const int x = (int)(i / Ty), y = (int)(i - (size_t)x * Ty);
            pb[i] = (valid && y < ty && idxs[y] == x) ? 1.f : 0.f;
        }
    } else {
        int* pb = reinterpret_cast<int*>(a.path) + (size_t)b * Tx * Ty;
        if ((Ty & 3) == 0) {
            int4* pb4 = reinterpret_cast<int4*>(pb);
            const int Ty4 = Ty >> 2;
            for (size_t i = tid; i < (size_t)Tx * Ty4; i += MAS_NT) {
                const int x = (int)(i / Ty4), y = (int)(i - (size_t)x * Ty4) << 2;
                int4 o;
                o.x = (valid && y + 0 < ty && idxs[y + 0] == x) ? 1 : 0;
                o.y = (valid && y + 1 < ty && idxs[y + 1] == x) ? 1 : 0;
                o.z = (valid && y + 2 < ty && idxs[y + 2] == x) ? 1 : 0;
                o.w = (valid && y + 3 < ty && idxs[y + 3] == x) ? 1 : 0;
                pb4[i] = o;
            }
        } else {
            for (size_t i = tid; i < (size_t)Tx * Ty; i += MAS_NT) {
                const int x = (int)(i / Ty), y = (int)(i - (size_t)x * Ty);
                pb[i] = (valid && y < ty && idxs[y] == x) ? 1 : 0;
            }
        }
    }
}

// ------------------------------------------------------------------ lean kernel for Tx <= 256 (one thread per text position)
// Same semantics as mas_kernel, ~3x fewer instructions per DP step: the stored column lives in a register, the left
// neighbour comes from __shfl_up (only warp-boundary values go through shared memory), band limits are warp-uniform,
// and value tiles are staged transposed ([yy][x], pitch odd mod 32) so both the 4-byte cp.async writes and the
// per-step reads are bank-conflict free.
constexpr int MAS2_YT = 16;

template <bool HAS_MASK, bool DIRS_SMEM>
__global__ void __launch_bounds__(MAS_NT) mas_kernel2(const MasArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int Tx = a.Tx, Ty = a.Ty, W = a.W;
    constexpr int YT = MAS2_YT, NW = MAS_NT / 32;
    const int TxP = (Tx | 31) + 2;                 // pitch == 1 (mod 32)
    int tx = min(max(a.t_x[b], 0), Tx), ty = min(max(a.t_y[b], 0), Ty);
    constexpr bool has_mask = HAS_MASK;
    float* tileV = reinterpret_cast<float*>(smem_raw);                    // [2][YT][TxP]
    float* tileM = tileV + 2 * YT * TxP;                                  // [2][YT][TxP] or empty
    float* bound = tileM + (has_mask ? 2 * YT * TxP : 0);                 // [2][NW]
    int* idxs = reinterpret_cast<int*>(bound + 2 * NW);                   // [Ty]
    unsigned* dirs_s = reinterpret_cast<unsigned*>(idxs + Ty);             // [Ty][W] when DIRS_SMEM
    unsigned* dirs_g = a.dirs_global + (size_t)b * Ty * W;
    const float* vb = a.value + (size_t)b * Tx * Ty;
    const float* mbp = has_mask ? a.mask + (size_t)b * Tx * Ty : nullptr;

    // loader mapping: lane -> (yy, row-in-group); a warp covers 32/YT rows per iteration
    const int l_yy = lane % YT, l_xs = lane / YT;
    constexpr int RPI = 32 / YT;                                          // rows per warp iteration
    auto load_tile = [&](int tile, int buf) {
        const int y = tile * YT + l_yy;
        float* dv = tileV + buf * YT * TxP + l_yy * TxP;
        float* dm = tileM + buf * YT * TxP + l_yy * TxP;
        if (y < ty) {
            for (int x = warp * RPI + l_xs; x < Tx; x += NW * RPI) {
                cp_async4(dv + x, vb + (size_t)x * Ty + y);
                if (has_mask) cp_async4(dm + x, mbp + (size_t)x * Ty + y);
            }
        }
        asm volatile("cp.async.commit_group;");
    };
    if (tid < 2 * NW) bound[tid] = 0.f;

    const int x = tid;
    const bool xin = x < Tx;
    // per-thread invariants of the band test  max(0, tx+y-ty) <= x < min(tx, y+1):
    //   x < tx (constant), x <= y, x - tx + ty >= y
    const bool x_lt_tx = x < tx;
    const int c1 = x - tx + ty;
    const bool is_x0 = (x == 0);
    const float neg = a.max_neg;
    float vc = 0.f;                                                       // stored[x, y-1]
    float* bnd_w = bound + warp;                                          // this warp's slot (written by lane 31)
    const float* bnd_r = bound + (warp > 0 ? warp - 1 : 0);               // left warp's slot (read by lane 0)
    const bool rd_bound = (lane == 0) && (warp > 0);
    const bool wr_bound = (lane == 31);
    const bool wr_dir = (lane == 0) && (warp < W);
    const unsigned a_bnd_w = (unsigned)__cvta_generic_to_shared(bnd_w);
    const unsigned a_bnd_r = (unsigned)__cvta_generic_to_shared(bnd_r);
    const unsigned a_dirs0 = (unsigned)__cvta_generic_to_shared(dirs_s + warp);
    const int ntiles = (ty + YT - 1) / YT;
    if (ntiles > 0) load_tile(0, 0);
    for (int tile = 0; tile < ntiles; ++tile) {
        const int buf = tile & 1;
        if (tile + 1 < ntiles) { load_tile(tile + 1, buf ^ 1); asm volatile("cp.async.wait_group 1;" ::: "memory"); }
        else asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();
        // raw 32-bit shared addresses kept in registers (the generic-pointer form recomputed the window base per step)
        unsigned a_tv = (unsigned)__cvta_generic_to_shared(tileV + buf * YT * TxP + (xin ? x : 0));
        unsigned a_tm = (unsigned)__cvta_generic_to_shared(tileM + buf * YT * TxP + (xin ? x : 0));
        const int y0 = tile * YT, ylim = min(YT, ty - y0);
        unsigned a_dir = a_dirs0 + (unsigned)(y0 * W) * 4u;
#pragma unroll 1
        for (int yy = 0; yy < ylim; ++yy) {
            const int y = y0 + yy;
            float raw = lds_f32(a_tv);
            if (HAS_MASK) raw = __fmul_rn(raw, lds_f32(a_tm));
            float left = __shfl_up_sync(0xffffffffu, vc, 1);
            const unsigned par = (unsigned)(y & 1) * (NW * 4u);
            if (rd_bound) left = lds_f32(a_bnd_r + par);
            // dir[x,y] = (y > 0) && (x != 0) && (x == y || stored[x,y-1] < stored[x-1,y-1])
            const bool x_eq_y = (x == y);
            const bool dir = xin && !is_x0 && (y > 0) && (x_eq_y || vc < left);
            const bool inband = x_lt_tx && (x <= y) && (c1 >= y);
            const float v_cur = x_eq_y ? neg : vc;
            const float v_prev = is_x0 ? (y == 0 ? 0.f : neg) : left;
            const float upd = __fadd_rn(fmaxf(v_cur, v_prev), raw);
            vc = inband ? upd : (xin ? raw : 0.f);
            const unsigned word = __ballot_sync(0xffffffffu, dir);
            if (wr_bound) sts_f32(a_bnd_w + (NW * 4u - par), vc);
            if (wr_dir) {
                if (DIRS_SMEM) sts_u32(a_dir, word);
                else dirs_g[(size_t)y * W + warp] = word;
            }
            a_tv += (unsigned)TxP * 4u; a_tm += (unsigned)TxP * 4u; a_dir += (unsigned)W * 4u;
            __syncthreads();
        }
    }
    const unsigned* dirs = DIRS_SMEM ? dirs_s : dirs_g;
    __syncthreads();
    if (warp == 0 && tx > 0) {
        int index = tx - 1;
        for (int ytop = ty - 1; ytop >= 0; ytop -= MAS_DEPTH) {
            unsigned rows[MAS_DEPTH];
#pragma unroll
            for (int d = 0; d < MAS_DEPTH; ++d) {
                const int y = ytop - d;
                rows[d] = (y >= 1 && lane < W) ? dirs[(size_t)y * W + lane] : 0u;
            }
#pragma unroll
            for (int d = 0; d < MAS_DEPTH; ++d) {
                const int y = ytop - d;
                if (y < 0) break;
                if (lane == 0) idxs[y] = index;
                if (y >= 1) {
                    const unsigned word = __shfl_sync(0xffffffffu, rows[d], index >> 5);
                    index -= (int)((word >> (index & 31)) & 1u);
                }
            }
        }
    }
    __syncthreads();
    const bool valid = tx > 0;
    if (a.path_is_f32) {
        float* pb = reinterpret_cast<float*>(a.path) + (size_t)b * Tx * Ty;
        if ((Ty & 3) == 0) {
            float4* pb4 = reinterpret_cast<float4*>(pb);
            const int Ty4 = Ty >> 2;
            for (int xx = warp; xx < Tx; xx += NW)
                for (int j = lane; j < Ty4; j += 32) {
                    const int y = j << 2;
                    float4 o;
                    o.x = (valid && y + 0 < ty && idxs[y + 0] == xx) ? 1.f : 0.f;
                    o.y = (valid && y + 1 < ty && idxs[y + 1] == xx) ? 1.f : 0.f;
                    o.z = (valid && y + 2 < ty && idxs[y + 2] == xx) ? 1.f : 0.f;
                    o.w = (valid && y + 3 < ty && idxs[y + 3] == xx) ? 1.f : 0.f;
                    pb4[(size_t)xx * Ty4 + j] = o;
                }
        } else {
            for (size_t i = tid; i < (size_t)Tx * Ty; i += MAS_NT) {
                const int xx = (int)(i / Ty), y = (int)(i - (size_t)xx * Ty);
                pb[i] = (valid && y < ty && idxs[y] == xx) ? 1.f : 0.f;
            }
        }
    } else {
        int* pb = reinterpret_cast<int*>(a.path) + (size_t)b * Tx * Ty;
        if ((Ty & 3) == 0) {
            int4* pb4 = reinterpret_cast<int4*>(pb);
            const int Ty4 = Ty >> 2;
            for (int xx = warp; xx < Tx; xx += NW)
                for (int j = lane; j < Ty4; j += 32) {
                    const int y = j << 2;
                    int4 o;
                    o.x = (valid && y + 0 < ty && idxs[y + 0] == xx) ? 1 : 0;
                    o.y = (valid && y + 1 < ty && idxs[y + 1] == xx) ? 1 : 0;
                    o.z = (valid && y + 2 < ty && idxs[y + 2] == xx) ? 1 : 0;
                    o.w = (valid && y + 3 < ty && idxs[y + 3] == xx) ? 1 : 0;
                    pb4[(size_t)xx * Ty4 + j] = o;
                }
        } else {
            for (size_t i = tid; i < (size_t)Tx * Ty; i += MAS_NT) {
                const int xx = (int)(i / Ty), y = (int)(i - (size_t)xx * Ty);
                pb[i] = (valid && y < ty && idxs[y] == xx) ? 1 : 0;
            }
        }
    }
}

// ------------------------------------------------------------------ third generation: no CTA barrier in the DP loop
// mas_kernel2 spends its time in one __syncthreads per DP column (ncu: the barrier is the top stall, issue slots 56 %
// busy).  The only cross-warp dependency of column y is ONE value: lane 0 of warp w needs stored[32w - 1, y - 1] from
// lane 31 of warp w - 1.  So the warps run as a skewed wavefront: each publishes that boundary value into a small ring
// in shared memory with a release store of its progress counter, its right neighbour acquires the counter (cached: it
// polls only when it has caught up) -- no barrier at all between the first column and the backtrack.
// Values never touch shared memory either: lane x streams row x as two LDG.128 per 8 columns (full 32-byte sectors),
// prefetched two groups ahead in registers.
constexpr int MAS3_RING = 64;          // boundary slots per warp (columns a producer may run ahead of its consumer)

__device__ __forceinline__ int ld_acquire_s32(unsigned addr) { int v; asm volatile("ld.acquire.cta.shared.s32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory"); return v; }
__device__ __forceinline__ void st_release_s32(unsigned addr, int v) { asm volatile("st.release.cta.shared.s32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }

template <bool HAS_MASK>
__global__ void __launch_bounds__(MAS_NT, 3) mas_kernel3(const MasArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int Tx = a.Tx, Ty = a.Ty, W = a.W;
    constexpr int NW = MAS_NT / 32;
    const int tx = min(max(a.t_x[b], 0), Tx), ty = min(max(a.t_y[b], 0), Ty);
    int* idxs = reinterpret_cast<int*>(smem_raw);                              // [Ty]
    unsigned* dirs = reinterpret_cast<unsigned*>(idxs + Ty);                   // [Ty][W]
    float* ring = reinterpret_cast<float*>(dirs + (size_t)Ty * W);             // [NW][MAS3_RING]
    int* prog = reinterpret_cast<int*>(ring + NW * MAS3_RING);                 // [NW] columns completed per warp
    if (tid < NW) prog[tid] = 0;
    __syncthreads();

    const int x = tid;
    const bool xin = x < Tx, active = warp < W;
    if (active && tx > 0 && ty > 0) {
        const size_t row = ((size_t)b * Tx + (size_t)(xin ? x : Tx - 1)) * Ty;
        const float4* vrow = reinterpret_cast<const float4*>(a.value + row);
        const float4* mrow = HAS_MASK ? reinterpret_cast<const float4*>(a.mask + row) : nullptr;
        const int ngroups = (ty + 7) / 8, Ty4 = Ty >> 2;
        auto load = [&](int g, float* v) {                 // columns [8g, 8g + 8) of this lane's row (masked on load)
            float4 p = make_float4(0.f, 0.f, 0.f, 0.f), q = p;
            if (g < ngroups) {
                p = __ldg(vrow + 2 * g);
                if (2 * g + 1 < Ty4) q = __ldg(vrow + 2 * g + 1);
                if (HAS_MASK) {
                    const float4 mp = __ldg(mrow + 2 * g);
                    float4 mq = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (2 * g + 1 < Ty4) mq = __ldg(mrow + 2 * g + 1);
                    p.x = __fmul_rn(p.x, mp.x); p.y = __fmul_rn(p.y, mp.y); p.z = __fmul_rn(p.z, mp.z); p.w = __fmul_rn(p.w, mp.w);
                    q.x = __fmul_rn(q.x, mq.x); q.y = __fmul_rn(q.y, mq.y); q.z = __fmul_rn(q.z, mq.z); q.w = __fmul_rn(q.w, mq.w);
                }
            }
            v[0] = p.x; v[1] = p.y; v[2] = p.z; v[3] = p.w; v[4] = q.x; v[5] = q.y; v[6] = q.z; v[7] = q.w;
        };
        const bool x_lt_tx = x < tx, is_x0 = (x == 0);
        const int c1 = x - tx + ty;
        const float neg = a.max_neg;
        const bool first = (warp == 0), last = (warp == W - 1);
        const unsigned a_ring_w = (unsigned)__cvta_generic_to_shared(ring + warp * MAS3_RING);
        const unsigned a_ring_r = (unsigned)__cvta_generic_to_shared(ring + (first ? 0 : warp - 1) * MAS3_RING);
        const unsigned a_prog_w = (unsigned)__cvta_generic_to_shared(prog + warp);
        const unsigned a_prog_l = (unsigned)__cvta_generic_to_shared(prog + (first ? 0 : warp - 1));
        const unsigned a_prog_r = (unsigned)__cvta_generic_to_shared(prog + (last ? warp : warp + 1));
        unsigned a_dir = (unsigned)__cvta_generic_to_shared(dirs + warp);
        int seen_left = 0, seen_right = 0;                // cached progress of the neighbours
        float vc = 0.f;                                   // stored[x, y - 1]
        float cur[8], n1[8], n2[8];
        load(0, cur); load(1, n1); load(2, n2);
#pragma unroll 1
        for (int g = 0; g < ngroups; ++g) {
            float n3[8];
            load(g + 3, n3);
            const int ylim = min(8, ty - 8 * g);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                if (j < ylim) {
                    const int y = 8 * g + j;
                    const float raw = xin ? cur[j] : 0.f;
                    float left = __shfl_up_sync(0xffffffffu, vc, 1);
                    if (lane == 0 && !first && y > 0) {                 // stored[32w - 1, y - 1] from the left warp
                        while (seen_left < y) seen_left = ld_acquire_s32(a_prog_l);
                        left = lds_f32(a_ring_r + (unsigned)((y - 1) & (MAS3_RING - 1)) * 4u);
                    }
                    const bool x_eq_y = (x == y);
                    const bool dir = xin && !is_x0 && (y > 0) && (x_eq_y || vc < left);
                    const bool inband = x_lt_tx && (x <= y) && (c1 >= y);
                    const float v_cur = x_eq_y ? neg : vc;
                    const float v_prev = is_x0 ? (y == 0 ? 0.f : neg) : left;
                    const float upd = __fadd_rn(fmaxf(v_cur, v_prev), raw);
                    vc = inband ? upd : raw;
                    const unsigned word = __ballot_sync(0xffffffffu, dir);
                    if (lane == 0) sts_u32(a_dir, word);
                    a_dir += (unsigned)W * 4u;
                    if (lane == 31) {
                        if (!last) {
                            // do not overwrite a slot the right warp has not read yet (it reads column c at its column c + 1)
                            while (seen_right < y - MAS3_RING + 2) seen_right = ld_acquire_s32(a_prog_r);
                            sts_f32(a_ring_w + (unsigned)(y & (MAS3_RING - 1)) * 4u, vc);
                        }
                        st_release_s32(a_prog_w, y + 1);
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) { cur[j] = n1[j]; n1[j] = n2[j]; n2[j] = n3[j]; }
        }
    }
    __syncthreads();
    if (warp == 0 && tx > 0) {
        int index = tx - 1;
        for (int ytop = ty - 1; ytop >= 0; ytop -= MAS_DEPTH) {
            unsigned rows[MAS_DEPTH];
#pragma unroll
            for (int d = 0; d < MAS_DEPTH; ++d) {
                const int y = ytop - d;
                rows[d] = (y >= 1 && lane < W) ? dirs[(size_t)y * W + lane] : 0u;
            }
#pragma unroll
            for (int d = 0; d < MAS_DEPTH; ++d) {
                const int y = ytop - d;
                if (y < 0) break;
                if (lane == 0) idxs[y] = index;
                if (y >= 1) {
                    const unsigned word = __shfl_sync(0xffffffffu, rows[d], index >> 5);
                    index -= (int)((word >> (index & 31)) & 1u);
                }
            }
        }
    }
    __syncthreads();
    const bool valid = tx > 0;
    const int Ty4 = Ty >> 2;                               // the launcher guarantees Ty % 4 == 0
    if (a.path_is_f32) {
        float4* pb4 = reinterpret_cast<float4*>(reinterpret_cast<float*>(a.path) + (size_t)b * Tx * Ty);
        for (int xx = warp; xx < Tx; xx += NW)
            for (int j = lane; j < Ty4; j += 32) {
                const int y = j << 2;
                float4 o;
                o.x = (valid && y + 0 < ty && idxs[y + 0] == xx) ? 1.f : 0.f;
                o.y = (valid && y + 1 < ty && idxs[y + 1] == xx) ? 1.f : 0.f;
                o.z = (valid && y + 2 < ty && idxs[y + 2] == xx) ? 1.f : 0.f;
                o.w = (valid && y + 3 < ty && idxs[y + 3] == xx) ? 1.f : 0.f;
                pb4[(size_t)xx * Ty4 + j] = o;
            }
    } else {
        int4* pb4 = reinterpret_cast<int4*>(reinterpret_cast<int*>(a.path) + (size_t)b * Tx * Ty);
        for (int xx = warp; xx < Tx; xx += NW)
            for (int j = lane; j < Ty4; j += 32) {
                const int y = j << 2;
                int4 o;
                o.x = (valid && y + 0 < ty && idxs[y + 0] == xx) ? 1 : 0;
                o.y = (valid && y + 1 < ty && idxs[y + 1] == xx) ? 1 : 0;
                o.z = (valid && y + 2 < ty && idxs[y + 2] == xx) ? 1 : 0;
                o.w = (valid && y + 3 < ty && idxs[y + 3] == xx) ? 1 : 0;
                pb4[(size_t)xx * Ty4 + j] = o;
            }
    }
}

static size_t mas3_smem(int Tx, int Ty) {
    const int W = (Tx + 31) / 32;
    return (size_t)Ty * 4 + (size_t)Ty * W * 4 + (size_t)(MAS_NT / 32) * MAS3_RING * 4 + (size_t)(MAS_NT / 32) * 4 + 16;
}

static size_t mas2_smem(int Tx, int Ty, bool has_mask, bool dirs_in_smem) {
    const int TxP = (Tx | 31) + 2, W = (Tx + 31) / 32;
    return (size_t)(has_mask ? 4 : 2) * MAS2_YT * TxP * 4 + 2 * (MAS_NT / 32) * 4 + (size_t)Ty * 4 +
           (dirs_in_smem ? (size_t)Ty * W * 4 : 0) + 16;
}

struct MasPlan { int YT; int dirs_in_smem; size_t smem; bool ok; };

MasPlan mas_plan(int Tx, int Ty, bool has_mask) {
    MasPlan p{32, 1, 0, false};
    const int W = (Tx + 31) / 32;
    const size_t fixed = (size_t)2 * (Tx + 1) * 4 + (size_t)Ty * 4;
    const size_t dirs = (size_t)Ty * W * 4;
    for (int yt = 32; yt >= 4; yt >>= 1) {
        const size_t tiles = (size_t)(has_mask ? 4 : 2) * Tx * (yt + 1) * 4;
        if (tiles + fixed + dirs <= 72 * 1024) { p = {yt, 1, tiles + fixed + dirs, true}; return p; }
    }
    for (int yt = 32; yt >= 4; yt >>= 1) {
        const size_t tiles = (size_t)(has_mask ? 4 : 2) * Tx * (yt + 1) * 4;
        if (tiles + fixed <= 200 * 1024) { p = {yt, 0, tiles + fixed, true}; return p; }
    }
    return p;
}

}  // namespace

size_t mas_workspace_bytes(int B, int Tx, int Ty) {
    const int W = (Tx + 31) / 32;
    return (size_t)B * Ty * W * 4 + 256;
}

int mas_forward(const float* value, const float* mask, const int* t_x, const int* t_y, int B, int Tx, int Ty,
                void* path, int path_is_f32, void* ws, size_t ws_bytes, cudaStream_t st) {
    B200_REQUIRE(B >= 0 && Tx >= 0 && Ty >= 0, "mas: negative size");
    if (B == 0 || Tx == 0 || Ty == 0) return 0;
    B200_REQUIRE(value && t_x && t_y && path, "mas: null pointer");
    static DeviceOnce attr2_once, attr_once, attr3_once;
    static int use3 = -1;
    // wavefront variant without the per-column CTA barrier: its per-lane row streaming (32 lines per LDG) and lower
    // occupancy work against it; kept as an opt-in experiment (B200TTS_MAS3=1), see DESIGN.md.
    if (use3 < 0) { const char* e = getenv("B200TTS_MAS3"); use3 = (e && atoi(e)) ? 1 : 0; }
    const bool aligned16 = (Ty % 4 == 0) && ((reinterpret_cast<uintptr_t>(value) & 15) == 0) &&
                           (!mask || (reinterpret_cast<uintptr_t>(mask) & 15) == 0) && ((reinterpret_cast<uintptr_t>(path) & 15) == 0);
    if (use3 && Tx <= MAS_NT && aligned16 && mas3_smem(Tx, Ty) <= 200 * 1024) {     // wavefront kernel (no CTA barrier per column)
        if (int rc = device_once(attr3_once, nullptr, [](int) -> int {
                B200_CUDA_OK(cudaFuncSetAttribute(mas_kernel3<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
                B200_CUDA_OK(cudaFuncSetAttribute(mas_kernel3<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
                return 0;
            })) return rc;
        MasArgs a3;
        a3.value = value; a3.mask = mask; a3.t_x = t_x; a3.t_y = t_y;
        a3.B = B; a3.Tx = Tx; a3.Ty = Ty; a3.YT = 8; a3.W = (Tx + 31) / 32;
        a3.path = path; a3.path_is_f32 = path_is_f32; a3.dirs_global = nullptr; a3.dirs_in_smem = 1; a3.max_neg = -1e9f;
        const size_t smem3 = mas3_smem(Tx, Ty);
        if (mask) mas_kernel3<true><<<B, MAS_NT, smem3, st>>>(a3);
        else mas_kernel3<false><<<B, MAS_NT, smem3, st>>>(a3);
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
        return 0;
    }
    if (Tx <= MAS_NT) {     // lean kernel
        bool dsm = mas2_smem(Tx, Ty, mask != nullptr, true) <= 72 * 1024;
        const size_t smem2 = mas2_smem(Tx, Ty, mask != nullptr, dsm);
        if (smem2 <= 200 * 1024 && (dsm || (ws && ws_bytes >= mas_workspace_bytes(B, Tx, Ty)))) {
            if (int rc = device_once(attr2_once, nullptr, [](int) -> int {
                    B200_CUDA_OK(cudaFuncSetAttribute(mas_kernel2<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
                    B200_CUDA_OK(cudaFuncSetAttribute(mas_kernel2<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
                    B200_CUDA_OK(cudaFuncSetAttribute(mas_kernel2<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
                    B200_CUDA_OK(cudaFuncSetAttribute(mas_kernel2<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
                    return 0;
                })) return rc;
            MasArgs a2;
            a2.value = value; a2.mask = mask; a2.t_x = t_x; a2.t_y = t_y;
            a2.B = B; a2.Tx = Tx; a2.Ty = Ty; a2.YT = MAS2_YT; a2.W = (Tx + 31) / 32;
            a2.path = path; a2.path_is_f32 = path_is_f32;
            a2.dirs_global = reinterpret_cast<unsigned*>(ws);
            a2.dirs_in_smem = dsm ? 1 : 0;
            a2.max_neg = -1e9f;
            if (mask) { if (dsm) mas_kernel2<true, true><<<B, MAS_NT, smem2, st>>>(a2); else mas_kernel2<true, false><<<B, MAS_NT, smem2, st>>>(a2); }
            else      { if (dsm) mas_kernel2<false, true><<<B, MAS_NT, smem2, st>>>(a2); else mas_kernel2<false, false><<<B, MAS_NT, smem2, st>>>(a2); }
            count_launch();
            B200_CUDA_OK(cudaGetLastError());
            return 0;
        }
    }
    MasPlan p = mas_plan(Tx, Ty, mask != nullptr);
    B200_REQUIRE(p.ok, "mas: Tx=%d Ty=%d does not fit the shared-memory plan", Tx, Ty);
    B200_REQUIRE(p.dirs_in_smem || (ws && ws_bytes >= mas_workspace_bytes(B, Tx, Ty)), "mas: workspace too small");
    if (int rc = device_once(attr_once, nullptr, [](int) -> int {
            B200_CUDA_OK(cudaFuncSetAttribute(mas_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
            return 0;
        })) return rc;
    MasArgs a;
    a.value = value; a.mask = mask; a.t_x = t_x; a.t_y = t_y;
    a.B = B; a.Tx = Tx; a.Ty = Ty; a.YT = p.YT; a.W = (Tx + 31) / 32;
    a.path = path; a.path_is_f32 = path_is_f32;
    a.dirs_global = reinterpret_cast<unsigned*>(ws);
    a.dirs_in_smem = p.dirs_in_smem;
    a.max_neg = -1e9f;
    mas_kernel<<<B, MAS_NT, p.smem, st>>>(a);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace b200tts

// ------------------------------------------------------------------ alignment from the prior statistics (training side)
// Vits.forward_mas, TTS/tts/models/vits.py:909-919: the log-likelihood of every (text position, frame) pair
//   logp = [sum_c o*(-0.5 z^2)] + [sum_c (m*o)*z] + sum_c(-0.5 log 2pi - logs) + sum_c(-0.5 m^2 o),   o = exp(-2 logs)
// (two einsums + two row sums, added in that order), then maximum_path(logp, mask).  Here one kernel forms logp
// ([64 x 64] tiles per CTA, 16-channel stages through shared memory, exp / squares computed on the way in, FP32 FMA in
// ascending channel order) and the MAS kernel above consumes it; the reference materialises five [B,Tx,Ty] / [B,C,*]
// temporaries and round-trips logp through the host.
namespace b200tts {
namespace {

constexpr int LP_T = 64, LP_KC = 16;

__global__ void __launch_bounds__(256) mas_logp_kernel(const float* __restrict__ z_p, const float* __restrict__ m_p,
                                                      const float* __restrict__ logs_p, float* __restrict__ logp, int C,
                                                      int Tx, int Ty) {
    __shared__ float sO[LP_KC][LP_T + 1], sMO[LP_KC][LP_T + 1], sL[LP_KC][LP_T + 1], sM2O[LP_KC][LP_T + 1];
    __shared__ float sZ[LP_KC][LP_T + 1], sZ2[LP_KC][LP_T + 1];
    const int b = blockIdx.z, x0 = blockIdx.y * LP_T, y0 = blockIdx.x * LP_T;
    const int tid = threadIdx.x, tx = tid >> 4, ty = tid & 15;          // thread -> 4 x-rows (tx*4..) x 4 y-columns (ty + 16 j)
    const float* zb = z_p + (size_t)b * C * Ty;
    const float* mb = m_p + (size_t)b * C * Tx;
    const float* lb = logs_p + (size_t)b * C * Tx;
    float acc2[4][4], acc3[4][4], l1[4], l4[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        l1[i] = 0.f; l4[i] = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) { acc2[i][j] = 0.f; acc3[i][j] = 0.f; }
    }
    const float half_log_2pi = 0.91893853320467274178f;                   // 0.5 * log(2 pi)
    for (int c0 = 0; c0 < C; c0 += LP_KC) {
        for (int i = tid; i < LP_KC * LP_T; i += 256) {
            const int c = i / LP_T, t = i - c * LP_T, cg = c0 + c;
            float o = 0.f, mo = 0.f, ls = 0.f, m2o = 0.f, z = 0.f, z2 = 0.f;
            if (cg < C) {
                if (x0 + t < Tx) {
                    const float lg = lb[(size_t)cg * Tx + x0 + t], m = mb[(size_t)cg * Tx + x0 + t];
                    o = expf(-2.f * lg);
                    mo = __fmul_rn(m, o);
                    ls = -half_log_2pi - lg;
                    m2o = __fmul_rn(__fmul_rn(-0.5f, __fmul_rn(m, m)), o);
                }
                if (y0 + t < Ty) {
                    z = zb[(size_t)cg * Ty + y0 + t];
                    z2 = __fmul_rn(-0.5f, __fmul_rn(z, z));
                }
            }
            sO[c][t] = o; sMO[c][t] = mo; sL[c][t] = ls; sM2O[c][t] = m2o; sZ[c][t] = z; sZ2[c][t] = z2;
        }
        __syncthreads();
#pragma unroll
        for (int c = 0; c < LP_KC; ++c) {
            float o[4], mo[4], zz[4], zz2[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) { o[i] = sO[c][tx * 4 + i]; mo[i] = sMO[c][tx * 4 + i]; l1[i] += sL[c][tx * 4 + i]; l4[i] += sM2O[c][tx * 4 + i]; }
#pragma unroll
            for (int j = 0; j < 4; ++j) { zz[j] = sZ[c][ty + 16 * j]; zz2[j] = sZ2[c][ty + 16 * j]; }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) { acc2[i][j] = fmaf(o[i], zz2[j], acc2[i][j]); acc3[i][j] = fmaf(mo[i], zz[j], acc3[i][j]); }
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int x = x0 + tx * 4 + i;
        if (x >= Tx) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int y = y0 + ty + 16 * j;
            if (y < Ty) logp[((size_t)b * Tx + x) * Ty + y] = __fadd_rn(__fadd_rn(__fadd_rn(acc2[i][j], acc3[i][j]), l1[i]), l4[i]);
        }
    }
}

}  // namespace

size_t mas_from_stats_workspace_bytes(int B, int Tx, int Ty) {
    return (((size_t)B * Tx * Ty * sizeof(float) + 255) & ~size_t(255)) + mas_workspace_bytes(B, Tx, Ty);
}

int mas_from_stats(const float* z_p, const float* m_p, const float* logs_p, const int* t_x, const int* t_y, int B, int C,
                   int Tx, int Ty, void* path, int path_is_f32, float* logp_out, void* ws, size_t ws_bytes, cudaStream_t st) {
    B200_REQUIRE(z_p && m_p && logs_p && t_x && t_y && path, "mas_from_stats: null pointer");
    if (B == 0 || Tx == 0 || Ty == 0) return 0;
    B200_REQUIRE(ws && ws_bytes >= mas_from_stats_workspace_bytes(B, Tx, Ty), "mas_from_stats: workspace too small");
    const size_t lp_bytes = ((size_t)B * Tx * Ty * sizeof(float) + 255) & ~size_t(255);
    float* logp = logp_out ? logp_out : reinterpret_cast<float*>(ws);
    dim3 grid((Ty + LP_T - 1) / LP_T, (Tx + LP_T - 1) / LP_T, B);
    B200_REQUIRE(grid.y <= 65535 && grid.z <= 65535, "mas_from_stats: grid too large");
    mas_logp_kernel<<<grid, 256, 0, st>>>(z_p, m_p, logs_p, logp, C, Tx, Ty);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return mas_forward(logp, nullptr, t_x, t_y, B, Tx, Ty, path, path_is_f32, reinterpret_cast<char*>(ws) + lp_bytes,
                       ws_bytes - lp_bytes, st);
}

}  // namespace b200tts
