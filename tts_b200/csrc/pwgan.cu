// Parallel WaveGAN generator engine.
// Reference semantics: TTS/vocoder/models/parallel_wavegan_generator.py:12-118, TTS/vocoder/layers/parallel_wavegan.py
// (ResidualBlock), TTS/vocoder/layers/upsample.py (ConvUpsample / UpsampleNetwork / Stretch2d).
//
// Per call:
//   A = [W_aux,0 W_in; ...; W_aux,L-1 W_in] c      one frame-rate conv (pwgan_aux_kernel), the replicate pad as clamped reads
//   x = first_conv(noise)                           element-wise (1 -> 64 channels)
//   per residual layer l (pwgan_layer_kernel, one launch): the dilated gate conv, + bias + U(A_l), tanh * sigmoid,
//     conv1x1_out | conv1x1_skip as one GEMM, x_new = (out + x) * 0.25, skip (+)= s; the last layer scales skip by
//     sqrt(1 / L)
//   ReLU -> 1x1 64 -> 64 (conv engine, the ReLU as its prologue) -> ReLU -> 1x1 64 -> 1 (FMA kernel)
//
// ConvUpsample is linear and works on each channel alone (conv_in is a bias-free 1x1; each stage is a nearest stretch and
// a zero-padded FIR), so it commutes with every layer's conv1x1_aux: W_aux U(W_in c) = U(W_aux W_in c).  The folded
// weights are formed in float64 at handle creation, and U -- a banded map from frames to samples -- is tabulated there
// by pushing unit impulses through the stage chain in float64: a polyphase table for interior samples and exact
// per-sample maps for the samples near either end, where the stages' zero padding changes the coefficients.  The
// audio-rate conditioning tensor is never formed.
#include <cuda_fp16.h>

#include <cmath>

#include "conv_tc.cuh"
#include "engines.cuh"

namespace b200tts {

namespace pw {
constexpr int RES = 64, GATE = 128, AUX = 80;
constexpr int NT = 128;                    // output columns per tile (the MMA N)
constexpr int NTHREADS = 256;              // two warpgroups: MMA rows 0-63 and 64-127
constexpr int BLK = 8192;                  // one pack_tc block: {hi, lo} x 2 slabs x 128 rows x 16 B
constexpr int SLAB_W = 128 * 16;           // weight slab: 128 rows of 8 fp16
constexpr int SLAB_X = NT * 16;            // activation slab: NT columns of 8 fp16
constexpr int X_HALF = 8 * SLAB_X;         // 64 channels = 8 slabs; the lo half follows the hi half
constexpr int W1_BYTES = 12 * BLK;         // gate conv: 4 chunks of 16 channels x 3 taps
constexpr int W2_BYTES = 4 * BLK;          // out | skip 1x1: 4 chunks
constexpr int X_BYTES = 2 * X_HALF;        // one tap window of x, split
constexpr int Z_BYTES = 2 * X_HALF;        // the gate output, split: GEMM 2's B operand
constexpr int SMEM = W1_BYTES + W2_BYTES + X_BYTES + Z_BYTES;
constexpr int MAX_TW = 8;                  // frames one output sample of U may read
constexpr int TB = 64;                     // frames of the impulse responses the U tables are read from
}  // namespace pw

// ------------------------------------------------------------------ the upsampler map U
struct UTab {
    const float* coef;   // [E0 + P + E1][TW]: left edge rows, the P interior phases, right edge rows
    int P, E0, E1, TW, off;
};

// coefficient row and first frame of output sample n (Ts = Tf * P samples); the host check in Pwgan::build_u uses it too
__host__ __device__ __forceinline__ int u_row(int P, int E0, int E1, int TW, int off, int n, int Ts, int Tf, int& f0) {
    if (n < E0) { f0 = 0; return n; }
    if (n >= Ts - E1) { f0 = Tf - TW; return E0 + P + n - (Ts - E1); }
    const int q = n / P;
    f0 = q - off;
    return E0 + n - q * P;
}

__device__ __forceinline__ float u_apply(const float* cf, int TW, const float* a_row, int f0, int Tf) {
    float s = 0.f;
#pragma unroll 1
    for (int j = 0; j < TW; ++j) s = fmaf(__ldg(cf + j), __ldg(a_row + min(max(f0 + j, 0), Tf - 1)), s);
    return s;
}

// U alone: a [rows][Tf] -> out [rows][Tf * P]
__global__ void pwgan_upsample_kernel(const float* __restrict__ a, int rows, int Tf, UTab u, float* __restrict__ out) {
    const int Ts = Tf * u.P;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)rows * Ts) return;
    const int r = (int)(i / Ts), n = (int)(i - (long long)r * Ts);
    int f0;
    const int row = u_row(u.P, u.E0, u.E1, u.TW, u.off, n, Ts, Tf, f0);
    out[i] = u_apply(u.coef + (size_t)row * u.TW, u.TW, a + (size_t)r * Tf, f0, Tf);
}

// ------------------------------------------------------------------ A = W_fold c (exact FP32 FMA, clamped columns)
// A[b, r, f] = sum_ci W[r, ci] c[b, ci, clamp(f - pad, 0, T - 1)]: the replicate pad of `pad` frames each side is an
// addressing mode.  64 x 64 output tile per CTA, 4 x 4 per thread, 16 input channels per step.
constexpr int AX_BM = 64, AX_BN = 64, AX_BK = 16;
__global__ void __launch_bounds__(256) pwgan_aux_kernel(const float* __restrict__ c, long long c_bs, int c_cs, int Cin, int T,
                                                        int pad, const float* __restrict__ W, int R, float* __restrict__ A,
                                                        int Tf) {
    __shared__ float ws[AX_BK][AX_BM + 4];
    __shared__ float xs[AX_BK][AX_BN + 4];
    const int b = blockIdx.z, r0 = blockIdx.y * AX_BM, f0 = blockIdx.x * AX_BN;
    const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    const float* cb = c + b * c_bs;
    for (int k0 = 0; k0 < Cin; k0 += AX_BK) {
        for (int i = threadIdx.x; i < AX_BK * AX_BM; i += blockDim.x) {
            const int wk = i % AX_BK, wr = i / AX_BK;
            ws[wk][wr] = (r0 + wr < R && k0 + wk < Cin) ? W[(size_t)(r0 + wr) * Cin + k0 + wk] : 0.f;
            const int xk = i / AX_BN, xf = i % AX_BN;
            const int src = min(max(f0 + xf - pad, 0), T - 1);
            xs[xk][xf] = (k0 + xk < Cin && f0 + xf < Tf) ? cb[(size_t)(k0 + xk) * c_cs + src] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < AX_BK; ++k) {
            float wv[4], xv[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) { wv[i] = ws[k][ty + 16 * i]; xv[i] = xs[k][tx + 16 * i]; }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(wv[i], xv[j], acc[i][j]);
        }
        __syncthreads();
    }
    float* Ab = A + (size_t)b * R * Tf;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int r = r0 + ty + 16 * i;
        if (r >= R) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int f = f0 + tx + 16 * j;
            if (f < Tf) Ab[(size_t)r * Tf + f] = acc[i][j];
        }
    }
}

// first_conv (1 -> 64, 1x1): x[b, c, n] = w[c] noise[b, n] + bias[c]
__global__ void pwgan_first_kernel(const float* __restrict__ noise, int Ts, const float* __restrict__ w,
                                   const float* __restrict__ bias, float* __restrict__ x, int pitch, int B) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)B * Ts) return;
    const int b = (int)(i / Ts), n = (int)(i - (long long)b * Ts);
    const float v = noise[i];
    float* xb = x + (size_t)b * pw::RES * pitch + n;
#pragma unroll 8
    for (int ch = 0; ch < pw::RES; ++ch) xb[(size_t)ch * pitch] = fmaf(w[ch], v, bias[ch]);
}

// ------------------------------------------------------------------ the fused residual layer
// m64n128k16 wgmma with fp16 operands (the m64n256 wrappers of conv_tc.cuh at half the width): d[4j + {0,1}] =
// D[16 w + lane/4][8j + 2(lane%4) + {0,1}], d[4j + {2,3}] the same columns of row + 8.  Always accumulates.
#define PW_D64                                                                                                                \
    "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31," \
    "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,"  \
    "%62,%63},"
#define PW_D64_OPS(d)                                                                                                          \
    "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),  \
    "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),      \
    "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),      \
    "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),      \
    "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),      \
    "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),      \
    "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])

__device__ __forceinline__ void wgmma_f16_m64n128(float* d, uint64_t adesc, uint64_t bdesc) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " PW_D64 " %64, %65, 1, 1, 1, 0, 0;\n"
                 : PW_D64_OPS(d)
                 : "l"(adesc), "l"(bdesc)
                 : "memory");
}
__device__ __forceinline__ void wgmma_f16_m64n128_rs(float* d, const uint32_t (&a)[4], uint64_t bdesc) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " PW_D64 " {%64, %65, %66, %67}, %68, 1, 1, 1, 0;\n"
                 : PW_D64_OPS(d)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc)
                 : "memory");
}

struct PwLayerArgs {
    const float* x;                 // [B][64][pitch], read
    float* xn;                      // [B][64][pitch], x_new (never the buffer x is)
    float* skip;                    // [B][64][pitch]
    long long bs;                   // batch stride of x / xn / skip (floats)
    int pitch, Ts, dil;
    const unsigned char* w1;        // gate conv, pack_tc PREC_F16X3 image (rows in gate order, see Pwgan::init)
    const unsigned char* w2;        // conv1x1_out | conv1x1_skip, pack_tc PREC_F16X3 image
    const float *rs1, *rs2;         // [128] row scales 2^-e_r of the two images
    const float *b1, *b2;           // [128] biases (b1 in gate order)
    const float* A;                 // this layer's conditioning [B][128 (gate order)][Tf], batch stride A_bs
    long long A_bs;
    int Tf;
    UTab u;
    int first;                      // 1: skip = s (store), else skip += s
    float skip_scale;               // != 0 (last layer): skip *= skip_scale after the sum
    int n_ttiles;
    long long n_tiles;
    int* err;                       // mapped error words ([ERR_RANGE]: an activation outside fp16's range)
};

// GEMM 1: D1[128 gate rows][NT] = W1 [128][64 ch x 3 taps] * x window, split-fp16 (3 products: W_hs X_lo, W_lo X_hi,
// W_hi X_hi), tap by tap: tap k's window starts at column t0 + (k - 1) dil, so any dilation takes the same 32 KB stage.
// Gate rows are ordered so that MMA rows 16g + i and 16g + 8 + i (i < 8) are channel 8g + i's tanh and sigmoid rows:
// both sit in the same thread (d[4j + e] and d[4j + 2 + e]), and z = tanh(a) sigmoid(b) is formed in registers and
// stored as GEMM 2's split K-major B operand.  GEMM 2: D2[128][NT] = [W_out; W_skip] * z.
__global__ void __launch_bounds__(pw::NTHREADS, 1) pwgan_layer_kernel(const PwLayerArgs a) {
    using namespace tc;
    using namespace pw;
    extern __shared__ __align__(128) unsigned char sm[];
    unsigned char* const sW1 = sm;
    unsigned char* const sW2 = sm + W1_BYTES;
    unsigned char* const sX = sW2 + W2_BYTES;
    unsigned char* const sZ = sX + X_BYTES;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wg = warp >> 2;
    {   // both weight images stay resident for all of this CTA's tiles
        const uint4* s1 = reinterpret_cast<const uint4*>(a.w1);
        const uint4* s2 = reinterpret_cast<const uint4*>(a.w2);
        uint4* d1 = reinterpret_cast<uint4*>(sW1);
        uint4* d2 = reinterpret_cast<uint4*>(sW2);
        for (int i = tid; i < W1_BYTES / 16; i += NTHREADS) d1[i] = __ldg(s1 + i);
        for (int i = tid; i < W2_BYTES / 16; i += NTHREADS) d2[i] = __ldg(s2 + i);
    }
    fence_async_smem();
    __syncthreads();
    const uint32_t w1s = smem_u32(sW1), w2s = smem_u32(sW2), xs = smem_u32(sX), zs = smem_u32(sZ);
    const int ra = 16 * warp + (lane >> 2), rb = ra + 8;          // this thread's two accumulator rows
    const float rs1a = a.rs1[ra], rs1b = a.rs1[rb], b1a = a.b1[ra], b1b = a.b1[rb];
    const float rs2a = a.rs2[ra], rs2b = a.rs2[rb], b2a = a.b2[ra], b2b = a.b2[rb];
    // ldmatrix row of W_hi (matrices {rows 0-7, 8-15} x {slab 0, 1} of the warp's 16 rows), as conv_tc3.cuh's consumers
    const uint32_t lds_off = (uint32_t)(lane >> 4) * SLAB_W + (uint32_t)(warp * 16 + (lane & 15)) * 16;
    const uint32_t wg_off = (uint32_t)wg * 64 * 16;                // this warpgroup's 64 weight rows
    const int tt = tid & (NT - 1), sg = tid >> 7;                  // staging: column tt, slabs sg, sg + 2, sg + 4, sg + 6
    float amax = 0.f;
#pragma unroll 1
    for (long long tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
        const int b = (int)(tile / a.n_ttiles), t0 = (int)(tile - (long long)b * a.n_ttiles) * NT;
        const float* xb = a.x + b * a.bs;
        float v[4][8];
        auto load = [&](int k) {                                   // tap k's window; zero outside the row
            const int n = t0 + tt + (k - 1) * a.dil;
            const bool in = n >= 0 && n < a.Ts;
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int e = 0; e < 8; ++e) v[i][e] = in ? __ldg(xb + (size_t)(8 * (sg + 2 * i) + e) * a.pitch + n) : 0.f;
        };
        float d[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) d[i] = 0.f;
        load(0);
#pragma unroll 1
        for (int k = 0; k < 3; ++k) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                uint32_t hi[4], lo[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    amax = fmaxf(amax, fmaxf(fabsf(v[i][2 * e]), fabsf(v[i][2 * e + 1])));
                    split_f16x2(v[i][2 * e], v[i][2 * e + 1], hi[e], lo[e]);
                }
                const int off = (sg + 2 * i) * SLAB_X + tt * 16;
                *reinterpret_cast<uint4*>(sX + off) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
                *reinterpret_cast<uint4*>(sX + X_HALF + off) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
            }
            fence_async_smem();                                    // generic-proxy stores -> visible to wgmma
            __syncthreads();
            if (k < 2) load(k + 1);                                // in flight during this tap's MMAs
            uint32_t whs[4][4];                                    // W_hs = W_hi * 2^-11, per 16-channel chunk
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                ldsm_x4(whs[c], w1s + (uint32_t)(c * 3 + k) * BLK + lds_off);
#pragma unroll
                for (int i = 0; i < 4; ++i) whs[c][i] = f16x2_times_2m11(whs[c][i]);
            }
            wgmma_fence();
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const uint32_t wb = w1s + (uint32_t)(c * 3 + k) * BLK + wg_off;
                const uint64_t w_hi = make_desc(wb, SLAB_W), w_lo = make_desc(wb + 2 * SLAB_W, SLAB_W);
                const uint64_t xh = make_desc(xs + 2 * c * SLAB_X, SLAB_X), xl = make_desc(xs + X_HALF + 2 * c * SLAB_X, SLAB_X);
                wgmma_f16_m64n128_rs(d, whs[c], xl);               // small terms first
                wgmma_f16_m64n128(d, w_lo, xh);
                wgmma_f16_m64n128(d, w_hi, xh);
            }
            wgmma_commit();
            wgmma_wait<0>();
            __syncthreads();                                       // every warpgroup is done with the stage
        }
        // ---- epilogue 1: bias + U(A), gate, z -> shared memory (K-major split B operand of GEMM 2)
        {
            const float* Ab = a.A + b * a.A_bs;
            const float* Aa = Ab + (size_t)ra * a.Tf;
            const float* Ag = Ab + (size_t)rb * a.Tf;
            unsigned char* const zhi = sZ + warp * SLAB_X + (lane >> 2) * 2;   // channel 8 warp + lane / 4: slab `warp`
#pragma unroll
            for (int j = 0; j < NT / 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int t = 8 * j + 2 * (lane & 3) + e, n = t0 + t;
                    float z = 0.f;
                    if (n < a.Ts) {
                        int f0;
                        const float* cf = a.u.coef + (size_t)u_row(a.u.P, a.u.E0, a.u.E1, a.u.TW, a.u.off, n, a.Ts, a.Tf, f0) * a.u.TW;
                        const float va = fmaf(d[4 * j + e], rs1a, b1a) + u_apply(cf, a.u.TW, Aa, f0, a.Tf);
                        const float vb = fmaf(d[4 * j + 2 + e], rs1b, b1b) + u_apply(cf, a.u.TW, Ag, f0, a.Tf);
                        z = tanhf(va) * (1.f / (1.f + expf(-vb)));
                    }
                    const __half h = __float2half_rn(z);
                    const __half l = __float2half_rn((z - __half2float(h)) * 2048.f);
                    *reinterpret_cast<__half*>(zhi + t * 16) = h;
                    *reinterpret_cast<__half*>(zhi + X_HALF + t * 16) = l;
                }
        }
        fence_async_smem();
        __syncthreads();
        // ---- GEMM 2
#pragma unroll
        for (int i = 0; i < 64; ++i) d[i] = 0.f;
        {
            uint32_t whs[4][4];
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                ldsm_x4(whs[c], w2s + (uint32_t)c * BLK + lds_off);
#pragma unroll
                for (int i = 0; i < 4; ++i) whs[c][i] = f16x2_times_2m11(whs[c][i]);
            }
            wgmma_fence();
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const uint32_t wb = w2s + (uint32_t)c * BLK + wg_off;
                const uint64_t w_hi = make_desc(wb, SLAB_W), w_lo = make_desc(wb + 2 * SLAB_W, SLAB_W);
                const uint64_t zh = make_desc(zs + 2 * c * SLAB_X, SLAB_X), zl = make_desc(zs + X_HALF + 2 * c * SLAB_X, SLAB_X);
                wgmma_f16_m64n128_rs(d, whs[c], zl);
                wgmma_f16_m64n128(d, w_lo, zh);
                wgmma_f16_m64n128(d, w_hi, zh);
            }
            wgmma_commit();
            wgmma_wait<0>();
        }
        // ---- epilogue 2: rows 0-63 x_new = (conv1x1_out(z) + x) * 0.5^2, rows 64-127 skip (+)= conv1x1_skip(z)
        if (wg == 0) {
            const float* x0 = xb + (size_t)ra * a.pitch;
            const float* x1 = xb + (size_t)rb * a.pitch;
            float* y0 = a.xn + b * a.bs + (size_t)ra * a.pitch;
            float* y1 = a.xn + b * a.bs + (size_t)rb * a.pitch;
#pragma unroll
            for (int j = 0; j < NT / 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int n = t0 + 8 * j + 2 * (lane & 3) + e;
                    if (n >= a.Ts) continue;
                    y0[n] = (fmaf(d[4 * j + e], rs2a, b2a) + x0[n]) * 0.25f;
                    y1[n] = (fmaf(d[4 * j + 2 + e], rs2b, b2b) + x1[n]) * 0.25f;
                }
        } else {
            float* s0 = a.skip + b * a.bs + (size_t)(ra - RES) * a.pitch;
            float* s1 = a.skip + b * a.bs + (size_t)(rb - RES) * a.pitch;
#pragma unroll
            for (int j = 0; j < NT / 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int n = t0 + 8 * j + 2 * (lane & 3) + e;
                    if (n >= a.Ts) continue;
                    float h0 = fmaf(d[4 * j + e], rs2a, b2a), h1 = fmaf(d[4 * j + 2 + e], rs2b, b2b);
                    if (!a.first) { h0 = s0[n] + h0; h1 = s1[n] + h1; }
                    if (a.skip_scale != 0.f) { h0 *= a.skip_scale; h1 *= a.skip_scale; }
                    s0[n] = h0;
                    s1[n] = h1;
                }
        }
    }
    // an activation fp16 cannot hold (|x| >= 65504) was split into an inf: the launch's output is invalid
    if (amax >= F16X3_MAX && a.err) { *reinterpret_cast<volatile int*>(a.err + ERR_RANGE) = 1; __threadfence_system(); }
}

static DeviceOnce g_pw_once;

// ------------------------------------------------------------------ engine
static inline int round4(int v) { return (v + 3) / 4 * 4; }

int Pwgan::dilation(int l) const { return 1 << (l % (c.num_res_blocks / c.stacks)); }

// The stage chain of UpsampleNetwork in float64 on one channel: per stage, Stretch2d (F.interpolate nearest, torch's index
// rule floorf(i * (float)(1 / u))) and the (1, 2u + 1) conv with zero padding u.
static void up_chain(const std::vector<int>& f, const std::vector<std::vector<double>>& fir, std::vector<double>& cur) {
    for (size_t s = 0; s < f.size(); ++s) {
        const int u = f[s], Lin = (int)cur.size(), Lout = Lin * u;
        const float sc = (float)(1.0 / u);
        std::vector<double> st(Lout), y(Lout, 0.0);
        for (int i = 0; i < Lout; ++i) {
            const int src = Lout == Lin ? i : Lout == 2 * Lin ? (i >> 1) : std::min((int)floorf((float)i * sc), Lin - 1);
            st[i] = cur[src];
        }
        for (int i = 0; i < Lout; ++i) {
            double acc = 0.0;
            for (int k = 0; k <= 2 * u; ++k) {
                const int j = i + k - u;
                if (j >= 0 && j < Lout) acc += fir[s][k] * st[j];
            }
            y[i] = acc;
        }
        cur.swap(y);
    }
}

static int floordiv(int a, int b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// U[f][n] for Tf frames: the response of frame f's unit impulse
static std::vector<std::vector<double>> u_matrix(const std::vector<int>& f, const std::vector<std::vector<double>>& fir, int Tf) {
    std::vector<std::vector<double>> U(Tf);
    for (int fr = 0; fr < Tf; ++fr) {
        U[fr].assign(Tf, 0.0);
        U[fr][fr] = 1.0;
        up_chain(f, fir, U[fr]);
    }
    return U;
}

int Pwgan::build_u(const std::vector<std::vector<double>>& fir) {
    using namespace pw;
    std::vector<int> fac(c.upsample_factors, c.upsample_factors + c.num_upsamples);
    const int Ns = TB * P, fm = TB / 2;
    const auto U = u_matrix(fac, fir, TB);
    double scale = 0.0;
    int lo = 0, hi = 1;
    bool any = false;
    for (int n = 0; n < Ns; ++n) {
        const double v = std::fabs(U[fm][n]);
        scale = std::max(scale, v);
        if (v != 0.0) {
            const int rel = n - fm * P;
            if (!any) lo = rel;
            hi = rel + 1;
            any = true;
        }
    }
    const double tol = 1e-12 * std::max(scale, 1e-300);
    B200_REQUIRE(hi - lo <= (TB / 4) * P, "pwgan: the upsampler's impulse response spans %d samples (factors too small)", hi - lo);
    uoff = floordiv(hi - 1, P);
    const int TWi = uoff + floordiv(P - 1 - lo, P) + 1;
    auto h = [&](int rel) { return (rel >= lo && rel < hi) ? U[fm][fm * P + rel] : 0.0; };
    // samples where the stationary (polyphase) form is exact, frames inside the row included
    std::vector<char> ok(Ns, 1);
    for (int n = 0; n < Ns; ++n) {
        const int q = n / P, p = n - q * P, f0 = q - uoff;
        if (f0 < 0 || f0 + TWi > TB) { ok[n] = 0; continue; }
        for (int fr = 0; fr < TB && ok[n]; ++fr) {
            const int j = fr - f0;
            const double want = (j >= 0 && j < TWi) ? h(p + (uoff - j) * P) : 0.0;
            if (std::fabs(U[fr][n] - want) > tol) ok[n] = 0;
        }
    }
    uE0 = 0;
    uE1 = 0;
    for (int n = 0; n < Ns / 2; ++n) if (!ok[n]) uE0 = n + 1;
    for (int n = Ns - 1; n >= Ns / 2; --n) if (!ok[n]) uE1 = Ns - n;
    B200_REQUIRE(uE0 + uE1 < Ns / 2, "pwgan: upsampler edge maps of %d + %d samples", uE0, uE1);
    int TWl = 0, TWr = 0;
    for (int fr = 0; fr < TB; ++fr)
        for (int n = 0; n < uE0; ++n) if (U[fr][n] != 0.0) TWl = std::max(TWl, fr + 1);
    for (int fr = 0; fr < TB; ++fr)
        for (int n = Ns - uE1; n < Ns; ++n) if (U[fr][n] != 0.0) TWr = std::max(TWr, TB - fr);
    uTW = std::max(TWi, std::max(TWl, TWr));
    B200_REQUIRE(uTW <= MAX_TW, "pwgan: one output sample of the upsampler reads %d frames (at most %d supported)", uTW, MAX_TW);
    const int rows = uE0 + P + uE1;
    std::vector<double> cf((size_t)rows * uTW, 0.0);
    for (int n = 0; n < uE0; ++n)
        for (int j = 0; j < uTW; ++j) cf[(size_t)n * uTW + j] = U[j][n];
    for (int p = 0; p < P; ++p)
        for (int j = 0; j < TWi; ++j) cf[(size_t)(uE0 + p) * uTW + j] = h(p + (uoff - j) * P);
    for (int i = 0; i < uE1; ++i)
        for (int j = 0; j < uTW; ++j) cf[(size_t)(uE0 + P + i) * uTW + j] = U[TB - uTW + j][Ns - uE1 + i];
    // the shortest input the tables are exact for: reconstruct U for Tf frames exactly as the kernels read the tables
    // (frames clamped into the row) and compare with the impulse responses at that length
    auto exact_at = [&](int Tf) {
        const auto V = u_matrix(fac, fir, Tf);
        const int Ts = Tf * P;
        std::vector<double> rec(Tf);
        for (int n = 0; n < Ts; ++n) {
            std::fill(rec.begin(), rec.end(), 0.0);
            int f0;
            const int row = u_row(P, uE0, uE1, uTW, uoff, n, Ts, Tf, f0);
            for (int j = 0; j < uTW; ++j) rec[std::min(std::max(f0 + j, 0), Tf - 1)] += cf[(size_t)row * uTW + j];
            for (int fr = 0; fr < Tf; ++fr)
                if (std::fabs(rec[fr] - V[fr][n]) > tol) return false;
        }
        return true;
    };
    min_frames = 0;
    for (int t = std::max(uTW, 1); t <= TB / 2 && !min_frames; ++t)
        if (exact_at(t) && exact_at(t + 1) && exact_at(t + 2) && exact_at(t + uTW + 1)) min_frames = t;
    B200_REQUIRE(min_frames > 0, "pwgan: no input length up to %d frames for which the upsampler tables are exact", TB / 2);
    std::vector<float> cf32(cf.begin(), cf.end());
    return upload(ucoef, cf32.data(), cf32.size());
}

int Pwgan::init(const b200tts_pwgan_config& cfg, const float* const* w, int nw) {
    using namespace pw;
    c = cfg;
    const int L = c.num_res_blocks, S = c.num_upsamples;
    B200_REQUIRE(L >= 1 && L <= 256 && c.stacks >= 1 && L % c.stacks == 0 && L / c.stacks <= 16 && S >= 1 && S <= 8,
                 "pwgan: unsupported config (num_res_blocks %d, stacks %d, %d upsample factors)", L, c.stacks, S);
    P = 1;
    for (int s = 0; s < S; ++s) {
        B200_REQUIRE(c.upsample_factors[s] >= 1 && c.upsample_factors[s] <= 64, "pwgan: upsample factor %d", c.upsample_factors[s]);
        P *= c.upsample_factors[s];
    }
    B200_REQUIRE(P <= 4096, "pwgan: upsampling %d samples per frame (at most 4096)", P);
    for (int i = 0; i < nw; ++i) B200_REQUIRE(w[i] != nullptr, "pwgan: weight tensor %d is null", i);
    WeightList wl(w, nw);
    int rc;
    if ((rc = upload(first_w, wl.take(), RES)) || (rc = upload(first_b, wl.take(), RES))) return rc;
    const float* W_in = wl.take();                                     // conv_in [80][80]
    std::vector<std::vector<double>> fir(S);
    for (int s = 0; s < S; ++s) {
        const float* f = wl.take();
        B200_REQUIRE(W_in && f, "pwgan: null conv_in or upsampler filter");
        fir[s].assign(f, f + 2 * c.upsample_factors[s] + 1);
    }
    // MMA row m of the gate: tanh row 8g + (m % 16) for m % 16 < 8, else sigmoid row 64 + 8g + (m % 16 - 8), g = m / 16
    auto gate_row = [](int m) { const int g = m / 16, q = m % 16; return q < 8 ? 8 * g + q : 64 + 8 * g + q - 8; };
    std::vector<float> aux((size_t)L * GATE * AUX), bias1((size_t)L * GATE), bias2((size_t)L * GATE);
    w1.resize(L); w2.resize(L); rs1.resize(L); rs2.resize(L);
    for (int l = 0; l < L; ++l) {
        const float *cw = wl.take(), *cb = wl.take(), *aw = wl.take(), *ow = wl.take(), *ob = wl.take(), *sw = wl.take(),
                    *sb = wl.take();
        B200_REQUIRE(cw && cb && aw && ow && ob && sw && sb, "pwgan: null residual layer weight or bias");
        std::vector<float> W1((size_t)GATE * RES * 3), W2((size_t)GATE * RES);
        for (int m = 0; m < GATE; ++m) {
            const int r = gate_row(m);
            std::copy(cw + (size_t)r * RES * 3, cw + (size_t)(r + 1) * RES * 3, W1.begin() + (size_t)m * RES * 3);
            bias1[(size_t)l * GATE + m] = cb[r];
            for (int ci = 0; ci < AUX; ++ci) {                         // (W_aux,l W_in)[r][ci] in float64
                double s = 0.0;
                for (int k = 0; k < AUX; ++k) s += (double)aw[(size_t)r * AUX + k] * (double)W_in[(size_t)k * AUX + ci];
                aux[((size_t)l * GATE + m) * AUX + ci] = (float)s;
            }
        }
        std::copy(ow, ow + RES * RES, W2.begin());
        std::copy(sw, sw + RES * RES, W2.begin() + RES * RES);
        for (int r = 0; r < RES; ++r) {
            bias2[(size_t)l * GATE + r] = ob[r];
            bias2[(size_t)l * GATE + RES + r] = sb[r];
        }
        if (pack_tc(w1[l], W1, GATE, RES, 3, tc::PREC_F16X3, 1, &rs1[l])) return 2;
        if (pack_tc(w2[l], W2, GATE, RES, 1, tc::PREC_F16X3, 1, &rs2[l])) return 2;
    }
    if (upload(aux_w, aux.data(), aux.size()) || upload(b1, bias1.data(), bias1.size()) ||
        upload(b2, bias2.data(), bias2.size()))
        return 2;
    tail1.tc_prec = B200TTS_PRECISION_FP32;
    const float *t1w = wl.take(), *t1b = wl.take(), *t2w = wl.take(), *t2b = wl.take();
    if ((rc = pack_conv(tail1, t1w, t1b, RES, RES, 1, 1, 0))) return rc;
    if ((rc = pack_conv(tail2, t2w, t2b, 1, RES, 1, 1, 0))) return rc;
    if ((rc = wl.finish("pwgan"))) return rc;
    return build_u(fir);
}

// A: the conditioning of every layer (forward) or of one (layer); forward() also takes X0 / X1 (the residual stream)
// and S (the skip sum)
struct PwganWs { float *A, *X0, *X1, *S; };
static PwganWs pwgan_carve(const Pwgan& m, Arena& ar, int B, int Tf, bool whole) {
    const size_t bs = (size_t)pw::RES * round4(Tf * m.P);
    PwganWs w{};
    w.A = ar.f32((size_t)B * (whole ? m.c.num_res_blocks : 1) * pw::GATE * Tf);
    if (whole) {
        w.X0 = ar.f32(B * bs);
        w.X1 = ar.f32(B * bs);
        w.S = ar.f32(B * bs);
    }
    return w;
}

size_t Pwgan::workspace_bytes(int B, int Tf) const {
    return arena_size([&](Arena& ar) { pwgan_carve(*this, ar, B, Tf, true); });
}

UTab Pwgan::utab() const { return UTab{ucoef, P, uE0, uE1, uTW, uoff}; }

int Pwgan::upsample(const float* a, int rows, int Tf, float* out, cudaStream_t st) const {
    B200_REQUIRE(a && out, "pwgan_upsample: null pointer");
    B200_REQUIRE(rows >= 0 && Tf >= min_frames, "pwgan_upsample: %d frames (at least %d)", Tf, min_frames);
    const long long n = (long long)rows * Tf * P;
    if (n == 0) return 0;
    pwgan_upsample_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a, rows, Tf, utab(), out);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

// the checks every call makes; Tf: frames after the pad
int Pwgan::check_call(const char* who, int B, int T, int pad, int* Tf) const {
    B200_REQUIRE(B >= 0 && B <= 65535 && T >= 1 && pad >= 0, "%s: B = %d, T = %d, pad = %d", who, B, T, pad);
    *Tf = T + 2 * pad;
    B200_REQUIRE(*Tf >= min_frames, "%s: %d frames after the pad; these upsample factors need at least %d", who, *Tf,
                 min_frames);
    B200_REQUIRE((long long)*Tf * P < (1LL << 30), "%s: %d frames is too long", who, *Tf);
    return 0;
}

// the tensor-core state of the device (error words, SM count) and the layer kernel's shared-memory attribute
static int layer_device(int** err, int* num_sms) {
    size_t max_smem = 0;
    if (int rc = tc_device(err, num_sms, &max_smem)) return rc;
    B200_REQUIRE(max_smem >= (size_t)pw::SMEM, "pwgan: the layer kernel needs %d B of shared memory per block", pw::SMEM);
    return device_once(g_pw_once, nullptr, [](int) -> int {
        B200_CUDA_OK(cudaFuncSetAttribute(pwgan_layer_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, pw::SMEM));
        return 0;
    });
}

// A[b] = [W_aux,l W_in]_l c for layers l0 .. l0 + nl - 1 ([B][nl * 128][Tf]), replicate-padded by `pad` frames (clamped
// reads)
int Pwgan::launch_aux(const float* mel, int B, int T, int pad, int l0, int nl, float* A, cudaStream_t st) const {
    using namespace pw;
    const int R = nl * GATE, Tf = T + 2 * pad;
    const dim3 grid((unsigned)((Tf + AX_BN - 1) / AX_BN), (unsigned)((R + AX_BM - 1) / AX_BM), (unsigned)B);
    pwgan_aux_kernel<<<grid, 256, 0, st>>>(mel, (long long)AUX * T, T, AUX, T, pad, aux_w + (size_t)l0 * GATE * AUX, R, A,
                                           Tf);
    count_launch();
    dispatch_note(DISPATCH_PWGAN_AUX);
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

// residual layer l: x, xn, skip [B][64][pitch] (Ts = Tf * P columns used), A this layer's [128][Tf] conditioning of row b
// at A + b * A_bs
int Pwgan::launch_layer(int l, const float* x, float* xn, float* skip, int B, int pitch, int Tf, const float* A,
                        long long A_bs, int* err, int num_sms, cudaStream_t st) const {
    using namespace pw;
    PwLayerArgs a;
    memset(&a, 0, sizeof(a));
    a.x = x; a.xn = xn; a.skip = skip;
    a.bs = (long long)RES * pitch; a.pitch = pitch; a.Ts = Tf * P; a.dil = dilation(l);
    a.w1 = w1[l]; a.w2 = w2[l];
    a.rs1 = rs1[l]; a.rs2 = rs2[l]; a.b1 = b1 + (size_t)l * GATE; a.b2 = b2 + (size_t)l * GATE;
    a.A = A; a.A_bs = A_bs; a.Tf = Tf; a.u = utab();
    a.first = l == 0;
    a.skip_scale = l == c.num_res_blocks - 1 ? (float)std::sqrt(1.0 / c.num_res_blocks) : 0.f;
    a.n_ttiles = (a.Ts + NT - 1) / NT;
    a.n_tiles = (long long)B * a.n_ttiles;
    a.err = err;
    const int grid = (int)std::max(1LL, std::min(a.n_tiles, (long long)num_sms));
    pwgan_layer_kernel<<<grid, NTHREADS, SMEM, st>>>(a);
    count_launch();
    dispatch_note(DISPATCH_PWGAN_TC);
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

int Pwgan::forward(const float* mel, const float* noise, int B, int T, int pad, float* out, void* ws, size_t ws_bytes,
                   cudaStream_t st) const {
    using namespace pw;
    B200_REQUIRE(mel && noise && out && ws, "pwgan_forward: null pointer");
    int Tf = 0;
    if (int rc = check_call("pwgan_forward", B, T, pad, &Tf)) return rc;
    if (B == 0) return 0;
    const size_t need = workspace_bytes(B, Tf);
    B200_REQUIRE(ws_bytes >= need, "pwgan_forward: workspace of %zu bytes, %zu needed", ws_bytes, need);
    Arena ar(ws, ws_bytes);
    const PwganWs w = pwgan_carve(*this, ar, B, Tf, true);
    float *A = w.A, *X0 = w.X0, *S = w.S;
    int* err = nullptr;
    int num_sms = 0;
    if (int rc = layer_device(&err, &num_sms)) return rc;
    const int L = c.num_res_blocks, Ts = Tf * P, pitch = round4(Ts);
    if (int rc = launch_aux(mel, B, T, pad, 0, L, A, st)) return rc;
    {
        const long long n = (long long)B * Ts;
        pwgan_first_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(noise, Ts, first_w, first_b, X0, pitch, B);
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
    }
    float *x = X0, *xn = w.X1;
    for (int l = 0; l < L; ++l) {
        if (int rc = launch_layer(l, x, xn, S, B, pitch, Tf, A + (size_t)l * GATE * Tf, (long long)L * GATE * Tf, err,
                                  num_sms, st))
            return rc;
        std::swap(x, xn);   // xn's buffer now holds x; the old x is the next layer's output
    }
    float* H = X0;          // x is no longer needed
    ConvIO io;
    io.x = dense(S, RES, pitch); io.Tin = Ts; io.in_slope = 0.f;   // ReLU as the prologue
    io.y = dense(H, RES, pitch); io.Tout = Ts; io.B = B;
    if (int rc = launch_conv(tail1, io, st)) return rc;
    io.x = dense(H, RES, pitch); io.y = dense(out, 1, Ts);
    return launch_conv(tail2, io, st);
}

int Pwgan::layer(int l, const float* mel, int B, int T, int pad, const float* x, float* skip, float* x_new, int pitch,
                 void* ws, size_t ws_bytes, cudaStream_t st) const {
    using namespace pw;
    B200_REQUIRE(mel && x && skip && x_new && ws, "pwgan_layer: null pointer");
    B200_REQUIRE(l >= 0 && l < c.num_res_blocks, "pwgan_layer: layer %d of %d", l, c.num_res_blocks);
    B200_REQUIRE(x != x_new, "pwgan_layer: x_new must not be the buffer x is (neighbouring tiles still read x)");
    int Tf = 0;
    if (int rc = check_call("pwgan_layer", B, T, pad, &Tf)) return rc;
    B200_REQUIRE(pitch >= Tf * P, "pwgan_layer: row pitch %d < %d samples", pitch, Tf * P);
    if (B == 0) return 0;
    const size_t need = arena_size([&](Arena& ar) { pwgan_carve(*this, ar, B, Tf, false); });
    B200_REQUIRE(ws_bytes >= need, "pwgan_layer: workspace of %zu bytes, %zu needed", ws_bytes, need);
    Arena ar(ws, ws_bytes);
    float* A = pwgan_carve(*this, ar, B, Tf, false).A;
    int* err = nullptr;
    int num_sms = 0;
    if (int rc = layer_device(&err, &num_sms)) return rc;
    if (int rc = launch_aux(mel, B, T, pad, l, 1, A, st)) return rc;
    return launch_layer(l, x, x_new, skip, B, pitch, Tf, A, (long long)GATE * Tf, err, num_sms, st);
}

}  // namespace b200tts
