// Multi-head self-attention over [B, 3C, T] q|k|v activations on the tensor cores (3xTF32 mma.sync), for the mel-frame
// transformer of ForwardTTS's FFTransformer decoder (TTS/tts/layers/generic/transformer.py:21-35, nn.MultiheadAttention
// without masks).  Per row b only the first lens[b] frames are queries and keys: a batched call equals the single-
// utterance call on every valid frame.
//
// Flash-style: one CTA owns FA_BQ queries of one (row, head) and streams the keys in tiles of FA_BK, keeping a running
// row max / row sum (online softmax), so shared memory does not grow with T (any T; the positional encoding caps the
// decoder at 5000 frames).  Both products are 3xTF32 (hi*hi + hi*lo + lo*hi, FP32 accumulation), each key tile's P.V
// and each 64-channel chunk of S in a fresh accumulator folded in with FP32 arithmetic, which keeps the result FP32-accurate:
//   S = (q * d^-1/2) . K     [FA_BQ x FA_BK]   warps: 2 query m-tiles x 4 groups of 2 key n-tiles
//   O = O * alpha + P . V^T  [FA_BQ x d]       warps: 2 query m-tiles x 4 groups of channel n-tiles (<= 12 each)
// q is scaled before the product, as torch does.  Key columns at or beyond lens[b] are never read (they may hold stale
// scratch, NaN included); they load as zero and score -inf.  Query columns in [lens[b], pitch) of the output are written
// as zero: the grid covers every query tile below the pitch, not only those below T.
// Heads need d % 8 == 0 and d <= FA_MAXD; the caller takes the FP32-FMA kernel otherwise.
#include <math.h>

#include "engines.cuh"

namespace b200tts {

namespace {

constexpr int FA_BQ = 32, FA_BK = 64, FA_WARPS = 8, FA_MAXD = 384;
constexpr int FA_NT = (FA_MAXD / 8 + 3) / 4;   // channel n-tiles per warp in the P.V product
// shared-memory row pitches, chosen so that every fragment load of a warp hits 32 distinct banks
constexpr int FA_QS = FA_BQ + 8;   // q  [d][FA_QS]   (A of S: stride = 8 mod 32)
constexpr int FA_KS = FA_BK + 8;   // k  [d][FA_KS]   (B of S: stride = 8 mod 32)
constexpr int FA_VS = FA_BK + 4;   // v  [d][FA_VS]   (B of P.V: stride = 4 mod 32), same buffer as k
constexpr int FA_PS = FA_BK + 4;   // p  [FA_BQ][FA_PS] (A of P.V: stride = 4 mod 32)

__device__ __forceinline__ uint32_t to_tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
    hi = to_tf32(x);
    lo = to_tf32(x - __uint_as_float(hi));
}
__device__ __forceinline__ void mma_tf32(float* c, const uint32_t* a, const uint32_t* b) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
// c += a * b in 3xTF32: the small cross terms first
__device__ __forceinline__ void mma3(float* c, const uint32_t* ah, const uint32_t* al, const float* b) {
    uint32_t bh[2], bl[2];
    split_tf32(b[0], bh[0], bl[0]);
    split_tf32(b[1], bh[1], bl[1]);
    mma_tf32(c, al, bh);
    mma_tf32(c, ah, bl);
    mma_tf32(c, ah, bh);
}

// rows [0, d) x columns [col0, col0 + FA_BK) of a [*, pitch] head slice into smem [d][sp]; columns >= len read as 0
__device__ __forceinline__ void load_tile(float* dst, int sp, const float* __restrict__ src, int pitch, int d, int col0,
                                          int len) {
    const int n = d * FA_BK;
    for (int base = threadIdx.x; base < n; base += 8 * 32 * FA_WARPS) {
        float v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const int idx = base + u * 32 * FA_WARPS;
            const int c = idx / FA_BK, jj = idx - c * FA_BK, j = col0 + jj;
            v[u] = (idx < n && j < len) ? src[(size_t)c * pitch + j] : 0.f;
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const int idx = base + u * 32 * FA_WARPS;
            const int c = idx / FA_BK, jj = idx - c * FA_BK;
            if (idx < n) dst[c * sp + jj] = v[u];
        }
    }
}

__global__ void __launch_bounds__(32 * FA_WARPS) attention_tc3_kernel(const float* __restrict__ qkv, long long qkv_bs,
                                                                      int pitch, const int* __restrict__ lens,
                                                                      float* __restrict__ out, long long out_bs, int C,
                                                                      int d, float scale) {
    extern __shared__ float sm[];
    float* qs = sm;                      // [d][FA_QS]
    float* kv = qs + d * FA_QS;          // [d][FA_KS] keys, then [d][FA_VS] values
    float* ps = kv + d * FA_KS;          // [FA_BQ][FA_PS] scores -> probabilities
    float* alpha_s = ps + FA_BQ * FA_PS; // [FA_BQ] rescale of the running output
    float* l_s = alpha_s + FA_BQ;        // [FA_BQ] final row sums
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, tig = lane & 3;
    const int b = blockIdx.z, h = blockIdx.y, i0 = blockIdx.x * FA_BQ;
    const int len = min(lens[b], pitch);
    const float* qb = qkv + (size_t)b * qkv_bs + (size_t)h * d * pitch;
    const float* kb = qb + (size_t)C * pitch;
    const float* vb = kb + (size_t)C * pitch;
    float* ob = out + (size_t)b * out_bs + (size_t)h * d * pitch;
    if (i0 >= len) {   // a tile of padded query columns
        for (int idx = tid; idx < d * FA_BQ; idx += 32 * FA_WARPS) {
            const int c = idx / FA_BQ, i = i0 + idx - c * FA_BQ;
            if (i < pitch) ob[(size_t)c * pitch + i] = 0.f;
        }
        return;
    }
    for (int idx = tid; idx < d * FA_BQ; idx += 32 * FA_WARPS) {
        const int c = idx / FA_BQ, q = idx - c * FA_BQ, i = i0 + q;
        qs[c * FA_QS + q] = i < len ? __fmul_rn(qb[(size_t)c * pitch + i], scale) : 0.f;
    }
    const int mt = warp & 1;                 // query m-tile of this warp in both products
    const int ng = warp >> 1;                // n-tile group
    const int nct = d >> 3;                  // channel n-tiles
    float o[FA_NT][4];
#pragma unroll
    for (int u = 0; u < FA_NT; ++u) o[u][0] = o[u][1] = o[u][2] = o[u][3] = 0.f;
    float m_run[4], l_run[4];                // softmax state of rows 4*warp + r (replicated over the warp)
#pragma unroll
    for (int r = 0; r < 4; ++r) { m_run[r] = -INFINITY; l_run[r] = 0.f; }

    for (int j0 = 0; j0 < len; j0 += FA_BK) {
        __syncthreads();   // the previous tile's P.V is done with kv and ps
        load_tile(kv, FA_KS, kb, pitch, d, j0, len);
        __syncthreads();
        {   // S = q . k for 16 queries x 16 keys per warp; each 64-channel chunk is summed in a fresh accumulator and
            // added in FP32, so few products pass through the MMA's own accumulation
            float s[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
            const float* qa = qs + mt * 16 + g;
            for (int kc = 0; kc < d; kc += 64) {
                float sp[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
                for (int k0 = kc; k0 < d && k0 < kc + 64; k0 += 8) {
                    uint32_t ah[4], al[4];
                    split_tf32(qa[(k0 + tig) * FA_QS], ah[0], al[0]);
                    split_tf32(qa[(k0 + tig) * FA_QS + 8], ah[1], al[1]);
                    split_tf32(qa[(k0 + tig + 4) * FA_QS], ah[2], al[2]);
                    split_tf32(qa[(k0 + tig + 4) * FA_QS + 8], ah[3], al[3]);
#pragma unroll
                    for (int n = 0; n < 2; ++n) {
                        const int col = (2 * ng + n) * 8 + g;
                        const float bb[2] = {kv[(k0 + tig) * FA_KS + col], kv[(k0 + tig + 4) * FA_KS + col]};
                        mma3(sp[n], ah, al, bb);
                    }
                }
#pragma unroll
                for (int n = 0; n < 2; ++n)
#pragma unroll
                    for (int e = 0; e < 4; ++e) s[n][e] += sp[n][e];
            }
#pragma unroll
            for (int n = 0; n < 2; ++n) {
                const int col = (2 * ng + n) * 8 + 2 * tig, row = mt * 16 + g;
                ps[row * FA_PS + col] = s[n][0];
                ps[row * FA_PS + col + 1] = s[n][1];
                ps[(row + 8) * FA_PS + col] = s[n][2];
                ps[(row + 8) * FA_PS + col + 1] = s[n][3];
            }
        }
        __syncthreads();
        // online softmax over this tile: warp w owns rows 4w..4w+3, lane covers key columns lane and lane + 32
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int row = 4 * warp + r;
            float v0 = ps[row * FA_PS + lane], v1 = ps[row * FA_PS + lane + 32];
            if (j0 + lane >= len) v0 = -INFINITY;
            if (j0 + lane + 32 >= len) v1 = -INFINITY;
            float mx = fmaxf(v0, v1);
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
            const float m_new = fmaxf(m_run[r], mx);          // finite: key column j0 < len is valid
            const float alpha = expf(m_run[r] - m_new);       // 0 on the first tile
            const float p0 = expf(v0 - m_new), p1 = expf(v1 - m_new);
            float sum = p0 + p1;
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
            l_run[r] = fmaf(l_run[r], alpha, sum);
            m_run[r] = m_new;
            ps[row * FA_PS + lane] = p0;
            ps[row * FA_PS + lane + 32] = p1;
            if (lane == 0) alpha_s[row] = alpha;
        }
        load_tile(kv, FA_VS, vb, pitch, d, j0, len);   // every warp finished reading k before the last barrier
        __syncthreads();
        {   // O = O * alpha + P . V^T: the tile's product in a fresh accumulator, folded into O with one FP32 fma
            float acc[FA_NT][4];
#pragma unroll
            for (int u = 0; u < FA_NT; ++u) acc[u][0] = acc[u][1] = acc[u][2] = acc[u][3] = 0.f;
            const float* pa = ps + (mt * 16 + g) * FA_PS;
#pragma unroll 2
            for (int k0 = 0; k0 < FA_BK; k0 += 8) {
                uint32_t ah[4], al[4];
                split_tf32(pa[k0 + tig], ah[0], al[0]);
                split_tf32(pa[8 * FA_PS + k0 + tig], ah[1], al[1]);
                split_tf32(pa[k0 + tig + 4], ah[2], al[2]);
                split_tf32(pa[8 * FA_PS + k0 + tig + 4], ah[3], al[3]);
#pragma unroll
                for (int u = 0; u < FA_NT; ++u) {
                    const int nt = ng + 4 * u;
                    if (nt < nct) {
                        const float* vr = kv + (nt * 8 + g) * FA_VS + k0 + tig;
                        const float bb[2] = {vr[0], vr[4]};
                        mma3(acc[u], ah, al, bb);
                    }
                }
            }
            const float a_lo = alpha_s[mt * 16 + g], a_hi = alpha_s[mt * 16 + g + 8];
#pragma unroll
            for (int u = 0; u < FA_NT; ++u) {
                o[u][0] = fmaf(o[u][0], a_lo, acc[u][0]); o[u][1] = fmaf(o[u][1], a_lo, acc[u][1]);
                o[u][2] = fmaf(o[u][2], a_hi, acc[u][2]); o[u][3] = fmaf(o[u][3], a_hi, acc[u][3]);
            }
        }
    }
    if (lane == 0) {
#pragma unroll
        for (int r = 0; r < 4; ++r) l_s[4 * warp + r] = l_run[r];
    }
    __syncthreads();
    const int row = mt * 16 + g;
    const float l_lo = l_s[row], l_hi = l_s[row + 8];
    const int i_lo = i0 + row, i_hi = i0 + row + 8;
#pragma unroll
    for (int u = 0; u < FA_NT; ++u) {
        const int nt = ng + 4 * u;
        if (nt < nct) {
            const int c = nt * 8 + 2 * tig;
            if (i_lo < len) {
                ob[(size_t)c * pitch + i_lo] = o[u][0] / l_lo;
                ob[(size_t)(c + 1) * pitch + i_lo] = o[u][1] / l_lo;
            } else if (i_lo < pitch) {
                ob[(size_t)c * pitch + i_lo] = 0.f;
                ob[(size_t)(c + 1) * pitch + i_lo] = 0.f;
            }
            if (i_hi < len) {
                ob[(size_t)c * pitch + i_hi] = o[u][2] / l_hi;
                ob[(size_t)(c + 1) * pitch + i_hi] = o[u][3] / l_hi;
            } else if (i_hi < pitch) {
                ob[(size_t)c * pitch + i_hi] = 0.f;
                ob[(size_t)(c + 1) * pitch + i_hi] = 0.f;
            }
        }
    }
}

size_t attention_tc3_smem(int d) {
    return sizeof(float) * ((size_t)d * FA_QS + (size_t)d * FA_KS + (size_t)FA_BQ * FA_PS + 2 * FA_BQ);
}

}  // namespace

bool attention_tc3_takes(int d) { return d >= 8 && d % 8 == 0 && d <= FA_MAXD; }

int launch_attention_tc3(const float* qkv, long long qkv_bs, int pitch, const int* lens, float* out, long long out_bs,
                         int B, int C, int num_heads, int T, cudaStream_t st) {
    B200_REQUIRE(qkv && lens && out, "attention_tc3: null pointer");
    B200_REQUIRE(num_heads >= 1 && C % num_heads == 0, "attention_tc3: %d channels not divisible by %d heads", C,
                 num_heads);
    const int d = C / num_heads;
    B200_REQUIRE(attention_tc3_takes(d), "attention_tc3: head dim %d needs d %% 8 == 0 and d <= %d", d, FA_MAXD);
    B200_REQUIRE(T >= 0 && T <= pitch, "attention_tc3: T=%d exceeds the row pitch %d", T, pitch);
    if (B == 0 || pitch == 0) return 0;
    const size_t smem = attention_tc3_smem(d);
    static DeviceOnce attr_once;
    if (int rc0 = device_once(attr_once, nullptr, [](int) -> int {
            B200_CUDA_OK(cudaFuncSetAttribute(attention_tc3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                              (int)attention_tc3_smem(FA_MAXD)));
            return 0;
        })) return rc0;
    // T only bounds the rows' lengths: the padded columns up to the pitch are zeroed too, so the grid spans the pitch
    dim3 grid((pitch + FA_BQ - 1) / FA_BQ, num_heads, B);
    attention_tc3_kernel<<<grid, 32 * FA_WARPS, smem, st>>>(qkv, qkv_bs, pitch, lens, out, out_bs, C, d,
                                                           (float)sqrt(1.0 / (double)d));
    count_launch();
    dispatch_note(DISPATCH_ATTN_TC3);
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace b200tts
