// Shared pieces of the Hopper (sm_90a) implicit-GEMM conv kernels in conv_tc3.cuh: mbarrier / bulk-copy /
// wgmma helpers and the operand-layout description (3xTF32 by default; bf16 / fp16 operands, see the end).
//
// conv1d as a wgmma implicit GEMM with 3xTF32 split precision.
//
//   D[row, t] += sum_ci W[row, ci, k] * A[t + k*dil - pad, ci]        for every tap k
//
// Both operands are K-major, no-swizzle ("interleave") canonical layouts: a 4-channel slab is a dense [rows][4 floats]
// array (16 B per row), so row r of K-chunk c lives at slab_c + r*16 -- 8-row core matrices are contiguous (SBO = 128 B)
// and the two 16-byte K chunks of one k8 MMA are LBO = slab stride apart.  Because rows are uniformly 16 B apart, the
// activation operand of tap k is THE SAME shared-memory tile with its descriptor start address advanced by k*dil rows:
// one staged window serves all taps (no im2col, no per-tap copies).
//
// fp32 accuracy: x = hi + lo with hi = x & 0xFFFFE000 (exactly representable in TF32) and lo = x - hi (exact in
// fp32; the tensor core keeps its top 11 bits).  D += A_hi*W_hi + A_lo*W_hi + A_hi*W_lo, accumulated in fp32; the
// dropped lo*lo term is 2^-22 relative.  Activations are split on the way into shared memory (together with the fused
// leaky-ReLU prologue); weights are split once at pack time.
//
// Opt-in 16-bit operands (bf16 or fp16, fp32 accumulation): no split, one m64n256k16 MMA per 16 input channels and tap.
// A slab row is still 16 bytes, now holding 8 channels of one time step, so a k16 step is two slabs LBO apart and the
// tap shift above still holds; activations are rounded (cvt.rn) on the way into shared memory, weights at pack time.
//
// 3-product fp16 split (PREC_F16X3, the HiFiGAN decoder's default): fp16 has TF32's 11-bit significand and twice its MMA
// rate, so the same hi/lo split costs 3 m64n256k16 MMAs per 16 channels instead of 6 m64n256k8.  fp16's small range is
// handled by scaling: weight row r is multiplied by 2^e_r (max |w'| in [2^14, 2^15)) at pack time and stored as W_hi =
// fp16(w'), W_lo = fp16(w' - W_hi); the kernel makes W_hs = fp16(W_hi * 2^-11) from W_hi in registers (register-A MMA,
// wgmma_f16_m64n256_rs); activations are split as X_hi = fp16(x), X_lo = fp16((x - X_hi)
// * 2^11) (subtraction and scaling exact).  D' = W_hs*X_lo + W_lo*X_hi + W_hi*X_hi = 2^e_r * D to 2^-22 relative, and the
// epilogue multiplies row r by 2^-e_r (exact) before the bias.  |x| >= 65504 cannot be represented: the producers report
// it (ERR_RANGE) instead of multiplying an inf.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200tts {
namespace tc {

// tensor-core operand type (the values of B200TTS_PRECISION_* in include/tts_b200.h; 3 is the header's TF32X3, which
// packs as PREC_FP32)
enum : int { PREC_FP32 = 0, PREC_BF16 = 1, PREC_FP16 = 2, PREC_F16X3 = 4 };
// the mapped error flags (conv1d.cu) are two words: err[0] a pipeline timeout, err[ERR_RANGE] an activation outside
// fp16's range (|x| >= F16X3_MAX) in PREC_F16X3
enum : int { ERR_RANGE = 1 };
constexpr float F16X3_MAX = 65504.f;
constexpr uint32_t SPIN_LIMIT = 1u << 22;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_wait(uint32_t bar, uint32_t parity, int* err) {
#pragma unroll 1
    for (uint32_t i = 0; i < SPIN_LIMIT; ++i) {
        uint32_t ok;
        asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}"
                     : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
        if (ok) return true;
    }
    if (err) { *reinterpret_cast<volatile int*>(err) = 1; __threadfence_system(); }   // mapped host flag (conv1d.cu)
    return false;
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// shared -> global bulk copy in the issuing thread's bulk async-group; `commit` closes the group.  `wait_read` returns
// once the thread's groups have finished reading shared memory (the source may be rewritten), `wait_all` once their writes
// are complete (visible to a grid that depends on this one).
__device__ __forceinline__ void bulk_s2g(void* dst, uint32_t src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// wgmma shared-memory descriptor: K-major, no swizzle; start address, LBO (between the two 16-byte K chunks),
// SBO = 128 B (next 8 rows), base offset 0
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((128u >> 4) & 0x3FFF) << 32;
    return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// The 128 accumulator operands of an m64n256 wgmma (%0 .. %127) and their constraints.
#define B200_WGMMA_D128                                                                                                       \
    "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"    \
    "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63," \
    "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95," \
    "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127},"
#define B200_WGMMA_D128_OPS(d)                                                                                                \
    "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),                          \
    "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),                    \
    "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),                  \
    "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),                  \
    "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),                  \
    "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),                  \
    "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),                  \
    "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),                  \
    "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),                  \
    "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),                  \
    "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),                  \
    "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),                  \
    "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),              \
    "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),          \
    "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),          \
    "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])

// D[64 x 256] (+)= A[64 x 8] * B[256 x 8]^T, tf32 inputs, fp32 accumulators in registers (128 per thread):
// d[4j + {0,1}] = D[16 w + lane/4][8j + 2(lane%4) + {0,1}], d[4j + {2,3}] = the same columns of row + 8 (w = warp of the
// warpgroup).  acc == 0 overwrites D.
__device__ __forceinline__ void wgmma_tf32_m64n256(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 " B200_WGMMA_D128
        " %128, %129, p, 1, 1;\n}"
        : B200_WGMMA_D128_OPS(d)
        : "l"(adesc), "l"(bdesc), "r"(acc)
        : "memory");
}

// The same tile with 16-bit operands: D[64 x 256] (+)= A[64 x 16] * B[256 x 16]^T, bf16 or fp16 inputs (both K-major,
// no transpose), fp32 accumulators in the layout above.  A K-major no-swizzle slab row is still 16 bytes, now 8 channels,
// so the k16 step reads two slabs LBO apart exactly as the tf32 k8 step does.
__device__ __forceinline__ void wgmma_bf16_m64n256(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 " B200_WGMMA_D128
        " %128, %129, p, 1, 1, 0, 0;\n}"
        : B200_WGMMA_D128_OPS(d)
        : "l"(adesc), "l"(bdesc), "r"(acc)
        : "memory");
}
__device__ __forceinline__ void wgmma_f16_m64n256(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 " B200_WGMMA_D128
        " %128, %129, p, 1, 1, 0, 0;\n}"
        : B200_WGMMA_D128_OPS(d)
        : "l"(adesc), "l"(bdesc), "r"(acc)
        : "memory");
}
// The fp16 tile with A from registers: a[0..3] is the warp's m16k16 fragment of its 16 rows (warp w of the warpgroup:
// rows 16 w ..), in mma.m16n8k16's A layout -- ldsm_x4's result.  The registers are read while the MMA is in flight:
// they must not be rewritten before the wgmma_wait that retires its group.
__device__ __forceinline__ void wgmma_f16_m64n256_rs(float* d, const uint32_t (&a)[4], uint64_t bdesc, uint32_t acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %133, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 " B200_WGMMA_D128
        " {%128, %129, %130, %131}, %132, p, 1, 1, 0;\n}"
        : B200_WGMMA_D128_OPS(d)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(acc)
        : "memory");
}

// Time-major tiles of the 32 / 64-channel layers (conv_tc3.cuh): D[64 time steps x N channels] (+)= A[64 x 16] *
// B[N x 16]^T, fp16 operands from shared memory (both K-major), fp32 accumulators in the m64nN layout:
// d[4j + {0,1}] = D[16 w + lane/4][8j + 2(lane%4) + {0,1}], d[4j + {2,3}] = the same columns of row + 8.
__device__ __forceinline__ void wgmma_f16_m64n64(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31},"
        " %32, %33, p, 1, 1, 0, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(acc)
        : "memory");
}
__device__ __forceinline__ void wgmma_f16_m64n32(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(adesc), "l"(bdesc), "r"(acc)
        : "memory");
}

// Four 8x8 b16 matrices from shared memory; lane l gives the address of row l % 8 of matrix l / 8, and r[i] is matrix
// i's element pair (row lane / 4, columns 2 (lane % 4) ..).  Matrices {rows 0-7, rows 8-15} x {k 0-7, k 8-15} in that
// order form an m16k16 A fragment.
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}
// two fp16 values times 2^-11, one round to nearest even (subnormal results kept): fp16(W_hi * 2^-11), as pack_tc's
// __float2half_rn(__half2float(hi) / 2048) rounds the exact product
__device__ __forceinline__ uint32_t f16x2_times_2m11(uint32_t v) {
    uint32_t r;
    asm("mul.rn.f16x2 %0, %1, %2;" : "=r"(r) : "r"(v), "r"(0x10001000u));
    return r;
}

// two fp32 values -> one register of two 16-bit values, round to nearest even; `lo` goes to the lower address
__device__ __forceinline__ uint32_t cvt_bf16x2(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}
__device__ __forceinline__ uint32_t cvt_f16x2(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}
// PREC_F16X3 activation split of two values (`a` at the lower address): hi = fp16(v), lo = fp16((v - hi) * 2^11).  v - hi is
// exact in fp32 (it is below half an fp16 ulp of v) and so is the scaling, so lo carries the next 11 bits of v.
__device__ __forceinline__ void split_f16x2(float a, float b, uint32_t& hi, uint32_t& lo) {
    hi = cvt_f16x2(a, b);
    float ha, hb;
    asm("{\n.reg .b16 l, h;\nmov.b32 {l, h}, %2;\ncvt.f32.f16 %0, l;\ncvt.f32.f16 %1, h;\n}" : "=f"(ha), "=f"(hb) : "r"(hi));
    lo = cvt_f16x2((a - ha) * 2048.f, (b - hb) * 2048.f);
}

}  // namespace tc
}  // namespace b200tts
