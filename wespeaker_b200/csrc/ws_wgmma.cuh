// Hopper warpgroup MMA (wgmma.mma_async, sm_90a): one instruction per (M = 64 rows, N, K = 32 bytes) block with both
// operands read from shared memory through matrix descriptors and the fp32 accumulator in the registers of the issuing
// warpgroup (4 consecutive warps, the first a multiple of 4).  Accumulator fragment of thread (warp w of the warpgroup,
// lane l) for an m64nN instruction: d[4j + 2h + e] = D[16w + l/4 + 8h][8j + 2(l%4) + e], j < N/8, h, e in {0, 1}.
#pragma once
#include <stdint.h>

namespace ws_wg {

// K-major shared-memory matrix descriptor: [0,14) start >> 4 | [16,30) LBO >> 4 (unused for swizzled K-major) |
// [32,46) SBO >> 4 = 8 rows | [62,64) swizzle (1 = 128 B, 2 = 64 B, 3 = 32 B).  Rows are `row_bytes` apart and the row
// byte count equals the swizzle span, as TMA writes the operand tiles.  One K step (32 bytes) is +2 in the start field.
__device__ __forceinline__ uint64_t desc(uint32_t saddr, int row_bytes) {
    const uint64_t layout = row_bytes == 128 ? 1ull : (row_bytes == 64 ? 2ull : 3ull);
    uint64_t d = (uint64_t)((saddr & 0x3FFFFu) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)((8 * row_bytes) >> 4) << 32;
    d |= layout << 62;
    return d;
}
// The wgmma instructions are .sync.aligned: every lane of the warp executes them convergently.  Spin waits on mbarriers
// and per-lane branches (an elected TMA thread, masked frames) can leave a warp diverged, so fence() and wait()
// reconverge it first; the MMAs between fence() and commit() are straight-line code.
__device__ __forceinline__ void fence() {
    __syncwarp();
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wait() {
    __syncwarp();
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads above the wait that completes them
template <int NR>
__device__ __forceinline__ void fence_regs(float* d) {
#pragma unroll
    for (int i = 0; i < NR; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define WS_WG_F8(o) "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7])
#define WS_WG_REGS_N32 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}"
#define WS_WG_OPS_N32 WS_WG_F8(0), WS_WG_F8(8)
#define WS_WG_REGS_N64 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}"
#define WS_WG_OPS_N64 WS_WG_F8(0), WS_WG_F8(8), WS_WG_F8(16), WS_WG_F8(24)
#define WS_WG_REGS_N128 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
#define WS_WG_OPS_N128 WS_WG_F8(0), WS_WG_F8(8), WS_WG_F8(16), WS_WG_F8(24), WS_WG_F8(32), WS_WG_F8(40), WS_WG_F8(48), WS_WG_F8(56)

__device__ __forceinline__ void wg_mma_bf16_n32(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\twgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 " WS_WG_REGS_N32
                 ", %16, %17, p, 1, 1, 0, 0;\n\t}" : WS_WG_OPS_N32 : "l"(da), "l"(db), "r"(acc));
}
__device__ __forceinline__ void wg_mma_f16_n32(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\twgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 " WS_WG_REGS_N32
                 ", %16, %17, p, 1, 1, 0, 0;\n\t}" : WS_WG_OPS_N32 : "l"(da), "l"(db), "r"(acc));
}
__device__ __forceinline__ void wg_mma_tf32_n32(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\twgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 " WS_WG_REGS_N32
                 ", %16, %17, p, 1, 1;\n\t}" : WS_WG_OPS_N32 : "l"(da), "l"(db), "r"(acc));
}
__device__ __forceinline__ void wg_mma_bf16_n64(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 " WS_WG_REGS_N64
                 ", %32, %33, p, 1, 1, 0, 0;\n\t}" : WS_WG_OPS_N64 : "l"(da), "l"(db), "r"(acc));
}
__device__ __forceinline__ void wg_mma_f16_n64(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " WS_WG_REGS_N64
                 ", %32, %33, p, 1, 1, 0, 0;\n\t}" : WS_WG_OPS_N64 : "l"(da), "l"(db), "r"(acc));
}
__device__ __forceinline__ void wg_mma_tf32_n64(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\twgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 " WS_WG_REGS_N64
                 ", %32, %33, p, 1, 1;\n\t}" : WS_WG_OPS_N64 : "l"(da), "l"(db), "r"(acc));
}
__device__ __forceinline__ void wg_mma_bf16_n128(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\twgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " WS_WG_REGS_N128
                 ", %64, %65, p, 1, 1, 0, 0;\n\t}" : WS_WG_OPS_N128 : "l"(da), "l"(db), "r"(acc));
}
__device__ __forceinline__ void wg_mma_f16_n128(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\twgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " WS_WG_REGS_N128
                 ", %64, %65, p, 1, 1, 0, 0;\n\t}" : WS_WG_OPS_N128 : "l"(da), "l"(db), "r"(acc));
}
__device__ __forceinline__ void wg_mma_tf32_n128(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\twgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 " WS_WG_REGS_N128
                 ", %64, %65, p, 1, 1;\n\t}" : WS_WG_OPS_N128 : "l"(da), "l"(db), "r"(acc));
}

// D[64 x N] (+)= A[64 x K32] * B[N x K32]^T for the activation dtype dt (0 fp32 -> tf32, 1 bf16, 2 fp16); acc = 0 starts a
// new accumulation.  dt is warp-uniform.
template <int N>
__device__ __forceinline__ void mma(int dt, float* d, uint64_t da, uint64_t db, uint32_t acc) {
    static_assert(N == 32 || N == 64 || N == 128, "wgmma N");
    if constexpr (N == 32) {
        if (dt == 1) wg_mma_bf16_n32(d, da, db, acc); else if (dt == 2) wg_mma_f16_n32(d, da, db, acc); else wg_mma_tf32_n32(d, da, db, acc);
    } else if constexpr (N == 64) {
        if (dt == 1) wg_mma_bf16_n64(d, da, db, acc); else if (dt == 2) wg_mma_f16_n64(d, da, db, acc); else wg_mma_tf32_n64(d, da, db, acc);
    } else {
        if (dt == 1) wg_mma_bf16_n128(d, da, db, acc); else if (dt == 2) wg_mma_f16_n128(d, da, db, acc); else wg_mma_tf32_n128(d, da, db, acc);
    }
}

// the same with N (128, 64 or 32) chosen at run time (warp-uniform); d holds at least n / 2 floats
__device__ __forceinline__ void mma_n(int n, int dt, float* d, uint64_t da, uint64_t db, uint32_t acc) {
    if (n == 128) mma<128>(dt, d, da, db, acc);
    else if (n == 64) mma<64>(dt, d, da, db, acc);
    else mma<32>(dt, d, da, db, acc);
}

// m64n256k16 with the 16-bit operand type fixed at compile time (DT: 1 bf16, 2 fp16): 128 accumulator registers per thread
#define WS_WG_REGS_N256                                                                                                     \
    "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, "  \
    "%25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "    \
    "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, "    \
    "%71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, "    \
    "%94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, "     \
    "%114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}"
#define WS_WG_OPS_N256                                                                                                       \
    WS_WG_F8(0), WS_WG_F8(8), WS_WG_F8(16), WS_WG_F8(24), WS_WG_F8(32), WS_WG_F8(40), WS_WG_F8(48), WS_WG_F8(56),          \
        WS_WG_F8(64), WS_WG_F8(72), WS_WG_F8(80), WS_WG_F8(88), WS_WG_F8(96), WS_WG_F8(104), WS_WG_F8(112), WS_WG_F8(120)
template <int DT>
__device__ __forceinline__ void mma16_n256(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    static_assert(DT == 1 || DT == 2, "16-bit wgmma");
    if constexpr (DT == 1)
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\twgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
                     WS_WG_REGS_N256 ", %128, %129, p, 1, 1, 0, 0;\n\t}" : WS_WG_OPS_N256 : "l"(da), "l"(db), "r"(acc));
    else
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\twgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
                     WS_WG_REGS_N256 ", %128, %129, p, 1, 1, 0, 0;\n\t}" : WS_WG_OPS_N256 : "l"(da), "l"(db), "r"(acc));
}

// per-thread register budget of the executing warpgroup (all four warps execute it): the producer warpgroup hands
// registers back to the CTA's pool, the consumer warpgroups take them
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// Row-wise access to an accumulator for epilogues written per output row: the warp's 16 rows x NC = 64 columns starting at
// column c0 of the fragment go through a per-warp shared-memory scratch of 16 x kScrPitch floats, after which lane l owns
// row (l & 15) and the 32 consecutive columns starting at (l >> 4) * 32.
constexpr int kScrPitch = 68;   // 16-byte rows reads are conflict-free per quarter warp (row offsets 4 banks apart)
constexpr int kScrFloats = 16 * kScrPitch;
template <int NC>
__device__ __forceinline__ void frag_to_rows(const float* d, int c0, float* scr, float* v) {
    const int lane = threadIdx.x & 31, r0 = lane >> 2, cq = (lane & 3) * 2;
    __syncwarp();
#pragma unroll
    for (int j = 0; j < NC / 8; ++j) {
        const int jj = c0 / 8 + j;
        *reinterpret_cast<float2*>(scr + r0 * kScrPitch + 8 * j + cq) = make_float2(d[4 * jj], d[4 * jj + 1]);
        *reinterpret_cast<float2*>(scr + (r0 + 8) * kScrPitch + 8 * j + cq) = make_float2(d[4 * jj + 2], d[4 * jj + 3]);
    }
    __syncwarp();
    const float4* src = reinterpret_cast<const float4*>(scr + (lane & 15) * kScrPitch + (lane >> 4) * (NC / 2));
#pragma unroll
    for (int i = 0; i < NC / 8; ++i) {
        const float4 x = src[i];
        v[4 * i] = x.x; v[4 * i + 1] = x.y; v[4 * i + 2] = x.z; v[4 * i + 3] = x.w;
    }
}

}  // namespace ws_wg
