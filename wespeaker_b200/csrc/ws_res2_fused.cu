// Fused Res2Conv1dReluBn chain (wespeaker/models/ecapa_tdnn.py:29-78) for 16-bit activations on the Hopper tensor cores
// (wgmma, sm_90a).
//
// The reference runs 7 *dependent* dilated k=3 convs on w-channel groups:  sp_i = BN_i(ReLU(conv_i(sp_{i-1} + x_i))).
// As separate launches each is latency-bound.  Here ONE persistent CTA owns a whole utterance and walks the chain on-chip:
//   * the conv input s_i = sp_{i-1} + x_i lives in shared memory as a K-major 128B-swizzled operand buffer with zero rows
//     around it; the three dilated taps are three wgmma operand reads of the SAME buffer at row offsets -d, 0, +d
//     (the descriptor start address is shifted by whole 128-B rows; the swizzle is a function of the absolute smem
//     address: a wrong row-shifted read fails the GPU parity test test_res2_fused_chain_matches_unfused), so there is no
//     im2col, no halo exchange, and the intermediate never goes to HBM;
//   * weights stream through a TMA ring (they are L2-resident, shared by all CTAs); each of the two consumer warpgroups
//     keeps the accumulator of its 64 rows of every 128-row M tile in registers;
//   * the epilogue (bias, ReLU, BN affine) writes sp_i to the output buffer through a swizzled staging tile + TMA store
//     and writes s_{i+1} = rnd(sp_i + x_{i+1}) straight back into the operand buffer for the next conv, from the rounded
//     16-bit sp_i it stores (the unfused chain's contract).
//   * utterances longer than 256 frames are walked in time tiles of 256 rows that overlap by 2 x 32: the chain's receptive
//     field is 7 x dilation <= 28 rows per side, so the inner 192 rows of a tile are exact and only those are stored (three
//     64-row TMA boxes per channel panel); rows before t = 0 and behind the utterance's end are forced to zero in the operand
//     buffer - they are the convs' zero padding.
// Warp roles (384 threads): w0 TMA producer, w1..w3 idle, w4..w11 two consumer warpgroups (MMAs + epilogue).
#include "ws_tc_common.cuh"

namespace {
using namespace ws_tcdev;

constexpr int kPadRows = 8;      // zero rows before t=0 (>= max dilation, multiple of 8 keeps the swizzle phase = t & 7)
constexpr int kSRows = 256 + 16; // operand buffer rows per K panel
constexpr int kWStages = 4;
constexpr int kNumConv = 7;

// DT = activation dtype, W8 = channels per group (64 / 128), both compile-time.  The epilogue sits on the serial
// conv_i -> conv_{i+1} chain, so its latency (not throughput) is what the kernel time is made of.
template <int DT, int W8>
__global__ void __launch_bounds__(384, 1) ws_res2_fused_kernel(const __grid_constant__ WsRes2Params p) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t s_bar[2 * kWStages + 3];
    __shared__ __align__(16) float s_par[3][128];
    // warp index through a shuffle: role branches are warp-uniform for the compiler
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    constexpr int npan = W8 >> 6;                     // K panels of 64 channels (128 B) per tap
    const int nmt = p.ntile > 1 ? 2 : (p.T + 127) >> 7;   // M tiles (128 rows) per work unit
    // work unit = (utterance, time tile); tile k covers rows [k * tstride - halo, +256); single-tile utterances: halo 0
    const int halo = p.ntile > 1 ? 32 : 0, tstride = 256 - 2 * halo, nunits = p.B * p.ntile;
    constexpr int wblk_bytes = W8 * 128;              // one weight k-block: w8 output rows x 128 B
    const uint32_t sS = base;                                             // [npan][kSRows][128 B]
    const uint32_t sW = sS + (uint32_t)(npan * kSRows * 128);             // [kWStages][wblk_bytes]
    const uint32_t sO = sW + (uint32_t)(kWStages * wblk_bytes);           // XO: [npan][256 rows][128 B]: x_{i+1} in, sp_i out
    const uint32_t bar_wfull = smem_u32(&s_bar[0]);
    const uint32_t bar_wempty = smem_u32(&s_bar[kWStages]);
    const uint32_t bar_x0 = smem_u32(&s_bar[2 * kWStages]);
    const uint32_t bar_sfree = smem_u32(&s_bar[2 * kWStages + 1]);
    const uint32_t bar_xn = smem_u32(&s_bar[2 * kWStages + 2]);   // x_{i+1} tile landed in the XO buffer

    // zero the whole operand buffer once: the pad rows (t < 0, t >= 128*nmt) are never written again
    {
        const int n16 = npan * kSRows * 128 / 16;
        for (int i = threadIdx.x; i < n16; i += blockDim.x)
            asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};" ::"r"(sS + (uint32_t)(i * 16)), "r"(0u) : "memory");
    }
    if (warp == 0 && lane == 0) {
        prefetch_tmap(&p.xmap); prefetch_tmap(&p.wmap); prefetch_tmap(&p.omap); prefetch_tmap(&p.omap64);
        for (int s = 0; s < kWStages; ++s) { mbar_init(bar_wfull + 8 * s, 1); mbar_init(bar_wempty + 8 * s, 2); }
        mbar_init(bar_x0, 1);
        mbar_init(bar_sfree, 2);
        mbar_init(bar_xn, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // zeros visible to the TMA / MMA proxy
    __syncthreads();

    if (warp == 0) {
        // ================================ producer: x_0 tiles and the weight ring ================================
        if (lane == 0) {
            int wit = 0, u = 0;
            for (int un = blockIdx.x; un < nunits; un += gridDim.x, ++u) {
                const int b = un / p.ntile, t0 = (un % p.ntile) * tstride - halo;
                mbar_wait(bar_sfree, ((uint32_t)u & 1u) ^ 1u);   // previous unit's last MMA no longer reads S
                mbar_expect_tx(bar_x0, (uint32_t)(npan * nmt * 128 * 128));
                for (int kp = 0; kp < npan; ++kp)
                    for (int mt = 0; mt < nmt; ++mt)
                        tma_load_3d(sS + (uint32_t)((kp * kSRows + kPadRows + mt * 128) * 128), &p.xmap, bar_x0, kp * 64,
                                    t0 + mt * 128, b);
                for (int i = 0; i < kNumConv; ++i)
                    for (int tap = 0; tap < 3; ++tap)
                        for (int kp = 0; kp < npan; ++kp, ++wit) {
                            const int s = wit % kWStages;
                            mbar_wait(bar_wempty + 8 * s, (((uint32_t)(wit / kWStages)) & 1u) ^ 1u);
                            mbar_expect_tx(bar_wfull + 8 * s, (uint32_t)wblk_bytes);
                            tma_load_2d(sW + (uint32_t)(s * wblk_bytes), &p.wmap, bar_wfull + 8 * s, tap * W8 + kp * 64,
                                        i * W8);
                        }
            }
        }
    } else if (warp >= 4) {
        // ================================ consumers ================================
        // Warpgroup wg runs the MMAs of rows [64 wg, 64 wg + 64) of each M tile and then the epilogue of exactly those
        // accumulator elements.  The XO buffer holds the next channel group x_{i+1} (TMA-loaded while the MMAs run); each
        // thread reads its elements, overwrites them with sp_i (stored to HBM by TMA afterwards) and writes
        // s_{i+1} = sp_i + x_{i+1} into the operand buffer.  The elected thread re-arms XO with the following group as soon
        // as the store has read it.
        const int wg = (warp - 4) >> 2, et = threadIdx.x - 128;   // et 0..255
        const int rw = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // first of this thread's two rows in an M tile (+8)
        const int cq = (lane & 3) * 2;                            // first of its column pairs inside an 8-column group
        const uint32_t xo_bytes = (uint32_t)(npan * nmt * 128 * 128);
        auto load_xn = [&](int un_, int grp) {
            const int bb = un_ / p.ntile, tt0 = (un_ % p.ntile) * tstride - halo;
            mbar_expect_tx(bar_xn, xo_bytes);
            for (int kp = 0; kp < npan; ++kp)
                for (int mt = 0; mt < nmt; ++mt)
                    tma_load_3d(sO + (uint32_t)((kp * 256 + mt * 128) * 128), &p.xmap, bar_xn, grp * W8 + kp * 64, tt0 + mt * 128, bb);
        };
        if (et == 0 && (int)blockIdx.x < nunits) load_xn(blockIdx.x, 1);
        int xc = 0, ws = 0, u = 0;
        uint32_t wph = 0;
        for (int un = blockIdx.x; un < nunits; un += gridDim.x, ++u) {
            const int b = un / p.ntile, t0 = (un % p.ntile) * tstride - halo;
            const int Tb = p.lens != nullptr ? min(p.T, p.lens[b]) : p.T;   // rows t >= Tb (and t < 0) are conv padding: stay zero everywhere
            for (int i = 0; i < kNumConv; ++i) {
                if (et < W8) {
                    s_par[0][et] = p.bias[i * W8 + et];
                    s_par[1][et] = p.scale[i * W8 + et];
                    s_par[2][et] = p.shift[i * W8 + et];
                }
                epi_bar_sync();   // s_i complete in the operand buffer (previous epilogue), parameters staged
                if (i == 0) mbar_wait(bar_x0, (uint32_t)u & 1u);
                float acc[2][W8 / 2];
                int prev = -1;
                for (int tap = 0; tap < 3; ++tap)
                    for (int kp = 0; kp < npan; ++kp) {
                        mbar_wait(bar_wfull + 8 * ws, wph);
                        const uint64_t bdesc = ws_wg::desc(sW + (uint32_t)(ws * wblk_bytes), 128);
                        ws_wg::fence();
#pragma unroll
                        for (int mt = 0; mt < 2; ++mt) {
                            if (mt < nmt) {
                                const int row = kPadRows + mt * 128 + wg * 64 + (tap - 1) * p.dil;   // dilated tap = row shift
                                const uint64_t adesc = ws_wg::desc(sS + (uint32_t)((kp * kSRows + row) * 128), 128);
#pragma unroll
                                for (int k = 0; k < 4; ++k)
                                    ws_wg::mma<W8>(DT, acc[mt], adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k),
                                                   (uint32_t)((tap | kp | k) != 0));
                            }
                        }
                        ws_wg::commit();
                        ws_wg::wait<1>();
                        if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(bar_wempty + 8 * prev);
                        prev = ws;
                        if (++ws == kWStages) { ws = 0; wph ^= 1u; }
                    }
                ws_wg::wait<0>();
                ws_wg::fence_regs<W8 / 2>(acc[0]);
                ws_wg::fence_regs<W8 / 2>(acc[1]);
                if ((threadIdx.x & 127) == 0) {
                    mbar_arrive(bar_wempty + 8 * prev);
                    if (i == kNumConv - 1) mbar_arrive(bar_sfree);   // conv 6 done: S may take the next utterance
                }
                epi_bar_sync();   // both warpgroups are done reading S: it may be overwritten with s_{i+1}
                const bool has_next = i < kNumConv - 1;
                if (has_next) { mbar_wait(bar_xn, (uint32_t)xc & 1u); ++xc; }
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    if (mt >= nmt) continue;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int t = mt * 128 + rw + 8 * h;              // row inside the tile (addresses the buffers)
                        const bool valid = t0 + t >= 0 && t0 + t < Tb;    // frame of the utterance
#pragma unroll
                        for (int jg = 0; jg < W8 / 8; ++jg) {
                            const int c = 8 * jg + cq;
                            const float2 bb = *reinterpret_cast<const float2*>(&s_par[0][c]);
                            const float2 sc = *reinterpret_cast<const float2*>(&s_par[1][c]);
                            const float2 sh = *reinterpret_cast<const float2*>(&s_par[2][c]);
                            const float a0 = valid ? fmaf(fmaxf(acc[mt][4 * jg + 2 * h] + bb.x, 0.f), sc.x, sh.x) : 0.f;
                            const float a1 = valid ? fmaf(fmaxf(acc[mt][4 * jg + 2 * h + 1] + bb.y, 0.f), sc.y, sh.y) : 0.f;
                            const int pn = c >> 6;      // panel; 16-B chunk (c & 63) >> 3 of the 128-B row, swizzled by t & 7
                            const uint32_t off = (uint32_t)(((((c & 63) >> 3) ^ (t & 7)) << 4) + (c & 7) * 2);
                            const uint32_t oa = sO + (uint32_t)((pn * 256 + t) * 128) + off;
                            uint32_t xs = 0u;
                            if (has_next) asm volatile("ld.shared.b32 %0, [%1];" : "=r"(xs) : "r"(oa));
                            const uint32_t sp = ws_pack2(a0, a1, DT);
                            asm volatile("st.shared.b32 [%0], %1;" ::"r"(oa), "r"(sp) : "memory");
                            if (has_next && valid) {   // rows >= T stay zero = conv padding
                                // s_{i+1} = rnd(sp_i + x_{i+1}) from the 16-bit sp_i that is stored (as the unfused chain's
                                // out2 = rnd(rnd(sp_i) + x_{i+1}) does), not from its fp32 value
                                const uint32_t o = ws_pack2(ws_16_to_f(sp & 0xffffu, DT) + ws_16_to_f(xs & 0xffffu, DT),
                                                            ws_16_to_f(sp >> 16, DT) + ws_16_to_f(xs >> 16, DT), DT);
                                asm volatile("st.shared.b32 [%0], %1;" ::"r"(sS + (uint32_t)((pn * kSRows + kPadRows + t) * 128) + off),
                                             "r"(o) : "memory");
                            }
                        }
                    }
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                epi_bar_sync();
                if (et == 0) {
                    for (int pn = 0; pn < npan; ++pn) {
                        if (p.ntile > 1) {   // only the exact inner rows [halo, 256 - halo) of the tile: three 64-row boxes
                            for (int q3 = 0; q3 < 3; ++q3)
                                tma_store_3d(&p.omap64, sO + (uint32_t)((pn * 256 + halo + 64 * q3) * 128), i * W8 + pn * 64,
                                             t0 + halo + 64 * q3, b);
                        } else {
                            for (int mt = 0; mt < nmt; ++mt)
                                tma_store_3d(&p.omap, sO + (uint32_t)((pn * 256 + mt * 128) * 128), i * W8 + pn * 64, mt * 128, b);
                        }
                    }
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // XO has been read by the store
                    if (i < kNumConv - 2) load_xn(un, i + 2);                         // group for the next conv's epilogue
                    else if (i == kNumConv - 1 && un + (int)gridDim.x < nunits) load_xn(un + gridDim.x, 1);
                }
            }
        }
        if (et == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
}

template <int DT, int W8>
const char* res2_go(const WsRes2Params* p, cudaStream_t s) {
    constexpr auto kernel = ws_res2_fused_kernel<DT, W8>;
    if (const char* m = ws_smem_opt_in<kernel>(kRes2MaxSmem)) return m;
    kernel<<<p->grid, 384, p->smem_bytes, s>>>(*p);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace

extern "C" const char* ws_res2_launch(const WsRes2Params* p, cudaStream_t s) {
    if (p->dtype != WS_BF16 && p->dtype != WS_F16) return "res2_fused: 16-bit activations only";
    if (p->w8 != 64 && p->w8 != 128) return "res2_fused: groups of 64 or 128 channels only";
    if (p->w8 == 128) return p->dtype == WS_BF16 ? res2_go<WS_BF16, 128>(p, s) : res2_go<WS_F16, 128>(p, s);
    return p->dtype == WS_BF16 ? res2_go<WS_BF16, 64>(p, s) : res2_go<WS_F16, 64>(p, s);
}
