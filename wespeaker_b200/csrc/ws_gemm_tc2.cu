// Persistent warp-specialised conv/GEMM on the Hopper tensor cores (wgmma + TMA, sm_90a).
//
// A conv is an implicit GEMM over output positions: each tap (kernel offset) is a rank-4 TMA map over the channels-last
// activations, shifted by the tap's time / frequency offset, whose out-of-bounds zero fill is the conv's zero padding.  A
// tile is 128 output positions x bn output channels; the k loop walks the taps in k-blocks of 128 / 64 / 32 bytes, with A
// (activations) and B (weights) K-major and swizzled in shared memory as TMA writes them.  On top of that:
//   * persistent CTAs (one per SM) walking a static tile schedule; the TMA producer runs ahead into the next tile's
//     operands while the consumers finish the current tile's epilogue;
//   * bn up to 128: each of the two consumer warpgroups keeps a 64 x bn fp32 accumulator in registers;
//   * BN = 256 (16-bit activations, lean epilogue without row bias, no epilogue-input tile): 128 x 256 tiles, which halve
//     the A-operand reads (L2 and shared memory) and the epilogue passes per FLOP.  The accumulator is 128 fp32 per
//     consumer thread, so the producer warpgroup gives registers back (setmaxnreg 40) and the consumers take them (232);
//     wgmma N and dtype are compile-time (m64n256k16, four per 128-byte k-block).  The consumers run the epilogue on
//     their accumulator fragments in place and write the whole tile into a 64 KB staging buffer in one pass; the
//     otherwise idle producer warps do the rest off the tensor cores' critical path: w1 stages the next tile's per-channel
//     parameters (two buffers) during the mainloop, w2 issues the TMA stores, and w2..w3 compute the SE column sums;
//   * coalesced, asynchronous epilogue: per-channel parameters staged in smem, residual / Res2 "add2" tiles fetched by
//     TMA into swizzled smem while the mainloop runs, outputs packed into 128-B-swizzled smem panels and written with
//     TMA stores (cp.async.bulk.tensor ... bulk_group), which also clips out-of-range rows/positions for free;
//   * CL > 1 (ws_tc3_launch, large layers): clusters of CL CTAs on adjacent position tiles and the same channel tile share
//     the weight tile - each CTA loads 1/CL of it and TMA-multicasts it to the whole cluster, so the L2 -> SM weight
//     traffic per CTA drops by CL; a ring stage is refilled once the consumers of every CTA of the cluster released it.
//
// Warp roles (384 threads): w0 TMA producer, w1..w3 idle (BN = 256: parameter, store and column-sum warps),
// w4..w11 two consumer warpgroups (MMA + epilogue).
//
// Replaces the library-dispatched cuDNN conv + elementwise launches of wespeaker/models/ecapa_tdnn.py:85-106,
// resnet.py:35-69, campplus.py:55-83,138-170.
#include "ws_tc_common.cuh"

namespace {
using namespace ws_tcdev;

constexpr int kThreads2 = 384;

__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the barrier at the same smem offset in CTA `rank` of the cluster
__device__ __forceinline__ void mbar_arrive_remote(uint32_t bar, uint32_t rank) {
    asm volatile(
        "{\n\t.reg .b32 ra;\n\t"
        "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
        "mbarrier.arrive.shared::cluster.b64 _, [ra];\n\t}" ::"r"(bar), "r"(rank)
        : "memory");
}
__device__ __forceinline__ void tma_load_2d_mc(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1,
                                               unsigned short mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, "
        "%4}], [%2], %5;" ::"r"(dst),
        "l"(map), "r"(bar), "r"(c0), "r"(c1), "h"(mask)
        : "memory");
}

// BN = 0: N tile p.bn <= 128 chosen at run time.  BN = 256: the wide 16-bit variant (p.bn == 256, p.bk_bytes == 128).
template <int KIND, int LEAN, int CL, int BN>
__global__ void __launch_bounds__(kThreads2, 1) ws_conv_gemm_tc2_kernel(const __grid_constant__ WsTc2Params p) {
    static_assert(BN == 0 || (BN == 256 && KIND == 1 && (LEAN == WS_BF16 + 1 || LEAN == WS_F16 + 1)), "wide tile: lean 16-bit");
    constexpr bool WIDE = BN == 256;
    extern __shared__ uint8_t smem_raw[];
    // ring full / empty, epilogue-input full / empty; wide tile: parameters full / free (two buffers each), staging
    // written / free
    __shared__ __align__(8) uint64_t s_bar[2 * WS_TC_MAX_STAGES + 8];

    const int warp = uniform_warp_idx(), lane = threadIdx.x & 31;
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const int a_bytes = 128 * p.bk_bytes, b_bytes = p.bn * p.bk_bytes;
    const int stage_bytes = a_bytes + b_bytes;
    const int es = KIND == 0 ? 4 : 2;
    const int panel_bytes = p.panel_bytes;               // row bytes of one staging panel (128 / 64)
    const int panel_cols = panel_bytes / es;
    const int npanels = p.bn / panel_cols;
    const int tile_out_bytes = 128 * p.bn * es;          // one staged output tile
    const uint32_t ring = base;
    const uint32_t stg_out = ring + (uint32_t)(p.nstages * stage_bytes);                  // p.nout output tiles
    const uint32_t stg_in = stg_out + (uint32_t)(p.nout * tile_out_bytes);                // only if p.has_epin
    const uint32_t s_par = stg_in + (uint32_t)(p.has_epin ? tile_out_bytes : 0);          // 3 * bn floats (wide: x2)
    const uint32_t s_scr = s_par + (uint32_t)(3 * p.bn * 4);                              // WS_TC_EPI_SCRATCH bytes (not wide)
    const uint32_t bar_full = smem_u32(&s_bar[0]);
    const uint32_t bar_empty = smem_u32(&s_bar[WS_TC_MAX_STAGES]);
    const uint32_t bar_ifull = smem_u32(&s_bar[2 * WS_TC_MAX_STAGES]);
    const uint32_t bar_iempty = smem_u32(&s_bar[2 * WS_TC_MAX_STAGES + 1]);
    const uint32_t bar_pfull = smem_u32(&s_bar[2 * WS_TC_MAX_STAGES + 2]);    // + 8 * parameter buffer
    const uint32_t bar_pfree = smem_u32(&s_bar[2 * WS_TC_MAX_STAGES + 4]);    // + 8 * parameter buffer
    const uint32_t bar_staged = smem_u32(&s_bar[2 * WS_TC_MAX_STAGES + 6]);
    const uint32_t bar_sfree = smem_u32(&s_bar[2 * WS_TC_MAX_STAGES + 7]);
    float* spar = reinterpret_cast<float*>(smem_raw + (s_par - smem_u32(smem_raw)));
    const uint32_t crank = CL > 1 ? cluster_ctarank() : 0u;
    const int ncl = (int)gridDim.x / CL, cid = (int)blockIdx.x / CL;
    // tile -> (first output channel, position tile of this CTA): the CL CTAs of a cluster take adjacent position tiles
    auto decode = [&](int tile, int& n0, int& t0, int& f0, int& b0) {
        int tt = (tile / p.tiles_n) * CL + (int)crank;
        n0 = (tile % p.tiles_n) * p.bn;
        t0 = (tt % p.tiles_t) << p.bt_log2; tt /= p.tiles_t;
        f0 = (tt % p.tiles_f) << p.bf_log2; tt /= p.tiles_f;
        b0 = tt << p.bb_log2;                            // >= B for a cluster's missing tail tile: all OOB
    };

    if (warp == 0 && lane == 0) {
        for (int i = 0; i < WS_MAX_SRC; ++i) prefetch_tmap(&p.amap[i]);
        prefetch_tmap(&p.wmap);
        for (int i = 0; i < p.nout; ++i) prefetch_tmap(&p.omap[i]);
        if (p.has_epin) prefetch_tmap(&p.imap);
        for (int s = 0; s < p.nstages; ++s) {
            mbar_init(bar_full + 8 * s, 1);
            mbar_init(bar_empty + 8 * s, 2 * CL);   // one arrive per consumer warpgroup of every CTA that writes the stage
        }
        mbar_init(bar_ifull, 1);
        mbar_init(bar_iempty, 8);                   // one arrive per consumer warp
        if constexpr (WIDE) {
            for (int i = 0; i < 2; ++i) {
                mbar_init(bar_pfull + 8 * i, 1);        // the parameter warp
                mbar_init(bar_pfree + 8 * i, 8);        // one arrive per consumer warp
            }
            mbar_init(bar_staged, 8);                   // one arrive per consumer warp
            mbar_init(bar_sfree, p.epi.colsum != nullptr ? 2 : 1);   // the store warp (+ the second column-sum warp)
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if constexpr (CL > 1) cluster_sync();   // the peers' barriers are initialised before any multicast or remote arrive

    if (warp < 4) {
        if constexpr (BN == 256) ws_wg::setmaxnreg_dec<40>();   // 128 x 40 + 256 x 232 <= 64 K registers
        // ================================ TMA producer ================================
        if (warp == 0 && lane == 0) {
            const int bk_elems = p.bk_bytes / es;
            const int wrows = p.bn / CL;             // weight rows this CTA fetches (and multicasts) per k-block
            int it = 0, j = 0;
            for (int tile = cid; tile < p.num_tiles; tile += ncl, ++j) {
                int n0, t0, f0, b0;
                decode(tile, n0, t0, f0, b0);
                for (int tp = 0; tp < p.ntaps; ++tp) {
                    const WsTcTap tap = p.taps[tp];
                    for (int kb = 0; kb < tap.nkb; ++kb) {
                        // 3xTF32: three passes per k-block, small terms first: x_lo*W, x*W_lo, x*W (fp32 operands are
                        // truncated to tf32 by the tensor core, so x and W themselves serve as the high parts)
                        for (int ps = 3 - p.nsplit; ps < 3; ++ps, ++it) {
                            const int s = it % p.nstages;
                            const uint32_t ph = (uint32_t)(it / p.nstages) & 1u;
                            mbar_wait(bar_empty + 8 * s, ph ^ 1u);
                            mbar_expect_tx(bar_full + 8 * s, (uint32_t)stage_bytes);
                            const uint32_t sa = ring + (uint32_t)(s * stage_bytes);
                            tma_load_4d(sa, ps == 0 ? &p.amap_lo[tap.map] : &p.amap[tap.map], bar_full + 8 * s,
                                        tap.c0 + kb * bk_elems, t0 + tap.dt, f0 + tap.df, b0);
                            if constexpr (CL == 1)
                                tma_load_2d(sa + (uint32_t)a_bytes, ps == 1 ? &p.wmap_lo : &p.wmap, bar_full + 8 * s,
                                            tap.wk + kb * bk_elems, n0);
                            else
                                tma_load_2d_mc(sa + (uint32_t)(a_bytes + (int)crank * wrows * p.bk_bytes), ps == 1 ? &p.wmap_lo : &p.wmap,
                                               bar_full + 8 * s, tap.wk + kb * bk_elems, n0 + (int)crank * wrows,
                                               (unsigned short)((1u << CL) - 1u));
                        }
                    }
                }
                // epilogue-input tile (residual / add2): issued after this tile's operand loads so that waiting for
                // the previous tile's epilogue to release the buffer never starves the MMA pipe
                if (p.has_epin) {
                    mbar_wait(bar_iempty, ((uint32_t)j & 1u) ^ 1u);
                    mbar_expect_tx(bar_ifull, (uint32_t)tile_out_bytes);
                    for (int pn = 0; pn < npanels; ++pn)
                        tma_load_4d(stg_in + (uint32_t)(pn * 128 * panel_bytes), &p.imap, bar_ifull, n0 + pn * panel_cols,
                                    t0, f0, b0);
                }
            }
        }
        if constexpr (WIDE) {
            const WsEpi& e = p.epi;
            if (warp == 1) {
                // ============ parameter warp: bias / BN scale / BN shift of tile j into buffer j & 1 ============
                // (filled during the tile's mainloop, so the epilogue finds them staged)
                int j = 0;
                for (int tile = cid; tile < p.num_tiles; tile += ncl, ++j) {
                    const int n0 = (tile % p.tiles_n) * BN, buf = j & 1;
                    float* sp = spar + buf * 3 * BN;
                    mbar_wait(bar_pfree + 8 * buf, ((uint32_t)(j >> 1) & 1u) ^ 1u);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        // all loads of a half before its stores, as in epi_stage_params
                        float pb[4], ps[4], ph[4];
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const int c = n0 + (4 * h + i) * 32 + lane;
                            pb[i] = e.bias ? __ldg(e.bias + c) : 0.f;
                            ps[i] = e.scale ? __ldg(e.scale + c) : 1.f;
                            ph[i] = e.scale ? __ldg(e.shift + c) : 0.f;
                        }
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const int c = (4 * h + i) * 32 + lane;
                            sp[c] = pb[i];
                            sp[BN + c] = ps[i];
                            sp[2 * BN + c] = ph[i];
                        }
                    }
                    __syncwarp();
                    if (lane == 0) mbar_arrive(bar_pfull + 8 * buf);
                }
            } else if (warp == 2 || (warp == 3 && e.colsum != nullptr)) {
                // ============ store warp (w2) and column-sum warps (w2, w3) ============
                // Per staged tile: w2 issues the four panel TMA stores; with column sums, thread q of w2..w3 sums columns
                // [4q, 4q + 4) over each 64-row unit, row by row in fp32 and split at the utterance boundary, in the order
                // of epi_colsum.  Then the staging buffer is handed back once the stores have read it.
                const bool sums = e.colsum != nullptr;
                const int q = (warp - 2) * 32 + lane;
                const uint32_t cbase = stg_out + (uint32_t)((q >> 4) * 128 * 128 + (q & 1) * 8);   // panel, 8-byte half of a chunk
                const int chunk = (q & 15) >> 1;
                const long long ldc = (long long)p.tiles_n * BN;
                int j = 0;
                for (int tile = cid; tile < p.num_tiles; tile += ncl, ++j) {
                    int n0, t0, f0, b0;
                    decode(tile, n0, t0, f0, b0);
                    mbar_wait(bar_staged, (uint32_t)j & 1u);
                    if (warp == 2 && lane == 0) {
                        for (int pn = 0; pn < npanels; ++pn)
                            tma_store_4d(&p.omap[0], stg_out + (uint32_t)(pn * 128 * panel_bytes), n0 + pn * panel_cols, t0, f0, b0);
                        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                    }
                    if (sums) {
                        for (int rh = 0; rh < 2; ++rh) {
                            const int pos0 = t0 + rh * 64;
                            if (b0 >= p.B || pos0 >= p.T) continue;   // units past the last position do not exist
                            const int nvalid = min(64, p.T - pos0);
                            const int split = min(nvalid, (pos0 / e.colsum_T + 1) * e.colsum_T - pos0);
                            float a[4] = {0.f, 0.f, 0.f, 0.f}, s[4] = {0.f, 0.f, 0.f, 0.f};
                            auto add_row = [&](float* acc4, int row) {
                                uint32_t w0, w1;
                                asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(w0), "=r"(w1)
                                             : "r"(cbase + (uint32_t)(row * 128 + ((chunk ^ (row & 7)) << 4))));
                                acc4[0] += ws_16_to_f(w0 & 0xffffu, LEAN - 1); acc4[1] += ws_16_to_f(w0 >> 16, LEAN - 1);
                                acc4[2] += ws_16_to_f(w1 & 0xffffu, LEAN - 1); acc4[3] += ws_16_to_f(w1 >> 16, LEAN - 1);
                            };
#pragma unroll 4
                            for (int rr = 0; rr < split; ++rr) add_row(a, rh * 64 + rr);
#pragma unroll 4
                            for (int rr = max(split, 0); rr < nvalid; ++rr) add_row(s, rh * 64 + rr);
                            float* dst = e.colsum + ((long long)(t0 >> 6) + rh) * 2 * ldc + n0 + 4 * q;
                            *reinterpret_cast<float2*>(dst) = make_float2(a[0], a[1]);
                            *reinterpret_cast<float2*>(dst + 2) = make_float2(a[2], a[3]);
                            *reinterpret_cast<float2*>(dst + ldc) = make_float2(s[0], s[1]);
                            *reinterpret_cast<float2*>(dst + ldc + 2) = make_float2(s[2], s[3]);
                        }
                    }
                    __syncwarp();
                    if (lane == 0) {
                        if (warp == 2) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                        mbar_arrive(bar_sfree);
                    }
                }
                if (warp == 2 && lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
            }
        }
    } else {
        if constexpr (WIDE) ws_wg::setmaxnreg_inc<232>();
        // ================================ consumers: mainloop + epilogue ================================
        const int wg = (warp - 4) >> 2;                  // accumulator rows [64 wg, 64 wg + 64) of the tile
        const int et = threadIdx.x - 128;                // 0..255
        const int r = wg * 64 + (warp & 3) * 16 + (lane & 15);   // tile row this lane owns in the epilogue
        const int dt = KIND == 0 ? WS_F32 : p.epi.dtype;
        const int kper = p.bk_bytes / 32;
        const WsEpi& e = p.epi;
        float* scr = reinterpret_cast<float*>(smem_raw + (s_scr - smem_u32(smem_raw))) + (warp - 4) * ws_wg::kScrFloats;
        auto release = [&](int s) {   // this warpgroup no longer reads ring stage s
            if ((threadIdx.x & 127) == 0) {
                if constexpr (CL == 1) mbar_arrive(bar_empty + 8 * s);
                else
                    for (int c = 0; c < CL; ++c) mbar_arrive_remote(bar_empty + 8 * s, (uint32_t)c);
            }
        };
        int s = 0, j = 0, last_n0 = -1;
        uint32_t ph = 0;
        for (int tile = cid; tile < p.num_tiles; tile += ncl, ++j) {
            int n0, t0, f0, b0;
            decode(tile, n0, t0, f0, b0);
            float acc[BN == 256 ? 128 : 64];
            const int nkit = p.nk_total * p.nsplit;
            int prev = -1;
            for (int kit = 0; kit < nkit; ++kit) {
                mbar_wait(bar_full + 8 * s, ph);
                const uint32_t sa = ring + (uint32_t)(s * stage_bytes) + (uint32_t)(wg * 64 * p.bk_bytes);
                const uint64_t adesc = ws_wg::desc(sa, p.bk_bytes);
                const uint64_t bdesc = ws_wg::desc(ring + (uint32_t)(s * stage_bytes + a_bytes), p.bk_bytes);
                ws_wg::fence();
                if constexpr (BN == 256) {
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        ws_wg::mma16_n256<LEAN - 1>(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (uint32_t)((kit | k) != 0));
                } else {
                    for (int k = 0; k < kper; ++k)
                        ws_wg::mma_n(p.bn, dt, acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (uint32_t)((kit | k) != 0));
                }
                ws_wg::commit();
                ws_wg::wait<1>();
                if (prev >= 0) release(prev);
                prev = s;
                if (++s == p.nstages) { s = 0; ph ^= 1u; }
            }
            ws_wg::wait<0>();
            ws_wg::fence_regs<BN == 256 ? 128 : 64>(acc);
            if (prev >= 0) release(prev);

            if constexpr (WIDE) {
                // One pass in fragment layout: thread (warp w, lane l) holds rows 16w + l/4 + {0, 8} of its warpgroup's
                // 64 and columns 8jj + 2(l%4) + {0, 1}; the arithmetic and its order are those of epi_chunk<LEAN>.
                const int buf = j & 1, cq = 2 * (lane & 3);
                const float* sp = spar + buf * 3 * BN;
                mbar_wait(bar_pfull + 8 * buf, (uint32_t)(j >> 1) & 1u);
#pragma unroll
                for (int jj = 0; jj < 32; ++jj) {
                    const float2 pb = *reinterpret_cast<const float2*>(sp + 8 * jj + cq);
                    acc[4 * jj] += pb.x; acc[4 * jj + 1] += pb.y; acc[4 * jj + 2] += pb.x; acc[4 * jj + 3] += pb.y;
                }
                if (e.act1 == WS_ACT_RELU) {
#pragma unroll
                    for (int i = 0; i < 128; ++i) acc[i] = fmaxf(acc[i], 0.f);
                } else if (e.act1 == WS_ACT_TANH) {
#pragma unroll
                    for (int i = 0; i < 128; ++i) acc[i] = tanh16(acc[i]);
                }
                if (e.scale != nullptr) {
#pragma unroll
                    for (int jj = 0; jj < 32; ++jj) {
                        const float2 a = *reinterpret_cast<const float2*>(sp + BN + 8 * jj + cq);
                        const float2 d = *reinterpret_cast<const float2*>(sp + 2 * BN + 8 * jj + cq);
                        acc[4 * jj] = fmaf(acc[4 * jj], a.x, d.x); acc[4 * jj + 1] = fmaf(acc[4 * jj + 1], a.y, d.y);
                        acc[4 * jj + 2] = fmaf(acc[4 * jj + 2], a.x, d.x); acc[4 * jj + 3] = fmaf(acc[4 * jj + 3], a.y, d.y);
                    }
                }
                if (e.act2 == WS_ACT_RELU) {
#pragma unroll
                    for (int i = 0; i < 128; ++i) acc[i] = fmaxf(acc[i], 0.f);
                }
                // the staging buffer is free once the previous tile's stores have read it and its column sums are done
                mbar_wait(bar_sfree, ((uint32_t)j & 1u) ^ 1u);
                // 128-byte-swizzled panels of 64 columns: the 8 rows of a store land in 8 different 16-byte chunks, so
                // the 32-bit stores of a warp are free of bank conflicts
                const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2);
                const uint32_t ra = stg_out + (uint32_t)(row * 128 + (lane & 3) * 4);
#pragma unroll
                for (int jj = 0; jj < 32; ++jj) {
                    const uint32_t a = ra + (uint32_t)((jj >> 3) * 128 * 128 + (((jj & 7) ^ (row & 7)) << 4));
                    asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(ws_pack2(acc[4 * jj], acc[4 * jj + 1], LEAN - 1)) : "memory");
                    asm volatile("st.shared.b32 [%0], %1;" ::"r"(a + 8 * 128), "r"(ws_pack2(acc[4 * jj + 2], acc[4 * jj + 3], LEAN - 1))
                                 : "memory");
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                __syncwarp();
                if (lane == 0) {
                    mbar_arrive(bar_pfree + 8 * buf);
                    mbar_arrive(bar_staged);
                }
                continue;
            }
            // row -> output position (for the per-row epilogue inputs that are not tile-shaped)
            const int t = t0 + (r & ((1 << p.bt_log2) - 1));
            const int f = f0 + ((r >> p.bt_log2) & ((1 << p.bf_log2) - 1));
            const int b = b0 + (r >> (p.bt_log2 + p.bf_log2));
            const bool valid = (t < p.T) && (f < p.F) && (b < p.B);
            const long long pos = ((long long)b * p.F + f) * p.T + t;
            int eb = 0, etm = 0;
            if (valid && (e.rowbias != nullptr || e.gate != nullptr)) {
                eb = (int)(pos / e.FT);
                etm = (int)(pos % e.T);
            }
            // staging buffers are free once the previous tile's TMA stores have finished reading them
            if (et == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
            if (n0 != last_n0) {
                epi_stage_params(p, spar, n0, et);
                last_n0 = n0;
            }
            epi_bar_sync();
            if (p.has_epin) mbar_wait(bar_ifull, (uint32_t)j & 1u);
            const EpiTile xt{spar, stg_in, stg_out, tile_out_bytes, panel_bytes, panel_cols, n0, r, valid, eb, etm};
            // 64-column blocks of the accumulator: lanes 0..15 take columns [0, 32) of their row, lanes 16..31 [32, 64)
#pragma unroll
            for (int cb = 0; cb < 2; ++cb) {
                if (cb * 64 < p.bn) {
                    uint32_t raw[32];
                    ws_wg::frag_to_rows<64>(acc, cb * 64, scr, reinterpret_cast<float*>(raw));
                    const int c = cb * 64 + (lane >> 4) * 32;
                    if (c < p.bn) epi_chunk<LEAN>(p, xt, raw, c);
                }
            }
            // the epilogue-input tile is drained: hand it back
            __syncwarp();
            if (lane == 0 && p.has_epin) mbar_arrive(bar_iempty);
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            epi_bar_sync();
            if (et == 0) {
                for (int o = 0; o < p.nout; ++o)
                    for (int pn = 0; pn < npanels; ++pn)
                        tma_store_4d(&p.omap[o], stg_out + (uint32_t)(o * tile_out_bytes + pn * 128 * panel_bytes),
                                     n0 + pn * panel_cols, t0, f0, b0);
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
            if constexpr (LEAN == WS_BF16 + 1 || LEAN == WS_F16 + 1) epi_colsum<LEAN>(p, stg_out, et, n0, p.bn, t0, b0);
        }
        if constexpr (!WIDE)
            if (et == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    if constexpr (CL > 1) cluster_sync();   // no peer may still multicast into this CTA's ring or arrive on its barriers
}

}  // namespace

namespace {
template <int KIND, int LEAN, int CL, int BN = 0>
const char* tc2_go(const WsTc2Params* p, cudaStream_t s) {
    constexpr auto kernel = ws_conv_gemm_tc2_kernel<KIND, LEAN, CL, BN>;
    if (const char* m = ws_smem_opt_in<kernel>(kMaxDynSmem2)) return m;
    cudaError_t e;
    if constexpr (CL == 1) {
        kernel<<<p->grid, kThreads2, p->smem_bytes, s>>>(*p);
        e = cudaGetLastError();
    } else {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned)p->grid); cfg.blockDim = dim3(kThreads2); cfg.dynamicSmemBytes = (size_t)p->smem_bytes; cfg.stream = s;
        cudaLaunchAttribute at;
        at.id = cudaLaunchAttributeClusterDimension;
        at.val.clusterDim.x = CL; at.val.clusterDim.y = 1; at.val.clusterDim.z = 1;
        cfg.attrs = &at; cfg.numAttrs = 1;
        e = cudaLaunchKernelEx(&cfg, kernel, *p);
    }
    return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}
template <int CL>
const char* tc2_dispatch(const WsTc2Params* p, cudaStream_t s, int lean) {
    if (p->bn == 256) return lean == WS_BF16 + 1 ? tc2_go<1, WS_BF16 + 1, CL, 256>(p, s) : tc2_go<1, WS_F16 + 1, CL, 256>(p, s);
    if (lean == WS_F32 + 1) return tc2_go<0, WS_F32 + 1, CL>(p, s);
    if (lean == WS_BF16 + 1) return tc2_go<1, WS_BF16 + 1, CL>(p, s);
    if (lean == WS_F16 + 1) return tc2_go<1, WS_F16 + 1, CL>(p, s);
    if (p->kind == 0) return tc2_go<0, 0, CL>(p, s);
    return tc2_go<1, 0, CL>(p, s);
}

// how many clusters of CL CTAs (at the kernel's maximum shared memory) the device keeps resident at once: GPCs whose SM
// count is not a multiple of CL leave SMs idle, so this can be below num_sms / CL
template <int CL>
int tc3_query_clusters() {
    constexpr auto kernel = ws_conv_gemm_tc2_kernel<1, WS_BF16 + 1, CL, 0>;
    if (ws_smem_opt_in<kernel>(kMaxDynSmem2) != nullptr) return 0;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(ws_num_sms() / CL * CL));
    cfg.blockDim = dim3(kThreads2);
    cfg.dynamicSmemBytes = kMaxDynSmem2;
    cudaLaunchAttribute at;
    at.id = cudaLaunchAttributeClusterDimension;
    at.val.clusterDim.x = CL; at.val.clusterDim.y = 1; at.val.clusterDim.z = 1;
    cfg.attrs = &at; cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, kernel, &cfg) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}
}  // namespace

extern "C" int ws_tc3_max_clusters(int cl) {
    static std::atomic<int> cache[64][2] = {};   // per device ordinal and cluster size; 0 = not yet queried
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64 || (cl != 2 && cl != 4)) return 0;
    std::atomic<int>& slot = cache[dev][cl == 4];
    int n = slot.load();
    if (n == 0) {
        n = cl == 4 ? tc3_query_clusters<4>() : tc3_query_clusters<2>();
        slot.store(n);
    }
    return n;
}

// the 256-wide instantiation has the lean 16-bit epilogue without row bias only and no room for an epilogue-input tile
static const char* ws_tc2_wide_check(const WsTc2Params* p, int lean) {
    if (p->bn == 256 && ((lean != WS_BF16 + 1 && lean != WS_F16 + 1) || p->has_epin || p->bk_bytes != 128 ||
                         p->epi.rowbias != nullptr))
        return "conv: 256-wide tiles need the lean 16-bit epilogue without row bias, 128-byte k-blocks and no residual / "
               "add2 tile";
    return nullptr;
}

extern "C" const char* ws_tc2_launch(const WsTc2Params* p, cudaStream_t s) {
    const int lean = p->epi_generic ? 0 : ws_tc_lean_kind(p);
    if (const char* m = ws_tc_colsum_check(p, lean)) return m;
    if (const char* m = ws_tc2_wide_check(p, lean)) return m;
    return tc2_dispatch<1>(p, s, lean);
}

extern "C" const char* ws_tc3_launch(const WsTc2Params* p, cudaStream_t s) {
    const int lean = p->epi_generic ? 0 : ws_tc_lean_kind(p);
    if (const char* m = ws_tc_colsum_check(p, lean)) return m;
    if (const char* m = ws_tc2_wide_check(p, lean)) return m;
    if (p->cl != 2 && p->cl != 4) return "ws_tc3_launch: cluster size must be 2 or 4";
    return p->cl == 4 ? tc2_dispatch<4>(p, s, lean) : tc2_dispatch<2>(p, s, lean);
}
