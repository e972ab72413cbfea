// Halo-resident 3x3 stride-1 convolution on the Hopper tensor cores (wgmma + TMA, sm_90a) for the low-channel 2-D stages:
// BasicBlock convs of ResNet layers 1-3 (wespeaker/models/resnet.py:35-69) and of CAM++'s FCM head
// (wespeaker/models/campplus.py:245-330), 16-bit activations, channels-last [B][F][T][C], C in {32, 64, 128}.
//
// The generic conv-GEMM kernel (ws_gemm_tc2.cu) fetches one A tile PER TAP: every input element crosses L2 -> SM nine
// times.  Here each input row of F is loaded ONCE into a shared-memory ring:
//   * one ring slot = one input row f of one utterance (or of `nb` short utterances side by side) including its two halo
//     columns t = -1 and t = T (TMA out-of-bounds zero fill = the conv's zero padding), stored as K-major swizzled operand
//     rows (one row per time step);
//   * output row f needs slots f-1, f, f+1; tap (df, dt) is a wgmma operand read of slot f+df starting (1 + dt) rows
//     into it - a descriptor start shifted by whole rows (the swizzle is a function of the absolute shared-memory address,
//     as in ws_res2_fused.cu), so there is no im2col and no per-tap reload;
//   * the CTA walks down F: each step loads one new row, retires one, and runs 9 * npan k-blocks of MMAs; each of the two
//     consumer warpgroups keeps the accumulator of its 64 rows of every M tile in registers; weights are resident in
//     shared memory (C <= 64) or streamed through a TMA ring;
//   * epilogue: folded-BN bias, optional residual (TMA-loaded into the staging tile), ReLU, swizzled staging + TMA store
//     (which also clips the halo / padding rows).
// Steps (output rows over all utterances) are split contiguously over one persistent CTA per SM.
//
// Warp roles (384 threads): w0 input-row producer, w1, w2 idle, w3 weight producer, w4..w11 two consumer warpgroups.
#include "ws_tc_common.cuh"

namespace {
using namespace ws_tcdev;

constexpr int kC3Threads = 384;

// Walk over this CTA's contiguous range of output-row steps.  The (f, b group, t tile, n tile) decomposition costs integer
// divisions only once; every role advances it incrementally (a 64-bit div/mod per step and role was ~5k cycles per step of
// pure overhead in the first version of this kernel).
struct C3Step {
    int f, bg, tt, nt;
    bool first, last;
};
struct C3Iter {
    int s, s_beg, s_end, f, bg, tt, nt;
    __device__ __forceinline__ C3Iter(const WsC3Params& p, int beg, int end) : s(beg), s_beg(beg), s_end(end) {
        f = beg % p.F;
        int img = beg / p.F;
        bg = img % p.n_bg; img /= p.n_bg;
        tt = img % p.n_tt;
        nt = img / p.n_tt;
    }
    __device__ __forceinline__ bool done() const { return s >= s_end; }
    __device__ __forceinline__ C3Step cur(const WsC3Params& p) const {
        C3Step x;
        x.f = f; x.bg = bg; x.tt = tt; x.nt = nt;
        x.first = (s == s_beg) || (f == 0);
        x.last = (s + 1 == s_end) || (f == p.F - 1);
        return x;
    }
    __device__ __forceinline__ void next(const WsC3Params& p) {
        ++s;
        if (++f == p.F) {
            f = 0;
            if (++bg == p.n_bg) { bg = 0; if (++tt == p.n_tt) { tt = 0; ++nt; } }
        }
    }
};

template <int DT, int ROWB, int NPAN, int NMT, int NN>
__global__ void __launch_bounds__(kC3Threads, 1) ws_conv3x3_kernel(const __grid_constant__ WsC3Params p) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t s_bar[2 * WS_C3_MAX_RING + 2 * WS_C3_MAX_WSTAGES + 4];

    // warp index through a shuffle: the compiler then knows the role branches are warp-uniform
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const int slot_bytes = p.npan * p.slot_rows * p.row_bytes;
    const int wblk_bytes = p.N * p.row_bytes;
    const int nwblk = 9 * p.npan;
    const uint32_t ring = base;
    const uint32_t wbuf = ring + (uint32_t)(p.R * slot_bytes);
    const uint32_t stg = (wbuf + (uint32_t)((p.w_resident ? nwblk : p.w_stages) * wblk_bytes) + 1023u) & ~1023u;
    const int npanels_out = p.N / p.panel_cols;
    const int panel_stride = p.stg_rows * p.panel_bytes;
    const int tile_bytes = npanels_out * panel_stride;
    const int obuf_bytes = p.n_mt * tile_bytes;                    // one staging buffer = the n_mt output tiles of a step
    const uint32_t s_par = stg + (uint32_t)(p.stg_bufs * obuf_bytes);
    const uint32_t bar_afull = smem_u32(&s_bar[0]);
    const uint32_t bar_aempty = smem_u32(&s_bar[WS_C3_MAX_RING]);
    const uint32_t bar_wfull = smem_u32(&s_bar[2 * WS_C3_MAX_RING]);
    const uint32_t bar_wempty = smem_u32(&s_bar[2 * WS_C3_MAX_RING + WS_C3_MAX_WSTAGES]);
    const uint32_t bar_wres = smem_u32(&s_bar[2 * WS_C3_MAX_RING + 2 * WS_C3_MAX_WSTAGES]);
    const uint32_t bar_rfull = smem_u32(&s_bar[2 * WS_C3_MAX_RING + 2 * WS_C3_MAX_WSTAGES + 1]);   // [buffer] residual panels landed

    const int s_beg = (int)((long long)p.total_steps * blockIdx.x / gridDim.x);
    const int s_end = (int)((long long)p.total_steps * (blockIdx.x + 1) / gridDim.x);

    if (warp == 0 && lane == 0) {
        prefetch_tmap(&p.amap); prefetch_tmap(&p.amap_tail); prefetch_tmap(&p.wmap); prefetch_tmap(&p.omap); prefetch_tmap(&p.rmap);
        // ring slots and weight stages are released by both consumer warpgroups
        for (int i = 0; i < p.R; ++i) { mbar_init(bar_afull + 8 * i, 1); mbar_init(bar_aempty + 8 * i, 2); }
        for (int i = 0; i < WS_C3_MAX_WSTAGES; ++i) { mbar_init(bar_wfull + 8 * i, 1); mbar_init(bar_wempty + 8 * i, 2); }
        mbar_init(bar_wres, 1);
        for (int i = 0; i < 3; ++i) mbar_init(bar_rfull + 8 * i, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 0) {
        // ================================ input-row producer ================================
        if (lane == 0) {
            const uint32_t tx = (uint32_t)(p.npan * p.rows_loaded * p.row_bytes);
            int slot = 0;
            uint32_t sphase = 1;                             // waits on the "previous" phase of a fresh barrier pass at once
            auto load_row = [&](int frow, int bg, int tt) {
                mbar_wait(bar_aempty + 8 * slot, sphase);
                mbar_expect_tx(bar_afull + 8 * slot, tx);
                const int tc = tt * p.tb - 1, b0 = bg * p.nb;
                for (int kp = 0; kp < p.npan; ++kp) {
                    const uint32_t dst = ring + (uint32_t)((slot * p.npan + kp) * p.slot_rows * p.row_bytes);
                    if (p.st == 2) {      // even plane from output column t0, odd plane shifted by one (O'[k] = x[2k - 1])
                        tma_load_4d(dst, &p.amap, bar_afull + 8 * slot, kp * p.kc, tc + 1, frow, b0);
                        tma_load_4d(dst + (uint32_t)(p.sub_rows * p.row_bytes), &p.amap_tail, bar_afull + 8 * slot, kp * p.kc, tc, frow, b0);
                    } else if (p.single_box) {
                        tma_load_4d(dst, &p.amap, bar_afull + 8 * slot, kp * p.kc, tc, frow, b0);
                    } else {
                        for (int m = 0; m < p.n_mt; ++m)
                            tma_load_4d(dst + (uint32_t)(m * 128 * p.row_bytes), &p.amap, bar_afull + 8 * slot, kp * p.kc,
                                        tc + 128 * m, frow, b0);
                        tma_load_4d(dst + (uint32_t)(p.n_mt * 128 * p.row_bytes), &p.amap_tail, bar_afull + 8 * slot,
                                    kp * p.kc, tc + 128 * p.n_mt, frow, b0);
                    }
                }
                if (++slot == p.R) { slot = 0; sphase ^= 1u; }
            };
            for (C3Iter it(p, s_beg, s_end); !it.done(); it.next(p)) {
                const C3Step st = it.cur(p);
                const int fi = p.sf * st.f;                  // input row under the centre tap
                if (st.first) load_row(fi - 1, st.bg, st.tt);
                if (st.first || p.sf == 2) load_row(fi, st.bg, st.tt);
                load_row(fi + 1, st.bg, st.tt);
            }
        }
    } else if (warp == 3) {
        // ================================ weight producer ================================
        if (lane == 0 && s_beg < s_end) {
            if (p.w_resident) {
                mbar_expect_tx(bar_wres, (uint32_t)(nwblk * wblk_bytes));
                for (int tap = 0; tap < 9; ++tap)
                    for (int kp = 0; kp < p.npan; ++kp)
                        tma_load_2d(wbuf + (uint32_t)((tap * p.npan + kp) * wblk_bytes), &p.wmap, bar_wres,
                                    tap * p.Cin + kp * p.kc, 0);
            } else {
                int ws = 0;
                uint32_t wphase = 1;
                for (C3Iter it(p, s_beg, s_end); !it.done(); it.next(p)) {   // one weight pass per step
                    const int nt = it.cur(p).nt;
                    for (int tap = 0; tap < 9; ++tap)
                        for (int kp = 0; kp < p.npan; ++kp) {
                            mbar_wait(bar_wempty + 8 * ws, wphase);
                            mbar_expect_tx(bar_wfull + 8 * ws, (uint32_t)wblk_bytes);
                            tma_load_2d(wbuf + (uint32_t)(ws * wblk_bytes), &p.wmap, bar_wfull + 8 * ws,
                                        tap * p.Cin + kp * p.kc, nt * p.N);
                            if (++ws == p.w_stages) { ws = 0; wphase ^= 1u; }
                        }
                }
            }
        }
    } else if (warp >= 4) {
        // ================================ consumers: MMAs + epilogue ================================
        // Both warpgroups walk the same steps; warpgroup wg issues the MMAs of rows [64 wg, 64 wg + 64) of every M tile and
        // runs the epilogue of exactly those accumulator elements.  One elected thread issues the residual loads and the
        // TMA stores of a step.
        constexpr int KPER = ROWB / 32;
        const int wg = (warp - 4) >> 2, et = threadIdx.x - 128;
        const int rw = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // first of this thread's two rows of an M tile (+8)
        const int cq = (lane & 3) * 2;                            // first column of its pair inside an 8-column group
        const bool tma_thread = et == 0;
        float* spar = reinterpret_cast<float*>(smem_raw + (s_par - smem_u32(smem_raw)));
        // operand start row of the three time taps inside a slot: consecutive rows, or (stride 2 along t) the shifted-odd,
        // even, shifted-odd+1 planes
        const int tap_row0 = p.st == 2 ? p.sub_rows : 0, tap_row1 = p.st == 2 ? 0 : 1, tap_row2 = p.st == 2 ? p.sub_rows + 1 : 2;
        const int R = p.R;
        const int nunits = p.n_mt * npanels_out;                 // store units per step (M tile, column panel)
        const bool has_res = p.res != nullptr;
        const int nbuf = p.stg_bufs;
        // The residual panel of a unit is TMA-loaded INTO that unit's output staging panel (same box geometry and swizzle);
        // the epilogue reads it from there and overwrites it in place.  With three staging buffers the load for step s+1 is
        // issued at the START of step s (its buffer was last read by the store of step s-2, long drained): a full step of
        // lead time.  With two it can only be issued at the end of step s, with one in line.
        const uint32_t unit_tx = (uint32_t)(p.panel_bytes * (p.case_b ? p.P * p.nb : 128));
        auto issue_res = [&](const C3Step& x, int ob) {
            mbar_expect_tx(bar_rfull + 8 * ob, unit_tx * (uint32_t)nunits);
            for (int u = 0; u < nunits; ++u) {
                const int mt = u / npanels_out, pn = u - mt * npanels_out;
                tma_load_4d(stg + (uint32_t)(ob * obuf_bytes + mt * tile_bytes + pn * panel_stride), &p.rmap,
                            bar_rfull + 8 * ob, x.nt * p.N + pn * p.panel_cols, p.case_b ? 0 : x.tt * p.tb + 128 * mt,
                            x.f, x.bg * p.nb);
            }
        };
        if (p.w_resident && s_beg < s_end) mbar_wait(bar_wres, 0);
        if (has_res && nbuf >= 2 && tma_thread && s_beg < s_end) issue_res(C3Iter(p, s_beg, s_end).cur(p), 0);
        int jslot = 0, wst = 0, last_nt = -1, ob = 0;    // ob == step % nbuf
        uint32_t jphase = 0, wph = 0, rph = 0;            // rph == (step / nbuf) & 1
        for (C3Iter it(p, s_beg, s_end); !it.done(); it.next(p)) {
            const C3Step st = it.cur(p);
            const int nnew = st.first ? 3 : p.sf;        // a new image segment starts with rows f-1, f, f+1
            // wait for the newly loaded rows: slot / phase of load i follow incrementally from (jslot, jphase)
            for (int i = 0; i < nnew; ++i) {
                mbar_wait(bar_afull + 8 * jslot, jphase);
                if (++jslot == R) { jslot = 0; jphase ^= 1u; }
            }
            // ---- mainloop: the three input rows (runtime loop), everything inside unrolled
            int sl0 = jslot - 3 < 0 ? jslot - 3 + R : jslot - 3;        // slot of row f-1
            const int slot_first = sl0;
            float acc[NMT][NN / 2];
            int prev = -1, wblk = 0;
#pragma unroll 1
            for (int df = 0; df < 3; ++df) {
                const uint32_t a_slot = ring + (uint32_t)(sl0 * slot_bytes) + (uint32_t)(wg * 64 * ROWB);
#pragma unroll
                for (int dt = 0; dt < 3; ++dt) {
                    const uint32_t a_tap = a_slot + (uint32_t)(dt == 0 ? tap_row0 : (dt == 1 ? tap_row1 : tap_row2)) * ROWB;
#pragma unroll
                    for (int kp = 0; kp < NPAN; ++kp, ++wblk) {
                        uint32_t b_addr;
                        if (!p.w_resident) {
                            mbar_wait(bar_wfull + 8 * wst, wph);
                            b_addr = wbuf + (uint32_t)(wst * wblk_bytes);
                        } else {
                            b_addr = wbuf + (uint32_t)(wblk * wblk_bytes);
                        }
                        const uint64_t bd = ws_wg::desc(b_addr, ROWB);
                        ws_wg::fence();
#pragma unroll
                        for (int mt = 0; mt < NMT; ++mt) {
                            const uint64_t ad = ws_wg::desc(a_tap + (uint32_t)(kp * p.slot_rows * ROWB + mt * 128 * ROWB), ROWB);
#pragma unroll
                            for (int k = 0; k < KPER; ++k)
                                ws_wg::mma<NN>(DT, acc[mt], ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k),
                                               (uint32_t)((df | dt | kp | k) != 0));
                        }
                        ws_wg::commit();
                        if (!p.w_resident) {
                            ws_wg::wait<1>();     // the previous weight stage is no longer read
                            if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(bar_wempty + 8 * prev);
                            prev = wst;
                            if (++wst == p.w_stages) { wst = 0; wph ^= 1u; }
                        }
                    }
                }
                ws_wg::wait<0>();
                if (++sl0 == R) sl0 = 0;                                     // next input row (ring wrap)
            }
#pragma unroll
            for (int mt = 0; mt < NMT; ++mt) ws_wg::fence_regs<NN / 2>(acc[mt]);
            if ((threadIdx.x & 127) == 0) {
                if (prev >= 0) mbar_arrive(bar_wempty + 8 * prev);
                int sl1 = slot_first + 1 == R ? 0 : slot_first + 1;
                const int sl2 = sl1 + 1 == R ? 0 : sl1 + 1;
                mbar_arrive(bar_aempty + 8 * slot_first);                   // row f-1 is not needed by later steps
                if (st.last || p.sf == 2) mbar_arrive(bar_aempty + 8 * sl1);  // stride 2: neither is the centre row
                if (st.last) mbar_arrive(bar_aempty + 8 * sl2);               // end of this image segment
            }

            // ---- epilogue
            const int n0 = st.nt * p.N, t0 = st.tt * p.tb, b0 = st.bg * p.nb;
            const uint32_t sbuf = stg + (uint32_t)(ob * obuf_bytes);
            const int ob_next = ob + 1 == nbuf ? 0 : ob + 1;
            if (tma_thread) {
                if (nbuf == 1) {          // single staging buffer: free once the previous store has read it
                    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                    if (has_res) issue_res(st, 0);
                } else if (nbuf == 3) {   // buffer of step s+1 == buffer of step s-2: drained unless 2 stores pend
                    asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
                    if (has_res) {
                        C3Iter nx = it;
                        nx.next(p);
                        if (!nx.done()) issue_res(nx.cur(p), ob_next);
                    }
                }
            }
            if (st.nt != last_nt) {
                for (int c = et; c < p.N; c += 256) spar[c] = p.bias ? __ldg(p.bias + n0 + c) : 0.f;
                last_nt = st.nt;
            }
            epi_bar_sync();
            if (has_res) mbar_wait(bar_rfull + 8 * ob, rph);
#pragma unroll
            for (int mt = 0; mt < NMT; ++mt) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int r = rw + 8 * h;                       // row inside the M tile
                    bool zero = false;
                    if (p.lens != nullptr) {   // length-masked batch: frames behind the utterance's end are the next conv's padding
                        const int i2 = mt * 128 + r, u = i2 / p.P, tti = i2 - u * p.P, bb = min(b0 + u, p.B - 1);
                        zero = t0 + tti >= p.lens[bb];
                    }
#pragma unroll
                    for (int jg = 0; jg < NN / 8; ++jg) {
                        const int c = 8 * jg + cq, pn = c / p.panel_cols, cc = c - pn * p.panel_cols;
                        const uint32_t a = sbuf + (uint32_t)(mt * tile_bytes + pn * panel_stride + r * p.panel_bytes +
                                                             (swz_chunk(cc >> 3, r, p.panel_bytes) << 4) + (cc & 7) * 2);
                        float v0 = acc[mt][4 * jg + 2 * h] + spar[c], v1 = acc[mt][4 * jg + 2 * h + 1] + spar[c + 1];
                        if (has_res) {
                            uint32_t w;
                            asm volatile("ld.shared.b32 %0, [%1];" : "=r"(w) : "r"(a));
                            v0 += ws_16_to_f(w & 0xffffu, DT); v1 += ws_16_to_f(w >> 16, DT);
                        }
                        if (p.relu) {
                            v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f);
                            if (p.relu == 2) { v0 = fminf(v0, 20.f); v1 = fminf(v1, 20.f); }   // Hardtanh(0, 20) (eres2net.py:43-52)
                        }
                        if (zero) { v0 = 0.f; v1 = 0.f; }
                        // rows that are no output position (halo columns, rows past T or B) hold junk: the TMA store clips them
                        asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(ws_pack2(v0, v1, DT)) : "memory");
                    }
                }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            epi_bar_sync();
            if (tma_thread) {
                for (int u = 0; u < nunits; ++u) {
                    const int mt = u / npanels_out, pn = u - mt * npanels_out;
                    tma_store_4d(&p.omap, sbuf + (uint32_t)(mt * tile_bytes + pn * panel_stride), n0 + pn * p.panel_cols,
                                 p.case_b ? 0 : t0 + 128 * mt, st.f, b0);
                }
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                if (nbuf == 2) {   // the other buffer (the store of step s-1) must be drained before anything lands in it
                    asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
                    if (has_res) {
                        C3Iter nx = it;
                        nx.next(p);
                        if (!nx.done()) issue_res(nx.cur(p), ob_next);
                    }
                }
            }
            ob = ob_next;
            if (ob == 0) rph ^= 1u;
        }
        if (tma_thread) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
}

}  // namespace

namespace {
template <int DT, int ROWB, int NPAN, int NMT, int NN>
const char* c3_launch_one(const WsC3Params* p, cudaStream_t s) {
    constexpr auto kernel = ws_conv3x3_kernel<DT, ROWB, NPAN, NMT, NN>;
    if (const char* m = ws_smem_opt_in<kernel>(kC3MaxSmem)) return m;
    kernel<<<p->grid, kC3Threads, p->smem_bytes, s>>>(*p);
    return nullptr;
}
template <int DT, int ROWB, int NPAN, int NMT>
const char* c3_dispatch_n(const WsC3Params* p, cudaStream_t s, int n) {
    if (n == 32) return c3_launch_one<DT, ROWB, NPAN, NMT, 32>(p, s);
    if (n == 64) return c3_launch_one<DT, ROWB, NPAN, NMT, 64>(p, s);
    if (n == 128) return c3_launch_one<DT, ROWB, NPAN, NMT, 128>(p, s);
    return "conv3x3: unsupported channel tile";
}
// (operand row bytes, K panels per tap, M tiles per step, output channels): 64-byte rows only exist with one panel (C = 32)
template <int DT>
const char* c3_dispatch(const WsC3Params* p, cudaStream_t s, int rowb, int npan, int nmt, int n) {
    if (rowb == 64 && npan == 1 && nmt == 1) return c3_dispatch_n<DT, 64, 1, 1>(p, s, n);
    if (rowb == 64 && npan == 1 && nmt == 2) return c3_dispatch_n<DT, 64, 1, 2>(p, s, n);
    if (rowb == 128 && npan == 1 && nmt == 1) return c3_dispatch_n<DT, 128, 1, 1>(p, s, n);
    if (rowb == 128 && npan == 1 && nmt == 2) return c3_dispatch_n<DT, 128, 1, 2>(p, s, n);
    if (rowb == 128 && npan == 2 && nmt == 1) return c3_dispatch_n<DT, 128, 2, 1>(p, s, n);
    if (rowb == 128 && npan == 2 && nmt == 2) return c3_dispatch_n<DT, 128, 2, 2>(p, s, n);
    return "conv3x3: unsupported (row bytes, K panels, M tiles) combination";
}
}  // namespace

extern "C" const char* ws_c3_launch(const WsC3Params* p, cudaStream_t s) {
    const char* m;
    if (p->dtype == WS_BF16) m = c3_dispatch<WS_BF16>(p, s, p->row_bytes, p->npan, p->n_mt, p->N);
    else if (p->dtype == WS_F16) m = c3_dispatch<WS_F16>(p, s, p->row_bytes, p->npan, p->n_mt, p->N);
    else return "conv3x3: 16-bit activations only";
    if (m) return m;
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}
