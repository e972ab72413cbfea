// Fused CAMDenseTDNNLayer of CAM++ (wespeaker/models/campplus.py:86-170) for 16-bit activations on the Hopper tensor
// cores (wgmma + TMA, sm_90a):
//
//     h   = ReLU(BN2(Conv1x1(ReLU(BN1(x)))))                      x: (T, Cin) slice of the block's concat buffer
//     ctx = mean_T(h) + segment_mean_100(h)                       (ceil-mode last segment divides by its own length)
//     m   = sigmoid(W2 ReLU(W1 ctx + b1) + b2)                    per segment, 128 -> 64 -> 32
//     y   = Conv_k3,dilated(h) * m                                32 new channels appended to the concat buffer
//
// Unfused this is 4 launches per layer (BN-ReLU pass that materialises the pre-activation, 1x1 conv-GEMM, context-gate
// kernel, dilated conv-GEMM): 52 layers x 4 latency-bound launches.  Here ONE CTA owns one utterance for a whole layer and
// nothing but the 32 new channels leaves the SM:
//   * BN1 + ReLU is applied IN PLACE on each TMA-loaded operand panel in shared memory (8 warps) before its MMAs are issued;
//   * h never goes to HBM: the first epilogue writes it as a K-major swizzled operand buffer with zero rows around it, its
//     column sums give the context vector, and the dilated taps are row-shifted wgmma reads of that buffer (as in
//     ws_res2_fused.cu);
//   * the gate is applied in the second epilogue, and the result leaves through a swizzled staging tile + TMA store.
// Each of the two consumer warpgroups issues the MMAs of rows [64 wg, 64 wg + 64) of every 128-row tile and applies the
// epilogues to exactly those accumulator elements (registers).  Layers [l0, l1) of a dense block can run back to back
// inside one launch (per-layer descriptors live in device memory).
//
// Warp roles (384 threads): w0 TMA producer, w1..w3 idle, w4..w11 two consumer warpgroups (transform, MMAs, epilogues).
#include "ws_tc_common.cuh"

namespace {
using namespace ws_tcdev;

constexpr int kCamThreads = 384;
constexpr int kCamMaxStages = 6;
constexpr int kStageBytes = 32 * 1024;       // 16 KB activation panel (128 rows x 64 ch) + 16 KB weight k-block (128 x 64)
constexpr int kHPad = 8;                     // zero rows in front of t = 0 (>= max dilation; multiple of 8 keeps the swizzle phase)
constexpr int kMaxSeg = 6;
constexpr int kParamFloats = 1024 + 1024 + 128 + 1536 + kMaxSeg * 128 + kMaxSeg * 64 + kMaxSeg * 32;

template <int DT>
__global__ void __launch_bounds__(kCamThreads, 1) ws_cam_dense_kernel(const __grid_constant__ WsCamParams p) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t s_bar[2 * kCamMaxStages + 3];

    const int warp = uniform_warp_idx(), lane = threadIdx.x & 31;
    const int b = blockIdx.x;
    const int nmt = p.nmt, nst = p.nstages;
    // frames of THIS utterance (length-masked batch) or of every utterance; memory extents stay p.T
    const int T = p.lens != nullptr ? max(1, min(p.T, p.lens[b])) : p.T;
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t sH = base;                                          // [2 panels][hrows][128 B] hidden operand buffer
    const uint32_t hpanel = (uint32_t)(p.hrows * 128);
    const uint32_t ring = sH + 2 * hpanel;                             // [nst][32 KB]; phase 2: local-conv weights + out staging
    const uint32_t sWl = ring;                                         // 6 blocks of 32 rows x 128 B
    const uint32_t sOut = ring + 6 * 4096;                             // nmt tiles of 128 rows x 64 B
    const uint32_t sPar = ring + (uint32_t)(nst * kStageBytes);
    float* par = reinterpret_cast<float*>(smem_raw + (sPar - smem_u32(smem_raw)));
    float* s_scale = par;                  // [1024]
    float* s_shift = par + 1024;           // [1024]
    float* s_bias2 = par + 2048;           // [128]
    float* s_scratch = par + 2176;         // [1536] partial sums (two phases)
    float* s_ctx = s_scratch + 1536;       // [kMaxSeg][128]
    float* s_hid = s_ctx + kMaxSeg * 128;  // [kMaxSeg][64]
    float* s_gate = s_hid + kMaxSeg * 64;  // [kMaxSeg][32]
    const uint32_t bar_full = smem_u32(&s_bar[0]);
    const uint32_t bar_empty = smem_u32(&s_bar[kCamMaxStages]);
    const uint32_t bar_acc1 = smem_u32(&s_bar[2 * kCamMaxStages]);       // every 1x1 MMA of the layer has retired
    const uint32_t bar_wl = smem_u32(&s_bar[2 * kCamMaxStages + 1]);
    const uint32_t bar_ldone = smem_u32(&s_bar[2 * kCamMaxStages + 2]);

    // zero the hidden operand buffer once: the pad rows in front of t = 0 and behind the last tile are never written again
    for (int i = threadIdx.x; i < (int)(2 * hpanel / 16); i += blockDim.x)
        asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};" ::"r"(sH + (uint32_t)(i * 16)), "r"(0u) : "memory");
    if (warp == 0 && lane == 0) {
        prefetch_tmap(&p.xmap); prefetch_tmap(&p.omap);
        for (int i = 0; i < nst; ++i) { mbar_init(bar_full + 8 * i, 1); mbar_init(bar_empty + 8 * i, 2); }
        mbar_init(bar_acc1, 2); mbar_init(bar_wl, 1); mbar_init(bar_ldone, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();

    if (warp == 0) {
        // ================================ TMA producer ================================
        if (lane == 0) {
            int s = 0;
            uint32_t ph = 1;                                    // empty-barrier parity of the current pass over the ring
            for (int l = p.l0; l < p.l1; ++l) {
                const WsCamLayer* L = p.layers + l;
                const uint32_t lph = (uint32_t)(l - p.l0) & 1u;
                // the previous layer's 32 channels are in global memory and the ring (its phase-2 tenant) is idle again
                if (l > p.l0) mbar_wait(bar_ldone, lph ^ 1u);
                const int npan = (L->cin + 63) >> 6;
                for (int tile = 0; tile < nmt; ++tile)
                    for (int kp = 0; kp < npan; ++kp) {
                        mbar_wait(bar_empty + 8 * s, ph);
                        mbar_expect_tx(bar_full + 8 * s, (uint32_t)kStageBytes);
                        const uint32_t dst = ring + (uint32_t)(s * kStageBytes);
                        tma_load_3d(dst, &p.xmap, bar_full + 8 * s, kp * 64, tile * 128, b);
                        tma_load_2d(dst + 16384u, &L->w1map, bar_full + 8 * s, kp * 64, 0);
                        if (++s == nst) { s = 0; ph ^= 1u; }
                    }
                // phase 2: the local-conv weights take over the front of the ring once every 1x1 MMA has retired
                mbar_wait(bar_acc1, lph);
                mbar_expect_tx(bar_wl, 6u * 4096u);
                for (int tap = 0; tap < 3; ++tap)
                    for (int k2 = 0; k2 < 2; ++k2)
                        tma_load_2d(sWl + (uint32_t)((tap * 2 + k2) * 4096), &L->wlmap, bar_wl, tap * 128 + k2 * 64, 0);
            }
        }
    } else if (warp >= 4) {
        // ================================ consumers: transform, MMAs, epilogues (256 threads) ================================
        const int wg = (warp - 4) >> 2, et = threadIdx.x - 128;
        const int rw = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // first of this thread's two rows of a tile (+8)
        const int cq = (lane & 3) * 2;                            // first column of its pair inside an 8-column group
        const int seg_len = p.seg_len, nseg = (T + seg_len - 1) / seg_len;
        int s = 0;
        uint32_t ph = 0;
        for (int l = p.l0; l < p.l1; ++l) {
            const WsCamLayer* L = p.layers + l;
            const uint32_t lph = (uint32_t)(l - p.l0) & 1u;
            const int cin = L->cin, npan = (cin + 63) >> 6, dil = L->dil;
            for (int c = et; c < npan * 64; c += 256) {
                s_scale[c] = c < cin ? __ldg(L->bn1_scale + c) : 0.f;
                s_shift[c] = c < cin ? __ldg(L->bn1_shift + c) : 0.f;
            }
            if (et < 128) s_bias2[et] = __ldg(L->bias2 + et);
            epi_bar_sync();
            for (int tile = 0; tile < nmt; ++tile) {
                float acc[64];
                for (int kp = 0; kp < npan; ++kp) {
                    mbar_wait(bar_full + 8 * s, ph);
                    // ---- BN1 + ReLU in place on the operand panel (16-byte chunk = 8 channels; physical chunk pc of row r
                    //      holds logical chunk pc ^ (r & 7) under the 128-byte swizzle)
                    const uint32_t pa = ring + (uint32_t)(s * kStageBytes);
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const int idx = et + 256 * i, row = idx >> 3, pc = idx & 7;
                        const int ch0 = kp * 64 + ((pc ^ (row & 7)) << 3);
                        const uint32_t a = pa + (uint32_t)(row * 128 + pc * 16);
                        uint4 x = make_uint4(0u, 0u, 0u, 0u);
                        if (ch0 < cin) {          // channels past cin belong to later layers: whatever is there must not leak in
                            asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(x.x), "=r"(x.y), "=r"(x.z), "=r"(x.w) : "r"(a));
                            float v[8];
                            ws_unpack8(x, DT, v);
                            const float4 s0 = *reinterpret_cast<const float4*>(s_scale + ch0), s1 = *reinterpret_cast<const float4*>(s_scale + ch0 + 4);
                            const float4 h0 = *reinterpret_cast<const float4*>(s_shift + ch0), h1 = *reinterpret_cast<const float4*>(s_shift + ch0 + 4);
                            v[0] = fmaxf(fmaf(v[0], s0.x, h0.x), 0.f); v[1] = fmaxf(fmaf(v[1], s0.y, h0.y), 0.f);
                            v[2] = fmaxf(fmaf(v[2], s0.z, h0.z), 0.f); v[3] = fmaxf(fmaf(v[3], s0.w, h0.w), 0.f);
                            v[4] = fmaxf(fmaf(v[4], s1.x, h1.x), 0.f); v[5] = fmaxf(fmaf(v[5], s1.y, h1.y), 0.f);
                            v[6] = fmaxf(fmaf(v[6], s1.z, h1.z), 0.f); v[7] = fmaxf(fmaf(v[7], s1.w, h1.w), 0.f);
                            x.x = ws_pack2(v[0], v[1], DT); x.y = ws_pack2(v[2], v[3], DT);
                            x.z = ws_pack2(v[4], v[5], DT); x.w = ws_pack2(v[6], v[7], DT);
                        }
                        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(x.x), "r"(x.y), "r"(x.z), "r"(x.w) : "memory");
                    }
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    epi_bar_sync();
                    const uint64_t ad = ws_wg::desc(pa + (uint32_t)(wg * 64 * 128), 128), bd = ws_wg::desc(pa + 16384u, 128);
                    ws_wg::fence();
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        ws_wg::mma<128>(DT, acc, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (uint32_t)((kp | k) != 0));
                    ws_wg::commit();
                    ws_wg::wait<0>();
                    ws_wg::fence_regs<64>(acc);
                    if ((threadIdx.x & 127) == 0) mbar_arrive(bar_empty + 8 * s);
                    if (++s == nst) { s = 0; ph ^= 1u; }
                }
                // ---- epilogue 1: h = ReLU(acc + bias2) -> hidden operand buffer (rows past T stay zero: conv padding)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int t = tile * 128 + rw + 8 * h, row = kHPad + t;
#pragma unroll
                    for (int jg = 0; jg < 16; ++jg) {
                        const int c = 8 * jg + cq;
                        const float v0 = t < T ? fmaxf(acc[4 * jg + 2 * h] + s_bias2[c], 0.f) : 0.f;
                        const float v1 = t < T ? fmaxf(acc[4 * jg + 2 * h + 1] + s_bias2[c + 1], 0.f) : 0.f;
                        const uint32_t a = sH + (uint32_t)(c >> 6) * hpanel + (uint32_t)(row * 128) +
                                           (uint32_t)(((((c & 63) >> 3) ^ (row & 7)) << 4) + (c & 7) * 2);
                        asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(ws_pack2(v0, v1, DT)) : "memory");
                    }
                }
            }
            if ((threadIdx.x & 127) == 0) mbar_arrive(bar_acc1);   // the ring front may take the local-conv weights
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            epi_bar_sync();
            // ---- context: per-segment column sums of the STORED (rounded) h, like the unfused gate kernel reads them.
            //      thread = (16-byte chunk of 8 channels, 1 of 16 row groups); the two row groups of a warp are combined by a
            //      shuffle, the 8 warps through shared memory: deterministic summation order.
            {
                const int cc16 = et & 15, rg = et >> 4;                 // chunk column (panel = cc16 >> 3), row group
                const uint32_t pb = sH + (uint32_t)(cc16 >> 3) * hpanel;
                const int lc = cc16 & 7;
                float tot8[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                for (int sg = 0; sg < nseg; ++sg) {
                    const int ta = sg * seg_len, tb = min(T, ta + seg_len);
                    float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                    for (int t = ta + rg; t < tb; t += 16) {
                        const int row = kHPad + t;
                        uint4 x;
                        asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(x.x), "=r"(x.y), "=r"(x.z), "=r"(x.w)
                                     : "r"(pb + (uint32_t)(row * 128 + ((lc ^ (row & 7)) << 4))));
                        float v[8];
                        ws_unpack8(x, DT, v);
#pragma unroll
                        for (int k = 0; k < 8; ++k) a[k] += v[k];
                    }
#pragma unroll
                    for (int k = 0; k < 8; ++k) a[k] += __shfl_xor_sync(0xffffffffu, a[k], 16);
                    if ((et & 16) == 0) {
#pragma unroll
                        for (int k = 0; k < 8; ++k) s_scratch[(warp - 4) * 128 + cc16 * 8 + k] = a[k];
                    }
                    epi_bar_sync();
                    if (et < 128) {
                        float t_ = 0.f;
#pragma unroll
                        for (int w = 0; w < 8; ++w) t_ += s_scratch[w * 128 + et];
                        s_ctx[sg * 128 + et] = t_;       // segment sum for now
                    }
                    epi_bar_sync();
                }
                (void)tot8;
            }
            if (et < 128) {
                float tot = 0.f;
                for (int sg = 0; sg < nseg; ++sg) tot += s_ctx[sg * 128 + et];
                tot /= (float)T;
                for (int sg = 0; sg < nseg; ++sg) {
                    const int cnt = min(T, (sg + 1) * seg_len) - sg * seg_len;    // ceil_mode partial window: its own count
                    s_ctx[sg * 128 + et] = s_ctx[sg * 128 + et] / (float)cnt + tot;
                }
            }
            epi_bar_sync();
            {   // hidden = ReLU(W1 ctx + b1): thread = (output j, quarter of the 128 inputs); W1 transposed -> coalesced; all
                // 32 weight loads of a thread are in flight at once (they are L2 hits, ~700 cycles each if serialised)
                const int j = et & 63, qt = et >> 6;
                const float* w = L->w1c_t + (size_t)(qt * 32) * 64 + j;
                float wv[32];
#pragma unroll
                for (int c = 0; c < 32; ++c) wv[c] = __ldg(w + (size_t)c * 64);
                for (int sg = 0; sg < nseg; ++sg) {
                    float a = 0.f;
#pragma unroll
                    for (int c = 0; c < 32; ++c) a = fmaf(wv[c], s_ctx[sg * 128 + qt * 32 + c], a);
                    s_scratch[(qt * kMaxSeg + sg) * 64 + j] = a;
                }
            }
            // gate weights of this thread (8 of the 64 inputs of output g) are fetched before the barrier
            const int gg = et & 31, gp = et >> 5;
            float w2v[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) w2v[i] = __ldg(L->w2c_t + (gp * 8 + i) * 32 + gg);
            const float b2v = __ldg(L->b2c + gg);
            epi_bar_sync();
            for (int o = et; o < nseg * 64; o += 256) {
                const int sg = o >> 6, j = o & 63;
                float a = __ldg(L->b1c + j);
#pragma unroll
                for (int qt = 0; qt < 4; ++qt) a += s_scratch[(qt * kMaxSeg + sg) * 64 + j];
                s_hid[sg * 64 + j] = fmaxf(a, 0.f);
            }
            epi_bar_sync();
            for (int sg = 0; sg < nseg; ++sg) {     // gate partials: thread = (output g, eighth of the 64 hidden units)
                float a = 0.f;
#pragma unroll
                for (int i = 0; i < 8; ++i) a = fmaf(w2v[i], s_hid[sg * 64 + gp * 8 + i], a);
                s_scratch[(gp * kMaxSeg + sg) * 32 + gg] = a;
            }
            epi_bar_sync();
            for (int o = et; o < nseg * 32; o += 256) {
                const int sg = o >> 5, g = o & 31;
                float a = b2v;                       // (o & 31) == (et & 31): this thread's own bias
#pragma unroll
                for (int k = 0; k < 8; ++k) a += s_scratch[(k * kMaxSeg + sg) * 32 + g];
                s_gate[sg * 32 + g] = 1.f / (1.f + expf(-a));
            }
            epi_bar_sync();
            // ---- local conv: 3 dilated taps as row-shifted reads of the hidden operand buffer, K = 128 (2 panels), N = 32;
            //      epilogue 2: y = local_conv(h) * gate[segment(t)] -> 64-byte-row staging -> TMA store (clips rows >= T)
            mbar_wait(bar_wl, lph);
            for (int tile = 0; tile < nmt; ++tile) {
                float acc2[16];
                ws_wg::fence();
#pragma unroll 1
                for (int tap = 0; tap < 3; ++tap) {
                    const int row = kHPad + tile * 128 + wg * 64 + (tap - 1) * dil;
#pragma unroll
                    for (int k2 = 0; k2 < 2; ++k2) {
                        const uint64_t ad = ws_wg::desc(sH + (uint32_t)k2 * hpanel + (uint32_t)(row * 128), 128);
                        const uint64_t bd = ws_wg::desc(sWl + (uint32_t)((tap * 2 + k2) * 4096), 128);
#pragma unroll
                        for (int k = 0; k < 4; ++k)
                            ws_wg::mma<32>(DT, acc2, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (uint32_t)((tap | k2 | k) != 0));
                    }
                }
                ws_wg::commit();
                ws_wg::wait<0>();
                ws_wg::fence_regs<16>(acc2);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int r = rw + 8 * h, t = tile * 128 + r;
                    const float* g = s_gate + min(t / seg_len, nseg - 1) * 32;
#pragma unroll
                    for (int jg = 0; jg < 4; ++jg) {
                        const int c = 8 * jg + cq;
                        const uint32_t a = sOut + (uint32_t)(tile * 8192 + r * 64) + (uint32_t)((swz_chunk(c >> 3, r, 64) << 4) + (c & 7) * 2);
                        asm volatile("st.shared.b32 [%0], %1;" ::"r"(a),
                                     "r"(ws_pack2(acc2[4 * jg + 2 * h] * g[c], acc2[4 * jg + 2 * h + 1] * g[c + 1], DT)) : "memory");
                    }
                }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            epi_bar_sync();
            if (et == 0) {
                for (int tile = 0; tile < nmt; ++tile) tma_store_3d(&p.omap, sOut + (uint32_t)(tile * 8192), cin, tile * 128, b);
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // writes complete: the next layer may load them
                mbar_arrive(bar_ldone);
            }
        }
    }
}

// shared-memory bytes the kernel needs for (nmt tiles, nstages ring stages)
constexpr int cam_smem(int nmt, int nstages) { return 2 * (16 + 128 * nmt) * 128 + nstages * kStageBytes + kParamFloats * 4 + 2048; }
static_assert(cam_smem(4, 2) <= kCamMaxSmem, "the longest utterance (4 M tiles) must fit with the shortest ring");

template <int DT>
const char* cam_go(const WsCamParams* p, cudaStream_t s) {
    if (const char* m = ws_smem_opt_in<ws_cam_dense_kernel<DT>>(kCamMaxSmem)) return m;
    ws_cam_dense_kernel<DT><<<p->grid, kCamThreads, p->smem_bytes, s>>>(*p);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace

// cam_smem, or 0 if the geometry is not supported
extern "C" int ws_cam_smem_bytes(int nmt, int nstages) {
    if (nmt < 1 || nmt > 4 || nstages < 2 || nstages > kCamMaxStages) return 0;
    return cam_smem(nmt, nstages);
}

extern "C" const char* ws_cam_launch(const WsCamParams* p, cudaStream_t s) {
    if (p->dtype == WS_BF16) return cam_go<WS_BF16>(p, s);
    if (p->dtype == WS_F16) return cam_go<WS_F16>(p, s);
    return "cam_dense: 16-bit activations only";
}
