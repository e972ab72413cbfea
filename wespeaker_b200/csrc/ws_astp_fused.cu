// ASTP tail in one launch: attention logits + softmax over time + weighted mean / std (pooling_layers.py:119-144,
//   alpha = softmax(linear2(tanh(linear1(x))), dim=T);  mean = sum alpha x;  std = sqrt(clamp(sum alpha x^2 - mean^2, var_floor)),
//   var_floor 1e-7; SimAM-ResNet's ASP, pooling_layers.py:188-204, is the same tail with a ReLU -> BN hidden layer and 1e-5).
// linear1 (+tanh) stays a conv-GEMM launch that leaves H [B][T][128]; this kernel replaces the linear2 launch (which wrote
// the [B][T][C] logits, 157 MB at B = 256) and the statistics launch (which read them back together with x):
//
//   * the logits tile is computed TRANSPOSED: D[channel, t] = W2[channel, :] . H[t, :]  (A = a 128-channel block of W2,
//     B = 64 frames of the utterance's H rows), so an accumulator row is a channel and its columns are time: each thread
//     runs the softmax over time and the weighted sums over the frames it holds of its two channels, and the four threads
//     sharing a channel merge their partial statistics once per block; the logits never leave the SM (they also stay
//     fp32 instead of being rounded to 16 bits);
//   * linear2's bias is constant over time and cancels in the softmax: it is not applied;
//   * utterances longer than 256 frames run as chunks with an online (running-max) softmax, so any T works;
//   * a work unit is (utterance, g consecutive channel blocks): H is fetched once per unit and reused for its g blocks;
//   * x reaches the statistics through a TMA ring of [128 frames x 128 channels] tiles in shared memory (un-swizzled, so
//     thread reads its (frame, channel) elements from shared memory instead of with 2-byte global loads.
//
// Warp roles (384 threads): w0 TMA producer (H chunks, W2 blocks, x tiles), w1..w3 idle, w4..w11 two consumer warpgroups;
// warpgroup wg computes (wgmma) and reduces the logits of channels [64 wg, 64 wg + 64) of every block.
#include "ws_tc_common.cuh"

namespace {
using namespace ws_tcdev;

constexpr int kThreadsA = 384;
constexpr int kHPanelBytes = 256 * 128;   // one K panel (64 of the 128 hidden units) of a 256-frame H chunk
constexpr int kWPanelBytes = 128 * 128;   // one K panel of a 128-channel W2 block
constexpr int kXTileBytes = 128 * 256;   // 128 frames x 128 channels of x, row pitch 256 B, no swizzle
constexpr int kXSlots = 3;
constexpr int kSmemA = 2 * kHPanelBytes + 2 * 2 * kWPanelBytes + kXSlots * kXTileBytes + 1024;   // H chunk + two W2 blocks + x ring

__device__ __forceinline__ float ex2f(float v) {
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v));
    return r;
}
template <int DT>
__device__ __forceinline__ float cvt16(uint32_t v) {
    if (DT == WS_BF16) return __uint_as_float(v << 16);
    return __half2float(__ushort_as_half((unsigned short)v));
}

template <int DT>
__global__ void __launch_bounds__(kThreadsA, 1) ws_astp_fused_kernel(const __grid_constant__ WsAstpParams p) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t s_bar[6 + 2 * kXSlots];
    const int warp = uniform_warp_idx(), lane = threadIdx.x & 31;
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t hbuf = base, wbuf = base + 2u * kHPanelBytes, xbuf = wbuf + 4u * kWPanelBytes;
    const uint32_t bar_hfull = smem_u32(&s_bar[0]), bar_hempty = smem_u32(&s_bar[1]);
    const uint32_t bar_wfull = smem_u32(&s_bar[2]), bar_wempty = smem_u32(&s_bar[4]);     // [2] each
    const uint32_t bar_xfull = smem_u32(&s_bar[6]), bar_xempty = smem_u32(&s_bar[6 + kXSlots]);   // [kXSlots] each

    if (warp == 0 && lane == 0) {
        prefetch_tmap(&p.hmap); prefetch_tmap(&p.wmap); prefetch_tmap(&p.xmap);
        // H and W2 are released by both consumer warpgroups, the x tiles by all 8 consumer warps
        mbar_init(bar_hfull, 1); mbar_init(bar_hempty, 2);
        for (int i = 0; i < kXSlots; ++i) { mbar_init(bar_xfull + 8 * i, 1); mbar_init(bar_xempty + 8 * i, 8); }
        for (int i = 0; i < 2; ++i) { mbar_init(bar_wfull + 8 * i, 1); mbar_init(bar_wempty + 8 * i, 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int nblk = p.C / 128, upb = nblk / p.g, nunits = p.B * upb;

    if (warp == 0) {
        // ================================ TMA producer ================================
        if (lane == 0) {
            uint32_t h_it = 0, w_it = 0, x_it = 0;
            for (int u = blockIdx.x; u < nunits; u += gridDim.x) {
                const int b = u / upb, blk0 = (u % upb) * p.g;
                const int Tb = p.lens ? max(1, min(p.T, p.lens[b])) : p.T;
                const int nch = (Tb + 255) >> 8;
                auto load_h = [&](int ch) {
                    mbar_wait(bar_hempty, (h_it & 1u) ^ 1u);
                    mbar_expect_tx(bar_hfull, 2u * kHPanelBytes);
                    tma_load_3d(hbuf, &p.hmap, bar_hfull, 0, ch * 256, b);
                    tma_load_3d(hbuf + kHPanelBytes, &p.hmap, bar_hfull, 64, ch * 256, b);
                    ++h_it;
                };
                if (nch == 1) load_h(0);
                for (int j = 0; j < p.g; ++j) {
                    for (int ch = 0; ch < nch; ++ch) {
                        if (nch > 1) load_h(ch);
                        if (ch == 0) {
                            const uint32_t ws = w_it & 1u;
                            mbar_wait(bar_wempty + 8 * ws, ((w_it >> 1) & 1u) ^ 1u);
                            mbar_expect_tx(bar_wfull + 8 * ws, 2u * kWPanelBytes);
                            const uint32_t dst = wbuf + ws * 2u * kWPanelBytes;
                            tma_load_2d(dst, &p.wmap, bar_wfull + 8 * ws, 0, (blk0 + j) * 128);
                            tma_load_2d(dst + kWPanelBytes, &p.wmap, bar_wfull + 8 * ws, 64, (blk0 + j) * 128);
                            ++w_it;
                        }
                        // x tiles of this (block, chunk): 128 frames x 128 channels each, in the order the epilogue consumes them
                        const int rows = min(256, Tb - ch * 256);
                        for (int hf = 0; hf * 128 < rows; ++hf, ++x_it) {
                            const uint32_t xs = x_it % kXSlots;
                            mbar_wait(bar_xempty + 8 * xs, ((x_it / kXSlots) & 1u) ^ 1u);
                            mbar_expect_tx(bar_xfull + 8 * xs, (uint32_t)kXTileBytes);
                            tma_load_3d(xbuf + xs * kXTileBytes, &p.xmap, bar_xfull + 8 * xs, (blk0 + j) * 128, ch * 256 + hf * 128, b);
                        }
                    }
                }
            }
        }
    } else if (warp >= 4) {
        // ================================ consumers: logits (wgmma) + per-channel online softmax statistics ================================
        const int wg = (warp - 4) >> 2;
        const int cr = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's channels in the block: cr, cr + 8
        const int cq = (lane & 3) * 2;                            // its frames in an 8-frame group: cq, cq + 1
        const float kLog2e = 1.4426950408889634f;
        uint32_t h_it = 0, w_it = 0, x_it = 0;
        for (int u = blockIdx.x; u < nunits; u += gridDim.x) {
            const int b = u / upb, blk0 = (u % upb) * p.g;
            const int Tb = p.lens ? max(1, min(p.T, p.lens[b])) : p.T;
            const int nch = (Tb + 255) >> 8;
            if (nch == 1) { mbar_wait(bar_hfull, h_it & 1u); ++h_it; }
            for (int j = 0; j < p.g; ++j) {
                const uint32_t ws = w_it & 1u;
                float m[2] = {-INFINITY, -INFINITY}, s0[2] = {0.f, 0.f}, s1[2] = {0.f, 0.f}, s2[2] = {0.f, 0.f};
                for (int ch = 0; ch < nch; ++ch) {
                    if (nch > 1) { mbar_wait(bar_hfull, h_it & 1u); ++h_it; }
                    if (ch == 0) mbar_wait(bar_wfull + 8 * ws, (w_it >> 1) & 1u);
                    const int rows = min(256, Tb - ch * 256);
                    const uint32_t wa = wbuf + ws * 2u * kWPanelBytes + (uint32_t)(wg * 64 * 128);
                    const uint64_t a0 = ws_wg::desc(wa, 128), a1 = ws_wg::desc(wa + kWPanelBytes, 128);
                    for (int hf = 0; hf * 128 < rows; ++hf, ++x_it) {
                        const uint32_t xs = x_it % kXSlots;
                        mbar_wait(bar_xfull + 8 * xs, (x_it / kXSlots) & 1u);
                        const uint32_t xt = xbuf + xs * kXTileBytes;
#pragma unroll 1
                        for (int f0 = hf * 128; f0 < min(rows, hf * 128 + 128); f0 += 64) {
                            float acc[32];
                            const uint64_t b0 = ws_wg::desc(hbuf + (uint32_t)(f0 * 128), 128);
                            const uint64_t b1 = ws_wg::desc(hbuf + kHPanelBytes + (uint32_t)(f0 * 128), 128);
                            ws_wg::fence();
#pragma unroll
                            for (int k = 0; k < 4; ++k) ws_wg::mma<64>(DT, acc, a0 + (uint64_t)(2 * k), b0 + (uint64_t)(2 * k), (uint32_t)(k != 0));
#pragma unroll
                            for (int k = 0; k < 4; ++k) ws_wg::mma<64>(DT, acc, a1 + (uint64_t)(2 * k), b1 + (uint64_t)(2 * k), 1u);
                            ws_wg::commit();
                            ws_wg::wait<0>();
                            ws_wg::fence_regs<32>(acc);
                            // frames behind the end get logit -inf (weight 0) and x 0
                            const int nv = rows - f0;
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                float lg[16], xv[16];
#pragma unroll
                                for (int i = 0; i < 16; ++i) {
                                    const int fr = 8 * (i >> 1) + cq + (i & 1);          // frame inside the 64-frame chunk
                                    const bool ok = fr < nv;
                                    uint32_t xr = 0u;
                                    if (ok) asm volatile("ld.shared.u16 %0, [%1];" : "=r"(xr)
                                                         : "r"(xt + (uint32_t)((f0 - hf * 128 + fr) * 256 + (cr + 8 * h) * 2)));
                                    lg[i] = ok ? acc[4 * (i >> 1) + 2 * h + (i & 1)] : -INFINITY;
                                    xv[i] = cvt16<DT>(xr);
                                }
                                float gm = -INFINITY;
#pragma unroll
                                for (int i = 0; i < 16; ++i) gm = fmaxf(gm, lg[i]);
                                if (gm == -INFINITY) continue;                   // none of this thread's frames is valid
                                const float mn = fmaxf(m[h], gm);
                                const float sc = ex2f((m[h] - mn) * kLog2e);     // m = -inf on the first group: ex2(-inf) = 0
                                m[h] = mn;
                                const float moff = -mn * kLog2e;
                                float a0s = 0.f, a1s = 0.f, a2s = 0.f;
#pragma unroll
                                for (int i = 0; i < 16; ++i) {
                                    const float e = ex2f(fmaf(lg[i], kLog2e, moff));
                                    const float ex = e * xv[i];
                                    a0s += e;
                                    a1s += ex;
                                    a2s = fmaf(ex, xv[i], a2s);
                                }
                                s0[h] = fmaf(s0[h], sc, a0s);
                                s1[h] = fmaf(s1[h], sc, a1s);
                                s2[h] = fmaf(s2[h], sc, a2s);
                            }
                        }
                        __syncwarp();
                        if (lane == 0) mbar_arrive(bar_xempty + 8 * xs);
                    }
                    if (nch > 1 && (threadIdx.x & 127) == 0) mbar_arrive(bar_hempty);
                }
                if ((threadIdx.x & 127) == 0) mbar_arrive(bar_wempty + 8 * ws);
                ++w_it;
                // the four threads holding a channel merge their partial statistics
#pragma unroll
                for (int h = 0; h < 2; ++h) {
#pragma unroll
                    for (int o = 1; o <= 2; o <<= 1) {
                        const float mo = __shfl_xor_sync(0xffffffffu, m[h], o);
                        const float t0 = __shfl_xor_sync(0xffffffffu, s0[h], o);
                        const float t1 = __shfl_xor_sync(0xffffffffu, s1[h], o);
                        const float t2 = __shfl_xor_sync(0xffffffffu, s2[h], o);
                        const float mn = fmaxf(m[h], mo);
                        const float ca = m[h] == -INFINITY ? 0.f : ex2f((m[h] - mn) * kLog2e);
                        const float cb = mo == -INFINITY ? 0.f : ex2f((mo - mn) * kLog2e);
                        s0[h] = s0[h] * ca + t0 * cb;
                        s1[h] = s1[h] * ca + t1 * cb;
                        s2[h] = s2[h] * ca + t2 * cb;
                        m[h] = mn;
                    }
                    if ((lane & 3) == 0) {
                        const int c = (blk0 + j) * 128 + cr + 8 * h;
                        const float mean = s1[h] / s0[h];
                        const float var = s2[h] / s0[h] - mean * mean;
                        p.out[(long long)b * 2 * p.C + c] = mean;
                        p.out[(long long)b * 2 * p.C + p.C + c] = sqrtf(var < p.var_floor ? p.var_floor : var);   // torch clamp: NaN stays NaN
                    }
                }
            }
            if (nch == 1 && (threadIdx.x & 127) == 0) mbar_arrive(bar_hempty);
        }
    }
}

template <int DT>
const char* astp_go(const WsAstpParams* p, cudaStream_t s) {
    if (const char* m = ws_smem_opt_in<ws_astp_fused_kernel<DT>>(kSmemA)) return m;
    ws_astp_fused_kernel<DT><<<p->grid, kThreadsA, kSmemA, s>>>(*p);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

}  // namespace

extern "C" const char* ws_astp_launch(const WsAstpParams* p, cudaStream_t s) {
    if (p->dtype == WS_BF16) return astp_go<WS_BF16>(p, s);
    if (p->dtype == WS_F16) return astp_go<WS_F16>(p, s);
    return "ws_astp_launch: 16-bit activations only";
}
