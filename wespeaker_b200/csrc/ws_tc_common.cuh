// Device-side building blocks shared by the persistent wgmma kernels (ws_gemm_tc2.cu and the fused conv / pooling
// kernels): mbarrier / TMA wrappers, the swizzled staging helpers and the fused GEMM epilogue (one 32-column chunk of one
// accumulator row per call).  Everything is __forceinline__.
#pragma once
#include "ws_common.cuh"
#include "ws_wgmma.cuh"

namespace ws_tcdev {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(bar), "r"(parity)
            : "memory");
    } while (!done);
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1,
                                            int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, "
        "%6}], [%2];" ::"r"(dst),
        "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::
            "r"(dst),
        "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::
            "r"(dst),
        "l"(map), "r"(bar), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(map),
                 "r"(src), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(map),
                 "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
                 : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
// Warp index through a shuffle: the compiler then treats the role branches as warp-uniform.
__device__ __forceinline__ int uniform_warp_idx() { return __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0); }
// 16-byte chunk index after the TMA / wgmma swizzle for a row of `row_bytes` (128/64/32) inside a 1024-B aligned panel
__device__ __forceinline__ int swz_chunk(int chunk, int row, int row_bytes) {
    return row_bytes == 128 ? (chunk ^ (row & 7)) : (row_bytes == 64 ? (chunk ^ ((row >> 1) & 3)) : (chunk ^ ((row >> 2) & 1)));
}

// 32 consecutive fp32 values -> packed activation dtype -> swizzled staging panel row
__device__ __forceinline__ void stage_store32(uint32_t panel_base, int row, int row_bytes, int col_in_panel, int dt,
                                              const float* v) {
    const uint32_t rbase = panel_base + (uint32_t)(row * row_bytes);
    if (dt == WS_F32) {
        const int c0 = (col_in_panel * 4) >> 4;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const uint32_t a = rbase + (uint32_t)(swz_chunk(c0 + i, row, row_bytes) << 4);
            asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(a), "f"(v[4 * i]), "f"(v[4 * i + 1]),
                         "f"(v[4 * i + 2]), "f"(v[4 * i + 3])
                         : "memory");
        }
    } else {
        const int c0 = (col_in_panel * 2) >> 4;
        const bool bf = dt == WS_BF16;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            uint32_t w[4];
#pragma unroll
            for (int j = 0; j < 4; ++j)
                w[j] = bf ? ws_pack2(v[8 * i + 2 * j], v[8 * i + 2 * j + 1], WS_BF16)
                          : ws_pack2(v[8 * i + 2 * j], v[8 * i + 2 * j + 1], WS_F16);
            const uint32_t a = rbase + (uint32_t)(swz_chunk(c0 + i, row, row_bytes) << 4);
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(w[0]), "r"(w[1]), "r"(w[2]), "r"(w[3])
                         : "memory");
        }
    }
}
// inverse: read 32 consecutive values of a TMA-loaded swizzled panel row
__device__ __forceinline__ void stage_load32(uint32_t panel_base, int row, int row_bytes, int col_in_panel, int dt,
                                             float* v) {
    const uint32_t rbase = panel_base + (uint32_t)(row * row_bytes);
    if (dt == WS_F32) {
        const int c0 = (col_in_panel * 4) >> 4;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const uint32_t a = rbase + (uint32_t)(swz_chunk(c0 + i, row, row_bytes) << 4);
            asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                         : "=f"(v[4 * i]), "=f"(v[4 * i + 1]), "=f"(v[4 * i + 2]), "=f"(v[4 * i + 3])
                         : "r"(a));
        }
    } else {
        const int c0 = (col_in_panel * 2) >> 4;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            uint32_t w[4];
            const uint32_t a = rbase + (uint32_t)(swz_chunk(c0 + i, row, row_bytes) << 4);
            asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]) : "r"(a));
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                v[8 * i + 2 * j] = ws_16_to_f(w[j] & 0xffffu, dt);
                v[8 * i + 2 * j + 1] = ws_16_to_f(w[j] >> 16, dt);
            }
        }
    }
}

// per-tile epilogue context of one thread (row r of the 128-row tile)
struct EpiTile {
    const float* spar;             // staged per-channel bias / scale / shift: 3 x bn floats
    uint32_t stg_in, stg_out;      // smem staging: epilogue-input tile, output tile(s)
    int tile_out_bytes, panel_bytes, panel_cols;
    int n0, r;                     // first output channel of the tile, row inside the tile
    bool valid;                    // the row maps to an existing output position
    int eb, etm;                   // utterance / frame of the row (row-bias and gate lookups)
};

// stage bias / BN scale / BN shift of channels [n0, n0 + bn) into spar (the 256 epilogue threads, et = 0..255)
__device__ __forceinline__ void epi_stage_params(const WsTc2Params& p, float* spar, int n0, int et) {
    const WsEpi& e = p.epi;
    for (int c = et; c < p.bn; c += 256) {
        // all three loads are issued before the first store: interleaved load/store pairs were serialised by
        // the compiler (possible aliasing) and cost three L2 round trips per tile on the epilogue's critical path
        const float pb = e.bias ? __ldg(e.bias + n0 + c) : 0.f;
        const float ps = e.scale ? __ldg(e.scale + n0 + c) : 1.f;
        const float ph = e.scale ? __ldg(e.shift + n0 + c) : 0.f;
        spar[c] = pb;
        spar[p.bn + c] = ps;
        spar[2 * p.bn + c] = ph;
    }
}

// tanh for 16-bit outputs: tanh(x) = 1 - 2 / (e^{2x} + 1) on ex2.approx + rcp.approx (abs error ~1e-7, far below the
// output rounding), 5 instructions per element instead of the ~25 of tanhf
__device__ __forceinline__ float tanh16(float x) {
    float ex;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(ex) : "f"(x * 2.885390081777927f));
    return 1.f - __fdividef(2.f, ex + 1.f);
}

// LEAN != 0 (= WsDType of the activations + 1) compiles only the common epilogue: bias, ReLU, BN scale/shift, residual
// tile, ReLU, one output (+ its 3xTF32 low twin for fp32).  The generic epilogue (row bias, gates, Res2 second output,
// tanh/sigmoid, every dtype) is ~100 KB of SASS of which a given layer executes a few KB scattered between never-taken
// branches: its warps stall on instruction fetch, which makes the short-K 1x1 convs epilogue-bound.  The lean chunk body
// is ~4 KB and stays in the L0 instruction cache.
template <int LEAN>
__device__ __forceinline__ void epi_chunk(const WsTc2Params& p, const EpiTile& x, const uint32_t* raw, const int c) {
    const WsEpi& e = p.epi;
    float v[32];
    if constexpr (LEAN != 0) {
        constexpr int DT = LEAN - 1;                          // activation dtype of this instantiation
        // staging panels: 128-byte rows (32 fp32 / 64 16-bit columns), or 64-byte rows for 32-channel 16-bit tiles (bn = 32)
        const int PB = x.panel_bytes, PCOLS = x.panel_cols;
        const float4* sb = reinterpret_cast<const float4*>(x.spar + c);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float4 x = sb[i];
            v[4 * i] = __uint_as_float(raw[4 * i]) + x.x; v[4 * i + 1] = __uint_as_float(raw[4 * i + 1]) + x.y;
            v[4 * i + 2] = __uint_as_float(raw[4 * i + 2]) + x.z; v[4 * i + 3] = __uint_as_float(raw[4 * i + 3]) + x.w;
        }
        if (e.rowbias != nullptr && x.valid) {   // per-utterance bias row (ECAPA global-context attention)
            const float4* rb = reinterpret_cast<const float4*>(e.rowbias + (long long)x.eb * e.rowbias_ld + x.n0 + c);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float4 x = __ldg(rb + i);
                v[4 * i] += x.x; v[4 * i + 1] += x.y; v[4 * i + 2] += x.z; v[4 * i + 3] += x.w;
            }
        }
        if (e.act1 == WS_ACT_RELU) {
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] = fmaxf(v[i], 0.f);
        } else if (e.act1 == WS_ACT_TANH) {
            if constexpr (DT == WS_F32) {
                ws_act_vec<32>(v, WS_ACT_TANH);
            } else {
#pragma unroll
                for (int i = 0; i < 32; ++i) v[i] = tanh16(v[i]);
            }
        }
        if (e.scale != nullptr) {
            const float4* ss = reinterpret_cast<const float4*>(x.spar + p.bn + c);
            const float4* sh = reinterpret_cast<const float4*>(x.spar + 2 * p.bn + c);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float4 a = ss[i], d = sh[i];
                v[4 * i] = fmaf(v[4 * i], a.x, d.x); v[4 * i + 1] = fmaf(v[4 * i + 1], a.y, d.y);
                v[4 * i + 2] = fmaf(v[4 * i + 2], a.z, d.z); v[4 * i + 3] = fmaf(v[4 * i + 3], a.w, d.w);
            }
        }
        const uint32_t poff = (uint32_t)((c / PCOLS) * 128 * PB);
        if (p.has_epin) {  // residual
            float rin[32];
            stage_load32(x.stg_in + poff, x.r, PB, c % PCOLS, DT, rin);
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] += rin[i];
        }
        if (e.act2 == WS_ACT_RELU) {
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] = fmaxf(v[i], 0.f);
        }
        stage_store32(x.stg_out + poff, x.r, PB, c % PCOLS, DT, v);
        if constexpr (DT == WS_F32) {
            if (p.nsplit == 3) {  // 3xTF32: the low twin of the output feeds the next layer's x_lo pass
#pragma unroll
                for (int i = 0; i < 32; ++i) v[i] = ws_tf32_lo(v[i]);
                stage_store32(x.stg_out + (uint32_t)x.tile_out_bytes + poff, x.r, PB, c % PCOLS, DT, v);
            }
        }
        return;
    }
    {
        const float4* sb = reinterpret_cast<const float4*>(x.spar + c);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float4 x = sb[i];
            v[4 * i] = __uint_as_float(raw[4 * i]) + x.x; v[4 * i + 1] = __uint_as_float(raw[4 * i + 1]) + x.y;
            v[4 * i + 2] = __uint_as_float(raw[4 * i + 2]) + x.z; v[4 * i + 3] = __uint_as_float(raw[4 * i + 3]) + x.w;
        }
    }
    if (e.rowbias != nullptr && x.valid) {
        const float4* rb = reinterpret_cast<const float4*>(e.rowbias + (long long)x.eb * e.rowbias_ld + x.n0 + c);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float4 x = __ldg(rb + i);
            v[4 * i] += x.x; v[4 * i + 1] += x.y; v[4 * i + 2] += x.z; v[4 * i + 3] += x.w;
        }
    }
    ws_act_vec<32>(v, e.act1);
    if (e.scale != nullptr) {
        const float4* ss = reinterpret_cast<const float4*>(x.spar + p.bn + c);
        const float4* sh = reinterpret_cast<const float4*>(x.spar + 2 * p.bn + c);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float4 a = ss[i], d = sh[i];
            v[4 * i] = fmaf(v[4 * i], a.x, d.x); v[4 * i + 1] = fmaf(v[4 * i + 1], a.y, d.y);
            v[4 * i + 2] = fmaf(v[4 * i + 2], a.z, d.z); v[4 * i + 3] = fmaf(v[4 * i + 3], a.w, d.w);
        }
    }
    if (e.gate != nullptr && x.valid) {
        const float4* g = reinterpret_cast<const float4*>(
            e.gate + ((long long)x.eb * e.gate_nseg + x.etm / e.gate_seg) * e.gate_ld + x.n0 + c);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float4 x = __ldg(g + i);
            v[4 * i] *= x.x; v[4 * i + 1] *= x.y; v[4 * i + 2] *= x.z; v[4 * i + 3] *= x.w;
        }
    }
    const int pn = c / x.panel_cols, cin = c % x.panel_cols;
    float rin[32];
    if (p.has_epin) stage_load32(x.stg_in + (uint32_t)(pn * 128 * x.panel_bytes), x.r, x.panel_bytes, cin, e.dtype, rin);
    if (p.has_epin && !p.has_out2) {  // residual
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] += rin[i];
    }
    ws_act_vec<32>(v, e.act2);
    const uint32_t poff = (uint32_t)(pn * 128 * x.panel_bytes);
    int ob = 0;
    stage_store32(x.stg_out + poff, x.r, x.panel_bytes, cin, e.dtype, v);
    if (p.has_out2) {  // Res2: next conv's input = this output + the next channel group
#pragma unroll
        for (int i = 0; i < 32; ++i) rin[i] += v[i];
    }
    if (p.nsplit == 3) {
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = ws_tf32_lo(v[i]);
        stage_store32(x.stg_out + (uint32_t)(++ob * x.tile_out_bytes) + poff, x.r, x.panel_bytes, cin, e.dtype, v);
    }
    if (p.has_out2) {
        stage_store32(x.stg_out + (uint32_t)(++ob * x.tile_out_bytes) + poff, x.r, x.panel_bytes, cin, e.dtype, rin);
        if (p.nsplit == 3) {
#pragma unroll
            for (int i = 0; i < 32; ++i) rin[i] = ws_tf32_lo(rin[i]);
            stage_store32(x.stg_out + (uint32_t)(++ob * x.tile_out_bytes) + poff, x.r, x.panel_bytes, cin, e.dtype, rin);
        }
    }
}

// fused SE squeeze (WsEpi::colsum): column sums of the staged (already rounded) tile, read back from the swizzled staging
// panels while the TMA store drains them; thread = (column pair, 64-row half), pairs past the tile's ncols = bn <= 128
// columns idle.  16-bit lean instantiations only (the 256-wide tile sums on its helper warps, ws_gemm_tc2.cu).
template <int LEAN>
__device__ __forceinline__ void epi_colsum(const WsTc2Params& p, uint32_t stg_out, int et, int n0, int ncols, int t0, int b0) {
    const WsEpi& e = p.epi;
    if (e.colsum != nullptr && 2 * (et & 127) < ncols && b0 < p.B && t0 + (et >> 7) * 64 < p.T) {   // units past the last position do not exist
        const int cpair = et & 127, rh = et >> 7;
        const int pos0 = t0 + rh * 64;
        const int nvalid = min(64, p.T - pos0);
        const int split = min(nvalid, (pos0 / e.colsum_T + 1) * e.colsum_T - pos0);
        const int col = 2 * cpair;
        const uint32_t cbase = stg_out + (uint32_t)((col >> 6) * 128 * 128 + (col & 7) * 2);
        const int chunk = (col & 63) >> 3;
        float a0 = 0.f, a1 = 0.f, b0s = 0.f, b1s = 0.f;
#pragma unroll 4
        for (int rr = 0; rr < split; ++rr) {
            const int row = rh * 64 + rr;
            uint32_t w;
            asm volatile("ld.shared.b32 %0, [%1];" : "=r"(w) : "r"(cbase + (uint32_t)(row * 128 + ((chunk ^ (row & 7)) << 4))));
            a0 += ws_16_to_f(w & 0xffffu, LEAN - 1); a1 += ws_16_to_f(w >> 16, LEAN - 1);
        }
#pragma unroll 4
        for (int rr = max(split, 0); rr < nvalid; ++rr) {
            const int row = rh * 64 + rr;
            uint32_t w;
            asm volatile("ld.shared.b32 %0, [%1];" : "=r"(w) : "r"(cbase + (uint32_t)(row * 128 + ((chunk ^ (row & 7)) << 4))));
            b0s += ws_16_to_f(w & 0xffffu, LEAN - 1); b1s += ws_16_to_f(w >> 16, LEAN - 1);
        }
        const long long unit = (long long)(t0 >> 6) + rh;
        float* dst = e.colsum + unit * 2 * (long long)(p.tiles_n * p.bn) + n0 + col;
        *reinterpret_cast<float2*>(dst) = make_float2(a0, a1);
        *reinterpret_cast<float2*>(dst + (long long)(p.tiles_n * p.bn)) = make_float2(b0s, b1s);
    }
}

}  // namespace ws_tcdev

// 0 = generic epilogue, else activation dtype + 1 (see the LEAN template parameter)
inline int ws_tc_lean_kind(const WsTc2Params* p) {
    const WsEpi& e = p->epi;
    const bool common = !p->has_out2 && e.gate == nullptr &&
                        (e.act1 == WS_ACT_NONE || e.act1 == WS_ACT_RELU || e.act1 == WS_ACT_TANH) &&
                        (e.act2 == WS_ACT_NONE || e.act2 == WS_ACT_RELU);
    if (!common) return 0;
    // 16-bit: 128-byte panels, or the 64-byte panels of 32-channel tiles (CAM++ / ResNet 1x1 shortcut convs) when no column
    // sums are asked for (they read whole 128-byte rows)
    if (p->kind == 1 && p->nsplit == 1 && p->nout == 1 && (e.dtype == WS_BF16 || e.dtype == WS_F16) &&
        ((p->bn >= 64 && p->panel_bytes == 128) || (p->bn == 32 && p->panel_bytes == 64 && e.colsum == nullptr)))
        return e.dtype + 1;
    if (p->panel_bytes != 128) return 0;
    if (p->kind == 0 && e.dtype == WS_F32 && p->bn >= 32 &&
        ((p->nsplit == 1 && p->nout == 1) || (p->nsplit == 3 && p->nout == 2)))
        return WS_F32 + 1;
    return 0;
}

// launch-time guard shared by both kernels: column sums exist only in the lean 16-bit epilogue on flat 1x1 tiles
inline const char* ws_tc_colsum_check(const WsTc2Params* p, int lean) {
    if (p->epi.colsum != nullptr && (lean != WS_BF16 + 1 && lean != WS_F16 + 1 || p->tiles_f != 1 || p->tiles_b != 1 ||
                                     p->bt_log2 != 7 || p->epi.colsum_T < 128))
        return "conv colsum: needs the lean 16-bit epilogue on a dense 1x1 conv (flat positions) and >= 128 frames per utterance";
    return nullptr;
}
