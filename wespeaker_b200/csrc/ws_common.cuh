// Shared device/host definitions for the wespeaker_b200 kernels (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>

enum WsDType : int { WS_F32 = 0, WS_BF16 = 1, WS_F16 = 2 };
// RELU20 = Hardtanh(0, 20), the "ReLU" of the Res2Net / ERes2Net families (eres2net.py:43-52); SILU = v * sigmoid(v) (AFF)
enum WsAct : int { WS_ACT_NONE = 0, WS_ACT_RELU = 1, WS_ACT_TANH = 2, WS_ACT_SIGMOID = 3, WS_ACT_RELU20 = 4, WS_ACT_SILU = 5 };

__host__ __device__ inline int ws_esize(int dt) { return dt == WS_F32 ? 4 : 2; }

// Fused epilogue of every conv/GEMM launch (applied on the fp32 accumulator, in this order):
//   v  = acc + bias[c] + rowbias[b][c]
//   v  = act1(v)
//   v  = v * scale[c] + shift[c]
//   v *= gate[b][t / gate_seg][c]
//   v += res[pos][c]
//   v  = act2(v)
//   out[pos][c] = v ;  out2[pos][c] = v + add2[pos][c]
// ECAPA's conv->relu->bn (ecapa_tdnn.py:105-106) is {bias, relu, scale/shift}; folded-BN conv->bn->relu
// (resnet.py:64-69, campplus.py:65-83) is {scale/shift folded into W, shift as bias, relu}.
struct WsEpi {
    const float* bias;
    const float* rowbias;
    int rowbias_ld;
    int act1;
    const float* scale;
    const float* shift;
    const float* gate;
    int gate_ld, gate_seg, gate_nseg;
    const void* res;
    long long res_ld;
    int act2;
    void* out;
    long long out_ld;
    void* out2;
    long long out2_ld;
    const void* add2;
    long long add2_ld;
    void* out_lo;   // 3xTF32 mode: out_lo = out - tf32_trunc(out) (same ld); null otherwise
    void* out2_lo;
    int dtype;  // dtype of res/out/out2/add2 (activation dtype)
    int FT;     // F*T of the output tensor (pos / FT = b)
    int T;      // T of the output tensor   (pos % T = t)
    // SE squeeze fused into a dense 1x1 conv (lean 16-bit tensor-core epilogue only): per 64-position unit u and slot s,
    // colsum[(2u + s) * Cout + c] = sum of the STORED (rounded) outputs of channel c over the unit's positions that belong
    // to utterance (64u / colsum_T) + s.  colsum_T >= 128 frames, so a unit touches at most two utterances.
    float* colsum;
    int colsum_T;
};

__device__ __forceinline__ float ws_act(float v, int act) {
    switch (act) {
        case WS_ACT_RELU: return fmaxf(v, 0.f);
        case WS_ACT_TANH: return tanhf(v);
        case WS_ACT_SIGMOID: return 1.f / (1.f + expf(-v));
        case WS_ACT_RELU20: return fminf(fmaxf(v, 0.f), 20.f);
        case WS_ACT_SILU: return v / (1.f + expf(-v));
        default: return v;
    }
}

// activation over a register vector with the (warp-uniform) switch hoisted OUT of the element loop: a per-element
// switch with inlined tanhf/expf made the GEMM epilogues instruction-issue bound (round-1 profile: ~4500 SASS
// instructions per 32-column chunk).
template <int NV>
__device__ __forceinline__ void ws_act_vec(float* v, int act) {
    if (act == WS_ACT_NONE) return;
    if (act == WS_ACT_RELU) {
#pragma unroll
        for (int j = 0; j < NV; ++j) v[j] = fmaxf(v[j], 0.f);
    } else if (act == WS_ACT_TANH) {
#pragma unroll 4
        for (int j = 0; j < NV; ++j) v[j] = tanhf(v[j]);
    } else if (act == WS_ACT_SIGMOID) {
#pragma unroll 4
        for (int j = 0; j < NV; ++j) v[j] = 1.f / (1.f + expf(-v[j]));
    } else if (act == WS_ACT_RELU20) {
#pragma unroll
        for (int j = 0; j < NV; ++j) v[j] = fminf(fmaxf(v[j], 0.f), 20.f);
    } else {
#pragma unroll 4
        for (int j = 0; j < NV; ++j) v[j] = v[j] / (1.f + expf(-v[j]));
    }
}

__device__ __forceinline__ uint32_t ws_pack2(float a, float b, int dt) {
    if (dt == WS_BF16) {
        __nv_bfloat162 h = __float22bfloat162_rn(make_float2(a, b));
        return *reinterpret_cast<uint32_t*>(&h);
    }
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}

__device__ __forceinline__ float ws_bf16_bits_to_f(uint32_t u16) { return __uint_as_float(u16 << 16); }
__device__ __forceinline__ float ws_f16_bits_to_f(uint32_t u16) {
    return __half2float(__ushort_as_half((unsigned short)u16));
}
__device__ __forceinline__ uint32_t ws_f_to_16(float v, int dt) {
    return dt == WS_BF16 ? (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(v))
                         : (uint32_t)__half_as_ushort(__float2half_rn(v));
}
__device__ __forceinline__ float ws_16_to_f(uint32_t u, int dt) {
    return dt == WS_BF16 ? ws_bf16_bits_to_f(u) : ws_f16_bits_to_f(u);
}

// low part of the 3xTF32 split: v - tf32_trunc(v) (exact in fp32; the tensor core truncates fp32 operands to tf32)
__device__ __forceinline__ float ws_tf32_lo(float v) { return v - __uint_as_float(__float_as_uint(v) & 0xffffe000u); }

// scalar typed load/store (any alignment)
__device__ __forceinline__ float ws_ld(const void* p, int dt, long long i) {
    if (dt == WS_F32) return ((const float*)p)[i];
    return ws_16_to_f(((const unsigned short*)p)[i], dt);
}
__device__ __forceinline__ void ws_st(void* p, int dt, long long i, float v) {
    if (dt == WS_F32) ((float*)p)[i] = v;
    else ((unsigned short*)p)[i] = (unsigned short)ws_f_to_16(v, dt);
}

// NV consecutive elements starting at element offset `off` (off % 4 == 0, base 16B aligned).
template <int NV>
__device__ __forceinline__ void ws_ldv(const void* p, int dt, long long off, float* v) {
    static_assert(NV % 4 == 0, "NV % 4");
    if (dt == WS_F32) {
        const float4* q = reinterpret_cast<const float4*>((const float*)p + off);
#pragma unroll
        for (int i = 0; i < NV / 4; ++i) {
            float4 x = q[i];
            v[4 * i] = x.x; v[4 * i + 1] = x.y; v[4 * i + 2] = x.z; v[4 * i + 3] = x.w;
        }
    } else {
        const uint2* q = reinterpret_cast<const uint2*>((const unsigned short*)p + off);
#pragma unroll
        for (int i = 0; i < NV / 4; ++i) {
            uint2 x = q[i];
            v[4 * i] = ws_16_to_f(x.x & 0xffffu, dt); v[4 * i + 1] = ws_16_to_f(x.x >> 16, dt);
            v[4 * i + 2] = ws_16_to_f(x.y & 0xffffu, dt); v[4 * i + 3] = ws_16_to_f(x.y >> 16, dt);
        }
    }
}
template <int NV>
__device__ __forceinline__ void ws_stv(void* p, int dt, long long off, const float* v) {
    static_assert(NV % 4 == 0, "NV % 4");
    if (dt == WS_F32) {
        float4* q = reinterpret_cast<float4*>((float*)p + off);
#pragma unroll
        for (int i = 0; i < NV / 4; ++i) q[i] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
    } else {
        uint2* q = reinterpret_cast<uint2*>((unsigned short*)p + off);
        if (dt == WS_BF16) {
#pragma unroll
            for (int i = 0; i < NV / 4; ++i)
                q[i] = make_uint2(ws_pack2(v[4 * i], v[4 * i + 1], WS_BF16), ws_pack2(v[4 * i + 2], v[4 * i + 3], WS_BF16));
        } else {
#pragma unroll
            for (int i = 0; i < NV / 4; ++i)
                q[i] = make_uint2(ws_pack2(v[4 * i], v[4 * i + 1], WS_F16), ws_pack2(v[4 * i + 2], v[4 * i + 3], WS_F16));
        }
    }
}

// 8 consecutive elements (off % 8 == 0): one 16-byte access for 16-bit types, two for fp32
__device__ __forceinline__ void ws_ldv8(const void* p, int dt, long long off, float* v) {
    if (dt == WS_F32) {
        ws_ldv<8>(p, dt, off, v);
    } else {
        const uint4 x = *reinterpret_cast<const uint4*>((const unsigned short*)p + off);
        const uint32_t w[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            v[2 * i] = ws_16_to_f(w[i] & 0xffffu, dt);
            v[2 * i + 1] = ws_16_to_f(w[i] >> 16, dt);
        }
    }
}
// 8 packed 16-bit values (one 16-byte load) -> fp32
__device__ __forceinline__ void ws_unpack8(const uint4& x, int dt, float* v) {
    const uint32_t w[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        v[2 * i] = ws_16_to_f(w[i] & 0xffffu, dt);
        v[2 * i + 1] = ws_16_to_f(w[i] >> 16, dt);
    }
}
__device__ __forceinline__ void ws_stv8(void* p, int dt, long long off, const float* v) {
    if (dt == WS_F32) {
        ws_stv<8>(p, dt, off, v);
    } else {
        uint4 x;
        x.x = ws_pack2(v[0], v[1], dt); x.y = ws_pack2(v[2], v[3], dt);
        x.z = ws_pack2(v[4], v[5], dt); x.w = ws_pack2(v[6], v[7], dt);
        *reinterpret_cast<uint4*>((unsigned short*)p + off) = x;
    }
}
// 2 consecutive elements (off % 2 == 0)
__device__ __forceinline__ void ws_ld2(const void* p, int dt, long long off, float* v) {
    if (dt == WS_F32) {
        const float2 x = *reinterpret_cast<const float2*>((const float*)p + off);
        v[0] = x.x; v[1] = x.y;
    } else {
        const uint32_t w = *reinterpret_cast<const uint32_t*>((const unsigned short*)p + off);
        v[0] = ws_16_to_f(w & 0xffffu, dt); v[1] = ws_16_to_f(w >> 16, dt);
    }
}

// Apply the fused epilogue to NV consecutive output channels [col0, col0+NV) of output position `pos`.
template <int NV>
__device__ __forceinline__ void ws_epilogue(const WsEpi& e, long long pos, int col0, float* v) {
    int b = 0, t = 0;
    if (e.rowbias != nullptr || e.gate != nullptr) {
        b = (int)(pos / e.FT);
        t = (int)(pos % e.T);
    }
    if (e.bias != nullptr) {
#pragma unroll
        for (int j = 0; j < NV; ++j) v[j] += __ldg(e.bias + col0 + j);
    }
    if (e.rowbias != nullptr) {
        const float* rb = e.rowbias + (long long)b * e.rowbias_ld + col0;
#pragma unroll
        for (int j = 0; j < NV; ++j) v[j] += __ldg(rb + j);
    }
    ws_act_vec<NV>(v, e.act1);
    if (e.scale != nullptr) {
#pragma unroll
        for (int j = 0; j < NV; ++j) v[j] = fmaf(v[j], __ldg(e.scale + col0 + j), __ldg(e.shift + col0 + j));
    }
    if (e.gate != nullptr) {
        const float* g = e.gate + ((long long)b * e.gate_nseg + t / e.gate_seg) * e.gate_ld + col0;
#pragma unroll
        for (int j = 0; j < NV; ++j) v[j] *= __ldg(g + j);
    }
    if (e.res != nullptr) {
        float r[NV];
        ws_ldv<NV>(e.res, e.dtype, pos * e.res_ld + col0, r);
#pragma unroll
        for (int j = 0; j < NV; ++j) v[j] += r[j];
    }
    ws_act_vec<NV>(v, e.act2);
    ws_stv<NV>(e.out, e.dtype, pos * e.out_ld + col0, v);
    if (e.out2 != nullptr) {
        float r[NV];
        ws_ldv<NV>(e.add2, e.dtype, pos * e.add2_ld + col0, r);
#pragma unroll
        for (int j = 0; j < NV; ++j) r[j] += v[j];
        ws_stv<NV>(e.out2, e.dtype, pos * e.out2_ld + col0, r);
    }
}

// ------------------------------------------------------------------ conv-as-GEMM description
// Activations are channels-last [B][F][T][C]; one "tap" contributes  sum_c X_src[b, f+df, t+dt, c0+c] * W[co][wk+c]
// for c in [0, nch).  Strided convs use parity-plane source views so taps stay unit-stride.
#define WS_MAX_SRC 4
#define WS_MAX_TAPS 52

struct WsSrc {
    const void* ptr;
    const void* ptr_lo;      // 3xTF32 mode: x - tf32_trunc(x) twin of the same geometry (or null)
    int B, F, T, C;          // extents of the (possibly strided) view; reads outside are zero (conv padding)
    long long sB, sF, sT;    // element strides
};
struct WsTap {
    int src, c0, dt, df, wk, nch;
};

struct WsSimtParams {
    WsSrc src[WS_MAX_SRC];
    WsTap taps[WS_MAX_TAPS];
    int ntaps;
    const void* W;  // [Cout][Ktot], activation dtype
    int Ktot, Cout;
    int B, F, T;    // output extents
    int dtype;
    WsEpi epi;
};

#define WS_TC_MAX_STAGES 8
// per-warp accumulator scratch of the row-wise GEMM epilogues (ws_wgmma.cuh, frag_to_rows): 8 consumer warps x 16 x 68 floats
#define WS_TC_EPI_SCRATCH (8 * 16 * 68 * 4)
// one tap of the tensor-core conv: source map, first channel, time / frequency offset, first weight column, k-blocks
struct WsTcTap {
    int map, c0, dt, df, wk, nkb;
};

// persistent conv-GEMM on the tensor cores (ws_gemm_tc2.cu)
struct WsTc2Params {
    CUtensorMap amap[WS_MAX_SRC];
    CUtensorMap amap_lo[WS_MAX_SRC];  // 3xTF32: low parts of the activations
    CUtensorMap wmap;
    CUtensorMap wmap_lo;              // 3xTF32: low parts of the weights
    CUtensorMap omap[4];  // output tile stores: [0] out, then (if split) out_lo, (if has_out2) out2, (both) out2_lo
    CUtensorMap imap;     // epilogue input tile (residual, or add2 when has_out2), if has_epin
    WsTcTap taps[WS_MAX_TAPS];
    int ntaps, nk_total;
    int bk_bytes;                        // 128 / 64 / 32: k-block row bytes == TMA / wgmma swizzle span
    int bt_log2, bf_log2, bb_log2;       // output tile = 2^bt x 2^bf x 2^bb = 128 positions
    int tiles_t, tiles_f, tiles_b, tiles_n, num_tiles;
    int B, F, T;                         // output extents (flattened to 1 x 1 x B*F*T for a dense 1x1 conv)
    int bn, nstages;                     // N tile (output channels per tile), ring stages
    int kind;                            // 0 = tf32, 1 = f16/bf16
    int panel_bytes;     // 128 or 64: row bytes of one swizzled staging panel
    int has_out2, has_epin;
    int nsplit;          // 1, or 3 = 3xTF32 error-compensated passes (x_lo*W, x*W_lo, x*W)
    int nout;            // number of output tiles staged per tile (1..4)
    int epi_generic;     // always run the generic epilogue instantiation (ConvSpec::epi_generic, a test reference)
    int grid, smem_bytes;
    int cl;              // CTAs per cluster: 1, or 2 / 4 (ws_tc3_launch) sharing the weight tile by TMA multicast
    WsEpi epi;
};

// fused ASTP tail (ws_astp_fused.cu): attention logits (linear2) + softmax over time + weighted mean / std
struct WsAstpParams {
    CUtensorMap hmap;   // H = tanh(linear1(x)) [B][T][128], 16-bit: dims (128, T, B), box (64, 256, 1), SWIZZLE_128B
    CUtensorMap wmap;   // linear2 weight [C][128] K-major: dims (128, C), box (64, 128)
    CUtensorMap xmap;   // x [B][T][x_ld]: dims (C, T, B), box (128, 128, 1), no swizzle (row pitch 256 B in smem)
    const void* x;      // frame-level features [B][T][x_ld] (16-bit), the tensor the statistics are taken of
    long long x_ld;
    float* out;         // [B][2C]: weighted mean, then std
    int B, T, C, dtype;
    int g;              // channel blocks (of 128) per work unit: H is fetched once per unit
    int grid;
    const int* lens;    // length-masked batch: frames of each utterance, or null
    float var_floor;    // std = sqrt(max(var, var_floor))
};

// fused Res2 chain (ws_res2_fused.cu)
struct WsRes2Params {
    CUtensorMap xmap;   // block input  [B][T][C] (channels-last, 16-bit): dims (C, T, B), box (64, 128, 1), SWIZZLE_128B
    CUtensorMap wmap;   // 7 packed conv weights [7*w8][3*w8] K-major: box (64, w8)
    CUtensorMap omap;   // block output [B][T][C]: same geometry as xmap
    CUtensorMap omap64; // the same with 64-row boxes (time-tiled utterances store the exact inner rows of a tile)
    int ntile;          // time tiles per utterance: 1 (T <= 256), else ceil(T / 192) tiles of 256 rows overlapping by 2 x 32
    const void* x;      // raw pointer of the block input (x_{i+1} groups are read directly in the epilogue)
    long long ld;       // row stride (elements) of the block input
    const float* bias;  // [7][w8]
    const float* scale; // [7][w8] BN affine after ReLU
    const float* shift;
    int B, T, w8, dil, dtype;
    int grid, smem_bytes;
    const int* lens;    // length-masked batch: frames of each utterance (rows behind it are conv padding: kept zero), or null
};

// halo-resident 3x3 stride-1 conv (ws_conv3x3.cu): input rows of F live in a shared-memory ring, the 9 taps are row-shifted
// wgmma operand reads of that ring
#define WS_C3_MAX_RING 8
#define WS_C3_MAX_WSTAGES 4
struct WsC3Params {
    CUtensorMap amap;       // input  (C, T, F, B): box (kc, box_t, 1, box_b), swizzle = row_bytes
    CUtensorMap amap_tail;  // same tensor, box (kc, 2, 1, 1): the last two halo columns when a slot needs > 256 rows
    CUtensorMap wmap;       // weights [Cout][9*Cin] K-major: box (kc, N)
    CUtensorMap omap;       // output (Cout, T, F, B): box (panel_cols, obox_t, 1, obox_b), swizzle = panel_bytes
    CUtensorMap rmap;       // residual tensor, same geometry and box as omap (TMA-loaded into the output staging tile)
    const void* res;        // residual base pointer (null = no residual)
    long long res_ld;
    int stg_bufs;           // output staging tiles: 2 = the residual of step s+1 is prefetched while step s drains, 1 = in line
    int sf, st;             // conv strides along F and T (1 or 2).  B, F, T below are OUTPUT extents.  st == 2: a slot holds the
                            // even-t and the (shifted) odd-t plane of an input row (amap / amap_tail), sub_rows rows each
    int sub_rows;
    const float* bias;      // [Cout]
    int relu;               // 0 none, 1 ReLU, 2 Hardtanh(0, 20)
    int B, F, T, Cin, Cout, dtype;
    int row_bytes, npan, kc;       // bytes per smem operand row per K panel (64 / 128), K panels per tap, channels per panel
    int P, tb, n_tt;               // padded pitch (tb + 2), output columns per t tile, number of t tiles
    int nb, n_bg;                  // utterances per slot (case B: several short utterances share one M tile), b groups
    int n_mt;                      // M tiles (128 rows) per step; tile mt starts 128*mt rows into the slot
    int single_box;                // slot filled by one TMA box (rows = box_t * box_b) instead of n_mt x 128 rows + 2-row tail
    int rows_loaded, slot_rows;    // rows written per slot per panel / allocated rows per slot per panel (multiple of 8)
    int R;                         // ring depth in slots (>= 4)
    int N, n_nt;                   // output channels per CTA tile, number of n tiles
    int w_resident, w_stages;      // all 9*npan weight blocks resident in smem, or streamed through a ring
    int panel_bytes, panel_cols;   // output staging panel row bytes (128, or 64 when N == 32) and columns
    int stg_rows;                  // allocated rows per staging panel (128, or 136 in case B)
    int case_b;
    int total_steps;               // n_nt * n_tt * n_bg * F output-row steps, split contiguously over the CTAs
    int grid, smem_bytes;
    const int* lens;               // length-masked batch: output frames of each utterance (rows behind are stored as zeros), or null
};

// fused CAM++ dense layer (ws_cam_dense.cu).  One descriptor per CAMDenseTDNNLayer, device-resident (the tensor maps are
// read by the TMA unit from global memory), 64-byte aligned.
struct alignas(64) WsCamLayer {
    CUtensorMap w1map;        // linear1 weights with nonlinear2's BN folded in: [128][Cin] K-major, box (64, 128), SWIZZLE_128B
    CUtensorMap wlmap;        // cam_layer.linear_local weights [32][3*128] tap-major, box (64, 32), SWIZZLE_128B
    const float* bn1_scale;   // nonlinear1 (BN + ReLU on the growing concat), [Cin]
    const float* bn1_shift;
    const float* bias2;       // nonlinear2 shift, [128]
    const float* w1c_t;       // cam_layer.linear1 weight transposed to [128][64]
    const float* b1c;         // [64]
    const float* w2c_t;       // cam_layer.linear2 weight transposed to [64][32]
    const float* b2c;         // [32]
    int cin, dil;
    int pad_[12];
};
struct WsCamParams {
    CUtensorMap xmap;         // concat buffer (Cmax, T, B): box (64, 128, 1), SWIZZLE_128B (operand panels of the 1x1 conv)
    CUtensorMap omap;         // same buffer: box (32, 128, 1), SWIZZLE_64B (the layer's 32 new channels)
    const WsCamLayer* layers;
    int l0, l1;               // layers [l0, l1) run back to back inside one launch
    int B, T, nmt, seg_len, dtype;
    int nstages, hrows;       // ring stages (32 KB each); rows per panel of the hidden operand buffer (16 + 128 * nmt)
    int grid, smem_bytes;
    const int* lens;          // length-masked batch: frames of each utterance (statistics and padding follow them), or null
};

// Dynamic shared memory per CTA that the host geometry code plans within and the kernels are opted in to.
constexpr int kMaxDynSmem2 = 226 * 1024;   // conv-GEMM (ws_gemm_tc2.cu): ring + staging + per-channel parameters + scratch
constexpr int kC3MaxSmem = 222 * 1024;     // halo-resident 3x3 conv (ws_conv3x3.cu)
constexpr int kCamMaxSmem = 222 * 1024;    // fused CAM++ dense layers (ws_cam_dense.cu)
constexpr int kRes2MaxSmem = 220 * 1024;   // fused Res2 chain (ws_res2_fused.cu)

// Opts one kernel instance into `bytes` of dynamic shared memory on the current device.  The attribute is per device, so
// each instance keeps one bit per device ordinal, set once the call succeeded (ordinals >= 64 set it on every call).  Two
// threads may both set it; that is harmless.  On failure the runtime's last error is cleared and its message returned.
template <auto Kernel>
inline const char* ws_smem_opt_in(int bytes) {
    static std::atomic<unsigned long long> done{0};
    int dev = 0;
    cudaGetDevice(&dev);
    const unsigned long long bit = dev >= 0 && dev < 64 ? 1ull << dev : 0;
    if (done.load() & bit) return nullptr;
    const cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return cudaGetErrorString(e);
    }
    done.fetch_or(bit);
    return nullptr;
}

inline int ws_num_sms() {
    static std::atomic<int> sms[64] = {};   // per device ordinal; 0 = not yet queried
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) return 132;
    int n = sms[dev].load();
    if (n == 0) {
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 132;
        sms[dev].store(n);
    }
    return n;
}

#ifdef __cplusplus
extern "C" {
#endif
const char* ws_astp_launch(const WsAstpParams* p, cudaStream_t s);
const char* ws_res2_launch(const WsRes2Params* p, cudaStream_t s);
const char* ws_cam_launch(const WsCamParams* p, cudaStream_t s);
const char* ws_c3_launch(const WsC3Params* p, cudaStream_t s);
int ws_tc3_max_clusters(int cl);   // co-resident clusters of `cl` CTAs on this device (0 = query failed)
const char* ws_tc3_launch(const WsTc2Params* p, cudaStream_t s);
const char* ws_tc2_launch(const WsTc2Params* p, cudaStream_t s);
const char* ws_simt_launch(const WsSimtParams* p, cudaStream_t s);
#ifdef __cplusplus
}
#endif
