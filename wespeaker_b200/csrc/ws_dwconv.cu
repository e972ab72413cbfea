// Depthwise 3x3 conv (groups = channels, pad 1, stride 1) + folded BN + ReLU: conv2 / bn2 of Gemini DF-ResNet's inverted
// bottleneck (gemini_dfresnet.py:30-48).  On channels-last maps [B][F][T][ld]:
//
//   out[b,f,t,c] = relu(sum_{df,dt in {-1,0,1}} w[c][df+1][dt+1] * x[b,f+df,t+dt,c] + shift[c])
//
// with zero padding outside [0,F) x [0,T_b) (T_b = the utterance's frame count in a length-masked batch, else T).  The
// BN scale is folded into w on the host; w and shift are fp32, the sum runs in fp32 in a fixed tap order and is rounded
// once to the activation dtype.  Rows t >= T_b are read as zeros (the expand conv leaves relu(bias) there) and written
// as zeros, so the value at (b, f, t, c) never depends on the batch it is computed in.
//
// The op streams the 4x-expanded tensor of the block once in and once out, so it is HBM-bound.  A CTA owns one
// (utterance, band of <= 10 frequency rows, tile of <= 32 frames, 32 channels) block: the input block and its one-row /
// one-frame halo are staged once into shared memory with 16-byte cp.async copies (zero-filled where the halo falls into
// padding or behind the utterance's end), then each thread computes 4 channels of one frame for every row of the band,
// with their 9 taps of weights in registers.  4 channels per thread (64 registers, 4 CTAs per SM) measured 1.68 TB/s on
// the stage-3 shape (B 64, F 10, T 100, C 512, fp16) on an H100 80GB HBM3 at 400 W, 8 per thread (120 registers, 2 CTAs
// per SM) 1.63 TB/s.
// With an fp32 `out_lo`, the 3xTF32 low part out - tf32_trunc(out) is written beside the output for the next GEMM.
#include <algorithm>

#include "../../include/wespeaker_b200.h"
#include "ws_host.h"

namespace {

constexpr int kV = 4;          // channels per thread
constexpr int kLanes = 8;      // threads across the channel chunk of a CTA
constexpr int kCh = kLanes * kV;   // channels per CTA
constexpr int kTT = 32;        // frames per CTA (at most)
constexpr int kMaxFB = 10;     // frequency rows per CTA (at most)
constexpr int kThreads = kLanes * kTT;
constexpr int kMaxSmem = (kMaxFB + 2) * (kTT + 2) * kCh * 4;

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(valid ? 16 : 0) : "memory");
}

// 4 consecutive channels at p (aligned to their size) <-> fp32
template <int DT>
__device__ __forceinline__ void ld4(const void* p, float* v) {
    if constexpr (DT == WS_F32) {
        const float4 q = *reinterpret_cast<const float4*>(p);
        v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
    } else {
        const uint2 q = *reinterpret_cast<const uint2*>(p);
        v[0] = ws_16_to_f(q.x & 0xffffu, DT); v[1] = ws_16_to_f(q.x >> 16, DT);
        v[2] = ws_16_to_f(q.y & 0xffffu, DT); v[3] = ws_16_to_f(q.y >> 16, DT);
    }
}
template <int DT>
__device__ __forceinline__ void st4(void* p, const float* v) {
    if constexpr (DT == WS_F32) {
        *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
        *reinterpret_cast<uint2*>(p) = make_uint2(ws_pack2(v[0], v[1], DT), ws_pack2(v[2], v[3], DT));
    }
}

template <int DT>
__global__ void __launch_bounds__(kThreads, 4) dwconv3x3_kernel(const void* __restrict__ x, long long x_ld, const float* __restrict__ w,
                                                                const float* __restrict__ shift, void* __restrict__ out,
                                                                float* __restrict__ out_lo, long long out_ld, int F, int T, int C,
                                                                int fb, int tt, int nchunk, const int* __restrict__ lens) {
    constexpr int ES = DT == WS_F32 ? 4 : 2;
    constexpr int V = kV;
    constexpr int PB = kCh * ES;              // bytes of a position's channel chunk
    constexpr int U = PB / 16;                // 16-byte copies per position
    extern __shared__ uint4 s_raw[];          // [fr + 2][tr + 2][PB bytes]
    char* s_x = reinterpret_cast<char*>(s_raw);
    const int chunk = blockIdx.x % nchunk, tile = blockIdx.x / nchunk, b = blockIdx.z;
    const int c0 = chunk * kCh, t0 = tile * tt, f0 = blockIdx.y * fb;
    const int fr = min(fb, F - f0), tr = min(tt, T - t0), pitch = tr + 2;
    const int Tb = lens != nullptr ? max(1, min(T, lens[b])) : T;
    const char* xb = reinterpret_cast<const char*>(x);
    const int n = (fr + 2) * pitch * U;
    for (int i = threadIdx.x; i < n; i += kThreads) {
        const int u = i % U, q = i / U;
        const int f = f0 - 1 + q / pitch, t = t0 - 1 + q % pitch, c = c0 + u * (16 / ES);
        const bool valid = f >= 0 && f < F && t >= 0 && t < Tb && c < C;
        const char* src = valid ? xb + ((((long long)b * F + f) * T + t) * x_ld + c) * ES : xb;
        cp_async16(s_x + (size_t)i * 16, src, valid);
    }
    asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;\n" ::: "memory");
    __syncthreads();

    const int v = threadIdx.x % kLanes, tl = threadIdx.x / kLanes;
    const int c = c0 + v * V, t = t0 + tl;
    if (tl >= tr || c >= C) return;
    float wr[V * 9], sh[V];   // wr[j * 9 + tap]: channel c + j, tap = (df + 1) * 3 + (dt + 1)
    {
        const float4* w4 = reinterpret_cast<const float4*>(w + (long long)c * 9);
#pragma unroll
        for (int i = 0; i < V * 9 / 4; ++i) {
            const float4 q = __ldg(w4 + i);
            wr[4 * i] = q.x; wr[4 * i + 1] = q.y; wr[4 * i + 2] = q.z; wr[4 * i + 3] = q.w;
        }
        const float4* s4 = reinterpret_cast<const float4*>(shift + c);
#pragma unroll
        for (int i = 0; i < V / 4; ++i) {
            const float4 q = __ldg(s4 + i);
            sh[4 * i] = q.x; sh[4 * i + 1] = q.y; sh[4 * i + 2] = q.z; sh[4 * i + 3] = q.w;
        }
    }
    const bool live = t < Tb;
#pragma unroll 1
    for (int fl = 0; fl < fr; ++fl) {
        float acc[V];
#pragma unroll
        for (int j = 0; j < V; ++j) acc[j] = 0.f;
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            float xv[V];
            ld4<DT>(s_x + ((fl + tap / 3) * pitch + tl + tap % 3) * PB + v * V * ES, xv);
#pragma unroll
            for (int j = 0; j < V; ++j) acc[j] = fmaf(wr[j * 9 + tap], xv[j], acc[j]);
        }
#pragma unroll
        for (int j = 0; j < V; ++j) acc[j] = live ? fmaxf(acc[j] + sh[j], 0.f) : 0.f;
        const long long o = (((long long)b * F + f0 + fl) * T + t) * out_ld + c;
        st4<DT>(reinterpret_cast<char*>(out) + o * ES, acc);
        if (DT == WS_F32 && out_lo != nullptr) {
#pragma unroll
            for (int j = 0; j < V; ++j) acc[j] = ws_tf32_lo(acc[j]);
            st4<WS_F32>(out_lo + o, acc);
        }
    }
}

inline const char* last_err() {
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace

const char* ws_launch_dwconv3x3(const WsDwconv3x3& a, cudaStream_t s) {
    const void *x = a.x.p, *w = a.w, *shift = a.shift;
    void* out = a.out.p;
    float* out_lo = (float*)a.out.plo;
    const long long x_ld = a.x.ld, out_ld = a.out.ld;
    const int dt = a.x.dt, B = a.x.B, F = a.x.F, T = a.x.T, C = a.x.C;
    if (dt != WS_F32 && dt != WS_BF16 && dt != WS_F16) return "dwconv3x3: dtype must be 0 (fp32), 1 (bf16) or 2 (fp16)";
    const int V = 16 / ws_esize(dt);   // channels per 16-byte copy
    if (C % V != 0 || x_ld % V != 0 || out_ld % V != 0 || x_ld < C || out_ld < C || !aligned16(x) || !aligned16(out) || !aligned16(w) ||
        !aligned16(shift) || (out_lo != nullptr && (dt != WS_F32 || !aligned16(out_lo))))
        return "dwconv3x3: C, x_ld and out_ld must be multiples of 8 (16-bit) / 4 (fp32), buffers 16-byte aligned, out_lo fp32 only";
    if (B < 1 || F < 1 || T < 1 || B > 65535) return "dwconv3x3: bad extents";
    // balanced bands and tiles: F = 10 is one band of 10 rows, F = 40 four; T = 100 is four tiles of 25 frames
    const int nband = (F + kMaxFB - 1) / kMaxFB, fb = (F + nband - 1) / nband;
    const int ntile = (T + kTT - 1) / kTT, tt = (T + ntile - 1) / ntile;
    const int nchunk = (C + kCh - 1) / kCh;
    if ((long long)nchunk * ntile > 0x7fffffffLL || nband > 65535) return "dwconv3x3: tensor too large";
    const dim3 grid(nchunk * ntile, nband, B);
    const int smem = (fb + 2) * (tt + 2) * kCh * ws_esize(dt);
    const char* m = dt == WS_BF16  ? ws_smem_opt_in<dwconv3x3_kernel<WS_BF16>>(kMaxSmem)
                    : dt == WS_F16 ? ws_smem_opt_in<dwconv3x3_kernel<WS_F16>>(kMaxSmem)
                                   : ws_smem_opt_in<dwconv3x3_kernel<WS_F32>>(kMaxSmem);
    if (m) return m;
    if (dt == WS_BF16)
        dwconv3x3_kernel<WS_BF16><<<grid, kThreads, smem, s>>>(x, x_ld, a.w, a.shift, out, nullptr, out_ld, F, T, C, fb, tt, nchunk, a.lens);
    else if (dt == WS_F16)
        dwconv3x3_kernel<WS_F16><<<grid, kThreads, smem, s>>>(x, x_ld, a.w, a.shift, out, nullptr, out_ld, F, T, C, fb, tt, nchunk, a.lens);
    else
        dwconv3x3_kernel<WS_F32><<<grid, kThreads, smem, s>>>(x, x_ld, a.w, a.shift, out, out_lo, out_ld, F, T, C, fb, tt, nchunk, a.lens);
    return last_err();
}

extern "C" int ws_dwconv(const ws_dwconv_desc* d, void* stream) {
    if (!d || !d->x || !d->w || !d->shift || !d->out) { ws::set_err("ws_dwconv: null argument"); return 1; }
    const WsView x{const_cast<void*>(d->x), nullptr, d->B, d->F, d->T, d->C, d->x_ld, d->dtype},
        out{d->out, d->out_lo, d->B, d->F, d->T, d->C, d->out_ld, d->dtype};
    WS_CKS(ws_launch_dwconv3x3(WsDwconv3x3{x, d->w, d->shift, out, d->lens}, (cudaStream_t)stream));
    return 0;
}
