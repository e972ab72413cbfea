// SimAM, the parameter-free attention inside every residual block of SimAM-ResNet (samresnet.py:57-70):
//   n = F*T - 1,  d = (X - mean_FT(X))^2,  v = sum_FT(d) / n,  out = X * sigmoid(d / (4 (v + lambda)) + 0.5)
// followed by the block's "out += shortcut; relu".  Two ops on channels-last maps [B][F][T][ld]:
//
//   * statistics: one CTA per (64-channel block, f, b) accumulates Welford (count, mean, centred sum of squares) per channel
//     in fp32 over its 32 time slices t = r, r + 32, ... (t < the utterance's frame count), merges the slices with Chan's
//     formula in a fixed tree order and writes one partial per (b, f, c); a second launch merges the F partials of each
//     (b, c) in fp64.  No atomics, and the order of every sum depends only on (f, t), never on the padded T of the batch:
//     a length-masked utterance sums exactly the partials it sums alone.  Centred squares throughout, never sum x^2 - n
//     mean^2: BN-shifted maps can have |mean| >> std.
//   * apply: out = relu(y * sigmoid((y - mean)^2 / (4 (v + lambda)) + 0.5) + res), 8 channels per thread.  res may alias
//     out (the block's downsample conv wrote its output there first), and out takes its own (b, f, t) strides, so the last
//     block of the trunk writes ASP's pooled frame [B][1][T][F*C] (feature f*C + c) directly.  Rows behind an utterance's
//     end are written as zeros (the next 3x3 conv reads across time).
#include <algorithm>

#include "../../include/wespeaker_b200.h"
#include "ws_host.h"

namespace {

constexpr int kSlices = 32;   // time slices per statistics CTA
constexpr int kCBlk = 64;     // channels per statistics CTA (8 threads x 8 channels)

__device__ __forceinline__ int frames_of(const int* lens, int b, int T) { return lens ? max(1, min(T, lens[b])) : T; }

template <int DT>
__global__ void __launch_bounds__(256) simam_partial_kernel(const void* __restrict__ y, int F, int T, int C, long long ld,
                                                            float* __restrict__ part, const int* __restrict__ lens) {
    __shared__ float s_mu[kSlices][kCBlk], s_m2[kSlices][kCBlk];
    __shared__ int s_n[kSlices];
    const int cg = threadIdx.x, r = threadIdx.y, f = blockIdx.y, b = blockIdx.z;
    const int c = blockIdx.x * kCBlk + cg * 8;
    const bool cv = c < C;
    const int Tb = frames_of(lens, b, T);
    const long long base = ((long long)b * F + f) * T * ld + c;
    float mu[8], m2[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { mu[k] = 0.f; m2[k] = 0.f; }
    int n = 0;
    if (cv) {
#pragma unroll 2
        for (int t = r; t < Tb; t += kSlices) {
            float v[8];
            ws_ldv8(y, DT, base + (long long)t * ld, v);
            ++n;
            const float inv = 1.f / (float)n;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const float d = v[k] - mu[k];
                mu[k] = fmaf(d, inv, mu[k]);
                m2[k] = fmaf(d, v[k] - mu[k], m2[k]);
            }
        }
    }
    // slice r + s is merged into slice r, s = 16, 8, 4, 2, 1
    for (int s = kSlices / 2; s >= 1; s >>= 1) {
        if (r >= s && r < 2 * s) {
#pragma unroll
            for (int k = 0; k < 8; ++k) { s_mu[r][cg * 8 + k] = mu[k]; s_m2[r][cg * 8 + k] = m2[k]; }
            if (cg == 0) s_n[r] = n;
        }
        __syncthreads();
        if (r < s) {
            const int nb = s_n[r + s];
            if (nb > 0) {
                const int nn = n + nb;
                const float wb = (float)nb / (float)nn, wab = (float)n * wb;
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const float d = s_mu[r + s][cg * 8 + k] - mu[k];
                    mu[k] = fmaf(d, wb, mu[k]);
                    m2[k] = m2[k] + s_m2[r + s][cg * 8 + k] + d * d * wab;
                }
                n = nn;
            }
        }
        __syncthreads();
    }
    if (r == 0 && cv) {
        float4* o = reinterpret_cast<float4*>(part + (((long long)b * F + f) * C + c) * 2);
#pragma unroll
        for (int k = 0; k < 4; ++k) o[k] = make_float4(mu[2 * k], m2[2 * k], mu[2 * k + 1], m2[2 * k + 1]);
    }
}

// the F partials of (b, c), each over the utterance's Tb frames, in fp64: mean, then the centred sum of squares
__global__ void __launch_bounds__(128) simam_merge_kernel(const float* __restrict__ part, int F, int T, int C,
                                                          float* __restrict__ stats, const int* __restrict__ lens) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (c >= C) return;
    const int Tb = frames_of(lens, b, T);
    const float2* p = reinterpret_cast<const float2*>(part) + (long long)b * F * C + c;
    double s = 0.0;
    for (int f = 0; f < F; ++f) s += (double)p[(long long)f * C].x;
    const double mean = s / F;
    double m2 = 0.0;
    for (int f = 0; f < F; ++f) {
        const float2 q = p[(long long)f * C];
        const double d = (double)q.x - mean;
        m2 += (double)q.y + (double)Tb * d * d;
    }
    stats[(long long)b * 2 * C + c] = (float)mean;
    stats[(long long)b * 2 * C + C + c] = (float)(m2 / (double)(F * Tb - 1));
}

template <int DT>
__global__ void __launch_bounds__(256) simam_apply_kernel(const void* __restrict__ y, long long y_ld, const float* __restrict__ stats,
                                                          float lambda_p, const void* res, WsMapStrides rs, void* out, float* out_lo,
                                                          WsMapStrides os, int F, int T, int C, const int* __restrict__ lens,
                                                          long long nvec) {
    // res and out may alias (in-place residual): every element is read and then written by the same thread
    const unsigned cv = (unsigned)C >> 3;
    unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned stride = gridDim.x * blockDim.x, n = (unsigned)nvec;   // launcher guarantees nvec < 2^31
    for (; i < n; i += stride) {
        const unsigned upos = i / cv;
        const int c = (int)(i - upos * cv) * 8;
        const unsigned bf = upos / (unsigned)T;
        const int t = (int)(upos - bf * (unsigned)T);
        const int b = (int)(bf / (unsigned)F), f = (int)(bf - (unsigned)b * F);
        const long long oo = (long long)b * os.b + (long long)f * os.f + (long long)t * os.t + c;
        float v[8];
        if (t >= frames_of(lens, b, T)) {
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] = 0.f;
            ws_stv8(out, DT, oo, v);
            if (out_lo != nullptr) ws_stv8(out_lo, WS_F32, oo, v);
            continue;
        }
        float rv[8], mu[8], var[8];
        ws_ldv8(y, DT, (long long)upos * y_ld + c, v);
        ws_ldv8(res, DT, (long long)b * rs.b + (long long)f * rs.f + (long long)t * rs.t + c, rv);
        ws_ldv<8>(stats, WS_F32, (long long)b * 2 * C + c, mu);
        ws_ldv<8>(stats, WS_F32, (long long)b * 2 * C + C + c, var);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float d = v[k] - mu[k];
            float g;
            if (DT == WS_F32) {   // the fp32-class paths keep IEEE division and expf
                const float z = d * d / (4.f * (var[k] + lambda_p)) + 0.5f;
                g = 1.f / (1.f + expf(-z));
            } else {
                const float z = __fdividef(d * d, 4.f * (var[k] + lambda_p)) + 0.5f;
                g = __frcp_rn(1.f + __expf(-z));
            }
            v[k] = fmaxf(fmaf(v[k], g, rv[k]), 0.f);
        }
        ws_stv8(out, DT, oo, v);
        if (out_lo != nullptr) {
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] = ws_tf32_lo(v[k]);
            ws_stv8(out_lo, WS_F32, oo, v);
        }
    }
}

inline const char* last_err() {
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace

const char* ws_launch_simam_stats(const WsSimamStats& a, cudaStream_t s) {
    const WsView& y = a.y;
    const int B = y.B, F = y.F, T = y.T, C = y.C;
    if (C % 8 != 0 || y.ld % 8 != 0 || !aligned16(y.p) || !aligned16(a.partial)) return "simam_stats: C and ld must be multiples of 8, buffers 16-byte aligned";
    if (F < 1 || T < 1 || F > 65535 || B > 65535 || (long long)F * T < 2) return "simam_stats: bad extents";
    const dim3 grid((C + kCBlk - 1) / kCBlk, F, B), block(8, kSlices);
    if (y.dt == WS_BF16) simam_partial_kernel<WS_BF16><<<grid, block, 0, s>>>(y.p, F, T, C, y.ld, a.partial, a.lens);
    else if (y.dt == WS_F16) simam_partial_kernel<WS_F16><<<grid, block, 0, s>>>(y.p, F, T, C, y.ld, a.partial, a.lens);
    else simam_partial_kernel<WS_F32><<<grid, block, 0, s>>>(y.p, F, T, C, y.ld, a.partial, a.lens);
    simam_merge_kernel<<<dim3((C + 127) / 128, B), 128, 0, s>>>(a.partial, F, T, C, a.stats, a.lens);
    return last_err();
}

const char* ws_launch_simam_apply(const WsSimamApply& a, cudaStream_t s) {
    const WsView& y = a.y;
    const WsMapStrides &rs = a.rs, &os = a.os;
    const int F = y.F, T = y.T, C = y.C;
    if (C % 8 != 0 || y.ld % 8 != 0 || rs.b % 8 || rs.f % 8 || rs.t % 8 || os.b % 8 || os.f % 8 || os.t % 8 ||
        !aligned16(y.p) || !aligned16(a.res) || !aligned16(a.out) || !aligned16(a.stats) || (a.out_lo && !aligned16(a.out_lo)))
        return "simam_apply: C and every stride must be multiples of 8, buffers 16-byte aligned";
    const long long nvec = y.npos() * (C / 8);
    if (nvec >= (1LL << 31)) return "simam_apply: tensor too large for 32-bit vector indices";
    const int g = (int)std::min<long long>((nvec + 255) / 256, (long long)ws_num_sms() * 16);
    if (y.dt == WS_BF16) simam_apply_kernel<WS_BF16><<<g, 256, 0, s>>>(y.p, y.ld, a.stats, a.lambda, a.res, rs, a.out, a.out_lo, os, F, T, C, a.lens, nvec);
    else if (y.dt == WS_F16) simam_apply_kernel<WS_F16><<<g, 256, 0, s>>>(y.p, y.ld, a.stats, a.lambda, a.res, rs, a.out, a.out_lo, os, F, T, C, a.lens, nvec);
    else simam_apply_kernel<WS_F32><<<g, 256, 0, s>>>(y.p, y.ld, a.stats, a.lambda, a.res, rs, a.out, a.out_lo, os, F, T, C, a.lens, nvec);
    return last_err();
}

extern "C" int ws_simam(const ws_simam_desc* d, void* stream) {
    if (!d || !d->y || !d->res || !d->out || !d->stats || !d->partial) { ws::set_err("ws_simam: null argument"); return 1; }
    cudaStream_t s = (cudaStream_t)stream;
    const WsView y{const_cast<void*>(d->y), nullptr, d->B, d->F, d->T, d->C, d->y_ld, d->dtype};
    WS_CKS(ws_launch_simam_stats(WsSimamStats{y, d->partial, d->stats, d->lens}, s));
    WS_CKS(ws_launch_simam_apply(WsSimamApply{y, d->stats, d->lambda_p, d->res, {d->res_sb, d->res_sf, d->res_st}, d->out, (float*)d->out_lo,
                                              {d->out_sb, d->out_sf, d->out_st}, d->lens}, s));
    return 0;
}
