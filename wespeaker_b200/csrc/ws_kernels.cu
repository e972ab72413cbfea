// Bandwidth-bound kernels of the embedding path: statistics pooling (TSTP / ASTP), SE gating, small
// fully-connected layers, BN-ReLU pre-activation, the 1-channel stem conv.  All operate on channels-last
// activations so that a warp always touches 32 consecutive channels (coalesced 128-B / 64-B rows); the
// reductions over T are split over 8 warps per block and merged through shared memory, reductions over
// input features in the FC kernel use warp shuffles.
#include "ws_kernels.cuh"
#include <cstdlib>

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__global__ void convert_kernel(const float* __restrict__ in, void* __restrict__ out, float* __restrict__ lo, int dt,
                               long long n) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        ws_st(out, dt, i, in[i]);
        if (lo != nullptr) lo[i] = ws_tf32_lo(in[i]);
    }
}

// block (32, 8): x = channel lane, y = T slice.
__global__ void __launch_bounds__(256) tstats_kernel(const void* __restrict__ x, int dt, int F, int T, int C,
                                                     long long ld, const float* __restrict__ pre_scale,
                                                     const float* __restrict__ pre_shift, void* __restrict__ out,
                                                     int odt, long long out_ld, int std_off, float eps,
                                                     const int* __restrict__ lens) {
    __shared__ float red[8][33];
    const int c = blockIdx.x * 32 + threadIdx.x;
    const int f = blockIdx.y, b = blockIdx.z;
    const bool cv = c < C;
    const long long base = ((long long)b * F + f) * T * ld + c;
    const int Ts = T;                                   // memory stride between utterances stays the padded T
    if (lens != nullptr) T = max(1, min(T, lens[b]));   // length-masked batch: statistics over this utterance's own frames
    (void)Ts;
    float ps = 1.f, ph = 0.f;
    const bool pre = pre_scale != nullptr;
    if (pre && cv) { ps = pre_scale[c]; ph = pre_shift[c]; }
    float s = 0.f;
    if (cv)
        for (int t = threadIdx.y; t < T; t += 8) {
            float v = ws_ld(x, dt, base + (long long)t * ld);
            if (pre) v = fmaxf(fmaf(v, ps, ph), 0.f);
            s += v;
        }
    red[threadIdx.y][threadIdx.x] = s;
    __syncthreads();
    float mean = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) mean += red[i][threadIdx.x];
    mean /= (float)T;
    __syncthreads();
    float ss = 0.f;
    if (cv && std_off >= 0)
        for (int t = threadIdx.y; t < T; t += 8) {
            float v = ws_ld(x, dt, base + (long long)t * ld);
            if (pre) v = fmaxf(fmaf(v, ps, ph), 0.f);
            const float d = v - mean;
            ss = fmaf(d, d, ss);
        }
    red[threadIdx.y][threadIdx.x] = ss;
    __syncthreads();
    if (threadIdx.y == 0 && cv) {
        float tot = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) tot += red[i][threadIdx.x];
        const long long o = (long long)b * out_ld + (long long)c * F + f;
        ws_st(out, odt, o, mean);
        if (std_off >= 0) ws_st(out, odt, o + std_off, sqrtf(tot / (float)(T - 1) + eps));  // torch.var: unbiased
    }
}

// 16-bit activations: 8 channels per thread (16-byte loads), 16 T slices per block of 128 channels, ONE pass with the
// utterance's first frame as a per-channel shift (sum (v - v0), sum (v - v0)^2: no cancellation for means far from zero).
// The scalar two-pass kernel above ran at 1.3 TB/s on the ECAPA global-context statistics (157 MB); it stays for fp32.
template <int DT>
__global__ void __launch_bounds__(256) tstats8_kernel(const void* __restrict__ x, int F, int T, int C, long long ld,
                                                      const float* __restrict__ pre_scale, const float* __restrict__ pre_shift,
                                                      void* __restrict__ out, int odt, long long out_ld, int std_off, float eps,
                                                      const int* __restrict__ lens) {
    __shared__ float red[2][16][128 + 4];
    __shared__ float shift[128];
    const int cg = threadIdx.x, sl = threadIdx.y;             // 16 channel groups of 8, 16 T slices
    const int c = blockIdx.x * 128 + cg * 8;
    const int f = blockIdx.y, b = blockIdx.z;
    const bool cv = c < C;
    const long long base = ((long long)b * F + f) * T * ld + c;
    if (lens != nullptr) T = max(1, min(T, lens[b]));
    float ps[8], ph[8], v0[8], s1[8], s2[8];
    const bool pre = pre_scale != nullptr;
#pragma unroll
    for (int k = 0; k < 8; ++k) { ps[k] = 1.f; ph[k] = 0.f; s1[k] = 0.f; s2[k] = 0.f; v0[k] = 0.f; }
    auto load8 = [&](int t, float* v) {
        const uint4 r = *reinterpret_cast<const uint4*>((const unsigned short*)x + base + (long long)t * ld);
        const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            v[2 * k] = ws_16_to_f(w[k] & 0xffffu, DT);
            v[2 * k + 1] = ws_16_to_f(w[k] >> 16, DT);
        }
        if (pre) {
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] = fmaxf(fmaf(v[k], ps[k], ph[k]), 0.f);
        }
    };
    if (cv) {
        if (pre) {
#pragma unroll
            for (int k = 0; k < 8; ++k) { ps[k] = pre_scale[c + k]; ph[k] = pre_shift[c + k]; }
        }
        load8(0, v0);
        int t = sl;
        for (; t + 48 < T; t += 64) {   // four independent 16-byte loads in flight per thread
            float va[8], vb[8], vc[8], vd[8];
            load8(t, va); load8(t + 16, vb); load8(t + 32, vc); load8(t + 48, vd);
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const float d0 = va[k] - v0[k], d1 = vb[k] - v0[k], d2 = vc[k] - v0[k], d3 = vd[k] - v0[k];
                s1[k] += (d0 + d1) + (d2 + d3);
                s2[k] = fmaf(d0, d0, fmaf(d1, d1, fmaf(d2, d2, fmaf(d3, d3, s2[k]))));
            }
        }
        for (; t < T; t += 16) {
            float v[8];
            load8(t, v);
#pragma unroll
            for (int k = 0; k < 8; ++k) { const float d = v[k] - v0[k]; s1[k] += d; s2[k] = fmaf(d, d, s2[k]); }
        }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) { red[0][sl][cg * 8 + k] = s1[k]; red[1][sl][cg * 8 + k] = s2[k]; }
    if (sl == 0) {
#pragma unroll
        for (int k = 0; k < 8; ++k) shift[cg * 8 + k] = v0[k];
    }
    __syncthreads();
    const int tid = sl * 16 + cg;
    if (tid < 128) {
        const int cc = blockIdx.x * 128 + tid;
        if (cc < C) {
            float a1 = 0.f, a2 = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) { a1 += red[0][i][tid]; a2 += red[1][i][tid]; }
            const float n = (float)T, dmean = a1 / n;
            const long long o = (long long)b * out_ld + (long long)cc * F + f;
            ws_st(out, odt, o, shift[tid] + dmean);
            // sum (d - dmean)^2 = sum d^2 - dmean * sum d;  torch.var: unbiased
            if (std_off >= 0) ws_st(out, odt, o + std_off, sqrtf(fmaxf(a2 - a1 * dmean, 0.f) / (n - 1.f) + eps));
        }
    }
}

// mean over T only, 8 channels per thread (16-byte loads): the SE squeeze (ecapa_tdnn.py:120) reads a full activation map
// per stage.  block (64, 8): x = group of 8 channels, y = T slice.
__global__ void __launch_bounds__(512) tmean8_kernel(const void* __restrict__ x, int dt, int T, int C, long long ld,
                                                      float* __restrict__ out, long long out_ld) {
    __shared__ float red[8][64 * 8 + 8];
    const int c = (blockIdx.x * 64 + threadIdx.x) * 8;
    const int b = blockIdx.y;
    const bool cv = c < C;
    const long long base = (long long)b * T * ld + c;
    float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (cv)
        for (int t = threadIdx.y; t < T; t += 8) {
            float v[8];
            ws_ldv8(x, dt, base + (long long)t * ld, v);
#pragma unroll
            for (int k = 0; k < 8; ++k) a[k] += v[k];
        }
#pragma unroll
    for (int k = 0; k < 8; ++k) red[threadIdx.y][threadIdx.x * 8 + k] = a[k];
    __syncthreads();
    const int tid = threadIdx.y * 64 + threadIdx.x;   // 512 threads: one output channel each
    const int cc = blockIdx.x * 512 + tid;
    if (cc < C) {
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) s += red[i][tid];
        out[(long long)b * out_ld + cc] = s / (float)T;
    }
}

// Small fully-connected layers (SE, CAM context, global-context row bias, embedding head) as a shared-memory tiled
// fp32 GEMM: block = 16 rows x 32 outputs (thread: 1 row x 2 outputs), K streamed in chunks of 64 with coalesced loads.
__global__ void __launch_bounds__(256) linear_rows_kernel(const float* __restrict__ in, long long in_ld,
                                                          const float* __restrict__ in2, long long in2_ld,
                                                          int rows_per_b, const float* __restrict__ W,
                                                          const float* __restrict__ bias, float* __restrict__ out,
                                                          long long out_ld, int R, int I, int O, int act) {
    constexpr int TR = 16, TO = 32, TK = 64;
    __shared__ float Xs[TR][TK + 1];
    __shared__ float Ws[TO][TK + 1];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int r0 = blockIdx.y * TR, o0 = blockIdx.x * TO;
    // split-K: blockIdx.z owns the k range [kbeg, kend); partial sums go to out + z*R*out_ld (no bias/act), a second
    // kernel reduces them in a fixed order (deterministic, unlike atomics)
    const int nsplit = gridDim.z;
    const int kper = ((I + nsplit - 1) / nsplit + TK - 1) / TK * TK;
    const int kbeg = blockIdx.z * kper, kend = min(I, kbeg + kper);
    if (nsplit > 1) { out += (long long)blockIdx.z * R * out_ld; bias = nullptr; act = WS_ACT_NONE; }
    float acc0 = 0.f, acc1 = 0.f;
    for (int k0 = kbeg; k0 < kend; k0 += TK) {
        __syncthreads();
        for (int idx = tid; idx < TR * TK; idx += 256) {
            const int rr = idx / TK, kk = idx % TK, r = r0 + rr, k = k0 + kk;
            float v = 0.f;
            if (r < R && k < kend) {
                v = in[(long long)r * in_ld + k];
                if (in2 != nullptr) v += in2[(long long)(r / rows_per_b) * in2_ld + k];
            }
            Xs[rr][kk] = v;
        }
        for (int idx = tid; idx < TO * TK; idx += 256) {
            const int oo = idx / TK, kk = idx % TK, o = o0 + oo, k = k0 + kk;
            Ws[oo][kk] = (o < O && k < kend) ? __ldg(W + (long long)o * I + k) : 0.f;
        }
        __syncthreads();
#pragma unroll 16
        for (int kk = 0; kk < TK; ++kk) {
            const float x = Xs[ty][kk];
            acc0 = fmaf(x, Ws[tx][kk], acc0);
            acc1 = fmaf(x, Ws[tx + 16][kk], acc1);
        }
    }
    const int r = r0 + ty;
    if (r < R) {
        const int oa = o0 + tx, ob = o0 + tx + 16;
        if (oa < O) out[(long long)r * out_ld + oa] = ws_act(acc0 + (bias != nullptr ? bias[oa] : 0.f), act);
        if (ob < O) out[(long long)r * out_ld + ob] = ws_act(acc1 + (bias != nullptr ? bias[ob] : 0.f), act);
    }
}

// Larger FC layers (embedding head: 256 rows x 3072 -> 192): 64 x 64 output tile, 4 x 4 register tile per thread, K in
// chunks of 32 staged TRANSPOSED in smem (so the inner loop is two LDS.128 per 16 FMAs), split-K over blockIdx.z with the
// same fixed-order reduction kernel.  Needs 16-byte aligned rows (I, in_ld, in2_ld multiples of 4).
__global__ void __launch_bounds__(256) linear_rows64_kernel(const float* __restrict__ in, long long in_ld,
                                                            const float* __restrict__ in2, long long in2_ld,
                                                            int rows_per_b, const float* __restrict__ W,
                                                            const float* __restrict__ bias, float* __restrict__ out,
                                                            long long out_ld, int R, int I, int O, int act) {
    constexpr int TR = 64, TO = 64, TK = 32;
    __shared__ __align__(16) float Xs[TK][TR + 4];
    __shared__ __align__(16) float Ws[TK][TO + 4];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int r0 = blockIdx.y * TR, o0 = blockIdx.x * TO;
    const int nsplit = gridDim.z;
    const int kper = ((I + nsplit - 1) / nsplit + TK - 1) / TK * TK;
    const int kbeg = blockIdx.z * kper, kend = min(I, kbeg + kper);
    if (nsplit > 1) { out += (long long)blockIdx.z * R * out_ld; bias = nullptr; act = WS_ACT_NONE; }
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int k0 = kbeg; k0 < kend; k0 += TK) {
        float4 xv[2], wv[2];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int idx = tid + 256 * j, rr = idx >> 3, k = k0 + (idx & 7) * 4;
            const int r = r0 + rr, o = o0 + rr;
            xv[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            wv[j] = xv[j];
            if (k < kend) {   // kend - k is a multiple of 4 (I % 4 == 0, kper % 32 == 0)
                if (r < R) {
                    xv[j] = *reinterpret_cast<const float4*>(in + (long long)r * in_ld + k);
                    if (in2 != nullptr) {
                        const float4 y = *reinterpret_cast<const float4*>(in2 + (long long)(r / rows_per_b) * in2_ld + k);
                        xv[j].x += y.x; xv[j].y += y.y; xv[j].z += y.z; xv[j].w += y.w;
                    }
                }
                if (o < O) wv[j] = __ldg(reinterpret_cast<const float4*>(W + (long long)o * I + k));
            }
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int idx = tid + 256 * j, rr = idx >> 3, kk = (idx & 7) * 4;
            Xs[kk][rr] = xv[j].x; Xs[kk + 1][rr] = xv[j].y; Xs[kk + 2][rr] = xv[j].z; Xs[kk + 3][rr] = xv[j].w;
            Ws[kk][rr] = wv[j].x; Ws[kk + 1][rr] = wv[j].y; Ws[kk + 2][rr] = wv[j].z; Ws[kk + 3][rr] = wv[j].w;
        }
        __syncthreads();
#pragma unroll 8
        for (int kk = 0; kk < TK; ++kk) {
            const float4 a = *reinterpret_cast<const float4*>(&Xs[kk][4 * ty]);
            const float4 w = *reinterpret_cast<const float4*>(&Ws[kk][4 * tx]);
            const float av[4] = {a.x, a.y, a.z, a.w}, wv4[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], wv4[j], acc[i][j]);
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int r = r0 + 4 * ty + i;
        if (r >= R) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int o = o0 + 4 * tx + j;
            if (o < O) out[(long long)r * out_ld + o] = ws_act(acc[i][j] + (bias != nullptr ? bias[o] : 0.f), act);
        }
    }
}

__global__ void linear_reduce_kernel(const float* __restrict__ part, int nsplit, const float* __restrict__ bias,
                                     float* __restrict__ out, long long out_ld, int R, int O, int act) {
    const long long n = (long long)R * O;
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int r = (int)(i / O), o = (int)(i % O);
    float a = 0.f;
    for (int s = 0; s < nsplit; ++s) a += part[((long long)s * R + r) * O + o];
    out[(long long)r * out_ld + o] = ws_act(a + (bias != nullptr ? bias[o] : 0.f), act);
}

template <int dt>   // compile-time dtype: one conversion path instead of both + selects (the kernel was issue-limited)
__global__ void scale_residual_kernel(const void* __restrict__ x, long long x_ld, const float* __restrict__ gate,
                                      const void* __restrict__ res, long long res_ld, void* __restrict__ out,
                                      float* __restrict__ lo, long long out_ld, int T, int C, long long nvec) {
    const unsigned cv = (unsigned)C >> 3;  // 8 channels per thread: 16-byte accesses for 16-bit activations
    unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned stride = gridDim.x * blockDim.x, n = (unsigned)nvec;   // launcher guarantees nvec < 2^31
    for (; i < n; i += stride) {
        const unsigned upos = i / cv;          // 32-bit index math (64-bit divisions were most of the instruction stream)
        const int c = (int)(i - upos * cv) * 8;
        const int b = (int)(upos / (unsigned)T);
        const long long pos = upos;
        float v[8], r[8];
        ws_ldv8(x, dt, pos * x_ld + c, v);
        ws_ldv8(res, dt, pos * res_ld + c, r);
        const float4 g0 = *reinterpret_cast<const float4*>(gate + (long long)b * C + c);
        const float4 g1 = *reinterpret_cast<const float4*>(gate + (long long)b * C + c + 4);
        v[0] = fmaf(v[0], g0.x, r[0]); v[1] = fmaf(v[1], g0.y, r[1]); v[2] = fmaf(v[2], g0.z, r[2]); v[3] = fmaf(v[3], g0.w, r[3]);
        v[4] = fmaf(v[4], g1.x, r[4]); v[5] = fmaf(v[5], g1.y, r[5]); v[6] = fmaf(v[6], g1.z, r[6]); v[7] = fmaf(v[7], g1.w, r[7]);
        ws_stv8(out, dt, pos * out_ld + c, v);
        if (lo != nullptr) {
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] = ws_tf32_lo(v[k]);
            ws_stv8(lo, WS_F32, pos * out_ld + c, v);
        }
    }
}

// ERes2Net attentional feature fusion, the combine step (eres2net.py:97-100): att = 1 + t with t = tanh(local_att(x | y))
// already applied by the producing conv's epilogue; out = x * att + y * (2 - att).  8 channels per thread, 16-byte accesses.
template <int dt>
__global__ void aff_combine_kernel(const void* __restrict__ x, long long x_ld, const void* __restrict__ y, long long y_ld,
                                   const void* __restrict__ t, long long t_ld, void* __restrict__ out, float* __restrict__ lo,
                                   long long out_ld, int C, long long nvec) {
    const unsigned cv = (unsigned)C >> 3;
    unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned stride = gridDim.x * blockDim.x, n = (unsigned)nvec;   // launcher guarantees nvec < 2^31
    for (; i < n; i += stride) {
        const unsigned upos = i / cv;
        const int c = (int)(i - upos * cv) * 8;
        const long long pos = upos;
        float a[8], b[8], g[8];
        ws_ldv8(x, dt, pos * x_ld + c, a);
        ws_ldv8(y, dt, pos * y_ld + c, b);
        ws_ldv8(t, dt, pos * t_ld + c, g);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float att = 1.f + g[k];
            a[k] = a[k] * att + b[k] * (2.f - att);
        }
        ws_stv8(out, dt, pos * out_ld + c, a);
        if (lo != nullptr) {
#pragma unroll
            for (int k = 0; k < 8; ++k) a[k] = ws_tf32_lo(a[k]);
            ws_stv8(lo, WS_F32, pos * out_ld + c, a);
        }
    }
}

// block (32, 8), 2 channels per thread; ONE pass over (x, logits) with an online softmax per (b, c): running max m and
// sums rescaled by exp(m_old - m_new); the 8 T-slices are merged through shared memory.
__global__ void __launch_bounds__(256) astp_stats_kernel(const void* __restrict__ x, const void* __restrict__ lg,
                                                         int dt, int T, int C, long long ld, float* __restrict__ out,
                                                         float var_floor, const int* __restrict__ lens) {
    __shared__ float red[4][8][65];
    const int c = (blockIdx.x * 32 + threadIdx.x) * 2;
    const int b = blockIdx.y;
    const bool cv = c < C;
    const long long base = (long long)b * T * ld + c;
    if (lens != nullptr) T = max(1, min(T, lens[b]));   // softmax / weighted statistics over this utterance's own frames
    float m[2] = {-INFINITY, -INFINITY}, s0[2] = {0.f, 0.f}, s1[2] = {0.f, 0.f}, s2[2] = {0.f, 0.f};
    if (cv) {
        for (int t = threadIdx.y; t < T; t += 8) {   // this thread's slice maximum (logits only)
            float l[2];
            ws_ld2(lg, dt, base + (long long)t * ld, l);
            m[0] = fmaxf(m[0], l[0]); m[1] = fmaxf(m[1], l[1]);
        }
        for (int t = threadIdx.y; t < T; t += 8) {   // one expf per element (logits re-read hits L1/L2)
            float l[2], v[2];
            ws_ld2(lg, dt, base + (long long)t * ld, l);
            ws_ld2(x, dt, base + (long long)t * ld, v);
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const float e = expf(l[k] - m[k]);
                s0[k] += e;
                s1[k] = fmaf(e, v[k], s1[k]);
                s2[k] = fmaf(e * v[k], v[k], s2[k]);
            }
        }
    }
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        red[0][threadIdx.y][2 * threadIdx.x + k] = m[k];
        red[1][threadIdx.y][2 * threadIdx.x + k] = s0[k];
        red[2][threadIdx.y][2 * threadIdx.x + k] = s1[k];
        red[3][threadIdx.y][2 * threadIdx.x + k] = s2[k];
    }
    __syncthreads();
    if (threadIdx.y < 2) {
        const int col = 2 * threadIdx.x + threadIdx.y, cc = c + threadIdx.y;
        if (cv && cc < C) {
            float M = red[0][0][col];
#pragma unroll
            for (int i = 1; i < 8; ++i) M = fmaxf(M, red[0][i][col]);
            float a0 = 0.f, a1 = 0.f, a2 = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float w = red[0][i][col] == -INFINITY ? 0.f : expf(red[0][i][col] - M);
                a0 = fmaf(red[1][i][col], w, a0); a1 = fmaf(red[2][i][col], w, a1); a2 = fmaf(red[3][i][col], w, a2);
            }
            const float mean = a1 / a0;
            const float var = a2 / a0 - mean * mean;
            out[(long long)b * 2 * C + cc] = mean;
            out[(long long)b * 2 * C + C + cc] = sqrtf(var < var_floor ? var_floor : var);   // torch clamp: NaN stays NaN
        }
    }
}

// 16-bit activations, T <= 256, every load issued up front: block (16, 32) = 16 channel groups of 4 channels (8-byte loads) x 32 T slices,
// T <= 256: the thread's <= 8 logits rows AND x rows are loaded into registers before any arithmetic (16 independent
// loads in flight per thread), then max / exp sums run from registers.  The fp32-path kernel above turned out to be
// instruction-bound (full-precision expf + run-time dtype selects: ~25 instructions per element), so this one is compiled
// per dtype and uses ex2.approx (__expf, ~1e-6 relative error: far below the 16-bit activation rounding it operates on).
template <int dt>
__global__ void __launch_bounds__(512, 2) astp_stats4_kernel(const void* __restrict__ x, const void* __restrict__ lg,
                                                             int T, int C, long long ld, float* __restrict__ out,
                                                             float var_floor, const int* __restrict__ lens) {
    __shared__ float red[16][4][64];
    const int cg = threadIdx.x, sl = threadIdx.y, warp = sl >> 1;   // a warp = 2 slices x 16 channel groups
    const int c = (blockIdx.x * 16 + cg) * 4;
    const int b = blockIdx.y;
    const bool cv = c < C;
    const long long base = (long long)b * T * ld + c;
    if (lens != nullptr) T = max(1, min(T, lens[b]));   // softmax / weighted statistics over this utterance's own frames
    float m[4], s0[4], s1[4], s2[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) { m[k] = -INFINITY; s0[k] = 0.f; s1[k] = 0.f; s2[k] = 0.f; }
    if (cv) {
        uint2 lr[8], xr[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int t = sl + 32 * i;
            lr[i] = make_uint2(0u, 0u); xr[i] = lr[i];
            if (t < T) {
                lr[i] = *reinterpret_cast<const uint2*>((const unsigned short*)lg + base + (long long)t * ld);
                xr[i] = *reinterpret_cast<const uint2*>((const unsigned short*)x + base + (long long)t * ld);
            }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i)
            if (sl + 32 * i < T) {
                m[0] = fmaxf(m[0], ws_16_to_f(lr[i].x & 0xffffu, dt)); m[1] = fmaxf(m[1], ws_16_to_f(lr[i].x >> 16, dt));
                m[2] = fmaxf(m[2], ws_16_to_f(lr[i].y & 0xffffu, dt)); m[3] = fmaxf(m[3], ws_16_to_f(lr[i].y >> 16, dt));
            }
#pragma unroll
        for (int i = 0; i < 8; ++i)
            if (sl + 32 * i < T) {
                const float l[4] = {ws_16_to_f(lr[i].x & 0xffffu, dt), ws_16_to_f(lr[i].x >> 16, dt),
                                    ws_16_to_f(lr[i].y & 0xffffu, dt), ws_16_to_f(lr[i].y >> 16, dt)};
                const float v[4] = {ws_16_to_f(xr[i].x & 0xffffu, dt), ws_16_to_f(xr[i].x >> 16, dt),
                                    ws_16_to_f(xr[i].y & 0xffffu, dt), ws_16_to_f(xr[i].y >> 16, dt)};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const float e = __expf(l[k] - m[k]);
                    s0[k] += e;
                    s1[k] = fmaf(e, v[k], s1[k]);
                    s2[k] = fmaf(e * v[k], v[k], s2[k]);
                }
            }
    }
    // lanes l and l^16 hold the same channels for 2 different T slices
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float mo = __shfl_xor_sync(0xffffffffu, m[k], 16);
        const float a0 = __shfl_xor_sync(0xffffffffu, s0[k], 16);
        const float a1 = __shfl_xor_sync(0xffffffffu, s1[k], 16);
        const float a2 = __shfl_xor_sync(0xffffffffu, s2[k], 16);
        const float M = fmaxf(m[k], mo);
        const float wa = m[k] == -INFINITY ? 0.f : expf(m[k] - M);
        const float wb = mo == -INFINITY ? 0.f : expf(mo - M);
        s0[k] = s0[k] * wa + a0 * wb;
        s1[k] = s1[k] * wa + a1 * wb;
        s2[k] = s2[k] * wa + a2 * wb;
        m[k] = M;
    }
    if ((sl & 1) == 0) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            red[warp][0][cg * 4 + k] = m[k]; red[warp][1][cg * 4 + k] = s0[k];
            red[warp][2][cg * 4 + k] = s1[k]; red[warp][3][cg * 4 + k] = s2[k];
        }
    }
    __syncthreads();
    const int tid = sl * 16 + cg;
    if (tid < 64) {
        const int cc = blockIdx.x * 64 + tid;
        if (cc < C) {
            float M = red[0][0][tid];
#pragma unroll
            for (int i = 1; i < 16; ++i) M = fmaxf(M, red[i][0][tid]);
            float a0 = 0.f, a1 = 0.f, a2 = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const float w = red[i][0][tid] == -INFINITY ? 0.f : expf(red[i][0][tid] - M);
                a0 = fmaf(red[i][1][tid], w, a0); a1 = fmaf(red[i][2][tid], w, a1); a2 = fmaf(red[i][3][tid], w, a2);
            }
            const float mean = a1 / a0;
            const float var = a2 / a0 - mean * mean;
            out[(long long)b * 2 * C + cc] = mean;
            out[(long long)b * 2 * C + C + cc] = sqrtf(var < var_floor ? var_floor : var);   // torch clamp: NaN stays NaN
        }
    }
}

__global__ void bnrelu_kernel(const void* __restrict__ x, long long x_ld, const float* __restrict__ scale,
                              const float* __restrict__ shift, void* __restrict__ out, float* __restrict__ lo,
                              long long out_ld, int dt, int C, long long nvec) {
    const int cv = C >> 2;
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (; i < nvec; i += stride) {
        const long long pos = i / cv;
        const int c = (int)(i % cv) * 4;
        float v[4];
        ws_ldv<4>(x, dt, pos * x_ld + c, v);
        const float4 sc = *reinterpret_cast<const float4*>(scale + c);
        const float4 sh = *reinterpret_cast<const float4*>(shift + c);
        v[0] = fmaxf(fmaf(v[0], sc.x, sh.x), 0.f); v[1] = fmaxf(fmaf(v[1], sc.y, sh.y), 0.f);
        v[2] = fmaxf(fmaf(v[2], sc.z, sh.z), 0.f); v[3] = fmaxf(fmaf(v[3], sc.w, sh.w), 0.f);
        ws_stv<4>(out, dt, pos * out_ld + c, v);
        if (lo != nullptr) {
            v[0] = ws_tf32_lo(v[0]); v[1] = ws_tf32_lo(v[1]); v[2] = ws_tf32_lo(v[2]); v[3] = ws_tf32_lo(v[3]);
            ws_stv<4>(lo, WS_F32, pos * out_ld + c, v);
        }
    }
}

// Stem conv (1 -> COUT channels, 3x3, pad 1) + folded BN + ReLU.  A block owns an 8 (F) x 128 (T) output tile of one
// utterance.  The 10 x 130 input patch is staged through shared memory with F-contiguous (coalesced) global reads (the
// input is [B][T][F]).  A thread owns ONE group of 8 output channels - its 72 weights sit in registers, so the inner loop is
// 9 shared-memory reads per 72 FMAs instead of one read per FMA - and walks 4 x 8 positions; the COUT/8 channel groups of a
// position are adjacent lanes, so a warp's store instruction covers whole 64- / 128-byte position records back to back.
template <int COUT>
__global__ void __launch_bounds__(128) stem_kernel(const float* __restrict__ feats, const float* __restrict__ w9,
                                                   const float* __restrict__ shift, void* __restrict__ out,
                                                   float* __restrict__ lo, int dt, int B, int T, int Fdim,
                                                   const int* __restrict__ lens) {
    constexpr int NG = COUT / 8;            // channel groups per position (4 or 8)
    constexpr int PL = 128 / NG;            // position lanes per block
    __shared__ float sin_[10][132];
    const int t0 = blockIdx.x * 128, f0 = blockIdx.y * 8, b = blockIdx.z;
    const int Tb = lens != nullptr ? min(T, lens[b]) : T;   // length-masked batch: frames past the utterance's end are padding
    for (int i = threadIdx.x; i < 10 * 130; i += 128) {
        const int tl = i / 10, fl = i - tl * 10;           // consecutive threads: consecutive F of the same frame
        const int tt = t0 + tl - 1, ff = f0 + fl - 1;
        sin_[fl][tl] = (ff >= 0 && ff < Fdim && tt >= 0 && tt < Tb) ? __ldg(feats + ((long long)b * T + tt) * Fdim + ff) : 0.f;
    }
    const int cg = threadIdx.x % NG, pl = threadIdx.x / NG;
    float w[8][9], sh8[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        sh8[j] = __ldg(shift + cg * 8 + j);
#pragma unroll
        for (int k = 0; k < 9; ++k) w[j][k] = __ldg(w9 + (cg * 8 + j) * 9 + k);
    }
    __syncthreads();
#pragma unroll 1
    for (int tl = pl; tl < 128; tl += PL) {
        const int t = t0 + tl;
        if (t >= T) break;
        float r0[3], r1[3], r2[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) { r0[k] = sin_[0][tl + k]; r1[k] = sin_[1][tl + k]; }
#pragma unroll 1
        for (int fl = 0; fl < 8; ++fl) {
            const int f = f0 + fl;
            if (f >= Fdim) break;
#pragma unroll
            for (int k = 0; k < 3; ++k) r2[k] = sin_[fl + 2][tl + k];
            const float in[9] = {r0[0], r0[1], r0[2], r1[0], r1[1], r1[2], r2[0], r2[1], r2[2]};
            float v[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float a = sh8[j];
#pragma unroll
                for (int k = 0; k < 9; ++k) a = fmaf(in[k], w[j][k], a);
                v[j] = t < Tb ? fmaxf(a, 0.f) : 0.f;        // zero rows behind the utterance: the next conv's padding
            }
            const long long idx = ((long long)b * Fdim + f) * T + t;
            ws_stv8(out, dt, idx * COUT + cg * 8, v);
            if (lo != nullptr) {
#pragma unroll
                for (int j = 0; j < 8; ++j) v[j] = ws_tf32_lo(v[j]);
                ws_stv8(lo, WS_F32, idx * COUT + cg * 8, v);
            }
#pragma unroll
            for (int k = 0; k < 3; ++k) { r0[k] = r1[k]; r1[k] = r2[k]; }
        }
    }
}

// block (32, 8)
__global__ void __launch_bounds__(256) seg_means_kernel(const void* __restrict__ x, int dt, int T, int C, long long ld,
                                                        int seg_len, float* __restrict__ mean,
                                                        float* __restrict__ segmean) {
    __shared__ float red[8][33];
    const int c = blockIdx.x * 32 + threadIdx.x;
    const int b = blockIdx.y;
    const bool cv = c < C;
    const int nseg = (T + seg_len - 1) / seg_len;
    const long long base = (long long)b * T * ld + c;
    float total = 0.f;
    for (int sgi = 0; sgi < nseg; ++sgi) {
        const int ta = sgi * seg_len, tb = min(T, ta + seg_len);
        float s = 0.f;
        if (cv)
            for (int t = ta + threadIdx.y; t < tb; t += 8) s += ws_ld(x, dt, base + (long long)t * ld);
        red[threadIdx.y][threadIdx.x] = s;
        __syncthreads();
        if (threadIdx.y == 0) {
            float tot = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) tot += red[i][threadIdx.x];
            total += tot;
            if (cv) segmean[((long long)b * nseg + sgi) * C + c] = tot / (float)(tb - ta);  // ceil_mode partial window
        }
        __syncthreads();
    }
    if (threadIdx.y == 0 && cv) mean[(long long)b * C + c] = total / (float)T;
}

// ECAPA SE_Connect gate in ONE launch (ecapa_tdnn.py:113-126): gate[b] = sigmoid(W2 relu(W1 mean_T(x[b]) + b1) + b2).
// One block per 2 utterances: (1) mean over T with 16-byte loads (all 512 threads), (2) fc1: one warp per hidden unit, lanes
// over C (coalesced W1 rows, both utterances share each weight read), (3) fc2 from a TRANSPOSED W2 ([H][C]) so consecutive
// threads read consecutive weights.  Replaces the mean + split-K fc1 + reduce + fc2 launches (4 latency-bound launches).
template <int H>
__global__ void __launch_bounds__(512) se_gate_kernel(const void* __restrict__ x, int dt, int B, int T, int C, long long ld,
                                                      const float* __restrict__ W1, const float* __restrict__ b1,
                                                      const float* __restrict__ W2t, const float* __restrict__ b2,
                                                      float* __restrict__ gate /*[B][C]*/,
                                                      const float* __restrict__ colsum /* WsEpi::colsum or null */,
                                                      const int* __restrict__ lens /* length-masked batch or null */) {
    extern __shared__ float sm[];
    float* mean = sm;              // [2][C]
    float* part = mean + 2 * C;    // [slices][2][C] partial sums of the T slices (slices * C = 4096 floats)
    float* hid = part + 8192;      // [2][H]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int b0 = blockIdx.x * 2;
    const int nb = min(2, B - b0);
    const int groups = C >> 3;                 // 8-channel groups (C=1024 -> 128 groups x 4 T slices, C=512 -> 64 x 8)
    const int slices = 512 / groups;
    const int sl = tid / groups, gi = tid % groups;
    if (colsum != nullptr) {
        // the producing conv already summed its output per 64-position unit (two utterance slots per unit)
        for (int i = tid; i < nb * C; i += 512) {
            const int u = i / C, c = i % C, b = b0 + u;
            const int first = (b * T) >> 6, last = ((b + 1) * T - 1) >> 6;
            float sacc = 0.f;
            for (int un = first; un <= last; ++un) {
                const int slot = ((un << 6) / T == b) ? 0 : 1;
                sacc += colsum[(long long)(2 * un + slot) * C + c];
            }
            mean[u * C + c] = sacc / (float)T;
        }
    }
    for (int u = 0; u < nb && colsum == nullptr; ++u) {
        float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        const long long base = (long long)(b0 + u) * T * ld + gi * 8;
        const int Tu = lens != nullptr ? max(1, min(T, lens[b0 + u])) : T;
        for (int t = sl; t < Tu; t += slices) {
            float v[8];
            ws_ldv8(x, dt, base + (long long)t * ld, v);
#pragma unroll
            for (int k = 0; k < 8; ++k) a[k] += v[k];
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) part[(sl * 2 + u) * C + gi * 8 + k] = a[k];
    }
    __syncthreads();
    for (int i = tid; i < nb * C && colsum == nullptr; i += 512) {
        const int u = i / C, c = i % C;
        float s = 0.f;
        for (int k = 0; k < slices; ++k) s += part[(k * 2 + u) * C + c];   // fixed order: deterministic
        mean[u * C + c] = s / (float)(lens != nullptr ? max(1, min(T, lens[b0 + u])) : T);
    }
    __syncthreads();
    // fc1: two hidden units per warp pass, 16-byte weight loads (C % 128 == 0): 4x fewer dependent-latency steps
    for (int h = 2 * warp; h < H; h += 32) {
        const float4* w0 = reinterpret_cast<const float4*>(W1 + (long long)h * C);
        const float4* w1 = reinterpret_cast<const float4*>(W1 + (long long)(h + 1) * C);
        float a00 = 0.f, a01 = 0.f, a10 = 0.f, a11 = 0.f;
#pragma unroll 4
        for (int c4 = lane; c4 < (C >> 2); c4 += 32) {
            const float4 x0 = __ldg(w0 + c4), x1 = __ldg(w1 + c4);
            const float4 m0 = *reinterpret_cast<const float4*>(mean + 4 * c4);
            const float4 m1 = *reinterpret_cast<const float4*>(mean + C + 4 * c4);
            a00 = fmaf(x0.x, m0.x, a00); a00 = fmaf(x0.y, m0.y, a00); a00 = fmaf(x0.z, m0.z, a00); a00 = fmaf(x0.w, m0.w, a00);
            a01 = fmaf(x0.x, m1.x, a01); a01 = fmaf(x0.y, m1.y, a01); a01 = fmaf(x0.z, m1.z, a01); a01 = fmaf(x0.w, m1.w, a01);
            a10 = fmaf(x1.x, m0.x, a10); a10 = fmaf(x1.y, m0.y, a10); a10 = fmaf(x1.z, m0.z, a10); a10 = fmaf(x1.w, m0.w, a10);
            a11 = fmaf(x1.x, m1.x, a11); a11 = fmaf(x1.y, m1.y, a11); a11 = fmaf(x1.z, m1.z, a11); a11 = fmaf(x1.w, m1.w, a11);
        }
        a00 = warp_sum(a00); a01 = warp_sum(a01); a10 = warp_sum(a10); a11 = warp_sum(a11);
        if (lane == 0) {
            hid[h] = fmaxf(a00 + b1[h], 0.f); hid[H + h] = fmaxf(a01 + b1[h], 0.f);
            hid[h + 1] = fmaxf(a10 + b1[h + 1], 0.f); hid[H + h + 1] = fmaxf(a11 + b1[h + 1], 0.f);
        }
    }
    __syncthreads();
    // fc2: 4 channels per thread (16-byte loads of the transposed weights); threads beyond C/4 split the hidden range
    {
        const int nq = C >> 2;                    // channel quads
        const int parts = 512 / nq;               // 2 (C=1024), 4 (C=512), 8 (C=256); 1 for C=2048 (two rounds)
        float* acc = part;                        // [parts][2][C] partial sums (part is free after the squeeze)
        for (int q0 = 0; q0 < nq; q0 += 512) {
            const int q = q0 + (parts > 0 ? tid % nq : tid), hp = parts > 0 ? tid / nq : 0;
            const int np = parts > 0 ? parts : 1;
            if (q < nq) {
                const int hb = hp * (H / np), he = hb + H / np;
                float a0[4] = {0.f, 0.f, 0.f, 0.f}, a1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 8
                for (int h = hb; h < he; ++h) {
                    const float4 wv = __ldg(reinterpret_cast<const float4*>(W2t + (long long)h * C) + q);
                    const float h0 = hid[h], h1 = hid[H + h];
                    a0[0] = fmaf(wv.x, h0, a0[0]); a0[1] = fmaf(wv.y, h0, a0[1]); a0[2] = fmaf(wv.z, h0, a0[2]); a0[3] = fmaf(wv.w, h0, a0[3]);
                    a1[0] = fmaf(wv.x, h1, a1[0]); a1[1] = fmaf(wv.y, h1, a1[1]); a1[2] = fmaf(wv.z, h1, a1[2]); a1[3] = fmaf(wv.w, h1, a1[3]);
                }
                if (np == 1) {
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const int c = 4 * q + k;
                        gate[(long long)b0 * C + c] = 1.f / (1.f + expf(-(a0[k] + b2[c])));
                        if (nb > 1) gate[(long long)(b0 + 1) * C + c] = 1.f / (1.f + expf(-(a1[k] + b2[c])));
                    }
                } else {
#pragma unroll
                    for (int k = 0; k < 4; ++k) { acc[(hp * 2) * C + 4 * q + k] = a0[k]; acc[(hp * 2 + 1) * C + 4 * q + k] = a1[k]; }
                }
            }
        }
        if (parts > 1) {
            __syncthreads();
            for (int i = tid; i < nb * C; i += 512) {
                const int u = i / C, c = i % C;
                float a = b2[c];
                for (int k = 0; k < parts; ++k) a += acc[(k * 2 + u) * C + c];   // fixed order
                gate[(long long)(b0 + u) * C + c] = 1.f / (1.f + expf(-a));
            }
        }
    }
}

// CAM++ context gate in one launch (campplus.py:108-135): per utterance, mean over T + per-100-frame segment means of
// h (C=128), then for every segment  gate = sigmoid(W2 relu(W1 (mean + segmean) + b1) + b2).  One block per utterance;
// replaces seg_means + 2 tiny FC launches (3 latency-bound launches per dense layer, 52 layers).
template <int C, int H, int G>
__global__ void __launch_bounds__(256) cam_gate_kernel(const void* __restrict__ x, int dt, int T, long long ld, int seg_len,
                                                       const float* __restrict__ W1, const float* __restrict__ b1,
                                                       const float* __restrict__ W2, const float* __restrict__ b2,
                                                       float* __restrict__ gate /*[B][nseg][G]*/) {
    extern __shared__ float sm[];
    const int nseg = (T + seg_len - 1) / seg_len;
    float* w1s = sm;                  // [H][C] staged once (all loads in flight) instead of latency-bound __ldg chains
    float* ssum = w1s + H * C;        // [nseg][C] segment sums -> context vectors
    float* part = ssum + nseg * C;    // [16][C] partial sums of the 16 T-slices
    float* hid = part + 16 * C;       // [nseg][H]
    float* tot = hid + nseg * H;      // [C]
    const int b = blockIdx.x, tid = threadIdx.x;
    {
        const float4* src = reinterpret_cast<const float4*>(W1);
        float4* dst = reinterpret_cast<float4*>(w1s);
        for (int i = tid; i < H * C / 4; i += 256) dst[i] = __ldg(src + i);
    }
    const int c8 = (tid & 15) * 8, ts = tid >> 4;  // 16 groups of 8 channels x 16 T-slices
    const long long base = (long long)b * T * ld;
    for (int sg = 0; sg < nseg; ++sg) {
        const int ta = sg * seg_len, tb = min(T, ta + seg_len);
        float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        for (int t = ta + ts; t < tb; t += 16) {
            float v[8];
            ws_ldv8(x, dt, base + (long long)t * ld + c8, v);
#pragma unroll
            for (int k = 0; k < 8; ++k) a[k] += v[k];
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) part[ts * C + c8 + k] = a[k];
        __syncthreads();
        if (tid < C) {
            float t_ = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) t_ += part[i * C + tid];
            ssum[sg * C + tid] = t_;
        }
        __syncthreads();
    }
    if (tid < C) {
        float t_ = 0.f;
        for (int sg = 0; sg < nseg; ++sg) t_ += ssum[sg * C + tid];
        tot[tid] = t_ / (float)T;
    }
    __syncthreads();
    for (int i = tid; i < nseg * C; i += 256) {
        const int sg = i / C, c = i % C;
        const int cnt = min(T, (sg + 1) * seg_len) - sg * seg_len;   // ceil_mode partial window divides by its own count
        ssum[i] = ssum[i] / (float)cnt + tot[c];
    }
    __syncthreads();
    const int warp = tid >> 5, lane = tid & 31;
    for (int o = warp; o < nseg * H; o += 8) {       // hidden = relu(W1 ctx + b1): one warp per output, lanes over C
        const int sg = o / H, h = o % H;
        float a = 0.f;
#pragma unroll
        for (int c = lane; c < C; c += 32) a = fmaf(w1s[h * C + c], ssum[sg * C + c], a);
        a = warp_sum(a);
        if (lane == 0) hid[o] = fmaxf(a + b1[h], 0.f);
    }
    __syncthreads();
    for (int o = tid; o < nseg * G; o += 256) {      // gate: one thread per output, W2 row (H floats) read as float4
        const int sg = o / G, g = o % G;
        const float4* w = reinterpret_cast<const float4*>(W2 + g * H);
        float a = b2[g];
#pragma unroll
        for (int h4 = 0; h4 < H / 4; ++h4) {
            const float4 q = __ldg(w + h4);
            a = fmaf(q.x, hid[sg * H + 4 * h4], a); a = fmaf(q.y, hid[sg * H + 4 * h4 + 1], a);
            a = fmaf(q.z, hid[sg * H + 4 * h4 + 2], a); a = fmaf(q.w, hid[sg * H + 4 * h4 + 3], a);
        }
        gate[((long long)b * nseg + sg) * G + g] = 1.f / (1.f + expf(-a));
    }
}

// Length-masked batches: zero the rows t >= lens[b] of a channels-last tensor [B][F][T][ld] (channels [0, C)) so that the
// next time-mixing op sees the zero padding the reference's unpadded forward sees.  One block per (b, f) row strip; the
// cost is proportional to the padding only.
__global__ void __launch_bounds__(256) zero_tail_kernel(void* __restrict__ x, float* __restrict__ lo, int dt, int F, int T,
                                                        int C, long long ld, const int* __restrict__ lens) {
    const int b = blockIdx.y, f = blockIdx.x;
    const int t0 = max(0, min(T, lens[b]));
    const int es = dt == WS_F32 ? 4 : 2, cpr = C * es / 16;          // 16-byte chunks per row
    const long long n = (long long)(T - t0) * cpr;
    char* base = (char*)x + (((long long)b * F + f) * T + t0) * ld * es;
    char* base_lo = lo ? (char*)lo + (((long long)b * F + f) * T + t0) * ld * 4 : nullptr;
    for (long long i = threadIdx.x; i < n; i += 256) {
        const long long r = i / cpr, c = i - r * cpr;
        *reinterpret_cast<uint4*>(base + r * ld * es + c * 16) = make_uint4(0u, 0u, 0u, 0u);
        if (base_lo) *reinterpret_cast<uint4*>(base_lo + r * ld * 4 + c * 16) = make_uint4(0u, 0u, 0u, 0u);
    }
}
// lens[k + 1][b] = (lens[k][b] - 1) / 2 + 1 (stride-2 convs with kernel 3 / pad 1 or kernel 5 / pad 2), k < levels - 1;
// level 0 is clamped to [1, T]
__global__ void lens_derive_kernel(int* __restrict__ lens, int B, int T, int levels) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    int l = max(1, min(T, lens[b]));
    lens[b] = l;
    for (int k = 1; k < levels; ++k) { l = (l - 1) / 2 + 1; lens[k * B + b] = l; }
}
// frames of an utterance of n samples (snip_edges, frames of frame_len samples every shift samples)
// (clamped to [1, Tmax]: an utterance shorter than one frame is the caller's error, the reference's fbank fails on it too)
__global__ void frames_from_samples_kernel(const int* __restrict__ nsamp, int* __restrict__ lens, int B, int Tmax, int frame_len,
                                           int shift) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < B) lens[b] = max(1, min(Tmax, nsamp[b] < frame_len ? 0 : 1 + (nsamp[b] - frame_len) / shift));
}

inline const char* last_err() {
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}
inline int grid_for(long long n, int block, int cap = 0) {
    if (cap <= 0) cap = ws_num_sms() * 16;
    long long g = (n + block - 1) / block;
    if (g < 1) g = 1;
    return (int)(g > cap ? cap : g);
}

}  // namespace

const char* ws_launch_convert(const WsConvert& a, cudaStream_t s) {
    convert_kernel<<<grid_for(a.n, 256), 256, 0, s>>>(a.in, a.out, a.lo, a.dt, a.n);
    return last_err();
}

int ws_tstats_kernel(const WsTstats& a) {
    const WsView& x = a.x;
    if (a.std_off < 0 && x.F == 1 && a.pre_scale == nullptr && a.odt == WS_F32 && x.C % 8 == 0 && a.lens == nullptr) return WS_TSTATS_TMEAN8;
    if (x.dt != WS_F32 && x.C % 8 == 0 && x.ld % 8 == 0 && ((uintptr_t)x.p & 15) == 0) return WS_TSTATS_8;
    return WS_TSTATS_SCALAR;
}

const char* ws_launch_tstats(const WsTstats& a, cudaStream_t s) {
    const WsView& x = a.x;
    if (a.kernel == WS_TSTATS_TMEAN8) {
        dim3 g8((x.C + 511) / 512, x.B), b8(64, 8);
        tmean8_kernel<<<g8, b8, 0, s>>>(x.p, x.dt, x.T, x.C, x.ld, (float*)a.out, a.out_ld);
        return last_err();
    }
    if (a.kernel == WS_TSTATS_8) {
        dim3 g8((x.C + 127) / 128, x.F, x.B), b8(16, 16);
        if (x.dt == WS_BF16) tstats8_kernel<WS_BF16><<<g8, b8, 0, s>>>(x.p, x.F, x.T, x.C, x.ld, a.pre_scale, a.pre_shift, a.out, a.odt, a.out_ld, a.std_off, a.eps, a.lens);
        else tstats8_kernel<WS_F16><<<g8, b8, 0, s>>>(x.p, x.F, x.T, x.C, x.ld, a.pre_scale, a.pre_shift, a.out, a.odt, a.out_ld, a.std_off, a.eps, a.lens);
        return last_err();
    }
    dim3 grid((x.C + 31) / 32, x.F, x.B), block(32, 8);
    tstats_kernel<<<grid, block, 0, s>>>(x.p, x.dt, x.F, x.T, x.C, x.ld, a.pre_scale, a.pre_shift, a.out, a.odt, a.out_ld, a.std_off, a.eps, a.lens);
    return last_err();
}

static dim3 linear_rows_grid(const WsLinear& a) {
    const bool big = a.kernel == WS_LINEAR_ROWS64;
    return dim3(big ? (a.O + 63) / 64 : (a.O + 31) / 32, big ? (a.R + 63) / 64 : (a.R + 15) / 16, a.nsplit < 1 ? 1 : a.nsplit);
}

void ws_linear_rows_plan(WsLinear& a, int sms) {
    // the 64x64-tile kernel serves FC layers with enough rows and outputs to fill its tile and 16-byte aligned rows
    const bool big = a.R >= 48 && a.O >= 48 && a.I % 4 == 0 && a.in_ld % 4 == 0 && (a.in2 == nullptr || a.in2_ld % 4 == 0);
    a.kernel = big ? WS_LINEAR_ROWS64 : WS_LINEAR_ROWS16;
    a.nsplit = 1;
    const dim3 g = linear_rows_grid(a);
    const int blocks = (int)(g.x * g.y);
    if (big) while (blocks * a.nsplit < sms && a.I / (a.nsplit * 2) >= 96 && a.nsplit < 32) a.nsplit *= 2;
    else while (blocks * a.nsplit < 2 * sms && a.I / (a.nsplit * 2) >= 128 && a.nsplit < 16) a.nsplit *= 2;
}

const char* ws_launch_linear_rows(const WsLinear& a, cudaStream_t s) {
    const dim3 grid = linear_rows_grid(a);
    auto kern = a.kernel == WS_LINEAR_ROWS64 ? linear_rows64_kernel : linear_rows_kernel;
    const int rpb = a.rows_per_b < 1 ? 1 : a.rows_per_b;
    if (grid.z == 1) {
        kern<<<grid, 256, 0, s>>>(a.in, a.in_ld, a.in2, a.in2_ld, rpb, a.W, a.bias, a.out, a.out_ld, a.R, a.I, a.O, a.act);
        return last_err();
    }
    if (a.wsp == nullptr) return "linear_rows: split-K needs a workspace";
    kern<<<grid, 256, 0, s>>>(a.in, a.in_ld, a.in2, a.in2_ld, rpb, a.W, nullptr, a.wsp, a.O, a.R, a.I, a.O, WS_ACT_NONE);
    const long long n = (long long)a.R * a.O;
    linear_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(a.wsp, a.nsplit, a.bias, a.out, a.out_ld, a.R, a.O, a.act);
    return last_err();
}

const char* ws_launch_scale_residual(const WsScaleResidual& a, cudaStream_t s) {
    const int B = a.x.B, T = a.x.T, C = a.x.C;
    if (C % 8 != 0) return "scale_residual: C must be a multiple of 8";
    const long long nvec = (long long)B * T * (C / 8);
    if (nvec >= (1LL << 31)) return "scale_residual: tensor too large for 32-bit vector indices";
    const int g = grid_for(nvec, 256);
    const WsView &x = a.x, &r = a.res, &o = a.out;
    if (x.dt == WS_BF16) scale_residual_kernel<WS_BF16><<<g, 256, 0, s>>>(x.p, x.ld, a.gate, r.p, r.ld, o.p, (float*)o.plo, o.ld, T, C, nvec);
    else if (x.dt == WS_F16) scale_residual_kernel<WS_F16><<<g, 256, 0, s>>>(x.p, x.ld, a.gate, r.p, r.ld, o.p, (float*)o.plo, o.ld, T, C, nvec);
    else scale_residual_kernel<WS_F32><<<g, 256, 0, s>>>(x.p, x.ld, a.gate, r.p, r.ld, o.p, (float*)o.plo, o.ld, T, C, nvec);
    return last_err();
}

const char* ws_launch_aff_combine(const WsAffCombine& a, cudaStream_t s) {
    const WsView &x = a.x, &y = a.y, &t = a.t, &o = a.out;
    const int C = x.C;
    if (C % 8 != 0 || x.ld % 8 != 0 || y.ld % 8 != 0 || t.ld % 8 != 0 || o.ld % 8 != 0) return "aff_combine: C and the row pitches must be multiples of 8";
    const long long nvec = x.npos() * (C / 8);
    if (nvec >= (1LL << 31)) return "aff_combine: tensor too large for 32-bit vector indices";
    const int g = grid_for(nvec, 256);
    float* lo = (float*)o.plo;
    if (x.dt == WS_BF16) aff_combine_kernel<WS_BF16><<<g, 256, 0, s>>>(x.p, x.ld, y.p, y.ld, t.p, t.ld, o.p, lo, o.ld, C, nvec);
    else if (x.dt == WS_F16) aff_combine_kernel<WS_F16><<<g, 256, 0, s>>>(x.p, x.ld, y.p, y.ld, t.p, t.ld, o.p, lo, o.ld, C, nvec);
    else aff_combine_kernel<WS_F32><<<g, 256, 0, s>>>(x.p, x.ld, y.p, y.ld, t.p, t.ld, o.p, lo, o.ld, C, nvec);
    return last_err();
}

int ws_astp_stats_kernel(const WsAstpStats& a) {
    return a.x.C % 4 == 0 && a.x.ld % 4 == 0 && a.x.dt != WS_F32 && a.x.T <= 256 ? WS_ASTP_STATS4 : WS_ASTP_STATS_SCALAR;
}

const char* ws_launch_astp_stats(const WsAstpStats& a, cudaStream_t s) {
    const WsView& x = a.x;
    if (x.C % 2 != 0) return "astp_stats: C must be even";
    if (a.kernel == WS_ASTP_STATS4) {
        dim3 grid((x.C + 63) / 64, x.B), block(16, 32);
        if (x.dt == WS_BF16) astp_stats4_kernel<WS_BF16><<<grid, block, 0, s>>>(x.p, a.logits.p, x.T, x.C, x.ld, a.stats, a.var_floor, a.lens);
        else astp_stats4_kernel<WS_F16><<<grid, block, 0, s>>>(x.p, a.logits.p, x.T, x.C, x.ld, a.stats, a.var_floor, a.lens);
        return last_err();
    }
    dim3 grid((x.C + 63) / 64, x.B), block(32, 8);
    astp_stats_kernel<<<grid, block, 0, s>>>(x.p, a.logits.p, x.dt, x.T, x.C, x.ld, a.stats, a.var_floor, a.lens);
    return last_err();
}

const char* ws_launch_zero_tail(const WsZeroTail& a, cudaStream_t s) {
    const WsView& x = a.x;
    if ((x.C * (x.dt == WS_F32 ? 4 : 2)) % 16 != 0 || (x.ld * (x.dt == WS_F32 ? 4 : 2)) % 16 != 0) return "zero_tail: rows must be 16-byte multiples";
    zero_tail_kernel<<<dim3((unsigned)x.F, (unsigned)x.B), 256, 0, s>>>(x.p, (float*)x.plo, x.dt, x.F, x.T, x.C, x.ld, a.lens);
    return last_err();
}
const char* ws_launch_lens_derive(const WsLensDerive& a, cudaStream_t s) {
    lens_derive_kernel<<<(a.B + 127) / 128, 128, 0, s>>>(a.lens, a.B, a.T, a.levels);
    return last_err();
}
const char* ws_launch_frames_from_samples(const int* nsamp, int* lens, int B, int Tmax, int frame_len, int shift, cudaStream_t s) {
    frames_from_samples_kernel<<<(B + 127) / 128, 128, 0, s>>>(nsamp, lens, B, Tmax, frame_len, shift);
    return last_err();
}

const char* ws_launch_bnrelu(const WsBnRelu& a, cudaStream_t s) {
    const WsView &x = a.x, &o = a.out;
    const long long nvec = x.npos() * (x.C / 4);
    bnrelu_kernel<<<grid_for(nvec, 256), 256, 0, s>>>(x.p, x.ld, a.scale, a.shift, o.p, (float*)o.plo, o.ld, x.dt, x.C, nvec);
    return last_err();
}

const char* ws_launch_stem(const WsStem& a, cudaStream_t s) {
    const WsView& o = a.out;
    const int B = o.B, T = o.T, Fdim = o.F;
    const dim3 grid((unsigned)((T + 127) / 128), (unsigned)((Fdim + 7) / 8), (unsigned)B);
    if (B > 65535) return "stem conv: batch too large for one launch";
    if (o.C == 32) stem_kernel<32><<<grid, 128, 0, s>>>(a.feats, a.w9, a.shift, o.p, (float*)o.plo, o.dt, B, T, Fdim, a.lens);
    else if (o.C == 64) stem_kernel<64><<<grid, 128, 0, s>>>(a.feats, a.w9, a.shift, o.p, (float*)o.plo, o.dt, B, T, Fdim, a.lens);
    else return "stem conv supports 32 or 64 output channels";
    return last_err();
}

const char* ws_launch_seg_means(const WsSegMeans& a, cudaStream_t s) {
    const WsView& x = a.x;
    dim3 grid((x.C + 31) / 32, x.B), block(32, 8);
    seg_means_kernel<<<grid, block, 0, s>>>(x.p, x.dt, x.T, x.C, x.ld, a.seg_len, a.mean, a.segmean);
    return last_err();
}

const char* ws_launch_cam_gate(const WsCamGate& a, cudaStream_t s) {
    const WsView& x = a.x;
    const int C = x.C, H = a.H;
    if (C != 128 || H != 64 || a.G != 32) return "cam_gate: expected C=128, H=64, G=32 (CAM++ bn_channels / reduction / growth)";
    const int nseg = (x.T + a.seg_len - 1) / a.seg_len;
    const size_t smem = (size_t)(H * C + nseg * C + 16 * C + nseg * H + C) * sizeof(float);
    if (smem > 48 * 1024) return "cam_gate: utterance too long for the shared-memory context buffer";
    cam_gate_kernel<128, 64, 32><<<x.B, 256, smem, s>>>(x.p, x.dt, x.T, x.ld, a.seg_len, a.W1, a.b1, a.W2, a.b2, a.gate);
    return last_err();
}

const char* ws_launch_se_gate(const WsSeGate& a, cudaStream_t s) {
    const WsView& x = a.x;
    const int C = x.C, H = a.H;
    if (H != 128 || (C != 512 && C != 1024 && C != 2048 && C != 256)) return "se_gate: expected H=128 and C in {256,512,1024,2048}";
    const size_t smem = (size_t)(2 * C + 8192 + 2 * H) * sizeof(float);
    if (smem > 96 * 1024) return "se_gate: channel count too large for shared memory";
    if (a.colsum != nullptr && x.T < 128) return "se_gate: fused column sums need >= 128 frames per utterance";
    if (a.lens != nullptr && a.colsum != nullptr) return "se_gate: fused column sums are not available for length-masked batches";
    if (const char* m = ws_smem_opt_in<se_gate_kernel<128>>(96 * 1024)) return m;
    se_gate_kernel<128><<<(x.B + 1) / 2, 512, smem, s>>>(x.p, x.dt, x.B, x.T, C, x.ld, a.W1, a.b1, a.W2t, a.b2, a.gate, a.colsum, a.lens);
    return last_err();
}
