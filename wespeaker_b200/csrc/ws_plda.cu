// Two-covariance PLDA log-likelihood-ratio scoring in fp64 (the reference is numpy fp64:
// wespeaker/utils/plda/two_cov_plda.py:156-184).  The per-trial formula is refactored into a GEMM:
//
//   LLR(i,j) = sum_d t_jd * (m_id / v_id)  -  1/2 sum_d t_jd^2 / v_id  +  r_i  +  c_j
//     m_i = n_i psi/(n_i psi + 1) * e_i ,  v_i = 1 + psi/(n_i psi + 1)
//     r_i = -1/2 (sum log v_i + sum m_i^2 / v_i) ,  c_j = 1/2 (sum log(psi+1) + sum t_j^2/(psi+1))
//
// With a constant enroll count n the second term only depends on j and moves into c_j (K = D); with per-speaker
// counts it is a second K-block (K = 2D): P_i = [m_i/v_i , -1/(2 v_i)], Q_j = [t_j , t_j^2].
// fp64 keeps |error| ~1e-13, far inside the 1e-5 budget which fp32 accumulators cannot guarantee (sums of
// magnitude ~256 have ulp 3e-5).  The H100 runs DFMA at half the FFMA rate, so this is DFMA-bound, not HBM-bound:
// 128x64 block tile, 8x4 register tile per thread, K streamed through shared memory.
#include "ws_kernels.cuh"
#include <cstdlib>

namespace {

constexpr int TM = 128, TN = 64, TK = 8;

__global__ void __launch_bounds__(256) dgemm_nt_kernel(const double* __restrict__ A, const double* __restrict__ Bm,
                                                       const double* __restrict__ rowc, const double* __restrict__ colc,
                                                       void* __restrict__ out, int out_is_f64, long long M, long long N,
                                                       int K, long long out_ld) {
    __shared__ double As[TK][TM + 2];
    __shared__ double Bs[TK][TN + 2];
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;  // tx -> 4 columns, ty -> 8 rows
    const long long m0 = (long long)blockIdx.y * TM, n0 = (long long)blockIdx.x * TN;
    const int arow = tid >> 1, ak = (tid & 1) * 4;
    const int brow = tid >> 2, bk = (tid & 3) * 2;
    const bool av = (m0 + arow) < M, bv = (n0 + brow) < N;
    const double* ap = A + (m0 + arow) * (long long)K + ak;
    const double* bp = Bm + (n0 + brow) * (long long)K + bk;
    double acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;
    for (int k0 = 0; k0 < K; k0 += TK) {
        double a[4] = {0, 0, 0, 0}, bb[2] = {0, 0};
        if (av) {
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (k0 + ak + j < K) a[j] = ap[k0 + j];
        }
        if (bv) {
#pragma unroll
            for (int j = 0; j < 2; ++j)
                if (k0 + bk + j < K) bb[j] = bp[k0 + j];
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < 4; ++j) As[ak + j][arow] = a[j];
#pragma unroll
        for (int j = 0; j < 2; ++j) Bs[bk + j][brow] = bb[j];
        __syncthreads();
#pragma unroll
        for (int k = 0; k < TK; ++k) {
            double av8[8], bv4[4];
#pragma unroll
            for (int i = 0; i < 8; ++i) av8[i] = As[k][ty * 8 + i];
#pragma unroll
            for (int j = 0; j < 4; ++j) bv4[j] = Bs[k][tx * 4 + j];
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fma(av8[i], bv4[j], acc[i][j]);
        }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const long long r = m0 + ty * 8 + i;
        if (r >= M) continue;
        const double rc = rowc != nullptr ? rowc[r] : 0.0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const long long c = n0 + tx * 4 + j;
            if (c >= N) continue;
            const double v = acc[i][j] + rc + (colc != nullptr ? colc[c] : 0.0);
            if (out_is_f64) ((double*)out)[r * out_ld + c] = v;
            else ((float*)out)[r * out_ld + c] = (float)v;
        }
    }
}

// ---------------------------------------------------------------------------------------------- DMMA variant
// Same GEMM on the fp64 tensor path (mma.sync.m8n8k4.f64): one instruction = 8x8x4 FMAs per warp instead of 32, which is
// what lets a kernel approach the DFMA peak (the FFMA-style loop above is instruction-issue bound at ~0.4 of it).
// 128x128 block tile, 8 warps of 32x64 (4 x 8 m8n8 tiles, 64 accumulator doubles per thread), K streamed in chunks of 16
// through a cp.async double buffer; shared rows are padded to 20 doubles so the 8-row x 4-column fragment loads of a
// half-warp hit 32 distinct banks.
constexpr int DBM = 128, DBN = 128, DBK = 16, DPITCH = 20;
constexpr int kDmmaSmem = 2 * (DBM + DBN) * DPITCH * 8;

__device__ __forceinline__ void dmma_8x8x4(double (&c)[2], double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                 : "+d"(c[0]), "+d"(c[1])
                 : "d"(a), "d"(b));
}
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}

template <int OUT_F64>
__global__ void __launch_bounds__(256) dgemm_nt_dmma_kernel(const double* __restrict__ A, const double* __restrict__ Bm,
                                                            const double* __restrict__ rowc, const double* __restrict__ colc,
                                                            void* __restrict__ out, long long M, long long N, int K,
                                                            long long out_ld) {
    extern __shared__ __align__(16) double dsm[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wm = warp & 3, wn = warp >> 2;               // 4 warps along M (32 rows each) x 2 along N (64 columns each)
    const long long m0 = (long long)blockIdx.y * DBM, n0 = (long long)blockIdx.x * DBN;
    // loader: (128 + 128) rows x 8 chunks of 2 doubles per stage; rows past M / N are clamped (their outputs are never stored)
    const double* src[8];
    int dst[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int idx = tid + 256 * (i & 3), row = idx >> 3, ch = idx & 7;
        if (i < 4) {
            const long long g = m0 + row < M ? m0 + row : M - 1;
            src[i] = A + g * (long long)K + ch * 2;
            dst[i] = row * DPITCH + ch * 2;
        } else {
            const long long g = n0 + row < N ? n0 + row : N - 1;
            src[i] = Bm + g * (long long)K + ch * 2;
            dst[i] = (DBM + row) * DPITCH + ch * 2;
        }
    }
    auto load_stage = [&](int st, int k0) {
        double* base = dsm + st * (DBM + DBN) * DPITCH;
#pragma unroll
        for (int i = 0; i < 8; ++i) cp_async16(base + dst[i], src[i] + k0);
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    double acc[4][8][2];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
    const int nk = K / DBK;
    load_stage(0, 0);
    const int fr = lane >> 2, fk = lane & 3;                // fragment row (A: m, B: n) and k of this lane
    for (int kc = 0; kc < nk; ++kc) {
        if (kc + 1 < nk) {
            load_stage((kc + 1) & 1, (kc + 1) * DBK);
            asm volatile("cp.async.wait_group 1;" ::: "memory");
        } else {
            asm volatile("cp.async.wait_group 0;" ::: "memory");
        }
        __syncthreads();
        const double* As = dsm + (kc & 1) * (DBM + DBN) * DPITCH + (wm * 32 + fr) * DPITCH + fk;
        const double* Bs = dsm + (kc & 1) * (DBM + DBN) * DPITCH + (DBM + wn * 64 + fr) * DPITCH + fk;
#pragma unroll
        for (int k4 = 0; k4 < DBK / 4; ++k4) {
            double a[4], b[8];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = As[i * 8 * DPITCH + k4 * 4];
#pragma unroll
            for (int j = 0; j < 8; ++j) b[j] = Bs[j * 8 * DPITCH + k4 * 4];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) dmma_8x8x4(acc[i][j], a[i], b[j]);
        }
        __syncthreads();
    }
    // accumulator fragment: rows lane/4 of each m8 tile, columns 2*(lane%4) + {0,1} of each n8 tile -> 8-byte (fp32) or
    // 16-byte (fp64) stores, one full 32-byte sector per row and tile
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const long long r = m0 + wm * 32 + i * 8 + fr;
        if (r >= M) continue;
        const double rc = rowc != nullptr ? rowc[r] : 0.0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const long long c = n0 + wn * 64 + j * 8 + fk * 2;
            if (c >= N) continue;
            const double v0 = acc[i][j][0] + rc + (colc != nullptr ? colc[c] : 0.0);
            if (c + 1 < N) {
                const double v1 = acc[i][j][1] + rc + (colc != nullptr ? colc[c + 1] : 0.0);
                if (OUT_F64) {
                    double* o = (double*)out + r * out_ld + c;
                    if ((((uintptr_t)o) & 15) == 0) *reinterpret_cast<double2*>(o) = make_double2(v0, v1);
                    else { o[0] = v0; o[1] = v1; }
                } else {
                    float* o = (float*)out + r * out_ld + c;
                    if ((((uintptr_t)o) & 7) == 0) *reinterpret_cast<float2*>(o) = make_float2((float)v0, (float)v1);
                    else { o[0] = (float)v0; o[1] = (float)v1; }
                }
            } else {
                if (OUT_F64) ((double*)out)[r * out_ld + c] = v0;
                else ((float*)out)[r * out_ld + c] = (float)v0;
            }
        }
    }
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__global__ void f32_to_f64_kernel(const float* __restrict__ in, double* __restrict__ out, long long n) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += stride) out[i] = (double)in[i];
}

// one warp per row
__global__ void center_norm_kernel(double* __restrict__ x, const double* __restrict__ mean_vec, long long N, int D,
                                   int do_norm) {
    const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (r >= N) return;
    double* p = x + r * D;
    double ss = 0.0;
    for (int d = lane; d < D; d += 32) {
        double v = p[d] - (mean_vec != nullptr ? mean_vec[d] : 0.0);
        p[d] = v;
        ss = fma(v, v, ss);
    }
    if (do_norm) {
        ss = warp_sum_d(ss);
        const double sc = sqrt((double)D) / sqrt(ss);
        for (int d = lane; d < D; d += 32) p[d] *= sc;
    }
}

__global__ void prep_enroll_kernel(const double* __restrict__ e, const int* __restrict__ counts, int const_n,
                                   const double* __restrict__ psi, long long N, int D, int K, double* __restrict__ P,
                                   double* __restrict__ rowc) {
    const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (r >= N) return;
    const double n = counts != nullptr ? (double)counts[r] : (double)const_n;
    double acc = 0.0;
    for (int d = lane; d < D; d += 32) {
        const double ps = psi[d];
        const double den = n * ps + 1.0;
        const double m = n * ps / den * e[r * D + d];
        const double v = 1.0 + ps / den;
        P[r * K + d] = m / v;
        if (K == 2 * D) P[r * K + D + d] = -0.5 / v;
        acc += log(v) + m * m / v;
    }
    acc = warp_sum_d(acc);
    if (lane == 0) rowc[r] = -0.5 * acc;
}

__global__ void prep_test_kernel(const double* __restrict__ t, const double* __restrict__ psi, int const_n,
                                 long long M, int D, int K, double* __restrict__ Q, double* __restrict__ colc) {
    const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (r >= M) return;
    double acc = 0.0;
    for (int d = lane; d < D; d += 32) {
        const double ps = psi[d];
        const double tv = t[r * D + d];
        Q[r * K + d] = tv;
        acc += 0.5 * (log(ps + 1.0) + tv * tv / (ps + 1.0));
        if (K == 2 * D) {
            Q[r * K + D + d] = tv * tv;
        } else {
            const double n = (double)const_n;
            const double v = 1.0 + ps / (n * ps + 1.0);
            acc -= 0.5 * tv * tv / v;
        }
    }
    acc = warp_sum_d(acc);
    if (lane == 0) colc[r] = acc;
}

__global__ void trials_kernel(const double* __restrict__ P, const double* __restrict__ rowc,
                              const double* __restrict__ Q, const double* __restrict__ colc,
                              const long long* __restrict__ ei, const long long* __restrict__ ti, long long ntrials,
                              int K, double* __restrict__ out) {
    const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (r >= ntrials) return;
    const long long i = ei[r], j = ti[r];
    double acc = 0.0;
    for (int k = lane; k < K; k += 32) acc = fma(P[i * K + k], Q[j * K + k], acc);
    acc = warp_sum_d(acc);
    if (lane == 0) out[r] = acc + rowc[i] + colc[j];
}

inline const char* last_err() {
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}
inline unsigned rows_grid(long long rows) { return (unsigned)((rows + 7) / 8); }

}  // namespace

const char* ws_launch_f32_to_f64(const float* in, double* out, long long n, cudaStream_t s) {
    long long g = (n + 255) / 256;
    if (g > ws_num_sms() * 32) g = ws_num_sms() * 32;
    if (g < 1) g = 1;
    f32_to_f64_kernel<<<(unsigned)g, 256, 0, s>>>(in, out, n);
    return last_err();
}

const char* ws_launch_dgemm_nt(const double* A, const double* Bm, const double* rowc, const double* colc, void* out,
                               int out_is_f64, long long M, long long N, int K, long long out_ld, cudaStream_t s) {
    if (M <= 0 || N <= 0) return nullptr;
    const long long gy = (M + TM - 1) / TM, gx = (N + TN - 1) / TN;
    if (gy > 65535) return "dgemm_nt: M too large for one launch (tile the enroll rows)";
    // fp64 tensor path (mma.sync m8n8k4) whenever K is a multiple of the 16-deep k chunk and the operand rows are 16-byte
    // aligned; WS_PLDA_SIMT=1 keeps the FFMA-style kernel as a cross-check
    if (K % DBK == 0 && K >= DBK && ((uintptr_t)A & 15) == 0 && ((uintptr_t)Bm & 15) == 0 && getenv("WS_PLDA_SIMT") == nullptr) {
        const long long dy = (M + DBM - 1) / DBM, dx = (N + DBN - 1) / DBN;
        if (dy > 65535) return "dgemm_nt: M too large for one launch (tile the enroll rows)";
        dim3 dgrid((unsigned)dx, (unsigned)dy);
        if (const char* m = out_is_f64 ? ws_smem_opt_in<dgemm_nt_dmma_kernel<1>>(kDmmaSmem) : ws_smem_opt_in<dgemm_nt_dmma_kernel<0>>(kDmmaSmem))
            return m;
        if (out_is_f64) dgemm_nt_dmma_kernel<1><<<dgrid, 256, kDmmaSmem, s>>>(A, Bm, rowc, colc, out, M, N, K, out_ld);
        else dgemm_nt_dmma_kernel<0><<<dgrid, 256, kDmmaSmem, s>>>(A, Bm, rowc, colc, out, M, N, K, out_ld);
        return last_err();
    }
    dim3 grid((unsigned)gx, (unsigned)gy);
    dgemm_nt_kernel<<<grid, 256, 0, s>>>(A, Bm, rowc, colc, out, out_is_f64, M, N, K, out_ld);
    return last_err();
}

const char* ws_launch_plda_center_norm(double* x, const double* mean_vec, long long N, int D, int do_norm,
                                       cudaStream_t s) {
    if (N <= 0) return nullptr;
    center_norm_kernel<<<rows_grid(N), 256, 0, s>>>(x, mean_vec, N, D, do_norm);
    return last_err();
}
const char* ws_launch_plda_rownorm(double* x, long long N, int D, cudaStream_t s) {
    return ws_launch_plda_center_norm(x, nullptr, N, D, 1, s);
}
const char* ws_launch_plda_prep_enroll(const double* e, const int* counts, int const_n, const double* psi,
                                       long long N, int D, int K, double* P, double* rowc, cudaStream_t s) {
    if (N <= 0) return nullptr;
    prep_enroll_kernel<<<rows_grid(N), 256, 0, s>>>(e, counts, const_n, psi, N, D, K, P, rowc);
    return last_err();
}
const char* ws_launch_plda_prep_test(const double* t, const double* psi, int const_n, long long M, int D, int K,
                                     double* Q, double* colc, cudaStream_t s) {
    if (M <= 0) return nullptr;
    prep_test_kernel<<<rows_grid(M), 256, 0, s>>>(t, psi, const_n, M, D, K, Q, colc);
    return last_err();
}
const char* ws_launch_plda_trials(const double* P, const double* rowc, const double* Q, const double* colc,
                                  const long long* ei, const long long* ti, long long ntrials, int K, double* out,
                                  cudaStream_t s) {
    if (ntrials <= 0) return nullptr;
    trials_kernel<<<rows_grid(ntrials), 256, 0, s>>>(P, rowc, Q, colc, ei, ti, ntrials, K, out);
    return last_err();
}
