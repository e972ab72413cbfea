// Cosine trial scoring and S-norm / AS-norm cohort statistics on the GPU (SURVEY.md section 8(f) rank 2).
// Replaces wespeaker/bin/score.py:38-72 (trials_cosine_score: mean-subtract, cosine per listed trial) and
// wespeaker/bin/score_norm.py:26-37 (get_mean_std: L2-normalise, emb @ cohort.T, per-row top-N mean / std) plus the
// per-trial normalisation of score_norm.py:102-117.  Arithmetic in fp64 on fp32 embeddings (the reference runs numpy /
// sklearn in fp32); the N x M cohort score matrix is produced tile by tile by the PLDA fp64 GEMM (ws_plda.cu) into a
// caller-provided fp32 workspace and never leaves the device.
//
// Per-row top-N without sorting: 4-pass MSB radix select on order-preserving 32-bit keys finds the N-th largest score
// exactly; the sums then take every score above it plus as many copies of the threshold as are needed, which equals the
// sum over np.sort(row)[::-1][:N] whatever the order of ties.
#include <cstdint>

#include "../../include/wespeaker_b200.h"
#include "ws_host.h"
#include "ws_kernels.cuh"
#include "ws_select.cuh"

using namespace ws;

namespace {

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// one warp per row: unit[r] = (x[r] - mean) / |x[r] - mean|, norms[r] = |x[r] - mean|
__global__ void __launch_bounds__(256) unit_rows_kernel(const float* __restrict__ x, const double* __restrict__ mean_vec,
                                                        long long N, int D, double* __restrict__ unit,
                                                        double* __restrict__ norms) {
    const long long r = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (r >= N) return;
    const float* p = x + r * D;
    double ss = 0.0;
    for (int d = lane; d < D; d += 32) {
        const double v = (double)p[d] - (mean_vec != nullptr ? mean_vec[d] : 0.0);
        ss = fma(v, v, ss);
    }
    ss = warp_sum_d(ss);
    const double nrm = sqrt(ss);
    const double inv = nrm > 0.0 ? 1.0 / nrm : 0.0;   // zero vector -> zero row: cosine 0, as sklearn's cosine_similarity
    for (int d = lane; d < D; d += 32)
        unit[r * D + d] = ((double)p[d] - (mean_vec != nullptr ? mean_vec[d] : 0.0)) * inv;
    if (lane == 0 && norms != nullptr) norms[r] = nrm;
}

// one warp per trial: dot of two unit rows
__global__ void __launch_bounds__(256) cos_trials_kernel(const double* __restrict__ unit, const long long* __restrict__ ei,
                                                         const long long* __restrict__ ti, long long ntrials, int D,
                                                         double* __restrict__ out) {
    const long long r = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (r >= ntrials) return;
    const double* a = unit + ei[r] * D;
    const double* b = unit + ti[r] * D;
    double acc = 0.0;
    for (int d = lane; d < D; d += 32) acc = fma(a[d], b[d], acc);
    acc = warp_sum_d(acc);
    if (lane == 0) out[r] = acc;
}

// one block per row of the score tile: mean / population std of the top_n largest of M scores
__global__ void __launch_bounds__(256) topn_stats_kernel(const float* __restrict__ scores, long long M, int top_n,
                                                         double* __restrict__ mean_out, double* __restrict__ std_out) {
    __shared__ double red[2][8];
    const float* row = scores + (long long)blockIdx.x * M;
    const int tid = threadIdx.x;
    unsigned n_ties;
    const uint32_t thr_key = radix_select_kth(row, M, (unsigned)top_n, &n_ties);
    const double thr = (double)key_value(thr_key);
    double s1 = 0.0, s2 = 0.0;
    for (long long j = tid; j < M; j += 256) {
        const float v = row[j];
        if (order_key(v) > thr_key) { s1 += (double)v; s2 = fma((double)v, (double)v, s2); }
    }
    s1 = warp_sum_d(s1); s2 = warp_sum_d(s2);
    if ((tid & 31) == 0) { red[0][tid >> 5] = s1; red[1][tid >> 5] = s2; }
    __syncthreads();
    if (tid == 0) {
        double a = 0.0, b2 = 0.0;
        for (int i = 0; i < 8; ++i) { a += red[0][i]; b2 += red[1][i]; }
        const double ties = (double)n_ties;
        a += ties * thr; b2 += ties * thr * thr;
        const double n = (double)top_n;
        const double mean = a / n;
        const double var = b2 / n - mean * mean;
        mean_out[blockIdx.x] = mean;
        std_out[blockIdx.x] = sqrt(var > 0.0 ? var : 0.0);
    }
}

__global__ void asnorm_kernel(const double* __restrict__ s, const long long* __restrict__ ei,
                              const long long* __restrict__ ti, long long n, const double* __restrict__ em,
                              const double* __restrict__ es, const double* __restrict__ tm,
                              const double* __restrict__ ts, double* __restrict__ out) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const long long i = ei[k], j = ti[k];
    out[k] = 0.5 * ((s[k] - em[i]) / es[i] + (s[k] - tm[j]) / ts[j]);   // score_norm.py:104-107
}

inline int last_err(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) return 0;
    set_err(std::string(what) + ": " + cudaGetErrorString(e));
    return 1;
}
inline bool no_gpu(const char* what) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        set_err(std::string(what) + ": no CUDA device (the scorer has no CPU fallback)");
        return true;
    }
    return false;
}

}  // namespace

extern "C" {

int ws_score_unit_rows(const float* x_dev, long long N, int D, const double* mean_vec_dev, double* unit_dev,
                       double* norms_dev, void* stream) {
    if (!x_dev || !unit_dev || N < 0 || D <= 0) { set_err("ws_score_unit_rows: bad argument"); return 1; }
    if (no_gpu("ws_score_unit_rows")) return 1;
    if (N == 0) return 0;
    unit_rows_kernel<<<(unsigned)((N + 7) / 8), 256, 0, (cudaStream_t)stream>>>(x_dev, mean_vec_dev, N, D, unit_dev, norms_dev);
    return last_err("ws_score_unit_rows");
}

int ws_score_cosine_trials(const double* unit_dev, const long long* enroll_idx_dev, const long long* test_idx_dev,
                           long long ntrials, int D, double* out_dev, void* stream) {
    if (!unit_dev || !enroll_idx_dev || !test_idx_dev || !out_dev || ntrials < 0 || D <= 0) {
        set_err("ws_score_cosine_trials: bad argument"); return 1;
    }
    if (no_gpu("ws_score_cosine_trials")) return 1;
    if (ntrials == 0) return 0;
    cos_trials_kernel<<<(unsigned)((ntrials + 7) / 8), 256, 0, (cudaStream_t)stream>>>(unit_dev, enroll_idx_dev, test_idx_dev,
                                                                                  ntrials, D, out_dev);
    return last_err("ws_score_cosine_trials");
}

int ws_score_cohort_stats(const double* unit_emb_dev, long long N, const double* unit_cohort_dev, long long M, int D,
                          int top_n, float* work_dev, long long work_rows, double* mean_dev, double* std_dev,
                          void* stream) {
    if (!unit_emb_dev || !unit_cohort_dev || !work_dev || !mean_dev || !std_dev || N < 0 || M <= 0 || D <= 0 ||
        top_n <= 0 || work_rows <= 0) {
        set_err("ws_score_cohort_stats: bad argument"); return 1;
    }
    if (no_gpu("ws_score_cohort_stats")) return 1;
    const int n_eff = top_n < M ? top_n : (int)M;    // emb_cohort_score[:, :top_n] keeps all M columns when top_n > M
    cudaStream_t s = (cudaStream_t)stream;
    if (work_rows > 65535LL * 128) work_rows = 65535LL * 128;
    for (long long r0 = 0; r0 < N; r0 += work_rows) {
        const long long rows = (N - r0) < work_rows ? (N - r0) : work_rows;
        WS_CKS(ws_launch_dgemm_nt(unit_emb_dev + r0 * D, unit_cohort_dev, nullptr, nullptr, work_dev, 0, rows, M, D, M, s));
        topn_stats_kernel<<<(unsigned)rows, 256, 0, s>>>(work_dev, M, n_eff, mean_dev + r0, std_dev + r0);
        if (last_err("ws_score_cohort_stats")) return 1;
    }
    return 0;
}

int ws_score_asnorm(const double* scores_dev, const long long* enroll_idx_dev, const long long* test_idx_dev,
                    long long ntrials, const double* enroll_mean_dev, const double* enroll_std_dev,
                    const double* test_mean_dev, const double* test_std_dev, double* out_dev, void* stream) {
    if (!scores_dev || !enroll_idx_dev || !test_idx_dev || !enroll_mean_dev || !enroll_std_dev || !test_mean_dev ||
        !test_std_dev || !out_dev || ntrials < 0) {
        set_err("ws_score_asnorm: bad argument"); return 1;
    }
    if (no_gpu("ws_score_asnorm")) return 1;
    if (ntrials == 0) return 0;
    asnorm_kernel<<<(unsigned)((ntrials + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        scores_dev, enroll_idx_dev, test_idx_dev, ntrials, enroll_mean_dev, enroll_std_dev, test_mean_dev, test_std_dev,
        out_dev);
    return last_err("ws_score_asnorm");
}

}  // extern "C"
