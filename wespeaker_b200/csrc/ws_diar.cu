// Speaker diarization around the engine's forward (wespeaker/cli/speaker.py:213-270), the two device stages that are not the
// model: (A) sub-segment windows cut from one fbank pass per speech segment - gather, cyclic tiling to window_fs rows and
// CMN, diar/extract_emb.py:55-83 + cli/speaker.py:110-112 - and (B) the spectral clusterer's matrix up to the
// eigendecomposition - cosine affinity, per-row top-k pruning, symmetrisation, Laplacian, diar/spectral_clusterer.py:35-56.
//
// (B) never forms the fp32 similarity 0.5 (1 + cos): that map is monotone, so the k largest of a row are chosen on the
// cosines (fp64 GEMM of unit rows, tile by tile, as the AS-norm cohort statistics do).  The pruned matrix has entries in
// {0, 1}, its symmetrisation in {0, 1/2, 1} and the degrees are multiples of 1/2, so the fp64 Laplacian written here holds
// exactly the numbers of the reference's fp32 one and no sum depends on its order.
#include <cstdint>

#include "../../include/wespeaker_b200.h"
#include "ws_host.h"
#include "ws_kernels.cuh"
#include "ws_select.cuh"

using namespace ws;

namespace {

constexpr int kMaxFeatDim = 256;

// One CTA per table entry: mean over rows [row0, row0 + len) of each column, summed in a fixed order (row groups of the
// block in sequence, then the groups in sequence) in fp64.  An entry outside [0, total_rows) gives zeros.
__global__ void __launch_bounds__(256) col_means_kernel(const float* __restrict__ feats, long long total_rows, int F,
                                                        const int* __restrict__ row0s, const int* __restrict__ lens,
                                                        float* __restrict__ out) {
    __shared__ double part[256];
    const int s = blockIdx.x, tid = threadIdx.x;
    const int G = 256 / F, g = tid / F, c = tid - g * F;
    const long long row0 = row0s[s];
    const int len = lens[s];
    const bool ok = row0 >= 0 && len > 0 && row0 + len <= total_rows;
    double acc = 0.0;
    if (ok && g < G)
        for (int r = g; r < len; r += G) acc += (double)feats[(row0 + r) * F + c];
    part[tid] = acc;
    __syncthreads();
    if (tid < F) {
        double m = 0.0;
        for (int i = 0; i < G; ++i) m += part[i * F + tid];
        out[(long long)s * F + tid] = ok ? (float)(m / (double)len) : 0.f;
    }
}

// One CTA per window: out[w][r][c] = feats[row0 + (r mod len)][c] - mean[c].  mode 0: mean = 0; 1: the mean of the
// window_fs tiled rows (the reference tiles, then subtracts), fp32 in a fixed order; 2: seg_mean[seg_of[w]].  A table entry
// outside [0, total_rows) is written as zeros and nothing is read for it.
__global__ void __launch_bounds__(256) diar_windows_kernel(const float* __restrict__ feats, long long total_rows, int F,
                                                           const int* __restrict__ row0s, const int* __restrict__ lens,
                                                           int window_fs, int mode, const float* __restrict__ seg_mean,
                                                           const int* __restrict__ seg_of, int n_seg,
                                                           float* __restrict__ out) {
    __shared__ float part[256];
    __shared__ float mean[kMaxFeatDim];
    const int w = blockIdx.x, tid = threadIdx.x;
    const long long row0 = row0s[w];
    const int len = lens[w];
    float* o = out + (long long)w * window_fs * F;
    const int n = window_fs * F;
    bool ok = row0 >= 0 && len > 0 && row0 + len <= total_rows;
    if (mode == 2 && (seg_of[w] < 0 || seg_of[w] >= n_seg)) ok = false;
    if (!ok) {
        for (int i = tid; i < n; i += 256) o[i] = 0.f;
        return;
    }
    const float* src = feats + row0 * F;
    if (mode == 1) {
        const int G = 256 / F, g = tid / F, c = tid - g * F;
        float acc = 0.f;
        if (g < G)
            for (int r = g; r < window_fs; r += G) acc += src[(long long)(r % len) * F + c];
        part[tid] = acc;
        __syncthreads();
        if (tid < F) {
            float m = 0.f;
            for (int i = 0; i < G; ++i) m += part[i * F + tid];
            mean[tid] = m / (float)window_fs;
        }
    } else if (tid < F) {
        mean[tid] = mode == 2 ? seg_mean[(long long)seg_of[w] * F + tid] : 0.f;
    }
    __syncthreads();
    for (int i = tid; i < n; i += 256) {
        const int r = i / F, c = i - r * F;
        o[i] = src[(long long)(r % len) * F + c] - mean[c];
    }
}

// One CTA per row of the cosine tile: adj[j] = 1 for the `keep` largest entries.  Entries equal to the keep-th largest are
// taken from the lowest column upwards until the count is reached (a running count over 256-column strips).
__global__ void __launch_bounds__(256) prune_rows_kernel(const float* __restrict__ cos_tile, long long m, unsigned keep,
                                                         unsigned char* __restrict__ adj) {
    __shared__ unsigned s_warp[8];
    __shared__ unsigned s_base;
    const float* row = cos_tile + (long long)blockIdx.x * m;
    unsigned char* a = adj + (long long)blockIdx.x * m;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    unsigned n_ties;
    const uint32_t thr = radix_select_kth(row, m, keep, &n_ties);
    if (tid == 0) s_base = 0u;
    __syncthreads();
    for (long long j0 = 0; j0 < m; j0 += 256) {
        const long long j = j0 + tid;
        const uint32_t key = j < m ? order_key(row[j]) : 0u;
        const bool eq = j < m && key == thr;
        const unsigned bal = __ballot_sync(0xffffffffu, eq);
        if (lane == 0) s_warp[warp] = __popc(bal);
        __syncthreads();
        unsigned before = s_base + __popc(bal & ((1u << lane) - 1u));
        unsigned strip = 0u;
        for (int i = 0; i < 8; ++i) {
            if (i < warp) before += s_warp[i];
            strip += s_warp[i];
        }
        if (j < m) a[j] = (key > thr || (eq && before < n_ties)) ? 1 : 0;
        __syncthreads();
        if (tid == 0) s_base += strip;
    }
}

// 32 x 32 tiles, block (32, 8): L[i][j] = -(a[i][j] + a[j][i]) / 2 off the diagonal, 0 on it (set by degree_kernel)
__global__ void __launch_bounds__(256) sym_laplacian_kernel(const unsigned char* __restrict__ adj, long long m,
                                                            double* __restrict__ lap) {
    __shared__ unsigned char t[32][33];
    const long long i0 = (long long)blockIdx.y * 32, j0 = (long long)blockIdx.x * 32;
    for (int k = threadIdx.y; k < 32; k += 8) {   // t[k][x] = a[j0 + k][i0 + x]
        const long long r = j0 + k, c = i0 + threadIdx.x;
        t[k][threadIdx.x] = (r < m && c < m) ? adj[r * m + c] : (unsigned char)0;
    }
    __syncthreads();
    for (int k = threadIdx.y; k < 32; k += 8) {
        const long long i = i0 + k, j = j0 + threadIdx.x;
        if (i < m && j < m)
            lap[i * m + j] = i == j ? 0.0 : -0.5 * (double)((int)adj[i * m + j] + (int)t[threadIdx.x][k]);
    }
}

// one CTA per row: L[i][i] = -sum_j L[i][j] (every term a multiple of 1/2: exact in any order; the order here is fixed anyway)
__global__ void __launch_bounds__(256) degree_kernel(double* __restrict__ lap, long long m) {
    __shared__ double red[256];
    double* row = lap + (long long)blockIdx.x * m;
    double acc = 0.0;
    for (long long j = threadIdx.x; j < m; j += 256) acc += row[j];
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) row[blockIdx.x] = -red[0];
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
        set_err(std::string(what) + ": no CUDA device (diarization has no CPU fallback)");
        return true;
    }
    return false;
}

}  // namespace

extern "C" {

int ws_diar_col_means(const float* feats_dev, long long total_rows, int feat_dim, const int* row0_dev, const int* len_dev,
                      int S, float* out_dev, void* stream) {
    if (!feats_dev || !row0_dev || !len_dev || !out_dev || total_rows < 0 || S < 0 || feat_dim <= 0 || feat_dim > kMaxFeatDim) {
        set_err("ws_diar_col_means: bad argument"); return 1;
    }
    if (no_gpu("ws_diar_col_means")) return 1;
    if (S == 0) return 0;
    col_means_kernel<<<(unsigned)S, 256, 0, (cudaStream_t)stream>>>(feats_dev, total_rows, feat_dim, row0_dev, len_dev, out_dev);
    return last_err("ws_diar_col_means");
}

int ws_diar_windows(const float* feats_dev, long long total_rows, int feat_dim, const int* row0_dev, const int* len_dev,
                    int W, int window_fs, int subseg_cmn, const float* seg_mean_dev, const int* seg_of_dev, int S,
                    float* out_dev, void* stream) {
    if (!feats_dev || !row0_dev || !len_dev || !out_dev || total_rows < 0 || W < 0 || window_fs <= 0 || feat_dim <= 0 ||
        feat_dim > kMaxFeatDim || (seg_mean_dev != nullptr && (!seg_of_dev || S <= 0))) {
        set_err("ws_diar_windows: bad argument"); return 1;
    }
    if (subseg_cmn && seg_mean_dev) { set_err("ws_diar_windows: window CMN and segment means are exclusive"); return 1; }
    if (no_gpu("ws_diar_windows")) return 1;
    if (W == 0) return 0;
    const int mode = subseg_cmn ? 1 : (seg_mean_dev ? 2 : 0);
    diar_windows_kernel<<<(unsigned)W, 256, 0, (cudaStream_t)stream>>>(feats_dev, total_rows, feat_dim, row0_dev, len_dev, window_fs,
                                                                   mode, seg_mean_dev, seg_of_dev, S, out_dev);
    return last_err("ws_diar_windows");
}

int ws_diar_laplacian(const double* unit_dev, long long m, int D, long long keep_per_row, float* work_dev, long long work_rows,
                      unsigned char* adj_dev, double* lap_dev, void* stream) {
    if (!unit_dev || !work_dev || !adj_dev || !lap_dev || m <= 0 || D <= 0 || work_rows <= 0 || keep_per_row <= 0 ||
        keep_per_row > m) {
        set_err("ws_diar_laplacian: bad argument"); return 1;
    }
    if (m > WS_DIAR_MAX_M) {
        set_err("ws_diar_laplacian: more than " + std::to_string(WS_DIAR_MAX_M) + " embeddings: the dense m x m fp64 Laplacian "
                "and its full eigendecomposition are the wrong algorithm at this size");
        return 1;
    }
    if (no_gpu("ws_diar_laplacian")) return 1;
    cudaStream_t s = (cudaStream_t)stream;
    for (long long r0 = 0; r0 < m; r0 += work_rows) {
        const long long rows = (m - r0) < work_rows ? (m - r0) : work_rows;
        WS_CKS(ws_launch_dgemm_nt(unit_dev + r0 * D, unit_dev, nullptr, nullptr, work_dev, 0, rows, m, D, m, s));
        prune_rows_kernel<<<(unsigned)rows, 256, 0, s>>>(work_dev, m, (unsigned)keep_per_row, adj_dev + r0 * m);
        if (last_err("ws_diar_laplacian")) return 1;
    }
    const unsigned t = (unsigned)((m + 31) / 32);
    sym_laplacian_kernel<<<dim3(t, t), dim3(32, 8), 0, s>>>(adj_dev, m, lap_dev);
    degree_kernel<<<(unsigned)m, 256, 0, s>>>(lap_dev, m);
    return last_err("ws_diar_laplacian");
}

}  // extern "C"
