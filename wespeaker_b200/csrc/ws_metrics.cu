// Verification metrics on the GPU (SURVEY.md section 2 row 18): the rbst miss / false-alarm curves, the EER crossing and the
// minimum detection cost of wespeaker/utils/score_metrics.py:58-116 (compute_pmiss_pfa_rbst, compute_eer, compute_c_norm,
// compute_c_dcf), which every recipe's bin/compute_metrics.py and bin/compute_det.py end with.
//
// Order: the stable ascending order by (score, trial line) - what the reference computes with np.argsort(kind="stable");
// its default argsort leaves ties in an order that depends on numpy's sort and the CPU.  -0.0 and +0.0 are equal (ordered by
// line), +-inf are ordered, a NaN score is refused.
//
// Stages, all on one stream, no host synchronisation:
//   1. keys_kernel: fp64 score -> order-preserving 64-bit key, payload = trial index | label << 31; in the same read the
//      target count, the NaN / bad-label flags and the histograms of all eight 8-bit digits.
//   2. Eight stable LSD radix passes (reduce-then-scan): per-tile digit counts, a per-digit scan over the tiles, then a
//      scatter that ranks each element within its tile by warp match + a per-warp prefix.  A pass whose digit is the same for
//      every key (one histogram bin holds n) does nothing; the buffers then ping-pong over the active passes only, which each
//      kernel reads from the plan stage on the device.
//   3. eval_kernel over the sorted payloads: exact target-count prefix (tile counts, one scan), fnr = T / Tt and
//      fpr = 1 - F / Ft in fp64, the cost (c_miss * fnr) * p + (c_fa * fpr) * (1 - p) per operating point with explicit
//      _rn intrinsics (no FMA contraction: numpy's association, bit for bit), exact min reductions of the costs (non-negative
//      doubles order as their bit patterns) and of x1 = min{i: fnr - fpr >= 0}, x2 = max{i: fnr - fpr < 0}.
//   4. finish_kernel: fnr / fpr at x1 and x2, the score at x1 and the status word.
#include <cstdint>

#include "../../include/wespeaker_b200.h"
#include "ws_host.h"
#include "ws_kernels.cuh"

using namespace ws;

namespace {

constexpr int kThreads = 256;
constexpr int kTile = 4096;               // elements per tile: 16 rounds of 256
constexpr int kRounds = kTile / kThreads;
constexpr int kPasses = 8;                 // 8-bit digits of a 64-bit key
constexpr unsigned kLabelBit = 0x80000000u;

struct Hdr {
    unsigned long long n_tgt;
    unsigned int status;
    int x1, x2;
    int final_parity;                      // buffer (0: A, 1: B) that holds the sorted payloads
    int src_parity[kPasses];
    int active[kPasses];
    unsigned long long minc[WS_METRICS_MAX_POINTS];
    unsigned int hist[kPasses][256];
    unsigned int goff[kPasses][256];       // exclusive global digit offsets
};

struct Points {
    double p[WS_METRICS_MAX_POINTS], q[WS_METRICS_MAX_POINTS];    // p_target, 1 - p_target (as the host computes it)
    double cm[WS_METRICS_MAX_POINTS], cf[WS_METRICS_MAX_POINTS];  // c_miss, c_fa
    int n;
};

inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }
inline long long n_tiles(long long n) { return (n + kTile - 1) / kTile; }

struct Layout {
    size_t hdr, ka, kb, va, vb, cnt, tpre, total;
};
Layout layout(long long n) {
    Layout L;
    const long long nt = n_tiles(n);
    L.hdr = 0;
    L.ka = align256(sizeof(Hdr));
    L.kb = L.ka + align256(8 * (size_t)n);
    L.va = L.kb + align256(8 * (size_t)n);
    L.vb = L.va + align256(4 * (size_t)n);
    L.cnt = L.vb + align256(4 * (size_t)n);
    L.tpre = L.cnt + align256(4 * 256 * (size_t)nt);
    L.total = L.tpre + align256(8 * (size_t)(nt + 1));
    return L;
}

__device__ __forceinline__ unsigned long long order_key64(double s) {
    unsigned long long b = (unsigned long long)__double_as_longlong(s == 0.0 ? 0.0 : s);   // -0.0 -> +0.0
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

__device__ __forceinline__ unsigned long long block_sum_u64(unsigned long long v, unsigned long long* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    unsigned long long t = 0;
    for (int w = 0; w < kThreads / 32; ++w) t += red[w];
    __syncthreads();
    return t;
}

// ---------------------------------------------------------------------------------------------------- 1. keys + histograms
__global__ void __launch_bounds__(kThreads) keys_kernel(const double* __restrict__ scores,
                                                        const unsigned char* __restrict__ labels, long long n,
                                                        Hdr* __restrict__ h, unsigned long long* __restrict__ keys,
                                                        unsigned* __restrict__ vals) {
    __shared__ unsigned int hist[kPasses][256];
    __shared__ unsigned long long red[kThreads / 32];
    for (int i = threadIdx.x; i < kPasses * 256; i += kThreads) (&hist[0][0])[i] = 0;
    __syncthreads();
    unsigned long long tgt = 0;
    unsigned flags = 0;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
        const double s = scores[i];
        const unsigned lab = labels[i];
        if (s != s) flags |= WS_METRICS_NAN_SCORE;
        if (lab > 1) flags |= WS_METRICS_BAD_LABEL;
        const unsigned long long k = order_key64(s);
        keys[i] = k;
        vals[i] = (unsigned)i | (lab == 1 ? kLabelBit : 0u);
        tgt += (lab == 1);
#pragma unroll
        for (int p = 0; p < kPasses; ++p) atomicAdd(&hist[p][(k >> (8 * p)) & 255], 1u);
    }
    flags = __reduce_or_sync(0xffffffffu, flags);
    if ((threadIdx.x & 31) == 0 && flags) atomicOr(&h->status, flags);
    tgt = block_sum_u64(tgt, red);
    if (threadIdx.x == 0 && tgt) atomicAdd(&h->n_tgt, tgt);
    for (int i = threadIdx.x; i < kPasses * 256; i += kThreads) {
        const unsigned c = (&hist[0][0])[i];
        if (c) atomicAdd(&h->hist[0][0] + i, c);
    }
}

// One block: class check, global digit offsets, which passes run and where each one reads from, reduction identities.
__global__ void __launch_bounds__(kThreads) plan_kernel(long long n, Hdr* __restrict__ h) {
    __shared__ unsigned int scan[256];
    __shared__ int trivial[kPasses];
    const int t = threadIdx.x;
    if (t < kPasses) trivial[t] = 0;
    if (t == 0) {
        if (h->n_tgt == 0 || h->n_tgt == (unsigned long long)n) h->status |= WS_METRICS_EMPTY_CLASS;
        h->x1 = 0x7fffffff;
        h->x2 = -1;
    }
    if (t < WS_METRICS_MAX_POINTS) h->minc[t] = ~0ull;
    __syncthreads();
    for (int p = 0; p < kPasses; ++p) {
        const unsigned c = h->hist[p][t];
        if (c == (unsigned)n) trivial[p] = 1;
        scan[t] = c;
        __syncthreads();
        for (int o = 1; o < 256; o <<= 1) {            // inclusive Hillis-Steele scan
            const unsigned v = t >= o ? scan[t - o] : 0u;
            __syncthreads();
            scan[t] += v;
            __syncthreads();
        }
        h->goff[p][t] = scan[t] - c;
        __syncthreads();
    }
    if (t == 0) {
        const bool bad = h->status != 0;
        int parity = 0;
        for (int p = 0; p < kPasses; ++p) {
            const int a = !bad && !trivial[p];
            h->active[p] = a;
            h->src_parity[p] = parity;
            parity ^= a;
        }
        h->final_parity = parity;
    }
}

// ---------------------------------------------------------------------------------------------------- 2. radix passes
__global__ void __launch_bounds__(kThreads) tile_hist_kernel(const Hdr* __restrict__ h, int pass,
                                                             const unsigned long long* __restrict__ ka,
                                                             const unsigned long long* __restrict__ kb, long long n,
                                                             long long nt, unsigned* __restrict__ cnt) {
    if (!h->active[pass]) return;
    __shared__ unsigned int hist[256];
    const unsigned long long* keys = h->src_parity[pass] ? kb : ka;
    hist[threadIdx.x] = 0;
    __syncthreads();
    const long long tile = blockIdx.x, base = tile * kTile;
    const int shift = 8 * pass;
    for (int r = 0; r < kRounds; ++r) {
        const long long i = base + r * kThreads + threadIdx.x;
        if (i < n) atomicAdd(&hist[(keys[i] >> shift) & 255], 1u);
    }
    __syncthreads();
    cnt[(long long)threadIdx.x * nt + tile] = hist[threadIdx.x];
}

// One block per digit: exclusive scan of its tile counts, plus the digit's global offset.  In place.
__global__ void __launch_bounds__(kThreads) digit_scan_kernel(const Hdr* __restrict__ h, int pass, long long nt,
                                                              unsigned* __restrict__ cnt) {
    if (!h->active[pass]) return;
    __shared__ unsigned int ws[kThreads / 32];
    const int d = blockIdx.x, t = threadIdx.x, lane = t & 31, w = t >> 5;
    unsigned* row = cnt + (long long)d * nt;
    unsigned carry = h->goff[pass][d];
    for (long long c0 = 0; c0 < nt; c0 += kThreads) {
        const long long i = c0 + t;
        const unsigned v = i < nt ? row[i] : 0u;
        unsigned x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) ws[w] = x;
        __syncthreads();
        unsigned before = 0, total = 0;
        for (int k = 0; k < kThreads / 32; ++k) {
            if (k < w) before += ws[k];
            total += ws[k];
        }
        if (i < nt) row[i] = carry + before + x - v;
        carry += total;
        __syncthreads();
    }
}

// Stable scatter of one tile.  Each element's rank within the tile's run of its digit: 16 rounds of 256 consecutive elements;
// within a round, the digit's running offset + the counts of the digit in lower warps + the lower lanes of the digit in this
// warp.  The tile is then reordered in shared memory by (digit, rank) and written out run by run, so that consecutive
// threads store consecutive addresses of the destination.
__global__ void __launch_bounds__(kThreads) scatter_kernel(const Hdr* __restrict__ h, int pass, unsigned long long* ka,
                                                           unsigned long long* kb, unsigned* va, unsigned* vb, long long n,
                                                           long long nt, const unsigned* __restrict__ cnt) {
    if (!h->active[pass]) return;
    __shared__ unsigned long long sk[kTile];               // keys, then (as unsigned) payloads, in tile-local sorted order
    __shared__ unsigned char sd[kTile];                    // digit of each tile-local position
    __shared__ unsigned int run[256];                      // running tile-local offset of each digit
    __shared__ unsigned int lstart[256];                   // tile-local start of each digit's run
    __shared__ unsigned int gbase[256];                    // destination of each digit's run
    __shared__ unsigned int wc[kThreads / 32][256];
    const int sp = h->src_parity[pass];
    const unsigned long long* ks = sp ? kb : ka;
    unsigned long long* kd = sp ? ka : kb;
    const unsigned* vs = sp ? vb : va;
    unsigned* vd = sp ? va : vb;
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    const long long tile = blockIdx.x, tbase = tile * kTile;
    const int cnt_tile = (int)(n - tbase < kTile ? n - tbase : kTile);
    const int shift = 8 * pass;
    run[t] = 0;
    gbase[t] = cnt[(long long)t * nt + tile];
    for (int k = 0; k < kThreads / 32; ++k) wc[k][t] = 0;
    __syncthreads();
    unsigned long long key[kRounds];
    unsigned val[kRounds], lpos[kRounds];
#pragma unroll
    for (int r = 0; r < kRounds; ++r) {
        const int j = r * kThreads + t;
        key[r] = 0;
        val[r] = 0;
        if (j < cnt_tile) {
            key[r] = ks[tbase + j];
            val[r] = vs[tbase + j];
            atomicAdd(&run[(key[r] >> shift) & 255], 1u);
        }
    }
    __syncthreads();
    if (t < 32) {                                          // exclusive scan of the tile's 256 digit counts by one warp
        unsigned c[8], s = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) { c[k] = run[t * 8 + k]; s += c[k]; }
        unsigned x = s;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        x -= s;
#pragma unroll
        for (int k = 0; k < 8; ++k) { lstart[t * 8 + k] = x; run[t * 8 + k] = x; x += c[k]; }
    }
    __syncthreads();
    const unsigned lt = (1u << lane) - 1u;
#pragma unroll
    for (int r = 0; r < kRounds; ++r) {
        const bool ok = r * kThreads + t < cnt_tile;
        const int d = ok ? (int)((key[r] >> shift) & 255) : 256;   // out-of-range lanes form their own group
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        const unsigned rank = __popc(peers & lt);
        if (ok && rank == 0) wc[w][d] = __popc(peers);
        __syncthreads();
        {
            unsigned s = run[t];
#pragma unroll
            for (int q = 0; q < kThreads / 32; ++q) {
                const unsigned c = wc[q][t];
                wc[q][t] = s;
                s += c;
            }
            run[t] = s;
        }
        __syncthreads();
        if (ok) {
            lpos[r] = wc[w][d] + rank;
            sk[lpos[r]] = key[r];
            sd[lpos[r]] = (unsigned char)d;
        }
        __syncthreads();
#pragma unroll
        for (int q = 0; q < kThreads / 32; ++q) wc[q][t] = 0;
        __syncthreads();                                   // cleared before the next round's leaders write their counts
    }
    for (int j = t; j < cnt_tile; j += kThreads) {
        const int d = sd[j];
        kd[gbase[d] + (unsigned)j - lstart[d]] = sk[j];
    }
    __syncthreads();
    unsigned* sv = (unsigned*)sk;
#pragma unroll
    for (int r = 0; r < kRounds; ++r)
        if (r * kThreads + t < cnt_tile) sv[lpos[r]] = val[r];
    __syncthreads();
    for (int j = t; j < cnt_tile; j += kThreads) {
        const int d = sd[j];
        vd[gbase[d] + (unsigned)j - lstart[d]] = sv[j];
    }
}

// ---------------------------------------------------------------------------------------------------- 3. evaluation
__global__ void __launch_bounds__(kThreads) tile_targets_kernel(const Hdr* __restrict__ h, const unsigned* __restrict__ va,
                                                                const unsigned* __restrict__ vb, long long n,
                                                                unsigned* __restrict__ cnt) {
    if (h->status) return;
    __shared__ unsigned long long red[kThreads / 32];
    const unsigned* vals = h->final_parity ? vb : va;
    const long long base = (long long)blockIdx.x * kTile;
    unsigned long long c = 0;
    for (int r = 0; r < kRounds; ++r) {
        const long long i = base + r * kThreads + threadIdx.x;
        if (i < n) c += vals[i] >> 31;
    }
    c = block_sum_u64(c, red);
    if (threadIdx.x == 0) cnt[blockIdx.x] = (unsigned)c;
}

// One block: tpre[j] = targets in tiles [0, j), int64.
__global__ void __launch_bounds__(kThreads) tile_prefix_kernel(const Hdr* __restrict__ h, const unsigned* __restrict__ cnt,
                                                               long long nt, long long* __restrict__ tpre) {
    if (h->status) return;
    __shared__ long long ws[kThreads / 32];
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    long long carry = 0;
    for (long long c0 = 0; c0 < nt; c0 += kThreads) {
        const long long i = c0 + t;
        const long long v = i < nt ? (long long)cnt[i] : 0;
        long long x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const long long y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) ws[w] = x;
        __syncthreads();
        long long before = 0, total = 0;
        for (int k = 0; k < kThreads / 32; ++k) {
            if (k < w) before += ws[k];
            total += ws[k];
        }
        if (i < nt) tpre[i] = carry + before + x - v;
        carry += total;
        __syncthreads();
    }
    if (t == 0) tpre[nt] = carry;
}

__device__ __forceinline__ double fnr_at(long long T, double Tt) { return __ddiv_rn((double)T, Tt); }
__device__ __forceinline__ double fpr_at(long long i, long long T, double Ft) {
    return __dsub_rn(1.0, __ddiv_rn((double)(i + 1 - T), Ft));
}

// One tile per block, 16 consecutive elements per thread.
__global__ void __launch_bounds__(kThreads) eval_kernel(Hdr* __restrict__ h, const Points pts,
                                                        const unsigned* __restrict__ va, const unsigned* __restrict__ vb,
                                                        long long n, const long long* __restrict__ tpre,
                                                        int* __restrict__ order, double* __restrict__ fnr_out,
                                                        double* __restrict__ fpr_out) {
    if (h->status) return;
    constexpr int kItems = kTile / kThreads;
    __shared__ long long ws[kThreads / 32];
    __shared__ unsigned long long rmin[WS_METRICS_MAX_POINTS][kThreads / 32];
    __shared__ int rx[2][kThreads / 32];
    const unsigned* vals = h->final_parity ? vb : va;
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    const long long i0 = (long long)blockIdx.x * kTile + (long long)t * kItems;
    unsigned v[kItems];
    int mine = 0;
#pragma unroll
    for (int k = 0; k < kItems; ++k) {
        v[k] = i0 + k < n ? vals[i0 + k] : 0u;
        mine += v[k] >> 31;
    }
    long long x = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) ws[w] = x;
    __syncthreads();
    long long T = tpre[blockIdx.x] + x - mine;
    for (int k = 0; k < w; ++k) T += ws[k];
    const double Tt = (double)h->n_tgt, Ft = (double)(n - (long long)h->n_tgt);
    unsigned long long cmin[WS_METRICS_MAX_POINTS];
#pragma unroll
    for (int q = 0; q < WS_METRICS_MAX_POINTS; ++q) cmin[q] = ~0ull;
    int x1 = 0x7fffffff, x2 = -1;
#pragma unroll
    for (int k = 0; k < kItems; ++k) {
        const long long i = i0 + k;
        if (i >= n) break;
        T += v[k] >> 31;
        const double fnr = fnr_at(T, Tt), fpr = fpr_at(i, T, Ft);
        if (order) order[i] = (int)(v[k] & ~kLabelBit);
        if (fnr_out) fnr_out[i] = fnr;
        if (fpr_out) fpr_out[i] = fpr;
        const double diff = __dsub_rn(fnr, fpr);
        if (diff >= 0.0) { if (x1 == 0x7fffffff) x1 = (int)i; }
        else x2 = (int)i;
#pragma unroll
        for (int q = 0; q < WS_METRICS_MAX_POINTS; ++q) {
            if (q < pts.n) {
                const double c = __dadd_rn(__dmul_rn(__dmul_rn(pts.cm[q], fnr), pts.p[q]),
                                           __dmul_rn(__dmul_rn(pts.cf[q], fpr), pts.q[q]));
                const unsigned long long b = (unsigned long long)__double_as_longlong(c);
                cmin[q] = b < cmin[q] ? b : cmin[q];
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        x1 = min(x1, __shfl_xor_sync(0xffffffffu, x1, o));
        x2 = max(x2, __shfl_xor_sync(0xffffffffu, x2, o));
#pragma unroll
        for (int q = 0; q < WS_METRICS_MAX_POINTS; ++q) {
            const unsigned long long y = __shfl_xor_sync(0xffffffffu, cmin[q], o);
            cmin[q] = y < cmin[q] ? y : cmin[q];
        }
    }
    if (lane == 0) {
        rx[0][w] = x1;
        rx[1][w] = x2;
#pragma unroll
        for (int q = 0; q < WS_METRICS_MAX_POINTS; ++q) rmin[q][w] = cmin[q];
    }
    __syncthreads();
    if (t < pts.n) {
        unsigned long long m = rmin[t][0];
        for (int k = 1; k < kThreads / 32; ++k) m = rmin[t][k] < m ? rmin[t][k] : m;
        atomicMin(&h->minc[t], m);
    }
    if (t == 32) {
        int a = rx[0][0], b = rx[1][0];
        for (int k = 1; k < kThreads / 32; ++k) { a = min(a, rx[0][k]); b = max(b, rx[1][k]); }
        if (a != 0x7fffffff) atomicMin(&h->x1, a);
        if (b >= 0) atomicMax(&h->x2, b);
    }
}

// One block: fnr / fpr at x1 and x2 (the target count up to each, from its tile's prefix), the score at x1, the status.
// out = [fnr(x1), fpr(x1), fnr(x2), fpr(x2), scores[order[x1]], x1, x2, status, c_det[0 .. n_points)].
__global__ void __launch_bounds__(kThreads) finish_kernel(Hdr* __restrict__ h, int n_points, const double* __restrict__ scores,
                                                          const unsigned* __restrict__ va, const unsigned* __restrict__ vb,
                                                          long long n, const long long* __restrict__ tpre,
                                                          double* __restrict__ out) {
    __shared__ unsigned long long red[kThreads / 32];
    const int t = threadIdx.x;
    unsigned status = h->status;
    if (status == 0 && h->x2 < 0) status |= WS_METRICS_NO_X2;
    if (status) {
        if (t == 0) out[7] = (double)status;
        return;
    }
    const unsigned* vals = h->final_parity ? vb : va;
    const double Tt = (double)h->n_tgt, Ft = (double)(n - (long long)h->n_tgt);
    const int xs[2] = {h->x1, h->x2};
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        const long long x = xs[j], tile0 = (x / kTile) * kTile;
        unsigned long long c = 0;
        for (long long i = tile0 + t; i <= x; i += kThreads) c += vals[i] >> 31;
        c = block_sum_u64(c, red);
        const long long T = tpre[x / kTile] + (long long)c;
        if (t == 0) {
            out[2 * j] = fnr_at(T, Tt);
            out[2 * j + 1] = fpr_at(x, T, Ft);
        }
    }
    if (t == 0) {
        out[4] = scores[vals[xs[0]] & ~kLabelBit];
        out[5] = (double)xs[0];
        out[6] = (double)xs[1];
        out[7] = 0.0;
    }
    if (t < n_points) out[8 + t] = __longlong_as_double((long long)h->minc[t]);
}

inline int last_err(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) return 0;
    set_err(std::string(what) + ": " + cudaGetErrorString(e));
    return 1;
}

}  // namespace

extern "C" {

size_t ws_metrics_work_bytes(long long n) {
    if (n <= 0 || n > WS_METRICS_MAX_N) return 0;
    return layout(n).total;
}

int ws_metrics_eval(const double* scores_dev, const unsigned char* labels_dev, long long n, const double* p_target,
                    const double* c_miss, const double* c_fa, int n_points, void* work_dev, size_t work_bytes,
                    double* out_dev, int* order_dev, double* fnr_dev, double* fpr_dev, void* stream,
                    void* const* stage_events) {
    const char* what = "ws_metrics_eval";
    if (n <= 0 || n > WS_METRICS_MAX_N) { set_err("ws_metrics_eval: n must be in [1, 2^31 - 1]"); return 1; }
    if (n_points < 1 || n_points > WS_METRICS_MAX_POINTS) {
        set_err("ws_metrics_eval: n_points must be in [1, 16]"); return 1;
    }
    if (!scores_dev || !labels_dev || !p_target || !c_miss || !c_fa || !work_dev || !out_dev) {
        set_err("ws_metrics_eval: null pointer"); return 1;
    }
    Points pts{};
    pts.n = n_points;
    for (int q = 0; q < n_points; ++q) {
        if (!(p_target[q] > 0.0 && p_target[q] < 1.0)) { set_err("ws_metrics_eval: p_target must be in (0, 1)"); return 1; }
        if (!(c_miss[q] >= 0.0) || !(c_fa[q] >= 0.0) || c_miss[q] > 1.7e308 || c_fa[q] > 1.7e308) {
            set_err("ws_metrics_eval: costs must be finite and non-negative"); return 1;
        }
        pts.p[q] = p_target[q];
        pts.q[q] = 1.0 - p_target[q];
        pts.cm[q] = c_miss[q] + 0.0;   // -0.0 -> +0.0: every cost stays a non-negative double (bit order = value order)
        pts.cf[q] = c_fa[q] + 0.0;
    }
    const Layout L = layout(n);
    if (work_bytes < L.total) { set_err("ws_metrics_eval: workspace smaller than ws_metrics_work_bytes(n)"); return 1; }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        set_err("ws_metrics_eval: no CUDA device (the metrics have no CPU fallback)");
        return 1;
    }
    cudaStream_t s = (cudaStream_t)stream;
    char* wb = (char*)work_dev;
    Hdr* h = (Hdr*)(wb + L.hdr);
    auto* ka = (unsigned long long*)(wb + L.ka);
    auto* kb = (unsigned long long*)(wb + L.kb);
    auto* va = (unsigned*)(wb + L.va);
    auto* vb = (unsigned*)(wb + L.vb);
    auto* cnt = (unsigned*)(wb + L.cnt);
    auto* tpre = (long long*)(wb + L.tpre);
    const long long nt = n_tiles(n);
    auto mark = [&](int k) {
        if (stage_events && stage_events[k]) WS_CK(cudaEventRecord((cudaEvent_t)stage_events[k], s));
        return 0;
    };
    if (mark(0)) return 1;
    WS_CK(cudaMemsetAsync(h, 0, sizeof(Hdr), s));
    const unsigned kgrid = (unsigned)(nt < 1024 ? nt : 1024);
    keys_kernel<<<kgrid, kThreads, 0, s>>>(scores_dev, labels_dev, n, h, ka, va);
    plan_kernel<<<1, kThreads, 0, s>>>(n, h);
    if (last_err(what) || mark(1)) return 1;
    for (int p = 0; p < kPasses; ++p) {
        tile_hist_kernel<<<(unsigned)nt, kThreads, 0, s>>>(h, p, ka, kb, n, nt, cnt);
        digit_scan_kernel<<<256, kThreads, 0, s>>>(h, p, nt, cnt);
        scatter_kernel<<<(unsigned)nt, kThreads, 0, s>>>(h, p, ka, kb, va, vb, n, nt, cnt);
        if (last_err(what) || mark(2 + p)) return 1;
    }
    tile_targets_kernel<<<(unsigned)nt, kThreads, 0, s>>>(h, va, vb, n, cnt);
    tile_prefix_kernel<<<1, kThreads, 0, s>>>(h, cnt, nt, tpre);
    eval_kernel<<<(unsigned)nt, kThreads, 0, s>>>(h, pts, va, vb, n, tpre, order_dev, fnr_dev, fpr_dev);
    finish_kernel<<<1, kThreads, 0, s>>>(h, n_points, scores_dev, va, vb, n, tpre, out_dev);
    if (last_err(what) || mark(2 + kPasses)) return 1;
    return 0;
}

}  // extern "C"
