// Per-row k-th largest of M fp32 values without sorting: 4-pass MSB radix select on order-preserving 32-bit keys.
// Shared by the AS-norm cohort statistics (ws_score.cu) and the affinity pruning of the spectral clusterer (ws_diar.cu).
#pragma once
#include <cstdint>

namespace ws {

__device__ __forceinline__ uint32_t order_key(float v) {   // larger float <=> larger key
    const uint32_t u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_value(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// Called by all 256 threads of a block: the key of the k-th largest of row[0..M) (1 <= k <= M).  *ties = how many entries
// EQUAL to that key belong to the k largest; every entry with a larger key does.  Ends on a __syncthreads().
__device__ __forceinline__ uint32_t radix_select_kth(const float* __restrict__ row, long long M, unsigned k, unsigned* ties) {
    __shared__ unsigned hist[256];
    __shared__ uint32_t s_prefix;
    __shared__ unsigned s_need;
    const int tid = threadIdx.x;
    if (tid == 0) { s_prefix = 0u; s_need = k; }
    for (int pass = 0; pass < 4; ++pass) {
        const int shift = 24 - 8 * pass;
        hist[tid] = 0u;
        __syncthreads();
        const uint32_t prefix = s_prefix;
        const uint32_t hi_mask = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
        for (long long j = tid; j < M; j += 256) {
            const uint32_t key = order_key(row[j]);
            if ((key & hi_mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (tid == 0) {
            unsigned need = s_need;
            int b = 255;
            for (; b > 0; --b) {
                if (hist[b] >= need) break;
                need -= hist[b];
            }
            s_need = need;                       // how many of the selected bin (finally: of the threshold value) to take
            s_prefix = prefix | ((uint32_t)b << shift);
        }
        __syncthreads();
    }
    *ties = s_need;
    return s_prefix;
}

}  // namespace ws
