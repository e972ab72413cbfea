// Kaldi-compatible log-mel fbank + per-utterance CMN on the GPU (HBM-bound: 128 KB in, 63 KB out per 2 s utterance at
// 16 kHz / 80 bins).  Restates what the reference gets from torchaudio.compliance.kaldi.fbank with the arguments of
// wespeaker/dataset/processor.py:518-525 / cli/speaker.py:92-97 (SURVEY.md Appendix B); native twin of
// runtime/core/frontend/fbank.h:138-198.  Two sample rates: 16 kHz (400-sample frames, 160-sample shift, 512-point FFT)
// and 8 kHz (200 / 80 samples, 256-point FFT), the rates of the reference's recipes; 4..128 mel bins.
//
// One warp per 25 ms frame (8 frames per block): coalesced sample loads, DC removal via warp-shuffle sum, pre-emphasis,
// window, then an Nfft-point real FFT computed as an Nfft/2-point complex FFT in registers and warp shuffles + the
// real-input split step, power spectrum, triangular mel filters as short per-bin dot products (each lane owns bins lane,
// lane+32, lane+64, lane+96), log with the float-eps floor.
#include "ws_kernels.cuh"

namespace {

constexpr int kMaxBins = 128;
constexpr float kEps = 1.1920928955078125e-07f;

// frame geometry of the Nfft-point transform: 25 ms frames and a 10 ms shift at Nfft * 31.25 Hz
template <int NFFT> struct Geom {
    static constexpr int kFrameLen = NFFT * 25 / 32;   // 400 | 200 samples
    static constexpr int kShift = NFFT * 10 / 32;      // 160 | 80 samples
    static constexpr int kN2 = NFFT / 2;               // complex FFT length
    static constexpr int kR = kN2 / 32;                // complex values per lane
    static constexpr int kPairSlots = (kFrameLen / 2 + 31) / 32;   // sample-pair registers per lane
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float ld_sample(const void* wav, int is_i16, long long i) {
    return is_i16 ? (float)((const short*)wav)[i] : ((const float*)wav)[i];
}

__device__ __forceinline__ float2 ld_sample2(const void* wav, int is_i16, long long i) {   // samples i, i+1
    // the pair load needs an 8-byte (float) / 4-byte (int16) aligned ADDRESS: odd row strides and views whose base pointer
    // is offset by an odd element count (wavs[1:] of an odd-length batch) take the scalar path
    const uintptr_t addr = (uintptr_t)wav + (uintptr_t)i * (is_i16 ? 2u : 4u);
    if (addr & (is_i16 ? 3u : 7u)) return make_float2(ld_sample(wav, is_i16, i), ld_sample(wav, is_i16, i + 1));
    if (is_i16) {
        const short2 v = *reinterpret_cast<const short2*>((const short*)wav + i);
        return make_float2((float)v.x, (float)v.y);
    }
    return *reinterpret_cast<const float2*>((const float*)wav + i);
}

// The N2 = Nfft/2-point complex FFT never touches shared memory.  With R = N2/32, lane L holds z[L + 32k] (k < R), so
//   X[f1 + R f0] = sum_L W32^(L f0) * ( W_N2^(L f1) * sum_k z[L + 32k] W_R^(k f1) )
// = an R-point DFT in each lane's registers, one twiddle per register, and a 32-point DIF across the lanes done with
// __shfl_xor butterflies (distance 16, 8, 4, 2, 1; result for f0 = bitrev5(L)).  The spectrum goes to smem once for the
// real-input split step (which pairs bin k with bin N2-k).
__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ int zpad(int f) { return f + (f >> 3); }   // skewed smem index of spectrum bin f
// register i of the R-point DIF holds frequency bitrev_log2(R)(i)
template <int R> __device__ __forceinline__ int reg_freq(int i) {
    return R == 8 ? (((i & 1) << 2) | (i & 2) | ((i & 4) >> 2)) : (((i & 1) << 1) | ((i & 2) >> 1));
}

// melw: [nbins][mel_maxlen] filter taps, staged in dynamic shared memory in rows of 4 * mel_ld4(mel_maxlen) floats.  Lanes
// read the rows of consecutive bins in lockstep: 16-byte aligned rows allow 128-bit loads, and a row length of 4 mod 8
// floats puts the 8 lanes of each 128-bit load phase in distinct banks.
__host__ __device__ constexpr int mel_ld4(int mel_maxlen) { return ((mel_maxlen + 3) / 4) | 1; }
// NG = ceil(nbins / 32): the mel bins each lane owns
template <int NFFT, int NG>
__global__ void __launch_bounds__(256) fbank_kernel(const void* __restrict__ wav, int is_i16, long long wav_ld, int T,
                                                    const float* __restrict__ window, const float* __restrict__ melw,
                                                    const int* __restrict__ melstart, const int* __restrict__ mellen,
                                                    int nbins, int mel_maxlen, float* __restrict__ feats,
                                                    const long long* __restrict__ offs, const int* __restrict__ lens) {
    using G = Geom<NFFT>;
    constexpr int N2 = G::kN2, R = G::kR, FL = G::kFrameLen;
    static_assert(R == 8 || R == 4, "fbank: 256- or 512-point FFT");
    __shared__ float2 s_tw[N2];                 // W_Nfft^k = exp(-2*pi*i*k/Nfft)
    __shared__ float2 s_z[8][N2 + N2 / 8];      // per-warp spectrum, index zpad(f)
    __shared__ float s_p[8][N2];                // per-warp power spectrum (bins 0..N2-1; Nyquist has zero mel weight)
    __shared__ float s_win[FL];
    __shared__ short s_mels[kMaxBins], s_mell[kMaxBins];
    extern __shared__ __align__(16) float s_melw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    {
        if (threadIdx.x < N2) {
            float sn, cs;
            sincospif((float)threadIdx.x / (float)N2, &sn, &cs);
            s_tw[threadIdx.x] = make_float2(cs, -sn);
        }
        for (int i = threadIdx.x; i < FL; i += 256) s_win[i] = window[i];
        for (int i = threadIdx.x; i < nbins * mel_maxlen; i += 256) s_melw[(i / mel_maxlen) * 4 * mel_ld4(mel_maxlen) + i % mel_maxlen] = melw[i];
        if (threadIdx.x < nbins) { s_mels[threadIdx.x] = (short)melstart[threadIdx.x]; s_mell[threadIdx.x] = (short)mellen[threadIdx.x]; }
    }
    __syncthreads();
    const int b = blockIdx.y;
    const int frame = blockIdx.x * 8 + warp;
    if (frame >= T) return;
    // ragged / length-masked input: utterance b starts at offs[b] (else b * wav_ld) and has lens[b] frames; frames behind
    // the end are neither read nor written (cmn_kernel zeroes them), so a ragged buffer is never read past its last sample
    if (lens != nullptr && frame >= lens[b]) return;
    // frame starts are multiples of the (even) shift, so pair loads are aligned whenever the row start is even
    const long long base = (offs != nullptr ? offs[b] : (long long)b * wav_ld) + (long long)frame * G::kShift;

    // each lane owns sample pairs n = lane + 32k (n < FL/2): ONE pass over the samples (coalesced pair loads)
    float2 x[G::kPairSlots];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < G::kPairSlots; ++k) {
        const int n = lane + 32 * k;
        x[k] = n < FL / 2 ? ld_sample2(wav, is_i16, base + 2 * n) : make_float2(0.f, 0.f);
        s += x[k].x + x[k].y;
    }
    const float mu = warp_sum(s) / (float)FL;   // remove_dc_offset

    // a[k] = z[lane + 32k] = y[2n] + i*y[2n+1], y = window * ((x - mu) - 0.97 * (x_prev - mu)); x[2n-1] comes from the
    // neighbouring lane (lane-1 of the same k, or lane 31 of k-1 for lane 0; replicate-pad at n = 0)
    float2 a[R];
#pragma unroll
    for (int k = 0; k < R; ++k) {
        const int n = lane + 32 * k;
        float2 v = make_float2(0.f, 0.f);
        if (k < G::kPairSlots) {
            float prev_same = __shfl_up_sync(0xffffffffu, x[k].y, 1);
            float prev_wrap = __shfl_sync(0xffffffffu, k > 0 ? x[k > 0 ? k - 1 : 0].y : 0.f, 31);
            if (n < FL / 2) {
                const float xm1 = (lane > 0 ? prev_same : (k > 0 ? prev_wrap : x[0].x)) - mu;
                const float x0 = x[k].x - mu, x1 = x[k].y - mu;
                v.x = (x0 - 0.97f * xm1) * s_win[2 * n];
                v.y = (x1 - 0.97f * x0) * s_win[2 * n + 1];
            }
        }
        a[k] = v;
    }
    // ---- R-point DIF over k in registers; afterwards register i holds f1 = reg_freq<R>(i)
    {
        const float h = 0.70710678118654752440f;
        float2 t;
        if constexpr (R == 8) {
            // stage 1 of 8: (k, k+4), twiddles W8^k
            t = csub(a[0], a[4]); a[0] = cadd(a[0], a[4]); a[4] = t;
            t = csub(a[1], a[5]); a[1] = cadd(a[1], a[5]); a[5] = make_float2(h * (t.x + t.y), h * (t.y - t.x));
            t = csub(a[2], a[6]); a[2] = cadd(a[2], a[6]); a[6] = make_float2(t.y, -t.x);
            t = csub(a[3], a[7]); a[3] = cadd(a[3], a[7]); a[7] = make_float2(h * (t.y - t.x), -h * (t.x + t.y));
        }
        // 4-point DIF on each group of 4 - (k, k+2), twiddles 1, -i; then neighbours
#pragma unroll
        for (int hb = 0; hb < R; hb += 4) {
            t = csub(a[hb], a[hb + 2]); a[hb] = cadd(a[hb], a[hb + 2]); a[hb + 2] = t;
            t = csub(a[hb + 1], a[hb + 3]); a[hb + 1] = cadd(a[hb + 1], a[hb + 3]); a[hb + 3] = make_float2(t.y, -t.x);
        }
#pragma unroll
        for (int hb = 0; hb < R; hb += 2) {
            t = csub(a[hb], a[hb + 1]); a[hb] = cadd(a[hb], a[hb + 1]); a[hb + 1] = t;
        }
    }
    // ---- twiddle W_N2^(lane * f1) = W_Nfft^(2 * lane * f1)  (2 * 31 * (R-1) < Nfft: at most one half-turn to fold)
#pragma unroll
    for (int i = 1; i < R; ++i) {
        const int idx = 2 * lane * reg_freq<R>(i);
        float2 w = s_tw[idx & (N2 - 1)];
        if (idx >= N2) w = make_float2(-w.x, -w.y);
        a[i] = cmul(a[i], w);
    }
    // ---- 32-point DIF across the lanes
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) {
        const bool upper = (lane & d) == 0;
        const float sg = upper ? 1.f : -1.f;
        const float2 w = upper ? make_float2(1.f, 0.f) : s_tw[(lane & (d - 1)) * (N2 / d)];
#pragma unroll
        for (int i = 0; i < R; ++i) {
            const float ox = __shfl_xor_sync(0xffffffffu, a[i].x, d);
            const float oy = __shfl_xor_sync(0xffffffffu, a[i].y, d);
            const float2 t = make_float2(fmaf(sg, a[i].x, ox), fmaf(sg, a[i].y, oy));   // upper: a + o, lower: o - a
            a[i] = cmul(t, w);
        }
    }
    // lane L, register i holds Z[reg_freq(i) + R * bitrev5(L)]
    float2* z = s_z[warp];
    {
        const int f0 = (int)(__brev((unsigned)lane) >> 27);
#pragma unroll
        for (int i = 0; i < R; ++i) z[zpad(reg_freq<R>(i) + R * f0)] = a[i];
    }
    __syncwarp();
    // split step: X[k] = E[k] + W_Nfft^k * O[k],  E = (Z[k] + conj(Z[N2-k]))/2,  O = -i (Z[k] - conj(Z[N2-k]))/2
    float* pw = s_p[warp];
#pragma unroll
    for (int k8 = 0; k8 < R; ++k8) {
        const int k = lane + 32 * k8;
        const float2 za = z[zpad(k)];
        const float2 c = z[zpad((N2 - k) & (N2 - 1))];
        const float er = 0.5f * (za.x + c.x), ei = 0.5f * (za.y - c.y);
        const float orr = 0.5f * (za.y + c.y), oi = -0.5f * (za.x - c.x);
        const float2 w = s_tw[k];
        const float xr = er + (orr * w.x - oi * w.y);
        const float xi = ei + (orr * w.y + oi * w.x);
        pw[k] = xr * xr + xi * xi;
    }
    __syncwarp();
    float* out = feats + ((long long)b * T + frame) * nbins;
#pragma unroll
    for (int k = 0; k < NG; ++k) {
        const int m = lane + 32 * k;
        if (m < nbins) {
            const int st = s_mels[m], len = s_mell[m];
            const float* w = s_melw + 4 * (m * mel_ld4(mel_maxlen));
            float e = 0.f;
            for (int i = 0; i < len; ++i) e = fmaf(pw[st + i], w[i], e);
            out[m] = logf(fmaxf(e, kEps));
        }
    }
}

// block (32, 8): subtract the per-utterance mean over T from every bin (dataset_utils.py:19-26)
__global__ void __launch_bounds__(256) cmn_kernel(float* __restrict__ feats, int T, int Fdim, const int* __restrict__ lens) {
    __shared__ float red[8][33];
    const int c = blockIdx.x * 32 + threadIdx.x;
    const int b = blockIdx.y;
    const bool cv = c < Fdim;
    float* p = feats + (long long)b * T * Fdim + c;
    const int Tpad = T;
    if (lens != nullptr) T = max(1, min(T, lens[b]));   // length-masked batch: mean over the utterance's own frames
    float s = 0.f;
    if (cv)
        for (int t = threadIdx.y; t < T; t += 8) s += p[(long long)t * Fdim];
    red[threadIdx.y][threadIdx.x] = s;
    __syncthreads();
    float mean = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) mean += red[i][threadIdx.x];
    mean /= (float)T;
    if (cv) {
        for (int t = threadIdx.y; t < T; t += 8) p[(long long)t * Fdim] -= mean;
        for (int t = T + threadIdx.y; t < Tpad; t += 8) p[(long long)t * Fdim] = 0.f;   // padding frames
    }
}

template <int NFFT>
cudaError_t launch_fbank(const void* wav, int is_i16, long long wav_ld, int B, int T, const float* window, const float* melw,
                         const int* melstart, const int* mellen, int nbins, int mel_maxlen, float* feats, cudaStream_t s,
                         const long long* offs, const int* lens) {
    dim3 grid((T + 7) / 8, B);
    const size_t smem = (size_t)nbins * 4 * mel_ld4(mel_maxlen) * sizeof(float);
    auto kern = nbins <= 32 ? fbank_kernel<NFFT, 1> : nbins <= 64 ? fbank_kernel<NFFT, 2>
              : nbins <= 96 ? fbank_kernel<NFFT, 3> : fbank_kernel<NFFT, 4>;
    kern<<<grid, 256, smem, s>>>(wav, is_i16, wav_ld, T, window, melw, melstart, mellen, nbins, mel_maxlen, feats, offs, lens);
    return cudaGetLastError();
}

}  // namespace

int ws_fbank_frame_len(int sample_rate) { return sample_rate == 16000 ? 400 : sample_rate == 8000 ? 200 : 0; }
int ws_fbank_frame_shift(int sample_rate) { return sample_rate == 16000 ? 160 : sample_rate == 8000 ? 80 : 0; }

const char* ws_launch_fbank(const void* wav, int wav_is_i16, long long wav_ld, int nsamples, int B, int T, int sample_rate,
                            int nbins, const float* window, const float* melw, const int* melstart, const int* mellen,
                            int mel_maxlen, float* feats, cudaStream_t s, const long long* offs, const int* lens) {
    const int fl = ws_fbank_frame_len(sample_rate), sh = ws_fbank_frame_shift(sample_rate);
    if (fl == 0) return "fbank: sample rate must be 8000 or 16000";
    if (nbins < 4 || nbins > kMaxBins) return "fbank: mel bin count outside [4, 128]";
    if (T <= 0 || B <= 0) return nullptr;
    if ((long long)(T - 1) * sh + fl > nsamples) return "fbank: T frames do not fit in nsamples";
    if ((size_t)nbins * 4 * mel_ld4(mel_maxlen) * sizeof(float) > kFbankMaxMelBytes) return "fbank: mel filter table larger than the shared-memory limit";
    const cudaError_t e = sample_rate == 16000
        ? launch_fbank<512>(wav, wav_is_i16, wav_ld, B, T, window, melw, melstart, mellen, nbins, mel_maxlen, feats, s, offs, lens)
        : launch_fbank<256>(wav, wav_is_i16, wav_ld, B, T, window, melw, melstart, mellen, nbins, mel_maxlen, feats, s, offs, lens);
    return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

// ---- sinc resampling (torchaudio.transforms.Resample, the reference's `resample`: dataset/processor.py:242-262,
// cli/speaker.py:157-159): out[j * nf + i] = sum_k x[j * of + k - width] * K[i][k], K = [nf][2 * width + of] polyphase taps
// (Hann-windowed sinc built on the host in fp64 exactly as torchaudio builds it), samples outside [0, n_in) read as zero.
namespace {
__global__ void __launch_bounds__(256) resample_kernel(const void* __restrict__ wav, int is_i16, long long wav_ld, int n_in,
                                                       const float* __restrict__ K, int of, int nf, int width, int klen,
                                                       float* __restrict__ out, long long out_ld, int n_out) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (n >= n_out) return;
    const int j = n / nf, i = n - j * nf;
    const long long base = (long long)j * of - width;
    const float* k = K + (size_t)i * klen;
    const long long row = (long long)b * wav_ld;
    float acc = 0.f;
    for (int t = 0; t < klen; ++t) {
        const long long m = base + t;
        if (m >= 0 && m < n_in) {
            const float x = is_i16 ? (float)((const short*)wav)[row + m] : ((const float*)wav)[row + m];
            acc = fmaf(x, k[t], acc);
        }
    }
    out[(long long)b * out_ld + n] = acc;
}
}  // namespace

const char* ws_launch_resample(const void* wav, int wav_is_i16, long long wav_ld, int n_in, int B, const float* taps, int of,
                               int nf, int width, float* out, long long out_ld, int n_out, cudaStream_t s) {
    if (B <= 0 || n_out <= 0) return nullptr;
    dim3 grid((n_out + 255) / 256, B);
    resample_kernel<<<grid, 256, 0, s>>>(wav, wav_is_i16, wav_ld, n_in, taps, of, nf, width, 2 * width + of, out, out_ld, n_out);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

const char* ws_launch_cmn(float* feats, int B, int T, int Fdim, cudaStream_t s, const int* lens) {
    if (T <= 0 || B <= 0) return nullptr;
    dim3 grid((Fdim + 31) / 32, B), block(32, 8);
    cmn_kernel<<<grid, block, 0, s>>>(feats, T, Fdim, lens);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}
