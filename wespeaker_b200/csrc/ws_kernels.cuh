// Host-callable launchers for the bandwidth-bound kernels (ws_kernels.cu, ws_fbank.cu, ws_plda.cu).
// All return nullptr on success or a static error string.
#pragma once
#include "ws_common.cuh"

// ---- elementwise / reductions over channels-last activations [rows][ld]
// (`lo`: optional fp32 twin receiving v - tf32_trunc(v) for the 3xTF32 GEMM path; pass nullptr otherwise)
const char* ws_launch_convert(const float* in, void* out, float* lo, int dt, long long n, cudaStream_t s);
// mean (and optional unbiased std, sqrt(var + eps)) over T for every (b, f, c).  x: [B][F][T][ld], channels [0,C).
// Optional per-channel pre-affine + relu (CAM++ out_nonlinear, campplus.py:378-379).  Output (fp32 or `odt`):
//   mean -> out[b*out_ld + c*F + f],  std -> out[b*out_ld + std_off + c*F + f]   (std skipped if std_off < 0)
const char* ws_launch_tstats(const void* x, int dt, int B, int F, int T, int C, long long ld, const float* pre_scale,
                             const float* pre_shift, void* out, int odt, long long out_ld, int std_off, float eps,
                             cudaStream_t s, const int* lens = nullptr);
// length-masked batches (per-utterance frame counts `lens`, device int32): zero the rows t >= lens[b]; derive the frame
// counts behind stride-2 layers (lens is [levels][B], level 0 = input); frames from sample counts
const char* ws_launch_zero_tail(void* x, float* lo, int dt, int B, int F, int T, int C, long long ld, const int* lens,
                                cudaStream_t s);
const char* ws_launch_lens_derive(int* lens, int B, int T, int levels, cudaStream_t s);
const char* ws_launch_frames_from_samples(const int* nsamp, int* lens, int B, int Tmax, int frame_len, int shift, cudaStream_t s);
// out[r][o] = act( sum_i W[o][i] * (in[r][i] + in2[r / rows_per_b][i]) + bias[o] ),  fp32 in/out, W fp32 [O][I]
bool ws_linear_rows_big(long long in_ld, const float* in2, long long in2_ld, int R, int I, int O);
const char* ws_launch_linear_rows(const float* in, long long in_ld, const float* in2, long long in2_ld,
                                  int rows_per_b, const float* W, const float* bias, float* out, long long out_ld,
                                  int R, int I, int O, int act, float* workspace, int nsplit, cudaStream_t s);
// SE apply + residual (ecapa_tdnn.py:124,157): out[pos][c] = x[pos][c]*gate[b][c] + res[pos][c]
const char* ws_launch_scale_residual(const void* x, long long x_ld, const float* gate, const void* res,
                                     long long res_ld, void* out, float* lo, long long out_ld, int dt, int B, int T,
                                     int C, cudaStream_t s);
// ERes2Net AFF combine (eres2net.py:97-100): out[pos][c] = x * (1 + t) + y * (2 - (1 + t)), t = the tanh'd attention map
const char* ws_launch_aff_combine(const void* x, long long x_ld, const void* y, long long y_ld, const void* t, long long t_ld,
                                  void* out, float* lo, long long out_ld, int dt, long long npos, int C, cudaStream_t s);
// ASTP statistics (pooling_layers.py:138-144): softmax over T of logits, weighted mean / std = sqrt(max(var, var_floor)) of x
// (ECAPA's ASTP floors the variance at 1e-7, SimAM-ResNet's ASP at 1e-5, pooling_layers.py:198-203)
const char* ws_launch_astp_stats(const void* x, const void* logits, int dt, int B, int T, int C, long long ld,
                                 float* out /*[B][2C]*/, float var_floor, cudaStream_t s, const int* lens = nullptr);
// SimAM (ws_simam.cu, samresnet.py:65-70).  Statistics of y [B][F][T][ld] (channels [0,C)) per (b, c) over F x (its own
// frames): stats fp32 [B][2][C] = mean, variance over n = F*T_b - 1; partial: fp32 scratch [B][F][C][2] (two launches).
const char* ws_launch_simam_stats(const void* y, int dt, int B, int F, int T, int C, long long ld, float* partial, float* stats,
                                  cudaStream_t s, const int* lens = nullptr);
// element (b, f, t, c) of a map at b*sb.b + f*sb.f + t*sb.t + c (elements)
struct WsMapStrides {
    long long b, f, t;
};
// out = relu(y * sigmoid((y - mean)^2 / (4 (var + lambda_p)) + 0.5) + res); res may alias out; rows t >= lens[b] of out are
// zeroed; out_lo (optional, fp32 with out's strides) receives the 3xTF32 low part
const char* ws_launch_simam_apply(const void* y, long long y_ld, const float* stats, float lambda_p, const void* res, WsMapStrides rs,
                                  void* out, float* out_lo, WsMapStrides os, int dt, int B, int F, int T, int C, cudaStream_t s,
                                  const int* lens = nullptr);
// Depthwise 3x3 pad-1 conv + folded BN + ReLU (ws_dwconv.cu, gemini_dfresnet.py:37-44): out = relu(dwconv(x, w) + shift) with
// w fp32 [C][3][3], shift fp32 [C]; rows t >= lens[b] are read as zeros and written as zeros; out_lo (fp32 activations,
// optional) receives the 3xTF32 low part.  C % 8 == 0 in 16-bit, C % 4 == 0 in fp32.
const char* ws_launch_dwconv3x3(const void* x, long long x_ld, const float* w, const float* shift, void* out, float* out_lo,
                                long long out_ld, int dt, int B, int F, int T, int C, cudaStream_t s, const int* lens = nullptr);
// out[pos][c] = relu(x[pos][c]*scale[c] + shift[c])  (CAM++ pre-activation BN-ReLU, campplus.py:164-166,214)
const char* ws_launch_bnrelu(const void* x, long long x_ld, const float* scale, const float* shift, void* out,
                             float* lo, long long out_ld, int dt, long long npos, int C, cudaStream_t s);
// ResNet / FCM stem: Conv2d(1->Cout,3x3,pad 1) + folded BN + ReLU.  feats fp32 [B][T][Fdim] -> out [B][Fdim][T][Cout]
const char* ws_launch_stem(const float* feats, const float* w9 /*[Cout][9]*/, const float* shift, void* out, float* lo,
                           int dt, int B, int T, int Fdim, int Cout, cudaStream_t s, const int* lens = nullptr);
// CAM context (campplus.py:108-135): mean over T and per-segment (seg_len) means with ceil-mode partial segment
const char* ws_launch_seg_means(const void* x, int dt, int B, int T, int C, long long ld, int seg_len, float* mean,
                                float* segmean /*[B][nseg][C]*/, cudaStream_t s);

// fused SE gate: gate[b][c] = sigmoid(W2 relu(W1 mean_T(x[b]) + b1) + b2); W2t is W2 transposed to [H][C]
const char* ws_launch_se_gate(const void* x, int dt, int B, int T, int C, long long ld, const float* W1, const float* b1,
                              const float* W2t, const float* b2, int H, float* gate, const float* colsum, cudaStream_t s,
                              const int* lens = nullptr);
// fused CAM context gate: gate[b][seg][g] = sigmoid(W2 relu(W1 (mean_T(x) + segmean(x)) + b1) + b2)
const char* ws_launch_cam_gate(const void* x, int dt, int B, int T, int C, long long ld, int seg_len, const float* W1,
                               const float* b1, const float* W2, const float* b2, int H, int G, float* gate,
                               cudaStream_t s);

// ---- fbank + CMN (ws_fbank.cu)
// 25 ms frame length / 10 ms shift in samples at sample_rate 8000 or 16000 (0 for any other rate)
int ws_fbank_frame_len(int sample_rate);
int ws_fbank_frame_shift(int sample_rate);
// the largest mel filter table (nbins rows of mel_maxlen taps, padded to 4 mod 8 floats) ws_launch_fbank stages in shared memory
constexpr size_t kFbankMaxMelBytes = 16384;
// wav: [B][wav_ld] samples in int16 range (float32 if wav_is_i16 == 0 else int16).  feats fp32 [B][T][nbins], 4 <= nbins <= 128;
// window: ws_fbank_frame_len(sample_rate) taps; melw [nbins][mel_maxlen] taps of the filter that starts at FFT bin melstart[m]
const char* ws_launch_fbank(const void* wav, int wav_is_i16, long long wav_ld, int nsamples, int B, int T, int sample_rate,
                            int nbins, const float* window, const float* melw, const int* melstart, const int* mellen,
                            int mel_maxlen, float* feats, cudaStream_t s, const long long* offs = nullptr,
                            const int* lens = nullptr);   // offs: utterance b starts at wav + offs[b]; lens: frames per utterance
const char* ws_launch_cmn(float* feats, int B, int T, int Fdim, cudaStream_t s, const int* lens = nullptr);
// polyphase sinc resampling: taps [nf][2*width+of] (device), out fp32 [B][out_ld]
const char* ws_launch_resample(const void* wav, int wav_is_i16, long long wav_ld, int n_in, int B, const float* taps, int of,
                               int nf, int width, float* out, long long out_ld, int n_out, cudaStream_t s);

// ---- PLDA (ws_plda.cu), fp64 arithmetic
const char* ws_launch_f32_to_f64(const float* in, double* out, long long n, cudaStream_t s);
// out[i][j] = sum_k A[i][k]*Bm[j][k] + rowc[i] + colc[j]   (A: [M][K], Bm: [N][K], fp64; out fp32 or fp64)
const char* ws_launch_dgemm_nt(const double* A, const double* Bm, const double* rowc, const double* colc, void* out,
                               int out_is_f64, long long M, long long N, int K, long long out_ld, cudaStream_t s);
// row preparation: x <- (x - mean_vec); optional sqrt(D)-length-norm   (plda_utils.py:46-58, two_cov_plda.py:225-241)
const char* ws_launch_plda_center_norm(double* x, const double* mean_vec, long long N, int D, int do_norm,
                                       cudaStream_t s);
const char* ws_launch_plda_rownorm(double* x, long long N, int D, cudaStream_t s);
// build GEMM operands + additive constants for enroll rows / test rows (see ws_plda.cu)
const char* ws_launch_plda_prep_enroll(const double* e, const int* counts, int const_n, const double* psi,
                                       long long N, int D, int K, double* P, double* rowc, cudaStream_t s);
const char* ws_launch_plda_prep_test(const double* t, const double* psi, int const_n, long long M, int D, int K,
                                     double* Q, double* colc, cudaStream_t s);
const char* ws_launch_plda_trials(const double* P, const double* rowc, const double* Q, const double* colc,
                                  const long long* ei, const long long* ti, long long ntrials, int K, double* out,
                                  cudaStream_t s);
