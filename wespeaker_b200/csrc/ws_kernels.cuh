// Host-callable launchers for the bandwidth-bound kernels (ws_kernels.cu, ws_fbank.cu, ws_plda.cu).
// All return nullptr on success or a static error string.
#pragma once
#include "ws_common.cuh"

// ---- plan ops: one argument record per op kind, read by its launcher and by its plan-trace writer (ws_host.h).  Shape-dependent
// kernel choices (*_kernel / *_plan) are made once, at plan build.  (`lo` / `plo`: optional fp32 twin receiving v - tf32_trunc(v)
// for the 3xTF32 GEMM path; nullptr otherwise)

// channels-last activation view: element (b,f,t,c) at p[((b*F+f)*T+t)*ld + c]
struct WsView {
    void* p = nullptr;
    void* plo = nullptr;  // 3xTF32 mode: twin buffer holding x - tf32_trunc(x)
    int B = 0, F = 1, T = 0, C = 0;
    long long ld = 0;
    int dt = WS_F32;
    long long npos() const { return (long long)B * F * T; }
    // the same buffer as a dense (B, F, T, C) tensor
    WsView shaped(int b, int f, int t, int c) const {
        WsView v = *this;
        v.B = b; v.F = f; v.T = t; v.C = c; v.ld = c;
        return v;
    }
    WsView ch(int c0, int c) const {
        WsView v = *this;
        v.p = (char*)p + (size_t)c0 * ws_esize(dt);
        if (plo) v.plo = (char*)plo + (size_t)c0 * ws_esize(dt);
        v.C = c;
        return v;
    }
};

struct WsConvert { const float* in; void* out; float* lo; int dt; long long n; };
const char* ws_launch_convert(const WsConvert& a, cudaStream_t s);

// mean (and optional unbiased std, sqrt(var + eps)) over T for every (b, f, c) of x's channels.  Optional per-channel
// pre-affine + relu (CAM++ out_nonlinear, campplus.py:378-379).  Output (dtype odt):
//   mean -> out[b*out_ld + c*F + f],  std -> out[b*out_ld + std_off + c*F + f]   (std skipped if std_off < 0)
enum WsTstatsKernel { WS_TSTATS_SCALAR, WS_TSTATS_TMEAN8, WS_TSTATS_8 };
struct WsTstats { WsView x; const float* pre_scale; const float* pre_shift; void* out; int odt; long long out_ld; int std_off;
    float eps; const int* lens; int kernel = WS_TSTATS_SCALAR; };
int ws_tstats_kernel(const WsTstats& a);
const char* ws_launch_tstats(const WsTstats& a, cudaStream_t s);

// length-masked batches (per-utterance frame counts `lens`, device int32): zero the rows t >= lens[b]; derive the frame
// counts behind stride-2 layers (lens is [levels][B], level 0 = input); frames from sample counts
struct WsZeroTail { WsView x; const int* lens; };
const char* ws_launch_zero_tail(const WsZeroTail& a, cudaStream_t s);
struct WsLensDerive { int* lens; int B, T, levels; };
const char* ws_launch_lens_derive(const WsLensDerive& a, cudaStream_t s);
const char* ws_launch_frames_from_samples(const int* nsamp, int* lens, int B, int Tmax, int frame_len, int shift, cudaStream_t s);

// out[r][o] = act( sum_i W[o][i] * (in[r][i] + in2[r / rows_per_b][i]) + bias[o] ),  fp32 in/out, W fp32 [O][I]; split K
// over nsplit CTAs (then wsp: fp32 [nsplit][R][O] partial sums)
enum WsLinearKernel { WS_LINEAR_ROWS16, WS_LINEAR_ROWS64 };
struct WsLinear { const float* in; long long in_ld; const float* in2; long long in2_ld; int rows_per_b; const float* W;
    const float* bias; float* out; long long out_ld; int R, I, O, act; float* wsp; int nsplit = 1;
    int kernel = WS_LINEAR_ROWS16; };
// a.kernel and a.nsplit for a's shape: K is split so that the launch fills the `sms` SMs (these layers are latency-bound)
void ws_linear_rows_plan(WsLinear& a, int sms);
const char* ws_launch_linear_rows(const WsLinear& a, cudaStream_t s);

// SE apply + residual (ecapa_tdnn.py:124,157): out[pos][c] = x[pos][c]*gate[b][c] + res[pos][c]
struct WsScaleResidual { WsView x; const float* gate; WsView res, out; };
const char* ws_launch_scale_residual(const WsScaleResidual& a, cudaStream_t s);

// ERes2Net AFF combine (eres2net.py:97-100): out[pos][c] = x * (1 + t) + y * (2 - (1 + t)), t = the tanh'd attention map
struct WsAffCombine { WsView x, y, t, out; };
const char* ws_launch_aff_combine(const WsAffCombine& a, cudaStream_t s);

// ASTP statistics (pooling_layers.py:138-144): softmax over T of logits, weighted mean / std = sqrt(max(var, var_floor)) of x
// (ECAPA's ASTP floors the variance at 1e-7, SimAM-ResNet's ASP at 1e-5, pooling_layers.py:198-203); logits are read with
// x's row pitch
enum WsAstpStatsKernel { WS_ASTP_STATS_SCALAR, WS_ASTP_STATS4 };
struct WsAstpStats { WsView x, logits; float* stats /*[B][2C]*/; float var_floor; const int* lens;
    int kernel = WS_ASTP_STATS_SCALAR; };
int ws_astp_stats_kernel(const WsAstpStats& a);
const char* ws_launch_astp_stats(const WsAstpStats& a, cudaStream_t s);

// SimAM (ws_simam.cu, samresnet.py:65-70).  Statistics of y [B][F][T][ld] (channels [0,C)) per (b, c) over F x (its own
// frames): stats fp32 [B][2][C] = mean, variance over n = F*T_b - 1; partial: fp32 scratch [B][F][C][2] (two launches).
struct WsSimamStats { WsView y; float* partial; float* stats; const int* lens; };
const char* ws_launch_simam_stats(const WsSimamStats& a, cudaStream_t s);
// element (b, f, t, c) of a map at b*sb.b + f*sb.f + t*sb.t + c (elements)
struct WsMapStrides { long long b, f, t; };
// out = relu(y * sigmoid((y - mean)^2 / (4 (var + lambda)) + 0.5) + res) with y's extents; res may alias out; rows
// t >= lens[b] of out are zeroed; out_lo (optional, fp32 with out's strides) receives the 3xTF32 low part
struct WsSimamApply { WsView y; const float* stats; float lambda; const void* res; WsMapStrides rs; void* out; float* out_lo;
    WsMapStrides os; const int* lens; };
const char* ws_launch_simam_apply(const WsSimamApply& a, cudaStream_t s);

// Depthwise 3x3 pad-1 conv + folded BN + ReLU (ws_dwconv.cu, gemini_dfresnet.py:37-44): out = relu(dwconv(x, w) + shift) with
// w fp32 [C][3][3], shift fp32 [C], x's extents and dtype; rows t >= lens[b] are read as zeros and written as zeros; out.plo
// (fp32 activations, optional) receives the 3xTF32 low part.  C % 8 == 0 in 16-bit, C % 4 == 0 in fp32.
struct WsDwconv3x3 { WsView x; const float* w; const float* shift; WsView out; const int* lens; };
const char* ws_launch_dwconv3x3(const WsDwconv3x3& a, cudaStream_t s);

// out[pos][c] = relu(x[pos][c]*scale[c] + shift[c]) over x's channels (CAM++ pre-activation BN-ReLU, campplus.py:164-166,214)
struct WsBnRelu { WsView x; const float* scale; const float* shift; WsView out; };
const char* ws_launch_bnrelu(const WsBnRelu& a, cudaStream_t s);

// ResNet / FCM stem: Conv2d(1->Cout,3x3,pad 1) + folded BN + ReLU.  feats fp32 [B][T][Fdim] -> out (B, Fdim, T, Cout)
struct WsStem { const float* feats; const float* w9 /*[Cout][9]*/; const float* shift; WsView out; const int* lens; };
const char* ws_launch_stem(const WsStem& a, cudaStream_t s);

// CAM context (campplus.py:108-135): mean over T and per-segment (seg_len) means with ceil-mode partial segment
struct WsSegMeans { WsView x; int seg_len; float* mean; float* segmean /*[B][nseg][C]*/; };
const char* ws_launch_seg_means(const WsSegMeans& a, cudaStream_t s);

// fused SE gate: gate[b][c] = sigmoid(W2 relu(W1 mean_T(x[b]) + b1) + b2); W2t is W2 transposed to [H][C]; colsum: the
// per-unit column sums of x that the producing conv's epilogue wrote (instead of a pass over x), or nullptr
struct WsSeGate { WsView x; const float* W1; const float* b1; const float* W2t; const float* b2; int H; float* gate;
    const float* colsum; const int* lens; };
const char* ws_launch_se_gate(const WsSeGate& a, cudaStream_t s);
// fused CAM context gate: gate[b][seg][g] = sigmoid(W2 relu(W1 (mean_T(x) + segmean(x)) + b1) + b2)
struct WsCamGate { WsView x; int seg_len; const float* W1; const float* b1; const float* W2; const float* b2; int H, G;
    float* gate; };
const char* ws_launch_cam_gate(const WsCamGate& a, cudaStream_t s);

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
