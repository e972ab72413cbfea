/* wespeaker_b200 — C ABI of the H100 (sm_90a) speaker-embedding extraction + PLDA scoring engine.
 *
 * The reference (wenet-e2e/wespeaker) has no FFI layer for this path; the seams this library sits behind are
 * Python call signatures and one C++ virtual (SURVEY.md §8b).  Each entry point below cites the reference
 * interface it replaces.  Conventions: plain pointers and sizes, no torch types; every function returns 0 on
 * success and non-zero on failure with a message in ws_last_error() (thread-local); no exceptions cross the ABI.
 * "dev" pointers are CUDA device pointers owned by the caller (e.g. torch tensors' data_ptr()); `stream` is a
 * cudaStream_t passed as void* (NULL = legacy default stream).  Handles are bound to one device and are not
 * internally thread-safe (same contract as the reference's single-threaded callers, extract.py:109-139).
 */
#ifndef WESPEAKER_B200_H_
#define WESPEAKER_B200_H_

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ws_engine ws_engine;
typedef struct ws_plda ws_plda;

int ws_version(void);
const char* ws_last_error(void);

/* ---- model engine: replaces `get_speaker_model(name)(**model_args)` + `load_checkpoint` + `model(features)`
 *      (wespeaker/models/speaker_model.py:31-62, wespeaker/utils/checkpoint.py:20-85, wespeaker/bin/extract.py:68-79,133)
 *      and is the GPU back-end for `SpeakerModel::ExtractEmbedding` (runtime/core/speaker/speaker_model.h:25-32).
 * model_name: ECAPA_TDNN_c512 | ECAPA_TDNN_GLOB_c512 | ECAPA_TDNN_c1024 | ECAPA_TDNN_GLOB_c1024 | ResNet18 |
 *             ResNet34 | CAMPPlus; SURVEY section 8(f) rank 4: ResNet50 | ResNet101 | ResNet152 | ResNet221 | ResNet293 |
 *             XVEC | Res2Net34_Base | Res2Net34_Large | ERes2Net34_Base | ERes2Net34_Large | ERes2Net34_aug |
 *             SimAM_ResNet34_ASP | SimAM_ResNet100_ASP | Gemini_DF_ResNet60 | Gemini_DF_ResNet114 | Gemini_DF_ResNet183 |
 *             Gemini_DF_ResNet237.
 * precision:  "fp32" (exact IEEE fp32 FFMA path, parity <= 1e-4), "tf32x3" (tensor cores with 3xTF32 error compensation,
 *             fp32-grade accuracy), "tf32", "bf16", "fp16" (wgmma tensor cores). */
int ws_engine_create(const char* model_name, const char* precision, int feat_dim, int embed_dim, int device,
                     ws_engine** out);
/* Plan-check engine: needs NO device and never computes.  set_option / set_tensor / finalize / plan_op_name behave as on a
 * real engine - the launch plan is built with placeholder addresses and every tensor map is checked against the
 * cuTensorMapEncodeTiled rules - so a checkpoint (`load_checkpoint`, wespeaker/utils/checkpoint.py:20-85) can be validated
 * against the plan builder (missing keys, shapes, kernel envelopes) on a host without a GPU.  Every compute entry point
 * returns an error on such an engine. */
int ws_engine_create_plan_check(const char* model_name, const char* precision, int feat_dim, int embed_dim, ws_engine** out);
/* Engine options, "name" (default): what the option selects.  A flag takes any value, nonzero meaning on; an unknown name
 * or a value outside the listed ones is an error.  Setting any option but sample_rate drops the engine's cached plans.
 *   "two_emb_layer" (0)  model_args of ResNet, Res2Net / ERes2Net and Gemini DF-ResNet: two segment layers, not one
 *   "emb_bn" (0)         model_args of ECAPA-TDNN: the BatchNorm bn2 after the embedding layer
 *   "cuda_graph" (1)     replay each plan as one CUDA graph; 0 launches its kernels one by one
 *   "res2_fused" (1)     16-bit precisions: each ECAPA Res2 chain runs as one fused persistent kernel
 *   "se_fused" (1)       ECAPA with 512 or 1024 channels: each SE block's squeeze and gate run as one kernel
 *   "se_colsum" (1)      with se_fused, 16-bit precisions, T >= 128, no length mask: the SE squeeze reads column sums the
 *                        preceding conv's epilogue wrote
 *   "conv3x3" (1)        16-bit precisions: 3x3 pad-1 convs run on the halo-resident kernel where the shape fits
 *   "cam_fused" (1)      16-bit precisions, T <= 1024: CAM++ dense layers run on the fused kernel (length-masked CAM++
 *                        plans need it)
 *   "cam_block" (1)      with cam_fused: one launch per CAM++ dense block; 0: one per layer
 *   "astp_fused" (1)     16-bit precisions: attentive statistics pooling (linear2, softmax, statistics) runs as one kernel
 *   "plan_trace" (0)     real engines: ws_engine_plan_trace may write the plan with device addresses
 *   "tc_version" (3)     2: persistent / TMA-store tensor-core kernel; 3: + weight-sharing CTA clusters on the large layers.
 *                        fp32 runs FFMA whatever it says
 *   "sample_rate" (16000) 8000 or 16000: the rate of the waveforms the extract_wav entry points receive; their fbank writes
 *                        feat_dim mel bins, 4 <= feat_dim <= 128 (resample other rates first, as the reference does) */
int ws_engine_set_option(ws_engine* e, const char* key, long long value);
/* one reference state_dict entry (fp32 host data, reference key names, SURVEY.md Appendix C). */
int ws_engine_set_tensor(ws_engine* e, const char* key, const float* host_data, const long long* shape, int ndim);
/* packs / folds / converts weights once; errors if a required key is missing (strict for the forward path). */
int ws_engine_finalize(ws_engine* e);
int ws_engine_embed_dim(const ws_engine* e);
/* feats_dev: fp32 (B,T,feat_dim) already mean-normalised by the caller, as `model(features)` receives them
 * (extract.py:125-133); embs_dev: fp32 (B,embed_dim). */
int ws_engine_forward(ws_engine* e, const float* feats_dev, int B, int T, float* embs_dev, void* stream);
/* Length-masked batches (utterances of different lengths padded to a common T in ONE batch; the reference has no masking and
 * runs such sets at batch 1, extract_vox.sh:31): the result of every utterance equals what it produces alone - rows behind
 * its end stay zero wherever a convolution reads across time (the zero padding its own forward sees), SE / ASTP / TSTP /
 * CAM++ context statistics use its own frame count, CAM++'s ceil-mode segment pooling its own segment count
 * (campplus.py:117-135, pooling_layers.py:78-85,119-144).  n_frames_dev / n_samples_dev: int32[B] on the device.
 * ECAPA, ResNet and CAM++ (16-bit precisions for CAM++); XVEC is refused. */
int ws_engine_forward_masked(ws_engine* e, const float* feats_dev, const int* n_frames_dev, int B, int T, float* embs_dev,
                             void* stream);
int ws_engine_extract_wav_masked(ws_engine* e, const void* wav_dev, int wav_is_i16, long long wav_ld, const int* n_samples_dev,
                                 int max_samples, int B, const char* window_type, float* embs_dev, void* stream);
/* The same from a RAGGED buffer: utterance b is the n_samples_dev[b] samples starting at wav_dev + offsets_dev[b] samples
 * (int64[B] on the device) - concatenated PCM as a reader produces it, no padded copy.  max_samples >= every n_samples[b]
 * (it fixes the plan's T); frames behind an utterance's end are neither read nor computed.  Every utterance must hold at
 * least one 25 ms frame (400 samples; the reference's kaldi fbank fails below that too).  _async: see below. */
int ws_engine_extract_wav_ragged(ws_engine* e, const void* wav_dev, int wav_is_i16, const long long* offsets_dev,
                                 const int* n_samples_dev, int max_samples, int B, const char* window_type, float* embs_dev,
                                 void* stream);
int ws_engine_extract_wav_ragged_async(ws_engine* e, const void* wav_dev, int wav_is_i16, const long long* offsets_dev,
                                       const int* n_samples_dev, int max_samples, int B, const char* window_type,
                                       float* embs_dev, void* stream);

/* Variable-length jobs: one plan (and CUDA graph) per distinct (B, T); plans own disjoint buffers and are spread over a
 * few internal streams, so the buckets of such a job overlap on the GPU when they are enqueued with the *_async variants
 * (same arguments and semantics as ws_engine_forward / ws_engine_extract_wav, but `stream` is NOT made to wait for the
 * result) and closed with ONE ws_engine_join(e, stream).  Inputs are ordered behind `stream` as usual; outputs and inputs
 * must stay alive and untouched until the join.  The reference runs such sets at batch 1 (extract_vox.sh:31). */
int ws_engine_forward_async(ws_engine* e, const float* feats_dev, int B, int T, float* embs_dev, void* stream);
int ws_engine_extract_wav_async(ws_engine* e, const void* wav_dev, int wav_is_i16, long long wav_ld, int nsamples, int B,
                                const char* window_type, float* embs_dev, void* stream);
int ws_engine_join(ws_engine* e, void* stream);

/* same with HOST buffers (pinned or pageable): H2D + forward + D2H + stream sync; mirrors
 * `features.to(device)` ... `embeds.cpu()` (extract.py:116,135). */
int ws_engine_forward_host(ws_engine* e, const float* feats_host, int B, int T, float* embs_host);
/* waveform -> embedding on device: fbank (80 bins, 25/10 ms, dither 0) + CMN + forward.  Replaces
 * compute_fbank + apply_cmvn + model() (processor.py:496-526, dataset_utils.py:19-26, cli/speaker.py:130-167).
 * wav: (B, wav_ld) samples in int16 range — float32 (`wav * (1<<15)`) or int16 PCM; feats_out_dev optional. */
int ws_engine_extract_wav(ws_engine* e, const void* wav_dev, int wav_is_i16, long long wav_ld, int nsamples, int B,
                          const char* window_type, float* embs_dev, float* feats_out_dev, void* stream);
int ws_engine_extract_wav_host(ws_engine* e, const void* wav_host, int wav_is_i16, int nsamples, int B,
                               const char* window_type, float* embs_host);
/* Pipelined variant of ws_engine_extract_wav_host: submit() enqueues H2D (copy stream) + fbank + CMN + forward + D2H
 * for `slot` (0..3) and returns; collect() blocks until that slot's embs_host is filled.  Cycling through the slots
 * overlaps the H2D copies of the next batches with the kernels of batch i and rides out host scheduling jitter — the role DataLoader workers / prefetch_factor play
 * in extract.py:99-103.  Host buffers should be pinned and must stay valid until collect(). */
int ws_engine_submit_wav_host(ws_engine* e, int slot, const void* wav_host, int wav_is_i16, int nsamples, int B,
                              const char* window_type, float* embs_host);
int ws_engine_collect(ws_engine* e, int slot);
/* tuning aid: per-op device time (ms) of the (B,T) plan, measured with CUDA events in sequence context; returns #ops */
int ws_engine_profile_ops(ws_engine* e, int B, int T, int iters, float* ms_out, int max_ops);
const char* ws_engine_plan_op_name(ws_engine* e, int B, int T, int i, double* flops_out);   /* label + FLOPs of op i */
/* write the (B,T) launch plan as data (JSON op descriptions + allocation table) so that a test can re-evaluate the plan's
 * arithmetic on the host (tests/plan_interp.py).  Plan-check engines: placeholder addresses + fp32 weight sources.  Real
 * engines with the option plan_trace = 1: device addresses, every weight and plan-buffer allocation, no weight sources. */
int ws_engine_plan_trace(ws_engine* e, int B, int T, int masked, const char* path);   /* masked: the length-masked plan of (B,T) */
/* test aid: run ops [first, last) of the (B,T[,masked]) plan eagerly (no CUDA graph) on `stream`, building the plan if
 * needed; the caller fills the plan's inputs and orders `stream` against other uses of its buffers.  Refused on a plan-check
 * engine. */
int ws_engine_run_ops(ws_engine* e, int B, int T, int masked, int first, int last, void* stream);
/* number of this library's kernels launched by the most recent forward/extract call */
long long ws_engine_last_launches(const ws_engine* e);
void ws_engine_destroy(ws_engine* e);

/* ---- fbank + CMN: replaces torchaudio.compliance.kaldi.fbank as called at processor.py:518-525 /
 *      cli/speaker.py:92-99 and Fbank::Compute (runtime/core/frontend/fbank.h:138-198).  The entry points without a rate
 *      are 16 kHz / 80 bins; the _at variants take sample_rate 8000 or 16000 (25 ms frames every 10 ms: 200 / 80 or
 *      400 / 160 samples, a 256- or 512-point FFT) and 4 <= num_mel_bins <= 128, and refuse anything else before launching. */
int ws_fbank_num_frames(int nsamples);
/* frames of nsamples samples at sample_rate (0 below one frame); -1 for a rate other than 8000 / 16000 */
int ws_fbank_num_frames_at(int nsamples, int sample_rate);
/* Sinc resampling of (B, n_in) waveforms (int16 or float32) to new_freq: torchaudio.transforms.Resample(orig_freq, new_freq)
 * with its defaults, as the reference applies it before fbank (dataset/processor.py:242-262, cli/speaker.py:157-159).
 * out_dev: fp32 (B, out_ld), the first ws_resample_out_len(n_in, orig, new) = ceil(new * n_in / orig) samples of each row. */
int ws_resample_out_len(int n_in, int orig_freq, int new_freq);
int ws_resample(const void* wav_dev, int wav_is_i16, long long wav_ld, int n_in, int B, int orig_freq, int new_freq,
                float* out_dev, long long out_ld, void* stream);
int ws_fbank(const void* wav_dev, int wav_is_i16, long long wav_ld, int nsamples, int B, const char* window_type,
             int apply_cmn, float* feats_dev, void* stream);
/* feats_dev fp32 [B][ws_fbank_num_frames_at(nsamples, sample_rate)][num_mel_bins]; a waveform shorter than one frame is refused */
int ws_fbank_at(const void* wav_dev, int wav_is_i16, long long wav_ld, int nsamples, int B, const char* window_type,
                int sample_rate, int num_mel_bins, int apply_cmn, float* feats_dev, void* stream);
/* Ragged fbank, one launch: row b = n_frames_dev[b] frames starting at sample offsets_dev[b] of the flat buffer wav_dev
 * (total_samples samples); feats_dev fp32 [B][max_frames][80], rows behind n_frames_dev[b] are not written.  No CMN.  A frame
 * depends on its own 400 samples only, so a long segment may be presented as several rows (row k starting 160 * C * k samples
 * later) with identical results.  The caller guarantees offsets_dev[b] + 160 * (n_frames_dev[b] - 1) + 400 <= total_samples. */
int ws_fbank_ragged(const void* wav_dev, int wav_is_i16, long long total_samples, const long long* offsets_dev,
                    const int* n_frames_dev, int max_frames, int B, const char* window_type, float* feats_dev, void* stream);
/* the same at sample_rate with num_mel_bins: feats_dev [B][max_frames][num_mel_bins], frames of the rate's geometry */
int ws_fbank_ragged_at(const void* wav_dev, int wav_is_i16, long long total_samples, const long long* offsets_dev,
                       const int* n_frames_dev, int max_frames, int B, const char* window_type, int sample_rate, int num_mel_bins,
                       float* feats_dev, void* stream);

/* ---- generic fused conv operator (channels-last), the building block of the engine; exported for parity tests
 *      against torch conv1d/conv2d.  Replaces Conv1dReluBn (ecapa_tdnn.py:85-106), BasicBlock convs
 *      (resnet.py:35-69), TDNNLayer (campplus.py:55-83). */
typedef struct {
    const void* x;            /* [B][F][T][x_ld] activations, dtype below, channels [0,Cin) used */
    int B, F, T, Cin;
    long long x_ld;
    const void* w;            /* [Cout][kf*kt*Cin], tap-major (tap = jf*kt + jt), dtype below */
    int Cout, kf, kt, dil_f, dil_t, pad_f, pad_t, stride_f, stride_t;
    const float* bias;        /* added before act1 (or NULL) */
    int act1;                 /* 0 none 1 relu 2 tanh 3 sigmoid 4 hardtanh(0,20) 5 silu */
    const float* scale;       /* per-channel affine after act1 (or NULL) */
    const float* shift;
    const void* res;          /* residual added after the affine (or NULL), [positions][res_ld] */
    long long res_ld;
    int act2;
    void* out;                /* [B][Fo][To][out_ld] */
    long long out_ld;
    int dtype;                /* 0 fp32 (tf32 MMA when use_tc), 1 bf16, 2 fp16 */
    int use_tc;               /* 0: fp32 FFMA kernel, 2: persistent tensor-core kernel, 3: the same with weight-sharing clusters on
                                 large layers, 4: 3 with 3x3 convs on the halo-resident 3x3 kernel where it applies; 1 is an
                                 error */
    /* 3xTF32 (dtype 0, use_tc 2): low parts v - tf32_trunc(v) of x and w (inputs) and of out (written); all NULL = off */
    const void* x_lo;
    const void* w_lo;
    void* out_lo;
    /* fused SE squeeze (dense 1x1 conv, 16-bit dtype, use_tc >= 2, T >= 128; NULL = off): fp32 [2*ceil(B*T/64)][Cout];
     * row 2u+s = per-channel sum of the stored outputs over the positions of 64-position unit u that belong to
     * utterance floor(64u/T)+s.  Replaces the mean pass of SE_Connect (ecapa_tdnn.py:120-121). */
    float* colsum;
} ws_conv_desc;
int ws_conv(const ws_conv_desc* d, void* stream);

/* ---- SimAM attention + residual + ReLU of a SimAM-ResNet block (samresnet.py:57-70), exported for parity tests:
 *      out = relu(y * sigmoid((y - mean)^2 / (4 (var + lambda_p)) + 0.5) + res), mean / var per (b, c) over F x T_b
 *      (var divides by F*T_b - 1).  Element (b, f, t, c) of res / out is at b*sb + f*sf + t*st + c (elements); res may
 *      equal out.  All pointers are device pointers. */
typedef struct {
    const void* y;            /* [B][F][T][y_ld], channels [0,C), dtype below */
    long long y_ld;
    int B, F, T, C;
    const int* lens;          /* int32[B] frames per utterance (rows t >= lens[b] are ignored and written as zeros) or NULL */
    float lambda_p;           /* 1e-4 in the reference */
    const void* res;
    long long res_sb, res_sf, res_st;
    void* out;
    long long out_sb, out_sf, out_st;
    void* out_lo;             /* dtype 0 only, optional: out - tf32_trunc(out) with out's strides */
    int dtype;                /* 0 fp32, 1 bf16, 2 fp16 */
    float* stats;             /* fp32 [B][2][C] (written): mean, variance */
    float* partial;           /* fp32 scratch [B][F][C][2] */
} ws_simam_desc;
int ws_simam(const ws_simam_desc* d, void* stream);

/* ---- depthwise 3x3 conv + folded BN + ReLU of a Gemini DF-ResNet block (gemini_dfresnet.py:30-48), exported for parity
 *      tests: out[b,f,t,c] = relu(sum_{df,dt} w[c][df+1][dt+1] * x[b,f+df,t+dt,c] + shift[c]), zero padding outside
 *      [0,F) x [0,T_b).  fp32 accumulation in a fixed tap order, one rounding to the activation dtype.  Element (b, f, t, c)
 *      of x / out is at ((b*F + f)*T + t)*ld + c.  All pointers are device pointers, 16-byte aligned. */
typedef struct {
    const void* x;            /* [B][F][T][x_ld], channels [0,C), dtype below; C % 8 == 0 (16-bit) or C % 4 == 0 (fp32) */
    long long x_ld;
    int B, F, T, C;
    const int* lens;          /* int32[B] frames per utterance (rows t >= lens[b] are read as zeros and written as zeros) or NULL */
    const float* w;           /* fp32 [C][3][3], the BN scale folded in */
    const float* shift;       /* fp32 [C] */
    void* out;                /* [B][F][T][out_ld] */
    long long out_ld;
    void* out_lo;             /* dtype 0 only, optional: fp32 out - tf32_trunc(out) with out's layout */
    int dtype;                /* 0 fp32, 1 bf16, 2 fp16 */
} ws_dwconv_desc;
int ws_dwconv(const ws_dwconv_desc* d, void* stream);

/* ---- two-covariance PLDA scorer: replaces TwoCovPLDA.transform_embedding / log_likelihood_ratio / the trial
 *      loop of eval_sv (wespeaker/utils/plda/two_cov_plda.py:156-184,186-256), fp64 like the reference. */
int ws_plda_create(int dim, const double* mu, const double* transform, const double* psi, const double* offset,
                   int normalize_length, int device, ws_plda** out);
/* y = transform_embedding(pre(x - mean_vec)); pre = sqrt(D)-length-norm (norm_embeddings, plda_utils.py:46-58) iff
 * pre_norm != 0 — eval_sv (:225-241) pre-normalises exactly when normalize_length is set.
 * x_dev fp32 (N,D); mean_vec_host fp64 (D) or NULL; y_dev fp64 (N,D). */
int ws_plda_transform(ws_plda* p, const float* x_dev, long long N, const double* mean_vec_host, int pre_norm,
                      double* y_dev, void* stream);
/* same with fp64 rows that are already mean-subtracted (the per-speaker session means of eval_sv :218-233 stay fp64) */
int ws_plda_transform64(ws_plda* p, const double* x64_dev, long long N, int pre_norm, double* y_dev, void* stream);
/* all-pairs LLR: out[i*out_ld + j] = log_likelihood_ratio(enroll_t[i], test_t[j], n_i);  n_i = counts_dev[i] or const_n */
int ws_plda_score_matrix(ws_plda* p, const double* enroll_t_dev, const int* counts_dev, int const_n, long long N,
                         const double* test_t_dev, long long M, void* out_dev, int out_is_f64, long long out_ld,
                         void* stream);
/* listed trials only (eval_sv :248-256): out[k] = LLR(enroll_t[ei[k]], test_t[ti[k]], n_{ei[k]}) */
int ws_plda_score_trials(ws_plda* p, const double* enroll_t_dev, const int* counts_dev, int const_n, long long N,
                         const double* test_t_dev, long long M, const long long* ei_dev, const long long* ti_dev,
                         long long ntrials, double* out_dev, void* stream);
void ws_plda_destroy(ws_plda* p);

/* ---- cosine scoring + S-norm / AS-norm (SURVEY.md 8(f) rank 2): replaces trials_cosine_score (wespeaker/bin/score.py:38-72),
 *      get_mean_std (wespeaker/bin/score_norm.py:26-37) and the per-trial normalisation (score_norm.py:102-107).
 *      All pointers are device pointers; fp32 embeddings in, fp64 arithmetic. */
/* unit[r] = (x[r] - mean_vec) / |x[r] - mean_vec| (fp64, N x D); norms[r] = |x[r] - mean_vec| (the "mag" columns of
 * score_norm.py:109-110); mean_vec_dev (D fp64) and norms_dev may be NULL. */
int ws_score_unit_rows(const float* x_dev, long long N, int D, const double* mean_vec_dev, double* unit_dev,
                       double* norms_dev, void* stream);
/* out[k] = <unit[enroll_idx[k]], unit[test_idx[k]]>: cosine_similarity of the listed trials (score.py:62-63) */
int ws_score_cosine_trials(const double* unit_dev, const long long* enroll_idx_dev, const long long* test_idx_dev,
                           long long ntrials, int D, double* out_dev, void* stream);
/* mean / population std of the top_n largest cosine scores of each embedding against the M cohort rows
 * (get_mean_std; top_n >= M is S-norm).  work_dev: fp32 scratch of work_rows x M score tiles. */
int ws_score_cohort_stats(const double* unit_emb_dev, long long N, const double* unit_cohort_dev, long long M, int D,
                          int top_n, float* work_dev, long long work_rows, double* mean_dev, double* std_dev,
                          void* stream);
/* out[k] = 0.5 * ((s[k] - emean[ei[k]]) / estd[ei[k]] + (s[k] - tmean[ti[k]]) / tstd[ti[k]]) */
int ws_score_asnorm(const double* scores_dev, const long long* enroll_idx_dev, const long long* test_idx_dev,
                    long long ntrials, const double* enroll_mean_dev, const double* enroll_std_dev,
                    const double* test_mean_dev, const double* test_std_dev, double* out_dev, void* stream);

/* ---- diarization around the engine's forward (wespeaker/cli/speaker.py:213-270): sub-segment windows and the spectral
 *      clusterer's Laplacian.  All pointers are device pointers.  Tables index the rows of a flat [total_rows][feat_dim] fp32
 *      feature buffer; an entry that is not inside [0, total_rows) or has len <= 0 is never read and its output is zeros. */
#define WS_DIAR_MAX_M 16384
/* out[s][c] = mean over rows [row0[s], row0[s] + len[s]) of feats[.][c] (the segment CMN of diar/make_fbank.py:85-86) */
int ws_diar_col_means(const float* feats_dev, long long total_rows, int feat_dim, const int* row0_dev, const int* len_dev,
                      int S, float* out_dev /* [S][feat_dim] */, void* stream);
/* diar/extract_emb.py:55-83 + cli/speaker.py:110-112: out[w][r][c] = feats[row0[w] + (r mod len[w])][c] - mean_w[c], r in
 * [0, window_fs).  mean_w = the mean of the window_fs tiled rows when subseg_cmn != 0; else seg_mean[seg_of[w]] when
 * seg_mean_dev ([S][feat_dim]) is given, else 0.  feat_dim <= 256. */
int ws_diar_windows(const float* feats_dev, long long total_rows, int feat_dim, const int* row0_dev, const int* len_dev,
                    int W, int window_fs, int subseg_cmn, const float* seg_mean_dev, const int* seg_of_dev, int S,
                    float* out_dev /* [W][window_fs][feat_dim] */, void* stream);
/* diar/spectral_clusterer.py:35-56 on m unit rows (ws_score_unit_rows): cosine affinity, the keep_per_row largest of each row
 * (the diagonal competes, as there) set to 1 and the rest to 0 - ties at the boundary go to the lowest columns -, symmetrised,
 * diagonal cleared, lap = diag(row sums) - matrix in fp64.  work_dev: fp32 scratch of work_rows x m cosine tiles; adj_dev:
 * m x m bytes of scratch.  m > WS_DIAR_MAX_M is refused. */
int ws_diar_laplacian(const double* unit_dev, long long m, int D, long long keep_per_row, float* work_dev,
                      long long work_rows, unsigned char* adj_dev, double* lap_dev /* [m][m] */, void* stream);

/* ---- verification metrics (wespeaker/utils/score_metrics.py:58-116 behind bin/compute_metrics.py and bin/compute_det.py):
 *      the rbst miss / false-alarm curves over the trials in the stable ascending order of (score, trial line), the EER
 *      crossing and the minimum detection cost per operating point.  -0.0 == +0.0 (ordered by line), +-inf are ordered. */
#define WS_METRICS_MAX_POINTS 16
#define WS_METRICS_MAX_N 2147483647LL
/* status word bits (out[7]): refusals only the data can reveal; with any of the first three set nothing but out[7] is written */
#define WS_METRICS_NAN_SCORE 1u
#define WS_METRICS_BAD_LABEL 2u     /* a label other than 0 or 1 */
#define WS_METRICS_EMPTY_CLASS 4u   /* no target or no non-target trial */
#define WS_METRICS_NO_X2 8u         /* fnr - fpr is >= 0 everywhere: the EER has no lower crossing point */
/* device workspace for n trials; 0 when n is outside [1, WS_METRICS_MAX_N] */
size_t ws_metrics_work_bytes(long long n);
/* scores_dev fp64 [n], labels_dev uint8 [n] (1 target, 0 non-target); p_target / c_miss / c_fa: HOST arrays of n_points
 * (1..16) operating points, 0 < p_target < 1, finite costs >= 0.  out_dev fp64 [8 + n_points] = fnr(x1), fpr(x1), fnr(x2),
 * fpr(x2), the score at x1, x1, x2, status, then per point min_i (c_miss * fnr_i) * p + (c_fa * fpr_i) * (1 - p) (c_det; the
 * caller divides by c_def).  x1 = first i with fnr_i - fpr_i >= 0, x2 = last i with fnr_i - fpr_i < 0.  Optional (NULL to
 * skip): order_dev int32 [n] trial indices in sorted order, fnr_dev / fpr_dev fp64 [n] curves.  stage_events: NULL, or 11
 * cudaEvent_t recorded on the stream before the keys pass, after it, after each of the 8 radix passes and after the
 * evaluation (profiling).  Argument errors are refused before anything is launched; the host never waits on the device. */
int ws_metrics_eval(const double* scores_dev, const unsigned char* labels_dev, long long n, const double* p_target,
                    const double* c_miss, const double* c_fa, int n_points, void* work_dev, size_t work_bytes,
                    double* out_dev, int* order_dev, double* fnr_dev, double* fpr_dev, void* stream,
                    void* const* stage_events);

#ifdef __cplusplus
}
#endif
#endif /* WESPEAKER_B200_H_ */
