// Speaker-embedding engine: the model table, the per-(B,T) plan cache (plans built by the model families' builders,
// ws_build_*.cu), CUDA-graph replay, the engine's streams, fbank frontend and resampling tables, and the C ABI declared in
// include/wespeaker_b200.h.
//
// Reference behaviour being reproduced (file:line in wenet-e2e/wespeaker, wespeaker/):
//   utils/checkpoint.py:20-85, bin/extract.py:109-139.
#include <cstdio>
#include <cstdlib>

#include "ws_plan.h"

using namespace ws;

namespace {

// ------------------------------------------------------------------------------------------------ model table
ModelCfg ecapa(int channels, bool glob) { ModelCfg c; c.channels = channels; c.glob = glob; return c; }
ModelCfg blocks(int l1, int l2, int l3, int l4, bool bottleneck = false) { ModelCfg c; c.num_blocks = {l1, l2, l3, l4}; c.bottleneck = bottleneck; return c; }
// Res2Net / ERes2Net: stem width m, AFF fusion, baseWidth, scale, expansion (res2net.py:202-221, eres2net.py:393-431)
ModelCfg res2(int m, bool fuse, int base_width = 32, int scale = 2, int expansion = 2) {
    ModelCfg c = blocks(3, 4, 6, 3);
    c.m = m; c.fuse = fuse; c.base_width = base_width; c.scale = scale; c.expansion = expansion;
    return c;
}

struct ModelRow { const char* name; PlanBuilder build; ModelCfg cfg; };
// every model name the engine accepts (wespeaker_b200.models.SUPPORTED_MODELS), with its family's builder
const ModelRow kModels[] = {
    {"ECAPA_TDNN_c512", build_ecapa, ecapa(512, false)},
    {"ECAPA_TDNN_GLOB_c512", build_ecapa, ecapa(512, true)},
    {"ECAPA_TDNN_c1024", build_ecapa, ecapa(1024, false)},
    {"ECAPA_TDNN_GLOB_c1024", build_ecapa, ecapa(1024, true)},
    {"ResNet18", build_resnet, blocks(2, 2, 2, 2)},
    {"ResNet34", build_resnet, blocks(3, 4, 6, 3)},
    {"ResNet50", build_resnet, blocks(3, 4, 6, 3, true)},
    {"ResNet101", build_resnet, blocks(3, 4, 23, 3, true)},
    {"ResNet152", build_resnet, blocks(3, 8, 36, 3, true)},
    {"ResNet221", build_resnet, blocks(6, 16, 48, 3, true)},
    {"ResNet293", build_resnet, blocks(10, 20, 64, 3, true)},
    {"XVEC", build_xvec, {}},
    {"Res2Net34_Base", build_res2net, res2(32, false)},
    {"Res2Net34_Large", build_res2net, res2(64, false)},
    {"ERes2Net34_Base", build_res2net, res2(32, true)},
    {"ERes2Net34_Large", build_res2net, res2(64, true)},
    {"ERes2Net34_aug", build_res2net, res2(64, true, 24, 3, 4)},
    {"CAMPPlus", build_campplus, {}},
    {"SimAM_ResNet34_ASP", build_simam_resnet, blocks(3, 4, 6, 3)},
    {"SimAM_ResNet100_ASP", build_simam_resnet, blocks(6, 16, 24, 3)},
    {"Gemini_DF_ResNet60", build_gemini, blocks(3, 3, 9, 3)},
    {"Gemini_DF_ResNet114", build_gemini, blocks(3, 3, 27, 3)},
    {"Gemini_DF_ResNet183", build_gemini, blocks(3, 8, 45, 3)},
    {"Gemini_DF_ResNet237", build_gemini, blocks(3, 8, 63, 3)},
};

// every precision the engine accepts: activation dtype, tensor-core level (ws_engine::tc) and 3xTF32 error compensation
struct PrecisionRow { const char* name; int act_dt; int tc; bool split; };
const PrecisionRow kPrecisions[] = {
    {"fp32", WS_F32, 0, false},
    {"tf32", WS_F32, 3, false},
    {"tf32x3", WS_F32, 3, true},
    {"bf16", WS_BF16, 3, false},
    {"fp16", WS_F16, 3, false},
};

// every option ws_engine_set_option accepts, with the field it sets: a flag, or a number it checks first
struct OptionRow { const char* name; bool EngineOptions::*flag; int EngineOptions::*number; };
using O = EngineOptions;
const OptionRow kOptions[] = {
    {"two_emb_layer", &O::two_emb_layer}, {"emb_bn", &O::emb_bn}, {"cuda_graph", &O::cuda_graph}, {"plan_trace", &O::plan_trace},
    {"res2_fused", &O::res2_fused}, {"se_fused", &O::se_fused}, {"se_colsum", &O::se_colsum}, {"conv3x3", &O::conv3x3},
    {"cam_fused", &O::cam_fused}, {"cam_block", &O::cam_block}, {"astp_fused", &O::astp_fused},
    {"tc_version", nullptr, &O::tc_version}, {"sample_rate", nullptr, &O::sample_rate},
};

// the row of `table` named `name` (nullptr: none)
template <class Row, size_t N> const Row* row_named(const Row (&table)[N], const std::string& name) {
    for (const Row& r : table)
        if (name == r.name) return &r;
    return nullptr;
}

// ------------------------------------------------------------------------------------------------ plan cache
Plan* get_plan(ws_engine* e, int B, int T, bool masked = false) {
    auto key = std::make_pair(B, 2 * T + (masked ? 1 : 0));
    auto it = e->plans.find(key);
    if (it != e->plans.end()) {
        it->second->last_use = ++e->use_clock;
        return it->second.get();
    }
    if (B <= 0 || T <= 0) { set_err("forward: B and T must be positive"); return nullptr; }
    std::unique_ptr<Plan> p(new Plan());
    p->B = B; p->T = T; p->masked = masked; p->check = e->plan_check;
    PlanCheckScope check_scope(e->plan_check);
    Builder b(*e, *p);
    if (masked) {
        p->lens = (int*)b.raw((size_t)4 * B * sizeof(int));
        if (b.good()) b.push(WsLensDerive{p->lens, B, T, 4}, ws_launch_lens_derive, "lens_derive");
    }
    p->feats_in = b.f32((size_t)B * T * e->feat_dim);
    p->emb = b.f32((size_t)B * e->embed_dim);
    if (!b.good() || !e->build(b)) return nullptr;
    // Plan cache policy: one plan (buffers + CUDA graph) per distinct (B,T); evict least-recently-used plans beyond 64
    // entries or 48 GB of activation memory (variable-length workloads touch many shapes; 180 GB HBM is shared with the
    // caller's tensors).  Eviction waits for in-flight work on the engine stream.
    size_t total = p->bytes;
    for (auto& kv : e->plans) total += kv.second->bytes;
    while (!e->plans.empty() && (e->plans.size() >= 64 || total > (size_t)48 << 30)) {
        auto victim = e->plans.begin();
        for (auto i2 = e->plans.begin(); i2 != e->plans.end(); ++i2)
            if (i2->second->last_use < victim->second->last_use) victim = i2;
        if (!e->plan_check) cudaDeviceSynchronize();   // the victim may be in flight on any lane
        total -= victim->second->bytes;
        e->plans.erase(victim);
    }
    p->last_use = ++e->use_clock;
    p->lane = e->next_lane++ % ws_engine::kLanes;
    if (!e->plan_check && cudaEventCreateWithFlags(&p->done, cudaEventDisableTiming) != cudaSuccess) { set_err("plan event creation failed"); return nullptr; }
    Plan* raw = p.get();
    e->plans[key] = std::move(p);
    return raw;
}

// staged: kernels the entry point launched ahead of the plan (fbank, CMN, frame counts), counted in last_launches
int run_plan(ws_engine* e, Plan* p, cudaStream_t s, int staged) {
    const bool want_graph = e->opts.cuda_graph && !p->graph_failed;
    if (want_graph && p->gexec == nullptr) {
        cudaGraph_t g = nullptr;
        if (cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
            const char* m = nullptr;
            for (auto& op : p->ops) { m = op.run(s); if (m) break; }
            cudaError_t ce = cudaStreamEndCapture(s, &g);
            if (m == nullptr && ce == cudaSuccess && g != nullptr &&
                cudaGraphInstantiate(&p->gexec, g, 0) == cudaSuccess) {
            } else {
                p->gexec = nullptr;
                p->graph_failed = true;
                if (m) { set_err(std::string("kernel launch failed during capture: ") + m); if (g) cudaGraphDestroy(g); return 1; }
            }
            if (g) cudaGraphDestroy(g);
            cudaGetLastError();
        } else {
            p->graph_failed = true;
            cudaGetLastError();
        }
    }
    if (p->gexec != nullptr) {
        WS_CK(cudaGraphLaunch(p->gexec, s));
    } else {
        for (auto& op : p->ops) WS_CKS(op.run(s));
    }
    e->last_launches = (long long)p->ops.size() + p->extra_launches + staged;
    return 0;
}

// why the frontend cannot run at (sample_rate, bins) (nullptr = it can)
const char* fbank_unsupported(int sample_rate, int bins) {
    if (ws_fbank_frame_len(sample_rate) == 0) return "sample rate must be 8000 or 16000 (resample first)";
    if (bins < 4 || bins > 128) return "num_mel_bins must be in [4, 128]";
    return nullptr;
}

// Window and mel banks of one (window type, sample rate, bin count), uploaded on first use.  Restates torchaudio kaldi.py
// _feature_window_function (25 ms, non-periodic) and get_mel_banks (20 Hz .. Nyquist, FFT bin width sample_rate / Nfft) in
// float32 like the reference.
const FbankTables* fbank_tables(ws_engine* e, const char* window_type, int rate, int nb) {
    const std::string wt = window_type ? window_type : "hamming";
    if (const char* why = fbank_unsupported(rate, nb)) { set_err(std::string("fbank: ") + why); return nullptr; }
    const auto key = std::make_tuple(wt, rate, nb);
    auto it = e->fb.find(key);
    if (it != e->fb.end()) return &it->second;
    const int fl = ws_fbank_frame_len(rate), nfft = rate == 16000 ? 512 : 256, nbins_fft = nfft / 2;
    std::vector<float> win(fl);
    for (int j = 0; j < fl; ++j) {
        const double c = std::cos(2.0 * M_PI * j / (fl - 1));
        if (wt == "hamming") win[j] = (float)(0.54 - 0.46 * c);
        else if (wt == "povey") win[j] = (float)std::pow(0.5 - 0.5 * c, 0.85);
        else if (wt == "hanning") win[j] = (float)(0.5 - 0.5 * c);
        else if (wt == "rectangular") win[j] = 1.f;
        else { set_err("unknown window_type " + wt); return nullptr; }
    }
    const double mel_low = 1127.0 * std::log(1.0 + 20.0 / 700.0), mel_high = 1127.0 * std::log(1.0 + 0.5 * rate / 700.0);
    const float delta = (float)((mel_high - mel_low) / (nb + 1)), lowf = (float)mel_low;
    const float bin_width = (float)rate / (float)nfft;
    std::vector<std::vector<float>> rows(nb, std::vector<float>(nbins_fft, 0.f));
    std::vector<int> start(nb, 0), len(nb, 0);
    int maxlen = 1;
    for (int m = 0; m < nb; ++m) {
        const float left = lowf + (float)m * delta, center = lowf + ((float)m + 1.0f) * delta, right = lowf + ((float)m + 2.0f) * delta;
        int first = -1, last = -1;
        for (int k = 0; k < nbins_fft; ++k) {
            const float mel = 1127.0f * std::log(1.0f + (bin_width * (float)k) / 700.0f);
            const float up = (mel - left) / (center - left), down = (right - mel) / (right - center);
            const float wv = std::max(0.f, std::min(up, down));
            rows[m][k] = wv;
            if (wv > 0.f) { if (first < 0) first = k; last = k; }
        }
        if (first >= 0) { start[m] = first; len[m] = last - first + 1; maxlen = std::max(maxlen, len[m]); }
    }
    std::vector<float> melw((size_t)nb * maxlen, 0.f);
    for (int m = 0; m < nb; ++m)
        for (int i = 0; i < len[m]; ++i) melw[(size_t)m * maxlen + i] = rows[m][start[m] + i];
    FbankTables t;
    t.rate = rate; t.bins = nb; t.maxlen = maxlen;
    if (cudaMalloc(&t.window, fl * 4) != cudaSuccess || cudaMalloc(&t.melw, melw.size() * 4) != cudaSuccess ||
        cudaMalloc(&t.melstart, nb * 4) != cudaSuccess || cudaMalloc(&t.mellen, nb * 4) != cudaSuccess) {
        set_err("fbank tables: cudaMalloc failed");
        return nullptr;
    }
    cudaMemcpy(t.window, win.data(), fl * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(t.melw, melw.data(), melw.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(t.melstart, start.data(), nb * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(t.mellen, len.data(), nb * 4, cudaMemcpyHostToDevice);
    return &(e->fb[key] = t);
}

// engine-less fbank tables for ws_fbank()
ws_engine* fbank_holder(int device) {
    static std::map<int, ws_engine*> holders;
    ws_engine*& h = holders[device];
    if (h == nullptr) { h = new ws_engine(); h->device = device; }
    return h;
}

// fbank (+ CMN) of B waveforms of nsamples samples (the longest, with lens) into feats [B][T][t->bins]; offs / lens: ws_launch_fbank
int fbank_into(const FbankTables* t, const void* wav, int is_i16, long long wav_ld, int nsamples, int B, int apply_cmn, float* feats,
               cudaStream_t s, const long long* offs = nullptr, const int* lens = nullptr) {
    const int T = ws_fbank_num_frames_at(nsamples, t->rate);
    WS_CKS(ws_launch_fbank(wav, is_i16, wav_ld, nsamples, B, T, t->rate, t->bins, t->window, t->melw, t->melstart, t->mellen, t->maxlen,
                           feats, s, offs, lens));
    if (apply_cmn) WS_CKS(ws_launch_cmn(feats, B, T, t->bins, s, lens));
    return 0;
}

// grow the device staging buffer *buf (capacity *cap) to hold `bytes`; its contents are not kept
int grow(void** buf, size_t* cap, size_t bytes) {
    if (bytes <= *cap) return 0;
    if (*buf) cudaFree(*buf);
    *buf = nullptr; *cap = 0;
    WS_CK(cudaMalloc(buf, bytes));
    *cap = bytes;
    return 0;
}

// ------------------------------------------------------------------------------------------------ one run of a plan
// why a compute entry point cannot run on this engine (nullptr = it can)
const char* not_runnable(const ws_engine* e) {
    if (e->plan_check) return " on a plan-check engine (it builds launch plans without a device and never computes)";
    if (!e->finalized) return " before ws_engine_finalize";
    return nullptr;
}

// the (B, T[, masked]) plan, built on the engine's device (plan-check engines have none) unless it is cached
Plan* plan_of(ws_engine* e, int B, int T, bool masked) {
    const cudaError_t ce = e->plan_check ? cudaSuccess : cudaSetDevice(e->device);
    if (ce != cudaSuccess) { set_err(std::string("cudaSetDevice: ") + cudaGetErrorString(ce)); return nullptr; }
    return get_plan(e, B, T, masked);
}

// One run of a plan through a compute entry point.  The device-pointer entry points run on the plan's lane, ordered behind
// the caller's stream; the host-pointer ones run on e->st.
struct Run {
    ws_engine* e;
    const char* who;                   // the entry point, for error messages
    bool host;                         // host-pointer entry point
    cudaStream_t user = nullptr;       // device-pointer entry points: the caller's stream
    Plan* p = nullptr;
    cudaStream_t s = nullptr;          // where the run is enqueued: the plan's lane, or e->st
    const FbankTables* fb = nullptr;   // waveform entry points: the frontend's tables
};

// The start of every compute entry point: refuse on an engine that cannot compute; for waveform input (samples >= 0: T is
// derived from the longest one) check the bin and frame counts; get the plan and the fbank tables (uploaded on first use); then
// order the run behind the plan's previous use and, on the device-pointer paths, behind the caller's stream.
int begin_run(Run& r, int B, int T, bool masked, int samples = -1, const char* window_type = nullptr) {
    ws_engine* e = r.e;
    if (const char* nr = not_runnable(e)) { set_err(std::string(r.who) + nr); return 1; }
    if (samples >= 0) {
        // the fbank frontend writes feat_dim mel bins at the engine's sample rate
        if (const char* why = fbank_unsupported(e->opts.sample_rate, e->feat_dim)) { set_err(std::string(r.who) + ": " + why); return 1; }
        T = ws_fbank_num_frames_at(samples, e->opts.sample_rate);
        if (T <= 0) { set_err(std::string(r.who) + ": waveforms shorter than one 25 ms frame"); return 1; }
    }
    if ((r.p = plan_of(e, B, T, masked)) == nullptr) return 1;
    if (samples >= 0 && (r.fb = fbank_tables(e, window_type, e->opts.sample_rate, e->feat_dim)) == nullptr) return 1;
    r.s = r.host || !e->lanes[r.p->lane] ? e->st : e->lanes[r.p->lane];
    if (!r.host) {
        WS_CK(cudaEventRecord(e->ev_in, r.user));
        WS_CK(cudaStreamWaitEvent(r.s, e->ev_in, 0));
    }
    WS_CK(cudaStreamWaitEvent(r.s, r.p->done, 0));
    return 0;
}

// The end of every compute entry point: run the plan behind the `staged` kernels the entry point launched ahead of it, copy
// the embeddings out and record the plan's use; with wait, the caller's stream (host paths: the host) then waits for it.
int finish_run(Run& r, int staged, float* embs, bool wait) {
    if (run_plan(r.e, r.p, r.s, staged)) return 1;
    WS_CK(cudaMemcpyAsync(embs, r.p->emb, (size_t)r.p->B * r.e->embed_dim * 4, r.host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, r.s));
    WS_CK(cudaEventRecord(r.p->done, r.s));
    if (wait && r.host) WS_CK(cudaStreamSynchronize(r.s));
    else if (wait) WS_CK(cudaStreamWaitEvent(r.user, r.p->done, 0));
    return 0;
}

}  // namespace

// ================================================================================================= C ABI

extern "C" {

// model name + precision -> engine configuration (shared by ws_engine_create and ws_engine_create_plan_check)
static int configure_engine(ws_engine* e, const char* model_name, const char* precision, int feat_dim, int embed_dim, int device) {
    e->model = model_name; e->prec = precision; e->feat_dim = feat_dim; e->embed_dim = embed_dim; e->device = device;
    const ModelRow* row = row_named(kModels, e->model);
    if (row == nullptr) { set_err("unknown / out-of-scope model name: " + e->model); return 1; }
    e->build = row->build;
    e->cfg = row->cfg;
    const PrecisionRow* prec = row_named(kPrecisions, e->prec);
    if (prec == nullptr) { set_err("unknown precision (fp32|tf32x3|tf32|bf16|fp16): " + e->prec); return 1; }
    e->act_dt = prec->act_dt; e->tc = prec->tc; e->split = prec->split;
    if (feat_dim % 8 != 0) { set_err("feat_dim must be a multiple of 8"); return 1; }
    return 0;
}

int ws_engine_create(const char* model_name, const char* precision, int feat_dim, int embed_dim, int device,
                     ws_engine** out) {
    if (!model_name || !precision || !out) { set_err("ws_engine_create: null argument"); return 1; }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        set_err("ws_engine_create: no CUDA device (this engine has no CPU fallback)");
        return 1;
    }
    WS_CK(cudaSetDevice(device));
    int cc_major = 0, cc_minor = 0;
    WS_CK(cudaDeviceGetAttribute(&cc_major, cudaDevAttrComputeCapabilityMajor, device));
    WS_CK(cudaDeviceGetAttribute(&cc_minor, cudaDevAttrComputeCapabilityMinor, device));
    if (cc_major != 9 || cc_minor != 0) {   // sm_90a code runs on compute capability 9.0 only
        set_err("ws_engine_create: device " + std::to_string(device) + " has compute capability " + std::to_string(cc_major) + "." +
                std::to_string(cc_minor) + "; the kernels are built for sm_90a (compute capability 9.0) only");
        return 1;
    }
    std::unique_ptr<ws_engine> e(new ws_engine());
    if (configure_engine(e.get(), model_name, precision, feat_dim, embed_dim, device)) return 1;
    WS_CK(cudaStreamCreateWithFlags(&e->st, cudaStreamNonBlocking));
    e->lanes[0] = e->st;
    for (int i = 1; i < ws_engine::kLanes; ++i) WS_CK(cudaStreamCreateWithFlags(&e->lanes[i], cudaStreamNonBlocking));
    WS_CK(cudaEventCreateWithFlags(&e->ev_in, cudaEventDisableTiming));
    WS_CK(cudaEventCreateWithFlags(&e->ev_out, cudaEventDisableTiming));
    *out = e.release();
    return 0;
}

// An engine that only BUILDS launch plans: no device is touched, nothing is computed, every compute entry point refuses.
// ws_engine_set_tensor / ws_engine_set_option / ws_engine_finalize / ws_engine_plan_op_name work as on a real engine, so a
// checkpoint can be validated against the plan builder (missing keys, shapes, kernel envelopes, tensor-map alignment rules)
// on a host without a GPU.
int ws_engine_create_plan_check(const char* model_name, const char* precision, int feat_dim, int embed_dim, ws_engine** out) {
    if (!model_name || !precision || !out) { set_err("ws_engine_create_plan_check: null argument"); return 1; }
    std::unique_ptr<ws_engine> e(new ws_engine());
    e->plan_check = true;
    if (configure_engine(e.get(), model_name, precision, feat_dim, embed_dim, 0)) return 1;
    *out = e.release();
    return 0;
}

int ws_engine_set_option(ws_engine* e, const char* key, long long value) {
    if (!e || !key) { set_err("ws_engine_set_option: null argument"); return 1; }
    const OptionRow* row = row_named(kOptions, key);
    if (row == nullptr) { set_err(std::string("unknown option ") + key); return 1; }
    const bool rate = row->number == &O::sample_rate;
    if (row->number == &O::tc_version && value != 2 && value != 3) {
        set_err("tc_version must be 2 (persistent tensor-core kernel) or 3 (+ weight-sharing clusters); 1, the one-tile-per-CTA "
                "kernel, was removed");
        return 1;
    }
    if (rate && (ws_fbank_frame_len((int)value) == 0 || value != (int)value)) { set_err("sample_rate must be 8000 or 16000 (resample first)"); return 1; }
    if (row->flag) e->opts.*row->flag = value != 0;
    else e->opts.*row->number = (int)value;
    if (!rate) e->plans.clear();   // plans do not depend on the waveform entry points' rate, so they are kept
    return 0;
}

int ws_engine_set_tensor(ws_engine* e, const char* key, const float* host_data, const long long* shape, int ndim) {
    if (!e || !key || (!host_data && ndim > 0) || ndim < 0 || ndim > 8) { set_err("ws_engine_set_tensor: bad argument"); return 1; }
    if (e->finalized) { set_err("ws_engine_set_tensor after finalize"); return 1; }
    HostT t;
    t.shape.assign(shape, shape + ndim);
    const long long n = t.numel();
    t.v.assign(host_data, host_data + n);
    e->sd[key] = std::move(t);
    return 0;
}

int ws_engine_finalize(ws_engine* e) {
    if (!e) { set_err("ws_engine_finalize: null engine"); return 1; }
    // Build (and drop) a nominal plan: this packs/folds/uploads every weight and reports missing keys.
    if (plan_of(e, 1, 200, false) == nullptr) return 1;
    e->plans.clear();
    e->finalized = true;
    return 0;
}

int ws_engine_embed_dim(const ws_engine* e) { return e ? e->embed_dim : -1; }
long long ws_engine_last_launches(const ws_engine* e) { return e ? e->last_launches : -1; }

static int forward_impl(ws_engine* e, const float* feats_dev, int B, int T, float* embs_dev, void* stream, bool join, const char* who) {
    if (!e || !feats_dev || !embs_dev) { set_err(std::string(who) + ": null argument"); return 1; }
    Run r{e, who, false, (cudaStream_t)stream};
    if (begin_run(r, B, T, false)) return 1;
    WS_CK(cudaMemcpyAsync(r.p->feats_in, feats_dev, (size_t)B * T * e->feat_dim * 4, cudaMemcpyDeviceToDevice, r.s));
    return finish_run(r, 0, embs_dev, join);
}
int ws_engine_forward(ws_engine* e, const float* feats_dev, int B, int T, float* embs_dev, void* stream) {
    return forward_impl(e, feats_dev, B, T, embs_dev, stream, true, "ws_engine_forward");
}
int ws_engine_forward_async(ws_engine* e, const float* feats_dev, int B, int T, float* embs_dev, void* stream) {
    return forward_impl(e, feats_dev, B, T, embs_dev, stream, false, "ws_engine_forward_async");
}
// make `stream` wait for everything the engine has in flight on any of its lanes (closes a series of *_async calls)
int ws_engine_join(ws_engine* e, void* stream) {
    if (!e) { set_err("ws_engine_join: null engine"); return 1; }
    WS_CK(cudaSetDevice(e->device));
    for (int i = 0; i < ws_engine::kLanes; ++i) {
        if (!e->lanes[i]) continue;
        WS_CK(cudaEventRecord(e->ev_out, e->lanes[i]));
        WS_CK(cudaStreamWaitEvent((cudaStream_t)stream, e->ev_out, 0));
    }
    return 0;
}

// Length-masked batches: utterances of different lengths padded to a common T run as ONE batch and produce what each
// utterance produces alone (the reference has no masking, extract_vox.sh:31 runs test sets at batch 1): rows behind an
// utterance's end are kept zero wherever a convolution reads across time, and SE / ASTP / TSTP / CAM++ context statistics
// use the utterance's own frame count.  n_frames_dev: int32[B] on the device; feats rows t >= n_frames[b] are ignored.
int ws_engine_forward_masked(ws_engine* e, const float* feats_dev, const int* n_frames_dev, int B, int T, float* embs_dev,
                             void* stream) {
    if (!e || !feats_dev || !n_frames_dev || !embs_dev) { set_err("ws_engine_forward_masked: null argument"); return 1; }
    Run r{e, "ws_engine_forward_masked", false, (cudaStream_t)stream};
    if (begin_run(r, B, T, true)) return 1;
    WS_CK(cudaMemcpyAsync(r.p->lens, n_frames_dev, (size_t)B * sizeof(int), cudaMemcpyDeviceToDevice, r.s));
    WS_CK(cudaMemcpyAsync(r.p->feats_in, feats_dev, (size_t)B * T * e->feat_dim * 4, cudaMemcpyDeviceToDevice, r.s));
    return finish_run(r, 0, embs_dev, true);
}

// Same from waveforms with n_samples_dev[b] valid samples each (max_samples = the longest): fbank, CMN over each utterance's
// own frames, masked forward.  Rectangular layout: utterance b at wav + b * wav_ld (offsets_dev == nullptr); ragged layout:
// utterance b at wav + offsets_dev[b] samples (concatenated PCM, no padding copies).  Frames behind an utterance's end are
// neither read nor computed.
static int extract_wav_masked_impl(ws_engine* e, const void* wav_dev, int wav_is_i16, long long wav_ld, const long long* offsets_dev,
                                   const int* n_samples_dev, int max_samples, int B, const char* window_type, float* embs_dev,
                                   void* stream, bool join, const char* who, bool ragged = false) {
    if (!e || !wav_dev || !n_samples_dev || !embs_dev || (ragged && !offsets_dev)) { set_err(std::string(who) + ": null argument"); return 1; }
    Run r{e, who, false, (cudaStream_t)stream};
    if (begin_run(r, B, 0, true, max_samples, window_type)) return 1;
    WS_CKS(ws_launch_frames_from_samples(n_samples_dev, r.p->lens, B, r.p->T, ws_fbank_frame_len(e->opts.sample_rate),
                                         ws_fbank_frame_shift(e->opts.sample_rate), r.s));
    if (fbank_into(r.fb, wav_dev, wav_is_i16, wav_ld, max_samples, B, 1, r.p->feats_in, r.s, offsets_dev, r.p->lens)) return 1;
    return finish_run(r, 3, embs_dev, join);
}
int ws_engine_extract_wav_masked(ws_engine* e, const void* wav_dev, int wav_is_i16, long long wav_ld, const int* n_samples_dev,
                                 int max_samples, int B, const char* window_type, float* embs_dev, void* stream) {
    return extract_wav_masked_impl(e, wav_dev, wav_is_i16, wav_ld, nullptr, n_samples_dev, max_samples, B, window_type, embs_dev,
                                   stream, true, "ws_engine_extract_wav_masked");
}
int ws_engine_extract_wav_ragged(ws_engine* e, const void* wav_dev, int wav_is_i16, const long long* offsets_dev,
                                 const int* n_samples_dev, int max_samples, int B, const char* window_type, float* embs_dev,
                                 void* stream) {
    return extract_wav_masked_impl(e, wav_dev, wav_is_i16, 0, offsets_dev, n_samples_dev, max_samples, B, window_type, embs_dev,
                                   stream, true, "ws_engine_extract_wav_ragged", true);
}
int ws_engine_extract_wav_ragged_async(ws_engine* e, const void* wav_dev, int wav_is_i16, const long long* offsets_dev,
                                       const int* n_samples_dev, int max_samples, int B, const char* window_type,
                                       float* embs_dev, void* stream) {
    return extract_wav_masked_impl(e, wav_dev, wav_is_i16, 0, offsets_dev, n_samples_dev, max_samples, B, window_type, embs_dev,
                                   stream, false, "ws_engine_extract_wav_ragged_async", true);
}

int ws_engine_forward_host(ws_engine* e, const float* feats_host, int B, int T, float* embs_host) {
    if (!e || !feats_host || !embs_host) { set_err("ws_engine_forward_host: null argument"); return 1; }
    Run r{e, "ws_engine_forward_host", true};
    if (begin_run(r, B, T, false)) return 1;
    WS_CK(cudaMemcpyAsync(r.p->feats_in, feats_host, (size_t)B * T * e->feat_dim * 4, cudaMemcpyHostToDevice, r.s));
    return finish_run(r, 0, embs_host, true);
}

int ws_fbank_num_frames(int nsamples) { return ws_fbank_num_frames_at(nsamples, 16000); }

int ws_fbank_num_frames_at(int nsamples, int sample_rate) {
    const int fl = ws_fbank_frame_len(sample_rate), sh = ws_fbank_frame_shift(sample_rate);
    if (fl == 0) { set_err("ws_fbank_num_frames_at: sample rate must be 8000 or 16000"); return -1; }
    return nsamples < fl ? 0 : 1 + (nsamples - fl) / sh;
}

// the tables of (window_type, sample_rate, bins) on the current device, for the engine-less fbank entry points
static const FbankTables* device_fbank_tables(const char* window_type, int sample_rate, int bins) {
    int dev = 0;
    const cudaError_t ce = cudaGetDevice(&dev);
    if (ce != cudaSuccess) { set_err(std::string("cudaGetDevice: ") + cudaGetErrorString(ce)); return nullptr; }
    return fbank_tables(fbank_holder(dev), window_type, sample_rate, bins);
}

int ws_fbank(const void* wav_dev, int wav_is_i16, long long wav_ld, int nsamples, int B, const char* window_type,
             int apply_cmn, float* feats_dev, void* stream) {
    if (!wav_dev || !feats_dev) { set_err("ws_fbank: null argument"); return 1; }
    const FbankTables* t = device_fbank_tables(window_type, 16000, 80);
    if (!t) return 1;
    return fbank_into(t, wav_dev, wav_is_i16, wav_ld, nsamples, B, apply_cmn, feats_dev, (cudaStream_t)stream);
}

int ws_fbank_at(const void* wav_dev, int wav_is_i16, long long wav_ld, int nsamples, int B, const char* window_type,
                int sample_rate, int num_mel_bins, int apply_cmn, float* feats_dev, void* stream) {
    if (!wav_dev || !feats_dev || B < 0) { set_err("ws_fbank_at: bad argument"); return 1; }
    if (const char* why = fbank_unsupported(sample_rate, num_mel_bins)) { set_err(std::string("ws_fbank_at: ") + why); return 1; }
    if (nsamples < ws_fbank_frame_len(sample_rate)) { set_err("ws_fbank_at: waveform shorter than one 25 ms frame"); return 1; }
    const FbankTables* t = device_fbank_tables(window_type, sample_rate, num_mel_bins);
    if (!t) return 1;
    return fbank_into(t, wav_dev, wav_is_i16, wav_ld, nsamples, B, apply_cmn, feats_dev, (cudaStream_t)stream);
}

int ws_fbank_ragged_at(const void* wav_dev, int wav_is_i16, long long total_samples, const long long* offsets_dev,
                       const int* n_frames_dev, int max_frames, int B, const char* window_type, int sample_rate, int num_mel_bins,
                       float* feats_dev, void* stream) {
    if (!wav_dev || !offsets_dev || !n_frames_dev || !feats_dev || B < 0 || max_frames < 0 || total_samples < 0) {
        set_err("ws_fbank_ragged: bad argument"); return 1;
    }
    if (const char* why = fbank_unsupported(sample_rate, num_mel_bins)) { set_err(std::string("ws_fbank_ragged: ") + why); return 1; }
    if (B > 65535) { set_err("ws_fbank_ragged: more than 65535 rows in one launch"); return 1; }
    const FbankTables* t = device_fbank_tables(window_type, sample_rate, num_mel_bins);
    if (!t) return 1;
    // the launcher's size check is per row there; rows are placed by the caller here, which vouches for them
    const int fl = ws_fbank_frame_len(sample_rate), sh = ws_fbank_frame_shift(sample_rate);
    WS_CKS(ws_launch_fbank(wav_dev, wav_is_i16, 0, max_frames > 0 ? (max_frames - 1) * sh + fl : 0, B, max_frames, sample_rate,
                           num_mel_bins, t->window, t->melw, t->melstart, t->mellen, t->maxlen, feats_dev, (cudaStream_t)stream,
                           offsets_dev, n_frames_dev));
    return 0;
}

int ws_fbank_ragged(const void* wav_dev, int wav_is_i16, long long total_samples, const long long* offsets_dev,
                    const int* n_frames_dev, int max_frames, int B, const char* window_type, float* feats_dev, void* stream) {
    return ws_fbank_ragged_at(wav_dev, wav_is_i16, total_samples, offsets_dev, n_frames_dev, max_frames, B, window_type, 16000, 80,
                              feats_dev, stream);
}

// ---- resampling (torchaudio.transforms.Resample defaults: sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99)
namespace {
struct ResampleTaps { float* dev = nullptr; int of = 0, nf = 0, width = 0; };
int gcd_i(int a, int b) { while (b) { const int t = a % b; a = b; b = t; } return a; }
// torchaudio/functional/functional.py::_get_sinc_resample_kernel, in fp64 then rounded to fp32 like there
const ResampleTaps* resample_taps(int device, int orig, int neu) {
    static std::map<std::tuple<int, int, int>, ResampleTaps> cache;
    const auto key = std::make_tuple(device, orig, neu);
    auto it = cache.find(key);
    if (it != cache.end()) return &it->second;
    const int g = gcd_i(orig, neu), of = orig / g, nf = neu / g;
    const double rolloff = 0.99, lpw = 6.0, pi = 3.14159265358979323846;
    const double base = (double)(of < nf ? of : nf) * rolloff;
    const int width = (int)std::ceil(lpw * of / base), klen = 2 * width + of;
    std::vector<float> taps((size_t)nf * klen);
    for (int i = 0; i < nf; ++i)
        for (int k = 0; k < klen; ++k) {
            double t = ((double)(-i) / nf + (double)(k - width) / of) * base;
            t = t < -lpw ? -lpw : (t > lpw ? lpw : t);
            const double c = std::cos(t * pi / lpw / 2.0), window = c * c;
            const double tp = t * pi;
            const double sinc = tp == 0.0 ? 1.0 : std::sin(tp) / tp;
            taps[(size_t)i * klen + k] = (float)(sinc * window * (base / of));
        }
    ResampleTaps r;
    r.of = of; r.nf = nf; r.width = width;
    if (cudaMalloc((void**)&r.dev, taps.size() * 4) != cudaSuccess ||
        cudaMemcpy(r.dev, taps.data(), taps.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess) {
        set_err("ws_resample: tap table upload failed");
        return nullptr;
    }
    return &(cache[key] = r);
}
}  // namespace

int ws_resample_out_len(int n_in, int orig_freq, int new_freq) {
    if (n_in <= 0 || orig_freq <= 0 || new_freq <= 0) return 0;
    const int g = gcd_i(orig_freq, new_freq);
    const long long of = orig_freq / g, nf = new_freq / g;
    return (int)((nf * (long long)n_in + of - 1) / of);      // ceil(new * length / orig)
}

int ws_resample(const void* wav_dev, int wav_is_i16, long long wav_ld, int n_in, int B, int orig_freq, int new_freq,
                float* out_dev, long long out_ld, void* stream) {
    if (!wav_dev || !out_dev || n_in <= 0 || B <= 0 || orig_freq <= 0 || new_freq <= 0) { set_err("ws_resample: bad argument"); return 1; }
    int dev = 0;
    WS_CK(cudaGetDevice(&dev));
    const ResampleTaps* t = resample_taps(dev, orig_freq, new_freq);
    if (!t) return 1;
    const int n_out = ws_resample_out_len(n_in, orig_freq, new_freq);
    if (out_ld < n_out) { set_err("ws_resample: out_ld smaller than the output length"); return 1; }
    WS_CKS(ws_launch_resample(wav_dev, wav_is_i16, wav_ld, n_in, B, t->dev, t->of, t->nf, t->width, out_dev, out_ld, n_out,
                              (cudaStream_t)stream));
    return 0;
}

static int extract_wav_impl(ws_engine* e, const void* wav_dev, int wav_is_i16, long long wav_ld, int nsamples, int B,
                            const char* window_type, float* embs_dev, float* feats_out_dev, void* stream, bool join, const char* who) {
    if (!e || !wav_dev || !embs_dev) { set_err(std::string(who) + ": null argument"); return 1; }
    Run r{e, who, false, (cudaStream_t)stream};
    if (begin_run(r, B, 0, false, nsamples, window_type)) return 1;
    if (fbank_into(r.fb, wav_dev, wav_is_i16, wav_ld, nsamples, B, 1, r.p->feats_in, r.s)) return 1;
    if (feats_out_dev)
        WS_CK(cudaMemcpyAsync(feats_out_dev, r.p->feats_in, (size_t)B * r.p->T * e->feat_dim * 4, cudaMemcpyDeviceToDevice, r.s));
    return finish_run(r, 2, embs_dev, join);
}
int ws_engine_extract_wav(ws_engine* e, const void* wav_dev, int wav_is_i16, long long wav_ld, int nsamples, int B,
                          const char* window_type, float* embs_dev, float* feats_out_dev, void* stream) {
    return extract_wav_impl(e, wav_dev, wav_is_i16, wav_ld, nsamples, B, window_type, embs_dev, feats_out_dev, stream, true, "ws_engine_extract_wav");
}
int ws_engine_extract_wav_async(ws_engine* e, const void* wav_dev, int wav_is_i16, long long wav_ld, int nsamples, int B,
                                const char* window_type, float* embs_dev, void* stream) {
    return extract_wav_impl(e, wav_dev, wav_is_i16, wav_ld, nsamples, B, window_type, embs_dev, nullptr, stream, false, "ws_engine_extract_wav_async");
}

int ws_engine_extract_wav_host(ws_engine* e, const void* wav_host, int wav_is_i16, int nsamples, int B,
                               const char* window_type, float* embs_host) {
    if (!e || !wav_host || !embs_host) { set_err("ws_engine_extract_wav_host: null argument"); return 1; }
    Run r{e, "ws_engine_extract_wav_host", true};
    if (begin_run(r, B, 0, false, nsamples, window_type)) return 1;
    const size_t bytes = (size_t)B * nsamples * (wav_is_i16 ? 2 : 4);
    if (grow(&e->wav_dev, &e->wav_bytes, bytes)) return 1;
    WS_CK(cudaMemcpyAsync(e->wav_dev, wav_host, bytes, cudaMemcpyHostToDevice, r.s));
    if (fbank_into(r.fb, e->wav_dev, wav_is_i16, nsamples, nsamples, B, 1, r.p->feats_in, r.s)) return 1;
    return finish_run(r, 2, embs_host, true);
}

// Pipelined host path: submit() enqueues H2D of batch i on a copy stream and the fbank+CMN+forward+D2H on the compute
// stream behind it, then returns immediately; collect() blocks until that slot's embeddings are in embs_host.  With two
// slots the H2D copy of batch i+1 overlaps the kernels of batch i (the reference overlaps with DataLoader workers and
// prefetch_factor=4, extract.py:99-103).
int ws_engine_submit_wav_host(ws_engine* e, int slot, const void* wav_host, int wav_is_i16, int nsamples, int B,
                              const char* window_type, float* embs_host) {
    if (!e || !wav_host || !embs_host || slot < 0 || slot >= ws_engine::kSlots) { set_err("ws_engine_submit_wav_host: bad argument"); return 1; }
    Run r{e, "ws_engine_submit_wav_host", true};
    if (begin_run(r, B, 0, false, nsamples, window_type)) return 1;
    if (e->copy_st == nullptr) {
        WS_CK(cudaStreamCreateWithFlags(&e->copy_st, cudaStreamNonBlocking));
        for (int i = 0; i < ws_engine::kSlots; ++i) {
            WS_CK(cudaEventCreateWithFlags(&e->slot_copied[i], cudaEventDisableTiming));
            WS_CK(cudaEventCreateWithFlags(&e->slot_done[i], cudaEventDisableTiming));
        }
    }
    const size_t bytes = (size_t)B * nsamples * (wav_is_i16 ? 2 : 4);
    if (bytes > e->slot_bytes[slot]) WS_CK(cudaStreamSynchronize(e->st));
    if (grow(&e->slot_wav[slot], &e->slot_bytes[slot], bytes)) return 1;
    // the slot's staging buffer is free once the previous job that used it finished its fbank (slot_done covers it)
    WS_CK(cudaStreamWaitEvent(e->copy_st, e->slot_done[slot], 0));
    WS_CK(cudaMemcpyAsync(e->slot_wav[slot], wav_host, bytes, cudaMemcpyHostToDevice, e->copy_st));
    WS_CK(cudaEventRecord(e->slot_copied[slot], e->copy_st));
    WS_CK(cudaStreamWaitEvent(r.s, e->slot_copied[slot], 0));
    if (fbank_into(r.fb, e->slot_wav[slot], wav_is_i16, nsamples, nsamples, B, 1, r.p->feats_in, r.s)) return 1;
    if (finish_run(r, 2, embs_host, false)) return 1;
    WS_CK(cudaEventRecord(e->slot_done[slot], r.s));
    return 0;
}

int ws_engine_collect(ws_engine* e, int slot) {
    if (!e || slot < 0 || slot >= ws_engine::kSlots || e->slot_done[slot] == nullptr) { set_err("ws_engine_collect: bad argument"); return 1; }
    WS_CK(cudaEventSynchronize(e->slot_done[slot]));
    return 0;
}

// Tuning aid: run the (B,T) plan op by op (no CUDA graph) with CUDA events between ops, in sequence context (the L2 holds
// what the previous op left there, unlike ncu's cold-cache replays).  ms_out[i] = duration of op i; returns the op count.
int ws_engine_profile_ops(ws_engine* e, int B, int T, int iters, float* ms_out, int max_ops) {
    if (!e || !ms_out) { set_err("ws_engine_profile_ops: bad argument"); return -1; }
    Run r{e, "ws_engine_profile_ops", true};
    if (begin_run(r, B, T, false)) return -1;
    const Plan* p = r.p;
    const int n = (int)p->ops.size();
    if (n > max_ops) { set_err("ws_engine_profile_ops: output array too small"); return -1; }
    std::vector<cudaEvent_t> ev(n + 1);
    for (auto& x : ev) cudaEventCreate(&x);
    std::vector<double> acc(n, 0.0);
    for (int it = 0; it < iters + 1; ++it) {
        cudaEventRecord(ev[0], r.s);
        for (int i = 0; i < n; ++i) {
            const char* m = p->ops[i].run(r.s);
            if (m) { set_err(std::string("profile_ops launch: ") + m); return -1; }
            cudaEventRecord(ev[i + 1], r.s);
        }
        if (cudaStreamSynchronize(r.s) != cudaSuccess) { set_err("profile_ops: sync failed"); return -1; }
        if (it == 0) continue;  // warm-up pass
        for (int i = 0; i < n; ++i) {
            float ms = 0.f;
            cudaEventElapsedTime(&ms, ev[i], ev[i + 1]);
            acc[i] += ms;
        }
    }
    for (int i = 0; i < n; ++i) ms_out[i] = (float)(acc[i] / iters);
    for (auto& x : ev) cudaEventDestroy(x);
    return n;
}

// label of op i of the (B,T) plan ("conv_tc3 pos=.. K=.. N=..", "conv3x3 ...", "tstats", ...) and its FLOPs (0 = not GEMM-like)
const char* ws_engine_plan_op_name(ws_engine* e, int B, int T, int i, double* flops_out) {
    if (!e || !e->finalized) return nullptr;
    Plan* p = plan_of(e, B, T, false);
    if (!p || i < 0 || i >= (int)p->ops.size()) return nullptr;
    if (flops_out) *flops_out = p->ops[i].flops;
    return p->ops[i].label.c_str();
}

// Write the (B,T) launch plan as data - a JSON description of every op (operands as addresses, shapes, strides, epilogues),
// the allocation table and, on plan-check engines, the fp32 source of every weight - so that a test can re-evaluate the
// plan's arithmetic on the host (tests/plan_interp.py) and compare it with the oracle.  Plan-check engines write placeholder
// addresses.  Real engines with the option plan_trace = 1 write device addresses, every weight and plan-buffer allocation
// and no weight blobs (the weights are on the device, in the dtype the kernels read), so that a test can run the plan op by
// op (ws_engine_run_ops) and check what each kernel wrote.
// File layout: "WSPT1\n", uint64 JSON length, JSON, then the weight blobs (fp32) back to back; the JSON's "blobs" table
// holds [address, float offset into the blob area, float count].
int ws_engine_plan_trace(ws_engine* e, int B, int T, int masked, const char* path) {
    if (!e || !path) { set_err("ws_engine_plan_trace: null argument"); return 1; }
    if (!e->finalized || (!e->plan_check && !e->opts.plan_trace)) {
        set_err("ws_engine_plan_trace: needs a finalized plan-check engine, or a finalized engine with the option plan_trace = 1");
        return 1;
    }
    Plan* p = plan_of(e, B, T, masked != 0);
    if (!p) return 1;
    std::vector<std::pair<unsigned long long, unsigned long long>> allocs = e->check_allocs;
    if (!e->plan_check) {
        allocs = e->weight_allocs;
        allocs.insert(allocs.end(), p->trace_allocs.begin(), p->trace_allocs.end());
    }
    std::string j = "{";
    j += ti("B", B) + "," + ti("T", T) + "," + ti("feat_dim", e->feat_dim) + "," + ti("embed_dim", e->embed_dim) + "," +
         ti("act_es", ws_esize(e->act_dt)) + "," + tp("feats_in", p->feats_in) + "," + tp("emb", p->emb) + "," + tp("lens", p->lens) + ",\"model\":\"" + e->model +
         "\",\"precision\":\"" + e->prec + "\",\"allocs\":[";
    for (size_t i = 0; i < allocs.size(); ++i)
        j += std::string(i ? "," : "") + "[" + std::to_string(allocs[i].first) + "," + std::to_string(allocs[i].second) + "]";
    j += "],\"blobs\":[";
    unsigned long long off = 0;
    bool first = true;
    for (auto& kv : e->check_blobs) {
        j += std::string(first ? "" : ",") + "[" + std::to_string(kv.first) + "," + std::to_string(off) + "," + std::to_string(kv.second.size()) + "]";
        off += kv.second.size();
        first = false;
    }
    j += "],\"ops\":[";
    for (size_t i = 0; i < p->ops.size(); ++i) {
        std::string lab = p->ops[i].label;
        for (char& ch : lab) if (ch == '"' || ch == '\\') ch = ' ';
        j += std::string(i ? "," : "") + "{\"label\":\"" + lab + "\",\"trace\":" + (p->ops[i].trace ? p->ops[i].trace() : std::string("null")) + "}";
    }
    j += "]}";
    FILE* f = fopen(path, "wb");
    if (!f) { set_err(std::string("ws_engine_plan_trace: cannot open ") + path); return 1; }
    const unsigned long long n = j.size();
    bool okw = fwrite("WSPT1\n", 1, 6, f) == 6 && fwrite(&n, 8, 1, f) == 1 && fwrite(j.data(), 1, j.size(), f) == j.size();
    for (auto& kv : e->check_blobs)
        okw = okw && (kv.second.empty() || fwrite(kv.second.data(), 4, kv.second.size(), f) == kv.second.size());
    okw = (fclose(f) == 0) && okw;
    if (!okw) { set_err(std::string("ws_engine_plan_trace: write failed: ") + path); return 1; }
    return 0;
}

// Test aid: run ops [first, last) of the (B,T[,masked]) plan eagerly (no CUDA graph) on `stream`, building the plan if needed.
// The caller fills the plan's inputs (ws_engine_plan_trace names feats_in and lens) and orders `stream` after whatever else
// touches the plan's buffers; nothing is synchronised here.
int ws_engine_run_ops(ws_engine* e, int B, int T, int masked, int first, int last, void* stream) {
    if (!e) { set_err("ws_engine_run_ops: null engine"); return 1; }
    if (const char* nr = not_runnable(e)) { set_err(std::string("ws_engine_run_ops") + nr); return 1; }
    Plan* p = plan_of(e, B, T, masked != 0);
    if (!p) return 1;
    if (first < 0 || last > (int)p->ops.size() || first > last) { set_err("ws_engine_run_ops: op range outside the plan"); return 1; }
    for (int i = first; i < last; ++i) {
        const char* m = p->ops[i].run((cudaStream_t)stream);
        if (m) { set_err("ws_engine_run_ops: op " + std::to_string(i) + " (" + p->ops[i].label + "): " + m); return 1; }
    }
    return 0;
}

void ws_engine_destroy(ws_engine* e) {
    if (!e) return;
    if (e->plan_check) { delete e; return; }
    cudaSetDevice(e->device);
    cudaDeviceSynchronize();
    delete e;
}

}  // extern "C"
