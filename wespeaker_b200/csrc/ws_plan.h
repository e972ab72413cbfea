// Launch plans and the engine that owns them, shared by the engine (ws_engine.cu) and the plan builders of the model
// families (ws_build_ecapa.cu, ws_build_2d.cu, ws_build_tdnn.cu): state_dict tensors, the plan, the engine, weight ingest and
// the Builder every family builds its plan with.
#pragma once
#include <algorithm>
#include <array>
#include <cmath>
#include <cstring>
#include <memory>
#include <tuple>

#include "../../include/wespeaker_b200.h"
#include "ws_host.h"

namespace ws {

struct HostT {
    std::vector<float> v;
    std::vector<long long> shape;
    long long numel() const {
        long long n = 1;
        for (long long d : shape) n *= d;
        return n;
    }
};

// the fbank frontend's device tables for one (window type, sample rate, mel bin count)
struct FbankTables {
    int rate = 16000, bins = 80;
    float* window = nullptr;
    float* melw = nullptr;
    int* melstart = nullptr;
    int* mellen = nullptr;
    int maxlen = 0;
};

struct Plan {
    int B = 0, T = 0;
    std::vector<PlanOp> ops;
    std::vector<void*> bufs;
    int extra_launches = 0;     // ops that launch more than one kernel (split-K FC = 2)
    size_t bytes = 0;           // device memory held by this plan
    long long last_use = 0;     // LRU stamp
    float* feats_in = nullptr;  // fp32 [B][T][feat_dim]
    float* emb = nullptr;       // fp32 [B][embed_dim]
    cudaGraphExec_t gexec = nullptr;
    bool graph_failed = false;
    bool masked = false;        // length-masked plan: per-utterance frame counts arrive with every run (see `lens`)
    int* lens = nullptr;        // device [4][B]: frames per utterance at the input and behind each stride-2 level
    int lane = 0;               // which of the engine's streams runs this plan through the device-pointer entry points
    cudaEvent_t done = nullptr; // recorded after every use: a later use on another stream waits for it
    bool check = false;         // built by a plan-check engine: buffers are placeholder addresses, nothing to release
    // every device buffer this plan allocated, (address, bytes), for ws_engine_plan_trace on real engines
    std::vector<std::pair<unsigned long long, unsigned long long>> trace_allocs;
    ~Plan() {
        if (done) cudaEventDestroy(done);
        if (gexec) cudaGraphExecDestroy(gexec);
        if (!check) for (void* p : bufs) cudaFree(p);
    }
};

struct Builder;
// A model family's plan builder: appends the ops of one forward pass at (b.p.B, b.p.T) to b.p; false with the error set
using PlanBuilder = bool (*)(Builder&);

// Hyper-parameters of a model, one row of the model table (ws_engine.cu); each family reads its own fields.
struct ModelCfg {
    std::array<int, 4> num_blocks{};   // blocks per stage: ResNet, Res2Net / ERes2Net, SimAM-ResNet, Gemini DF-ResNet
    int channels = 512;                // ECAPA-TDNN
    bool glob = false;                 // ECAPA-TDNN: global context in the attentive pooling
    bool bottleneck = false;           // ResNet50..293: Bottleneck blocks (expansion 4) instead of BasicBlocks
    // Res2Net / ERes2Net (res2net.py:202-221, eres2net.py:393-431): stem width, baseWidth, scale, expansion, AFF fusion
    int m = 32, base_width = 32, scale = 2, expansion = 2;
    bool fuse = false;
};

// The engine options at their defaults (ws_engine_set_option; include/wespeaker_b200.h documents each)
struct EngineOptions {
    bool two_emb_layer = false, emb_bn = false;   // model_args
    bool cuda_graph = true, plan_trace = false;
    // the fused kernels the plan builders may take
    bool res2_fused = true, se_fused = true, se_colsum = true, conv3x3 = true, cam_fused = true, cam_block = true, astp_fused = true;
    int tc_version = 3, sample_rate = 16000;   // sample_rate: the waveform entry points' rate (the mel bin count is feat_dim)
};

}  // namespace ws

struct ws_engine {
    std::string model, prec;
    int feat_dim = 80, embed_dim = 0, device = 0;
    int act_dt = WS_F32;
    int tc = 0;          // the precision's tensor-core level: 0 FFMA, 3 tensor cores
    bool split = false;  // 3xTF32: fp32 activations/weights carry lo twins, GEMMs run 3 error-compensated passes
    ws::EngineOptions opts;
    // the level plans use (2 persistent tensor-core kernel, 3 + weight-sharing clusters): fp32 stays on FFMA
    int use_tc() const { return std::min(tc, opts.tc_version); }
    std::map<const void*, const void*> wlo;  // packed weight -> its lo twin
    std::map<std::string, ws::HostT> sd;
    bool finalized = false;
    bool plan_check = false;   // ws_engine_create_plan_check: builds launch plans without a device, never computes
    // plan-check engines: every placeholder allocation (address, bytes) and the fp32 source of every weight upload, for
    // ws_engine_plan_trace
    std::vector<std::pair<unsigned long long, unsigned long long>> check_allocs;
    std::map<unsigned long long, std::vector<float>> check_blobs;
    // real engines: every weight allocation (address, bytes), written by ws_engine_plan_trace under the option plan_trace (the
    // weights are usually uploaded by ws_engine_finalize, before any option is set; a plan's own buffers are in
    // Plan::trace_allocs: they go away with the plan)
    std::vector<std::pair<unsigned long long, unsigned long long>> weight_allocs;
    std::map<std::string, void*> wcache;  // packed device weights by id
    std::map<std::pair<int, int>, std::unique_ptr<ws::Plan>> plans;   // key: (B, 2 * T + masked)
    long long last_launches = 0;
    long long use_clock = 0;             // LRU clock for the plan cache
    cudaStream_t st = nullptr;
    // Plans of different (B, T) own disjoint buffers, so the device-pointer entry points spread them over a few streams:
    // the buckets of a variable-length job (one plan per distinct length) then overlap on the GPU instead of running one
    // small batch at a time.  lanes[0] == st.
    static constexpr int kLanes = 4;
    cudaStream_t lanes[kLanes] = {nullptr, nullptr, nullptr, nullptr};
    int next_lane = 0;
    cudaEvent_t ev_in = nullptr, ev_out = nullptr;
    std::map<std::tuple<std::string, int, int>, ws::FbankTables> fb;   // key: (window type, sample rate, mel bins)
    void* wav_dev = nullptr;
    size_t wav_bytes = 0;
    // double-buffered host->device pipeline (ws_engine_submit_wav_host / ws_engine_collect)
    cudaStream_t copy_st = nullptr;
    static constexpr int kSlots = 4;
    void* slot_wav[kSlots] = {nullptr, nullptr, nullptr, nullptr};
    size_t slot_bytes[kSlots] = {0, 0, 0, 0};
    cudaEvent_t slot_copied[kSlots] = {nullptr, nullptr, nullptr, nullptr}, slot_done[kSlots] = {nullptr, nullptr, nullptr, nullptr};
    // the model's row of the model table: its family's plan builder and hyper-parameters
    ws::PlanBuilder build = nullptr;
    ws::ModelCfg cfg;
    ~ws_engine() {
        plans.clear();
        if (plan_check) return;   // placeholder addresses only, no streams / events were created
        for (auto& kv : wcache) cudaFree(kv.second);
        for (auto& kv : fb) {
            cudaFree(kv.second.window); cudaFree(kv.second.melw); cudaFree(kv.second.melstart); cudaFree(kv.second.mellen);
        }
        if (wav_dev) cudaFree(wav_dev);
        for (int i = 0; i < kSlots; ++i) {
            if (slot_wav[i]) cudaFree(slot_wav[i]);
            if (slot_copied[i]) cudaEventDestroy(slot_copied[i]);
            if (slot_done[i]) cudaEventDestroy(slot_done[i]);
        }
        if (copy_st) cudaStreamDestroy(copy_st);
        if (ev_in) cudaEventDestroy(ev_in);
        if (ev_out) cudaEventDestroy(ev_out);
        for (int i = 1; i < kLanes; ++i)
            if (lanes[i]) cudaStreamDestroy(lanes[i]);
        if (st) cudaStreamDestroy(st);
    }
};

namespace ws {

// ------------------------------------------------------------------------------------------------ weights
struct Weights {
    ws_engine& e;
    bool ok = true;
    explicit Weights(ws_engine& eng) : e(eng) {}

    const HostT* get(const std::string& key) {
        auto it = e.sd.find(key);
        if (it == e.sd.end()) {
            if (ok) set_err("missing tensor in state_dict: " + key);
            ok = false;
            return nullptr;
        }
        return &it->second;
    }
    // f32src: the fp32 values `host` was converted from (kept by plan-check engines for ws_engine_plan_trace)
    void* upload(const std::string& id, const void* host, size_t bytes, const std::vector<float>* f32src = nullptr) {
        auto it = e.wcache.find(id);
        if (it != e.wcache.end()) return it->second;
        void* d = nullptr;
        if (plan_check_mode()) {
            d = plan_check_alloc(bytes);
            e.check_allocs.push_back({(unsigned long long)d, (unsigned long long)bytes});
            if (f32src) e.check_blobs[(unsigned long long)d] = *f32src;
        } else if (cudaMalloc(&d, bytes ? bytes : 16) != cudaSuccess || cudaMemcpy(d, host, bytes, cudaMemcpyHostToDevice) != cudaSuccess) {
            if (ok) set_err("device allocation/copy failed for weight " + id);
            ok = false;
            return nullptr;
        } else {
            e.weight_allocs.push_back({(unsigned long long)d, (unsigned long long)bytes});
        }
        e.wcache[id] = d;
        return d;
    }
    bool cached(const std::string& id, void** out) {
        auto it = e.wcache.find(id);
        if (it == e.wcache.end()) return false;
        *out = it->second;
        return true;
    }
    float* f32(const std::string& id, const std::vector<float>& v) { return (float*)upload(id, v.data(), v.size() * 4, &v); }
    void* act(const std::string& id, const std::vector<float>& v) {
        void* c;
        if (cached(id, &c)) return c;
        if (e.act_dt == WS_F32) {
            void* hi = upload(id, v.data(), v.size() * 4, &v);
            if (e.split && hi != nullptr) {
                std::vector<float> lo(v.size());
                for (size_t i = 0; i < v.size(); ++i) {
                    uint32_t u;
                    memcpy(&u, &v[i], 4);
                    u &= 0xffffe000u;
                    float t;
                    memcpy(&t, &u, 4);
                    lo[i] = v[i] - t;
                }
                e.wlo[hi] = upload(id + ":lo", lo.data(), lo.size() * 4);
            }
            return hi;
        }
        std::vector<unsigned short> h(v.size());
        for (size_t i = 0; i < v.size(); ++i)
            h[i] = e.act_dt == WS_BF16 ? __bfloat16_as_ushort(__float2bfloat16_rn(v[i]))
                                       : __half_as_ushort(__float2half_rn(v[i]));
        return upload(id, h.data(), h.size() * 2, &v);
    }
    const float* vec(const std::string& key) {
        void* c;
        if (cached("v:" + key, &c)) return (const float*)c;
        const HostT* t = get(key);
        return t ? f32("v:" + key, t->v) : nullptr;
    }
    // eval-mode BatchNorm as per-channel affine: scale = w / sqrt(var + eps), shift = b - mean * scale
    bool bn(const std::string& p, bool affine, std::vector<float>& scale, std::vector<float>& shift) {
        const HostT* m = get(p + ".running_mean");
        const HostT* v = get(p + ".running_var");
        const HostT* w = affine ? get(p + ".weight") : nullptr;
        const HostT* b = affine ? get(p + ".bias") : nullptr;
        if (!m || !v || (affine && (!w || !b))) return false;
        const size_t n = m->v.size();
        scale.resize(n); shift.resize(n);
        for (size_t i = 0; i < n; ++i) {
            const double s = (affine ? (double)w->v[i] : 1.0) / std::sqrt((double)v->v[i] + 1e-5);
            scale[i] = (float)s;
            shift[i] = (float)((affine ? (double)b->v[i] : 0.0) - (double)m->v[i] * s);
        }
        return true;
    }
    // conv weight (Cout, Cin, k) or (Cout, Cin, kf, kt) -> [Cout][tap][Cin] (tap-major), optional per-row scale and shape
    bool pack_conv(const std::string& key, const std::vector<float>* rowscale, std::vector<float>& out, int* Cout = nullptr,
                   int* Cin = nullptr, int* ntap = nullptr) {
        const HostT* t = get(key);
        if (!t) return false;
        const int co = (int)t->shape[0], ci = (int)t->shape[1];
        int taps = 1;
        for (size_t i = 2; i < t->shape.size(); ++i) taps *= (int)t->shape[i];
        out.resize((size_t)co * ci * taps);
        for (int o = 0; o < co; ++o) {
            const float sc = rowscale ? (*rowscale)[o] : 1.f;
            for (int c = 0; c < ci; ++c)
                for (int j = 0; j < taps; ++j)
                    out[((size_t)o * taps + j) * ci + c] = t->v[((size_t)o * ci + c) * taps + j] * sc;
        }
        if (Cout) *Cout = co;
        if (Cin) *Cin = ci;
        if (ntap) *ntap = taps;
        return true;
    }
};

// ------------------------------------------------------------------------------------------------ plan builder
struct Builder {
    ws_engine& e;
    Plan& p;
    Weights w;
    bool ok = true;
    Builder(ws_engine& eng, Plan& pl) : e(eng), p(pl), w(eng) {}
    bool good() const { return ok && w.ok; }
    // may a fused 16-bit tensor-core kernel build an op: the precision runs those kernels and the option selecting it is on
    bool fused(bool option) const { return e.use_tc() >= 2 && e.act_dt != WS_F32 && option; }

    void* raw(size_t bytes) {
        void* d = nullptr;
        if (plan_check_mode()) {
            d = plan_check_alloc(bytes);
            e.check_allocs.push_back({(unsigned long long)d, (unsigned long long)bytes});
        } else if (cudaMalloc(&d, bytes ? bytes : 16) != cudaSuccess) {
            if (ok) set_err("cudaMalloc failed for an activation buffer");
            ok = false;
            return nullptr;
        } else {
            p.trace_allocs.push_back({(unsigned long long)d, (unsigned long long)bytes});
        }
        p.bufs.push_back(d);
        p.bytes += bytes;
        return d;
    }
    View act(int B, int F, int T, int C) {
        View v;
        v.B = B; v.F = F; v.T = T; v.C = C; v.ld = C; v.dt = e.act_dt;
        v.p = raw((size_t)B * F * T * C * ws_esize(e.act_dt));
        if (e.split) v.plo = raw((size_t)B * F * T * C * 4);
        return v;
    }
    float* f32(size_t n) { return (float*)raw(n * 4); }
    // n rotating activation buffers of `elems` elements each (with their 3xTF32 lo twins)
    std::vector<View> ring(int n, size_t elems) {
        std::vector<View> v((size_t)n);
        for (View& x : v) {
            x.dt = e.act_dt;
            x.p = raw(elems * ws_esize(e.act_dt));
            if (e.split) x.plo = raw(elems * 4);
        }
        return v;
    }
    void push(PlanOp op) { p.ops.push_back(std::move(op)); }
    // a bandwidth op: its argument record, which both its launch and its plan trace (trace_of, ws_host.h) read
    template <class Rec>
    void push(const Rec& a, const char* (*launch)(const Rec&, cudaStream_t), const char* label) {
        push(plan_op(a, launch, label));
    }
    // length-masked plans: frame counts of stride level k (nullptr in ordinary plans), and "zero the rows behind every
    // utterance's end" for tensors a time-mixing op is about to read (the reference's unpadded forward sees zero padding)
    const int* lens(int level) const { return p.masked ? p.lens + (size_t)level * p.B : nullptr; }
    void zero_tail(const View& v, int level) {
        if (p.masked) push(WsZeroTail{v, lens(level)}, ws_launch_zero_tail, "zero_tail");
    }
    void conv(const ConvSpec& s_in) {
        if (!good()) return;
        ConvSpec s = s_in;
        if (e.split) {
            auto it = e.wlo.find(s.W);
            if (it == e.wlo.end()) { set_err("internal: 3xTF32 weight without a lo twin"); ok = false; return; }
            s.W_lo = it->second;
            s.split = true;
        }
        PlanOp op;
        if (!make_conv_op(s, e.use_tc(), &op)) { ok = false; return; }
        push(std::move(op));
    }
    static WsSrc src_of(const View& v) {
        WsSrc s;
        s.ptr = v.p; s.ptr_lo = v.plo; s.B = v.B; s.F = v.F; s.T = v.T; s.C = v.C;
        s.sT = v.ld; s.sF = (long long)v.T * v.ld; s.sB = (long long)v.F * v.T * v.ld;
        return s;
    }
    // plain conv over one input view; returns output dims via out view (must be pre-sized by caller)
    void conv_simple(const View& x, const View& out, const void* W, int kf, int kt, int dil_f, int dil_t, int pad_f,
                     int pad_t, int sf, int st_, const WsEpi& epi_in) {
        if (!good()) return;
        ConvSpec s;
        s.dt = e.act_dt;
        int Fo, To;
        const int K = add_conv_taps(s, x, kf, kt, dil_f, dil_t, pad_f, pad_t, sf, st_, 0, &Fo, &To);
        if (K < 0 || Fo != out.F || To != out.T) { set_err("internal: conv shape mismatch"); ok = false; return; }
        s.W = W; s.Ktot = K; s.Cout = out.C; s.B = out.B; s.F = Fo; s.T = To;
        s.dense_pointwise = (kf == 1 && kt == 1 && sf == 1 && st_ == 1);
        s.epi = epi_in;
        fill_epi_out(s.epi, out);
        conv(s);
    }
    void tstats(const View& x, const float* pre_scale, const float* pre_shift, float* out, long long out_ld, int std_off,
                int level = 0) {
        WsTstats a{x, pre_scale, pre_shift, out, WS_F32, out_ld, std_off, 1e-7f, lens(level)};
        a.kernel = ws_tstats_kernel(a);
        push(a, ws_launch_tstats, "tstats");
    }
    void linear(const float* in, long long in_ld, const float* in2, long long in2_ld, int rows_per_b, const float* W,
                const float* bias, float* out, long long out_ld, int R, int I, int O, int act) {
        WsLinear a{in, in_ld, in2, in2_ld, rows_per_b, W, bias, out, out_ld, R, I, O, act, nullptr};
        ws_linear_rows_plan(a, ws_num_sms());
        if (a.nsplit > 1) {
            a.wsp = f32((size_t)a.nsplit * R * O);
            p.extra_launches += 1;
        }
        push(a, ws_launch_linear_rows, "linear_rows");
    }
    // the fp32 input features -> x0 (B,1,T,feat_dim) in the activation dtype
    void convert_input(const View& x0) {
        push(WsConvert{p.feats_in, x0.p, (float*)x0.plo, x0.dt, x0.npos() * x0.C}, ws_launch_convert, "convert");
    }
    // The halo-resident 3x3 pad-1 conv (ws_conv3x3.cu: every input row crosses L2 -> SM once instead of once per tap),
    // out = act(conv(x, W) + bias [+ res]).  halo_conv3x3 returns 1 with *op built (not pushed), 0 when the caller runs the
    // conv-GEMM instead (also when the shape is outside the kernel's envelope), -1 on error.  lvl: stride level of `out`.
    int halo_conv3x3(const View& x, const View& out, const void* W, const float* bias, const View* res, int act, int sf, int st, int lvl,
                     PlanOp* op) {
        if (!fused(e.opts.conv3x3)) return 0;
        const OpBuild r = make_conv3x3_op(x, out, W, bias, res, act == WS_ACT_RELU20 ? 2 : act == WS_ACT_RELU ? 1 : 0, op, sf, st, lens(lvl));
        if (r == OpBuild::error) ok = false;
        return r == OpBuild::built ? 1 : r == OpBuild::outside ? 0 : -1;
    }
    // 3x3 pad-1 conv, out = act(conv(x, W) + bias), act WS_ACT_RELU20, WS_ACT_RELU or WS_ACT_NONE: the halo-resident kernel where
    // it applies, else the conv-GEMM, followed (length-masked plans) by zeroing the rows behind every utterance's end unless the
    // caller's next reader does not mix time (`zero_tail_after` = false)
    bool conv3x3(const View& x, const View& out, const void* W, const float* bias, int act, int sf, int st, int lvl, bool zero_tail_after = true) {
        PlanOp op;
        const int r = halo_conv3x3(x, out, W, bias, nullptr, act, sf, st, lvl, &op);
        if (r > 0) push(std::move(op));
        if (r != 0) return good();
        WsEpi ep{};
        ep.bias = bias;
        ep.act1 = act;
        conv_simple(x, out, W, 3, 3, 1, 1, 1, 1, sf, st, ep);
        if (zero_tail_after) zero_tail(out, lvl);
        return good();
    }
    // The strided 1x1 shortcut conv `pfx`.shortcut.0 (with its BN `pfx`.shortcut.1 folded in) over x as one more K range of the
    // block's last conv `cs` (output o): its weights are appended to every row of wk ([o.C][K] -> [o.C][K + x.C]) and its BN
    // shift is added to bias.
    bool merge_shortcut(ConvSpec& cs, const std::string& pfx, const View& x, int sf, int st, const View& o, std::vector<float>& wk, int& K,
                        std::vector<float>& bias) {
        std::vector<float> ss, hs, wsv;
        int co = 0;
        if (!w.bn(pfx + ".shortcut.1", true, ss, hs) || !w.pack_conv(pfx + ".shortcut.0.weight", &ss, wsv, &co)) return false;
        int Fs, Ts;
        const int K2 = add_conv_taps(cs, x, 1, 1, 1, 1, 0, 0, sf, st, K, &Fs, &Ts);
        if (K2 != x.C || co != o.C || (int)wsv.size() != o.C * K2 || Fs != o.F || Ts != o.T) { set_err(pfx + ": shortcut shape mismatch"); ok = false; return false; }
        std::vector<float> wm((size_t)o.C * (K + K2));
        for (int r = 0; r < o.C; ++r) {
            memcpy(&wm[(size_t)r * (K + K2)], &wk[(size_t)r * K], (size_t)K * 4);
            memcpy(&wm[(size_t)r * (K + K2) + K], &wsv[(size_t)r * K2], (size_t)K2 * 4);
        }
        wk.swap(wm);
        K += K2;
        for (int i = 0; i < o.C; ++i) bias[i] += hs[i];
        return true;
    }
    // Attentive statistics (pooling_layers.py): logits = W2 h + bias2, softmax over time per channel, stats = [mean | sqrt(max(var,
    // eps))] of x under those weights.  The fused op where it applies (bias2 cancels in the softmax), else linear2 as a conv plus
    // astp_stats.  lvl: stride level of x
    bool astp_tail(const View& x, const View& h, const void* W2, const float* bias2, float* stats, double eps, int lvl) {
        const int* l = lens(lvl);
        if (fused(e.opts.astp_fused) && good()) {
            PlanOp op;
            const OpBuild r = make_astp_op(x, h, W2, stats, (float)eps, &op, l);
            if (r == OpBuild::built) { push(std::move(op)); return true; }
            if (r == OpBuild::error) { ok = false; return false; }
        }
        View logits = act(x.B, 1, x.T, x.C);
        WsEpi ep{};
        ep.bias = bias2;
        conv_simple(h, logits, W2, 1, 1, 1, 1, 0, 0, 1, 1, ep);
        if (!good()) return false;
        WsAstpStats a{x, logits, stats, (float)eps, l};
        a.kernel = ws_astp_stats_kernel(a);
        push(a, ws_launch_astp_stats, "astp_stats");
        return good();
    }
};

bool build_ecapa(Builder& b);
bool build_resnet(Builder& b);
bool build_res2net(Builder& b);
bool build_simam_resnet(Builder& b);
bool build_gemini(Builder& b);
bool build_xvec(Builder& b);
bool build_campplus(Builder& b);
// shared by the families: the ResNet-style stem, BasicBlock (also CAM++'s FCM head) and the TSTP + segment-layer tail
View stem(Builder& b, const std::string& convkey, const std::string& bnkey, View outbuf);
View basic_block(Builder& b, const std::string& p, const View& x, int cout, int sf, int st_, View hbuf, View obuf, int lvl = 0);
bool resnet_tail(Builder& b, const View& cur, bool two_layers, int lvl = 3);

}  // namespace ws
