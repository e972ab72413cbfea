// Speaker-embedding engine: weight ingest (reference state_dict keys), per-(B,T) launch plans for
// ECAPA-TDNN / ResNet / CAM++ built from the fused conv operator + bandwidth kernels, CUDA-graph replay, fbank
// frontend tables, and the C ABI declared in include/wespeaker_b200.h.
//
// Reference behaviour being reproduced (file:line in wenet-e2e/wespeaker, wespeaker/):
//   models/ecapa_tdnn.py:29-234, models/pooling_layers.py:67-148, models/resnet.py:35-204,
//   models/campplus.py:55-413, utils/checkpoint.py:20-85, bin/extract.py:109-139.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>

#include "../../include/wespeaker_b200.h"
#include "ws_host.h"

using namespace ws;

namespace {

struct HostT {
    std::vector<float> v;
    std::vector<long long> shape;
    long long numel() const {
        long long n = 1;
        for (long long d : shape) n *= d;
        return n;
    }
};

struct FbankTables {
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
    // plan-trace engines (option plan_trace): every buffer this plan allocated, (address, bytes), for ws_engine_plan_trace
    std::vector<std::pair<unsigned long long, unsigned long long>> trace_allocs;
    ~Plan() {
        if (done) cudaEventDestroy(done);
        if (gexec) cudaGraphExecDestroy(gexec);
        if (!check) for (void* p : bufs) cudaFree(p);
    }
};

}  // namespace

struct ws_engine {
    std::string model, prec;
    int feat_dim = 80, embed_dim = 0, device = 0;
    int act_dt = WS_F32;
    int use_tc = 0;  // 0 FFMA, 2 persistent tensor-core kernel, 3 the same + weight-sharing clusters on large layers (default)
    bool split = false;  // 3xTF32: fp32 activations/weights carry lo twins, GEMMs run 3 error-compensated passes
    std::map<const void*, const void*> wlo;  // packed weight -> its lo twin
    std::map<std::string, long long> opts;
    std::map<std::string, HostT> sd;
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
    std::map<std::pair<int, int>, std::unique_ptr<Plan>> plans;   // key: (B, 2 * T + masked)
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
    std::map<std::string, FbankTables> fb;
    void* wav_dev = nullptr;
    size_t wav_bytes = 0;
    // double-buffered host->device pipeline (ws_engine_submit_wav_host / ws_engine_collect)
    cudaStream_t copy_st = nullptr;
    static constexpr int kSlots = 4;
    void* slot_wav[kSlots] = {nullptr, nullptr, nullptr, nullptr};
    size_t slot_bytes[kSlots] = {0, 0, 0, 0};
    cudaEvent_t slot_copied[kSlots] = {nullptr, nullptr, nullptr, nullptr}, slot_done[kSlots] = {nullptr, nullptr, nullptr, nullptr};
    // model hyper-parameters
    int channels = 512;
    bool glob = false;
    bool bottleneck = false;   // ResNet50..293: Bottleneck blocks (expansion 4) instead of BasicBlocks
    std::vector<int> num_blocks;
    // Res2Net / ERes2Net (res2net.py:202-221, eres2net.py:393-431): stem width, baseWidth, scale, expansion, AFF fusion
    int r2_m = 0, r2_base_width = 32, r2_scale = 2, r2_expansion = 2;
    bool r2_fuse = false;
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
    long long opt(const char* k, long long dflt) const {
        auto it = opts.find(k);
        return it == opts.end() ? dflt : it->second;
    }
};

namespace {

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

    void* raw(size_t bytes) {
        void* d = nullptr;
        if (plan_check_mode()) {
            d = plan_check_alloc(bytes);
            e.check_allocs.push_back({(unsigned long long)d, (unsigned long long)bytes});
        } else if (cudaMalloc(&d, bytes ? bytes : 16) != cudaSuccess) {
            if (ok) set_err("cudaMalloc failed for an activation buffer");
            ok = false;
            return nullptr;
        } else if (plan_trace_mode()) {
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
    // a bandwidth op: launch closure, label, and its plan-trace description (kept in plan-trace mode only)
    void push(Op run, const char* label, std::string trace) {
        push(PlanOp{std::move(run), label, 0.0, plan_trace_mode() ? std::move(trace) : std::string()});
    }
    // length-masked plans: frame counts of stride level k (nullptr in ordinary plans), and "zero the rows behind every
    // utterance's end" for tensors a time-mixing op is about to read (the reference's unpadded forward sees zero padding)
    const int* lens(int level) const { return p.masked ? p.lens + (size_t)level * p.B : nullptr; }
    void zero_tail(const View& v, int level) {
        if (!p.masked) return;
        const View x = v;
        const int* l = lens(level);
        push([=](cudaStream_t s) { return ws_launch_zero_tail(x.p, (float*)x.plo, x.dt, x.B, x.F, x.T, x.C, x.ld, l, s); }, "zero_tail",
             "{\"kind\":\"zero_tail\"," + ti("es", ws_esize(x.dt)) + "," + tview("x", x) + "," + tp("lens", l) + "}");
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
        if (!make_conv_op(s, e.use_tc, &op)) { ok = false; return; }
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
        View xv = x;
        const int* l = lens(level);
        push([=](cudaStream_t s) {
            return ws_launch_tstats(xv.p, xv.dt, xv.B, xv.F, xv.T, xv.C, xv.ld, pre_scale, pre_shift, out, WS_F32, out_ld,
                                    std_off, 1e-7f, s, l);
        }, "tstats", "{\"kind\":\"tstats\"," + ti("es", ws_esize(x.dt)) + "," + tview("x", x) + "," + tp("pre_scale", pre_scale) + "," + tp("pre_shift", pre_shift) + "," +
                     tp("out", out) + "," + ti("out_ld", out_ld) + "," + ti("std_off", std_off) + "," + tp("lens", l) + "}");
    }
    void linear(const float* in, long long in_ld, const float* in2, long long in2_ld, int rows_per_b, const float* W,
                const float* bias, float* out, long long out_ld, int R, int I, int O, int act) {
        // split K so that the launch fills the machine (these layers are latency-bound otherwise)
        const bool big = ws_linear_rows_big(in_ld, in2, in2_ld, R, I, O);
        const int blocks = big ? ((O + 63) / 64) * ((R + 63) / 64) : ((O + 31) / 32) * ((R + 15) / 16);
        int nsplit = 1;
        const int sms = ws_num_sms();
        if (big) while (blocks * nsplit < sms && I / (nsplit * 2) >= 96 && nsplit < 32) nsplit *= 2;
        else while (blocks * nsplit < 2 * sms && I / (nsplit * 2) >= 128 && nsplit < 16) nsplit *= 2;
        float* wsp = nsplit > 1 ? f32((size_t)nsplit * R * O) : nullptr;
        if (nsplit > 1) p.extra_launches += 1;
        push([=](cudaStream_t s) {
            return ws_launch_linear_rows(in, in_ld, in2, in2_ld, rows_per_b, W, bias, out, out_ld, R, I, O, act, wsp,
                                         nsplit, s);
        }, "linear_rows", "{\"kind\":\"linear\"," + tp("in", in) + "," + ti("in_ld", in_ld) + "," + tp("in2", in2) + "," + ti("in2_ld", in2_ld) + "," + ti("rows_per_b", rows_per_b) + "," +
                     tp("W", W) + "," + tp("bias", bias) + "," + tp("out", out) + "," + ti("out_ld", out_ld) + "," + ti("R", R) + "," + ti("I", I) + "," + ti("O", O) + "," + ti("act", act) +
                     tplo("wsp", wsp) + "}");
    }
    // the fp32 input features -> x0 (B,1,T,feat_dim) in the activation dtype
    void convert_input(const View& x0) {
        const float* fin = p.feats_in;
        void* xo = x0.p;
        float* xlo = (float*)x0.plo;
        const int dt = x0.dt;
        const long long n = x0.npos() * x0.C;
        push([=](cudaStream_t s) { return ws_launch_convert(fin, xo, xlo, dt, n, s); }, "convert",
             "{\"kind\":\"convert\"," + ti("es", ws_esize(dt)) + "," + tp("in", fin) + "," + tp("out", xo) + "," + ti("n", n) + tplo("out_lo", xlo) + "}");
    }
    // out = relu(x * scale + shift), per channel over x's C channels
    void bnrelu(const View& x, const float* scale, const float* shift, const View& out) {
        const View xv = x, ov = out;
        const int C = x.C;
        const long long npos = x.npos();
        push([=](cudaStream_t s) { return ws_launch_bnrelu(xv.p, xv.ld, scale, shift, ov.p, (float*)ov.plo, ov.ld, xv.dt, npos, C, s); }, "bnrelu",
             "{\"kind\":\"bnrelu\"," + ti("es", ws_esize(x.dt)) + "," + tview("x", x) + "," + tp("scale", scale) + "," + tp("shift", shift) + "," +
             tview("out", out) + "," + ti("C", C) + "}");
    }
    // The halo-resident 3x3 pad-1 conv (ws_conv3x3.cu: every input row crosses L2 -> SM once instead of once per tap),
    // out = act(conv(x, W) + bias [+ res]).  halo3x3: whether the precision and the options let convs of strides (sf, st) use
    // it.  halo_conv3x3 returns 1 with *op built (not pushed), 0 when the caller runs the conv-GEMM instead (also when the
    // shape is outside the kernel's envelope), -1 on error.  lvl: stride level of `out`.
    bool halo3x3(int sf, int st) const {
        return e.use_tc >= 2 && e.act_dt != WS_F32 && e.opt("conv3x3", 1) != 0 && ((sf == 1 && st == 1) || e.opt("conv3x3_strided", 1) != 0);
    }
    int halo_conv3x3(const View& x, const View& out, const void* W, const float* bias, const View* res, int act, int sf, int st, int lvl,
                     PlanOp* op) {
        if (!halo3x3(sf, st)) return 0;
        bool unsupported = false;
        if (make_conv3x3_op(x, out, W, bias, res, act == WS_ACT_RELU20 ? 2 : act == WS_ACT_RELU ? 1 : 0, op, &unsupported, sf, st, lens(lvl)))
            return 1;
        if (unsupported) return 0;
        ok = false;
        return -1;
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
        if (e.use_tc >= 2 && e.opt("astp_fused", 1) && good()) {
            PlanOp op;
            bool unsupported = false;
            if (make_astp_op(x, h, W2, stats, (float)eps, &op, &unsupported, l)) { push(std::move(op)); return true; }
            if (!unsupported) { ok = false; return false; }
        }
        View logits = act(x.B, 1, x.T, x.C);
        WsEpi ep{};
        ep.bias = bias2;
        conv_simple(h, logits, W2, 1, 1, 1, 1, 0, 0, 1, 1, ep);
        if (!good()) return false;
        const View fr = x, lg = logits;
        const float var_floor = (float)eps;
        push([=](cudaStream_t s) { return ws_launch_astp_stats(fr.p, lg.p, fr.dt, fr.B, fr.T, fr.C, fr.ld, stats, var_floor, s, l); }, "astp_stats",
             "{\"kind\":\"astp_stats\"," + ti("es", ws_esize(fr.dt)) + "," + tview("x", fr) + "," + tview("logits", lg) + "," + tp("stats", stats) + "," +
             tp("lens", l) + "," + tf("eps", eps) + "}");
        return good();
    }
};

// ----------------------------------------------------------------------------------------------- ECAPA-TDNN
// ecapa_tdnn.py:160-234.  Channels-last buffers; torch.cat is free (layer outputs are written into slices of one
// (B,T,3C) buffer), Res2 "sp + spx[i]" is produced by the previous conv's epilogue (out2 = out + add2).
bool build_ecapa(Builder& b) {
    ws_engine& e = b.e;
    const int B = b.p.B, T = b.p.T, C = e.channels, w8 = C / 8, Fd = e.feat_dim, E = e.embed_dim;
    View x0 = b.act(B, 1, T, Fd);
    View out1 = b.act(B, 1, T, C), cat = b.act(B, 1, T, 3 * C);
    View tA = b.act(B, 1, T, C), tB = b.act(B, 1, T, C), tC = b.act(B, 1, T, C);
    View sc[2] = {b.act(B, 1, T, w8), b.act(B, 1, T, w8)};
    View frame = b.act(B, 1, T, 1536), hid = b.act(B, 1, T, 128);
    float* semean = b.f32((size_t)B * C);
    float* sehid = b.f32((size_t)B * 128);
    float* segate = b.f32((size_t)B * C);
    float* stats = b.f32((size_t)B * 3072);
    if (!b.good()) return false;
    b.convert_input(x0);
    b.zero_tail(x0, 0);   // (masked plans) the k=5 conv of layer1 must see zero padding behind each utterance
    // Conv1dReluBn (ecapa_tdnn.py:85-106): bn(relu(conv(x)+bias))
    auto conv_relu_bn = [&](const std::string& pfx, const View& x, const View& out, int k, int dil, int pad) {
        std::vector<float> wp, s, h;
        if (!b.w.pack_conv(pfx + ".conv.weight", nullptr, wp) || !b.w.bn(pfx + ".bn", true, s, h)) return;
        WsEpi ep{};
        ep.bias = b.w.vec(pfx + ".conv.bias");
        ep.act1 = WS_ACT_RELU;
        ep.scale = b.w.f32("bns:" + pfx, s);
        ep.shift = b.w.f32("bnh:" + pfx, h);
        b.conv_simple(x, out, b.w.act("w:" + pfx, wp), 1, k, 1, dil, 0, pad, 1, 1, ep);
    };
    conv_relu_bn("layer1", x0, out1, 5, 1, 2);
    View xin = out1;
    float* se_colsum = nullptr;
    if (e.use_tc >= 2 && e.act_dt != WS_F32 && !e.split && T >= 128 && (C == 512 || C == 1024) && e.opt("se_fused", 1) &&
        e.opt("se_colsum", 1) && getenv("WS_EPI_GENERIC") == nullptr && !b.p.masked)   // (column sums would include padding rows)
        se_colsum = b.f32((size_t)2 * (((size_t)B * T + 63) / 64) * C);
    for (int L = 2; L <= 4 && b.good(); ++L) {
        const int d = L;
        const std::string pf = "layer" + std::to_string(L) + ".se_res2block";
        conv_relu_bn(pf + ".0", xin, tA, 1, 1, 0);
        b.zero_tail(tA, 0);   // (masked plans) the dilated Res2 convs read tA across time
        // Res2Conv1dReluBn (ecapa_tdnn.py:29-78): 7 dependent dilated k=3 convs on w8-channel groups
        bool fused = false;
        if (e.use_tc >= 2 && e.act_dt != WS_F32 && e.opt("res2_fused", 1)) {
            // one persistent launch per stage: the chain stays in shared memory / registers (ws_res2_fused.cu)
            std::vector<float> w7((size_t)7 * w8 * 3 * w8), b7((size_t)7 * w8), s7((size_t)7 * w8), h7((size_t)7 * w8);
            bool okw = true;
            for (int i = 0; i < 7 && okw; ++i) {
                const std::string cp = pf + ".1.convs." + std::to_string(i), bp = pf + ".1.bns." + std::to_string(i);
                std::vector<float> wp, s, h;
                const HostT* bt = b.w.get(cp + ".bias");
                okw = bt && b.w.pack_conv(cp + ".weight", nullptr, wp) && b.w.bn(bp, true, s, h);
                if (!okw) break;
                memcpy(&w7[(size_t)i * w8 * 3 * w8], wp.data(), wp.size() * 4);
                memcpy(&b7[(size_t)i * w8], bt->v.data(), (size_t)w8 * 4);
                memcpy(&s7[(size_t)i * w8], s.data(), (size_t)w8 * 4);
                memcpy(&h7[(size_t)i * w8], h.data(), (size_t)w8 * 4);
            }
            if (!okw) break;
            PlanOp op;
            bool unsupported = false;
            if (make_res2_op(tA, tB, b.w.act("w7:" + pf, w7), b.w.f32("b7:" + pf, b7), b.w.f32("s7:" + pf, s7),
                             b.w.f32("h7:" + pf, h7), w8, d, &op, &unsupported, b.lens(0))) {
                b.push(std::move(op));
                fused = true;
            } else if (!unsupported) {
                b.ok = false;
                break;
            }
        }
        for (int i = 0; i < 7 && b.good() && !fused; ++i) {
            const std::string cp = pf + ".1.convs." + std::to_string(i), bp = pf + ".1.bns." + std::to_string(i);
            std::vector<float> wp, s, h;
            if (!b.w.pack_conv(cp + ".weight", nullptr, wp) || !b.w.bn(bp, true, s, h)) break;
            WsEpi ep{};
            ep.bias = b.w.vec(cp + ".bias");
            ep.act1 = WS_ACT_RELU;
            ep.scale = b.w.f32("bns:" + bp, s);
            ep.shift = b.w.f32("bnh:" + bp, h);
            if (i < 6) {
                View nx = tA.ch((i + 1) * w8, w8);
                ep.out2 = sc[i & 1].p; ep.out2_lo = sc[i & 1].plo; ep.out2_ld = sc[i & 1].ld;
                ep.add2 = nx.p; ep.add2_ld = nx.ld;
            }
            const View src = (i == 0) ? tA.ch(0, w8) : sc[(i - 1) & 1];
            b.conv_simple(src, tB.ch(i * w8, w8), b.w.act("w:" + cp, wp), 1, 3, 1, d, 0, d, 1, 1, ep);
            if (i < 6) b.zero_tail(sc[i & 1], 0);   // (masked plans) s_{i+1} feeds the next dilated conv
        }
        if (!b.good()) break;
        {   // third block: 1x1 conv over cat[sp_0..sp_6, spx_7]: two K ranges from two buffers
            const std::string cp = pf + ".2";
            std::vector<float> wp, s, h;
            if (!b.w.pack_conv(cp + ".conv.weight", nullptr, wp) || !b.w.bn(cp + ".bn", true, s, h)) break;
            ConvSpec cs;
            cs.dt = e.act_dt;
            cs.src[0] = Builder::src_of(tB.ch(0, 7 * w8));
            cs.src[1] = Builder::src_of(tA.ch(7 * w8, w8));
            cs.nsrc = 2;
            cs.taps.push_back(WsTap{0, 0, 0, 0, 0, 7 * w8});
            cs.taps.push_back(WsTap{1, 0, 0, 0, 7 * w8, w8});
            cs.W = b.w.act("w:" + cp, wp); cs.Ktot = C; cs.Cout = C; cs.B = B; cs.F = 1; cs.T = T;
            cs.dense_pointwise = true;
            cs.epi.bias = b.w.vec(cp + ".conv.bias");
            cs.epi.act1 = WS_ACT_RELU;
            cs.epi.scale = b.w.f32("bns:" + cp, s);
            cs.epi.shift = b.w.f32("bnh:" + cp, h);
            fill_epi_out(cs.epi, tC);
            // SE squeeze fused into this conv's epilogue (16-bit tensor-core path): per-unit column sums instead of a
            // second pass over the 100 MB output
            if (se_colsum != nullptr) { cs.epi.colsum = se_colsum; cs.epi.colsum_T = T; }
            b.conv(cs);
        }
        // SE_Connect (ecapa_tdnn.py:113-126) + residual (:157)
        if (e.opt("se_fused", 1) && (C == 512 || C == 1024)) {
            const HostT* w2 = b.w.get(pf + ".3.linear2.weight");   // (C, 128) -> transposed (128, C) for coalesced reads
            if (!w2) break;
            std::vector<float> w2t((size_t)128 * C);
            for (int c = 0; c < C; ++c)
                for (int h = 0; h < 128; ++h) w2t[(size_t)h * C + c] = w2->v[(size_t)c * 128 + h];
            const float* w1d = b.w.vec(pf + ".3.linear1.weight");
            const float* b1d = b.w.vec(pf + ".3.linear1.bias");
            const float* w2d = b.w.f32("w2t:" + pf, w2t);
            const float* b2d = b.w.vec(pf + ".3.linear2.bias");
            View tc = tC;
            const int dt = e.act_dt;
            const float* cs_in = se_colsum;
            const int* l0 = b.lens(0);
            b.push([=](cudaStream_t s) { return ws_launch_se_gate(tc.p, dt, B, T, C, tc.ld, w1d, b1d, w2d, b2d, 128, segate, cs_in, s, l0); }, "se_gate",
                   "{\"kind\":\"se_gate\"," + ti("es", ws_esize(dt)) + "," + tview("x", tc) + "," + tp("W1", w1d) + "," + tp("b1", b1d) + "," +
                   tp("W2t", w2d) + "," + tp("b2", b2d) + "," + ti("H", 128) + "," + tp("gate", segate) + "," + tp("lens", l0) + "}");
        } else {
            b.tstats(tC, nullptr, nullptr, semean, C, -1);
            b.linear(semean, C, nullptr, 0, 1, b.w.vec(pf + ".3.linear1.weight"), b.w.vec(pf + ".3.linear1.bias"), sehid, 128, B,
                     C, 128, WS_ACT_RELU);
            b.linear(sehid, 128, nullptr, 0, 1, b.w.vec(pf + ".3.linear2.weight"), b.w.vec(pf + ".3.linear2.bias"), segate, C,
                     B, 128, C, WS_ACT_SIGMOID);
        }
        {
            View o = cat.ch((L - 2) * C, C), xi = xin, tc = tC;
            const int dt = e.act_dt;
            b.push([=](cudaStream_t s) {
                return ws_launch_scale_residual(tc.p, tc.ld, segate, xi.p, xi.ld, o.p, (float*)o.plo, o.ld, dt, B, T, C, s);
            }, "scale_residual", "{\"kind\":\"scale_residual\"," + ti("es", ws_esize(dt)) + "," + tview("x", tc) + "," + tp("gate", segate) + "," +
                                 tview("res", xi) + "," + tview("out", o) + "}");
            xin = o;
        }
    }
    if (!b.good()) return false;
    {   // self.conv (1x1, 3C -> 1536) then F.relu (ecapa_tdnn.py:217-218,229)
        std::vector<float> wp;
        if (!b.w.pack_conv("conv.weight", nullptr, wp)) return false;
        WsEpi ep{};
        ep.bias = b.w.vec("conv.bias");
        ep.act1 = WS_ACT_RELU;
        b.conv_simple(cat, frame, b.w.act("w:conv", wp), 1, 1, 1, 1, 0, 0, 1, 1, ep);
    }
    // ASTP (pooling_layers.py:119-144).  Global context: W1 [x; mean; std] = W1x x + (W1m mean + W1s std): the
    // broadcast part becomes a per-utterance bias row added in the GEMM epilogue.
    const float* rowbias = nullptr;
    {
        const HostT* w1 = b.w.get("pool.linear1.weight");
        if (!w1) return false;
        const int in_dim = (int)w1->shape[1];
        std::vector<float> wx((size_t)128 * 1536);
        for (int o = 0; o < 128; ++o)
            for (int c = 0; c < 1536; ++c) wx[(size_t)o * 1536 + c] = w1->v[(size_t)o * in_dim + c];
        if (e.glob) {
            if (in_dim != 3 * 1536) { set_err("pool.linear1.weight: expected 4608 inputs for global_context_att"); return false; }
            std::vector<float> wc((size_t)128 * 3072);
            for (int o = 0; o < 128; ++o)
                for (int c = 0; c < 3072; ++c) wc[(size_t)o * 3072 + c] = w1->v[(size_t)o * in_dim + 1536 + c];
            float* ctx = b.f32((size_t)B * 3072);
            float* rb = b.f32((size_t)B * 128);
            b.tstats(frame, nullptr, nullptr, ctx, 3072, 1536);
            b.linear(ctx, 3072, nullptr, 0, 1, b.w.f32("w:pool.linear1.ctx", wc), nullptr, rb, 128, B, 3072, 128, WS_ACT_NONE);
            rowbias = rb;
        } else if (in_dim != 1536) {
            set_err("pool.linear1.weight: expected 1536 inputs"); return false;
        }
        WsEpi ep{};
        ep.bias = b.w.vec("pool.linear1.bias");
        ep.rowbias = rowbias; ep.rowbias_ld = 128;
        ep.act1 = WS_ACT_TANH;
        b.conv_simple(frame, hid, b.w.act("w:pool.linear1.x", wx), 1, 1, 1, 1, 0, 0, 1, 1, ep);
        std::vector<float> w2;
        if (!b.w.pack_conv("pool.linear2.weight", nullptr, w2)) return false;
        // linear2 + softmax over time + weighted statistics, fused into one launch where it applies: the logits never leave
        // the SM (ws_astp_fused.cu)
        if (!b.astp_tail(frame, hid, b.w.act("w:pool.linear2", w2), b.w.vec("pool.linear2.bias"), stats, 1e-7, 0)) return false;
    }
    {   // bn(3072) then linear (ecapa_tdnn.py:230-231): fold the affine into the linear; optional bn2 (emb_bn)
        std::vector<float> s, h;
        const HostT* lw = b.w.get("linear.weight");
        const HostT* lb = b.w.get("linear.bias");
        if (!lw || !lb || !b.w.bn("bn", true, s, h)) return false;
        if ((int)lw->shape[0] != E) { set_err("linear.weight: embed_dim mismatch"); return false; }
        std::vector<float> wf((size_t)E * 3072), bf(E);
        std::vector<float> s2(E, 1.f), h2(E, 0.f);
        if (e.opt("emb_bn", 0) && !b.w.bn("bn2", true, s2, h2)) return false;
        for (int o = 0; o < E; ++o) {
            double acc = lb->v[o];
            for (int i = 0; i < 3072; ++i) {
                wf[(size_t)o * 3072 + i] = (float)((double)lw->v[(size_t)o * 3072 + i] * s[i] * s2[o]);
                acc += (double)lw->v[(size_t)o * 3072 + i] * h[i];
            }
            bf[o] = (float)(acc * s2[o] + h2[o]);
        }
        b.linear(stats, 3072, nullptr, 0, 1, b.w.f32("w:linear.folded", wf), b.w.f32("b:linear.folded", bf), b.p.emb, E, B,
                 3072, E, WS_ACT_NONE);
    }
    return b.good();
}

// ----------------------------------------------------------------------------------------------- 2-D residual blocks
// BasicBlock (resnet.py:35-69) / BasicResBlock (campplus.py:245-279): eval BN folded into the conv weights, the
// 1x1 strided shortcut conv is merged into conv2's GEMM as one extra K range, residual/ReLU in the epilogue.
// `lvl`: stride level of the block's OUTPUT (length-masked plans: frame counts b.lens(lvl)); the time stride st_ is 1 or 2
View basic_block(Builder& b, const std::string& p, const View& x, int cout, int sf, int st_, View hbuf, View obuf, int lvl = 0) {
    std::vector<float> s1, h1, s2, h2, w1, w2;
    View none;
    if (!b.w.bn(p + ".bn1", true, s1, h1) || !b.w.bn(p + ".bn2", true, s2, h2) || !b.w.pack_conv(p + ".conv1.weight", &s1, w1) ||
        !b.w.pack_conv(p + ".conv2.weight", &s2, w2))
        return none;
    const int Fo = (x.F + 2 - 3) / sf + 1, To = (x.T + 2 - 3) / st_ + 1;
    const View h = hbuf.shaped(x.B, Fo, To, cout), o = obuf.shaped(x.B, Fo, To, cout);
    if (!b.conv3x3(x, h, b.w.act("w:" + p + ".conv1", w1), b.w.f32("bnh:" + p + ".bn1", h1), WS_ACT_RELU, sf, st_, lvl)) return none;
    const bool has_sc = b.e.sd.count(p + ".shortcut.0.weight") != 0;
    if (b.halo3x3(1, 1) && (cout == 32 || cout == 64 || cout == 128)) {
        // conv2 on the halo-resident kernel: the 1x1 strided shortcut conv (+ its BN) is written to `o` first and then
        // read back as the residual, in place (each output element is read and written by the same CTA step).  conv2's op is
        // built first: if the shape is outside the kernel's envelope nothing has been emitted yet.  (The channel counts the
        // kernel takes are checked here so that other blocks do not upload conv2's unmerged weights.)
        const View res = has_sc ? o : x;
        PlanOp op2;
        const int r = b.halo_conv3x3(h, o, b.w.act("w:" + p + ".conv2", w2), b.w.f32("bnh:" + p + ".bn2", h2), &res, WS_ACT_RELU, 1, 1, lvl, &op2);
        if (r < 0) return none;
        if (r > 0) {
            if (has_sc) {
                std::vector<float> ss, hs, wsv;
                if (!b.w.bn(p + ".shortcut.1", true, ss, hs) || !b.w.pack_conv(p + ".shortcut.0.weight", &ss, wsv)) return none;
                WsEpi es{};
                es.bias = b.w.f32("bnh:" + p + ".shortcut", hs);
                b.conv_simple(x, o, b.w.act("w:" + p + ".shortcut", wsv), 1, 1, 1, 1, 0, 0, sf, st_, es);
                if (!b.good()) return none;
            }
            b.push(std::move(op2));
            return o;
        }
    }
    ConvSpec cs;
    cs.dt = b.e.act_dt;
    int F2, T2;
    int K = add_conv_taps(cs, h, 3, 3, 1, 1, 1, 1, 1, 1, 0, &F2, &T2);
    std::vector<float> bias2 = h2;
    if (has_sc) {
        if (!b.merge_shortcut(cs, p, x, sf, st_, o, w2, K, bias2)) return none;
    } else {
        cs.epi.res = x.p;
        cs.epi.res_ld = x.ld;
    }
    cs.W = b.w.act("w:" + p + ".conv2m", w2); cs.Ktot = K; cs.Cout = cout; cs.B = x.B; cs.F = Fo; cs.T = To;
    cs.epi.bias = b.w.f32("bnh:" + p + ".bn2m", bias2);
    cs.epi.act2 = WS_ACT_RELU;
    fill_epi_out(cs.epi, o);
    b.conv(cs);
    b.zero_tail(o, lvl);
    return o;
}

// Bottleneck (resnet.py:72-107): 1x1 -> BN -> ReLU -> 3x3 (stride) -> BN -> ReLU -> 1x1 (x4) -> BN, + shortcut, ReLU.  BNs are
// folded into the conv weights; the 1x1 strided shortcut conv (+ BN) is merged into conv3's GEMM as one extra K range (same
// output positions), an identity shortcut is the residual input of conv3's epilogue.
View bottleneck_block(Builder& b, const std::string& p, const View& x, int planes, int s, View h1buf, View h2buf, View obuf,
                      int lvl_in = 0, int lvl = 0) {
    std::vector<float> s1, h1, s2, h2, s3, h3, w1, w2, w3;
    View none;
    if (!b.w.bn(p + ".bn1", true, s1, h1) || !b.w.bn(p + ".bn2", true, s2, h2) || !b.w.bn(p + ".bn3", true, s3, h3) ||
        !b.w.pack_conv(p + ".conv1.weight", &s1, w1) || !b.w.pack_conv(p + ".conv2.weight", &s2, w2) || !b.w.pack_conv(p + ".conv3.weight", &s3, w3))
        return none;
    const int cout = 4 * planes;
    const int Fo = (x.F + 2 - 3) / s + 1, To = (x.T + 2 - 3) / s + 1;
    const View a = h1buf.shaped(x.B, x.F, x.T, planes), c = h2buf.shaped(x.B, Fo, To, planes), o = obuf.shaped(x.B, Fo, To, cout);
    WsEpi e1{};
    e1.bias = b.w.f32("bnh:" + p + ".bn1", h1);
    e1.act1 = WS_ACT_RELU;
    b.conv_simple(x, a, b.w.act("w:" + p + ".conv1", w1), 1, 1, 1, 1, 0, 0, 1, 1, e1);
    b.zero_tail(a, lvl_in);   // (masked plans) the 3x3 conv reads `a` across time
    if (!b.good()) return none;
    // (conv3 is 1x1: its input needs no zero rows behind the utterance's end)
    if (!b.conv3x3(a, c, b.w.act("w:" + p + ".conv2", w2), b.w.f32("bnh:" + p + ".bn2", h2), WS_ACT_RELU, s, s, lvl, false)) return none;
    ConvSpec cs;
    cs.dt = b.e.act_dt;
    int F3, T3;
    int K = add_conv_taps(cs, c, 1, 1, 1, 1, 0, 0, 1, 1, 0, &F3, &T3);
    std::vector<float> bias3 = h3;
    if (b.e.sd.count(p + ".shortcut.0.weight") != 0) {
        if (!b.merge_shortcut(cs, p, x, s, s, o, w3, K, bias3)) return none;
    } else {
        cs.epi.res = x.p;
        cs.epi.res_ld = x.ld;
        cs.dense_pointwise = true;
    }
    cs.W = b.w.act("w:" + p + ".conv3m", w3); cs.Ktot = K; cs.Cout = cout; cs.B = x.B; cs.F = Fo; cs.T = To;
    cs.epi.bias = b.w.f32("bnh:" + p + ".bn3m", bias3);
    cs.epi.act2 = WS_ACT_RELU;
    fill_epi_out(cs.epi, o);
    b.conv(cs);
    return o;
}

View stem(Builder& b, const std::string& convkey, const std::string& bnkey, View outbuf) {
    std::vector<float> s, h, w9;
    int co, ci, nt;
    View none;
    if (!b.w.bn(bnkey, true, s, h) || !b.w.pack_conv(convkey, &s, w9, &co, &ci, &nt)) return none;
    if (ci != 1 || nt != 9) { set_err(convkey + ": expected (Cout,1,3,3)"); b.ok = false; return none; }
    const int B = b.p.B, T = b.p.T, Fd = b.e.feat_dim;
    const View o = outbuf.shaped(B, Fd, T, co);
    const float* wd = b.w.f32("w:" + convkey + ".stem", w9);   // [Cout][9] (tap = df*3 + dt)
    const float* hd = b.w.f32("bnh:" + bnkey, h);
    const float* fin = b.p.feats_in;
    const int dt = b.e.act_dt;
    void* op = o.p;
    float* olo = (float*)o.plo;
    const int* l0 = b.lens(0);
    b.push([=](cudaStream_t st) { return ws_launch_stem(fin, wd, hd, op, olo, dt, B, T, Fd, co, st, l0); }, "stem",
           "{\"kind\":\"stem\"," + ti("es", ws_esize(dt)) + "," + tp("feats", fin) + "," + tp("w9", wd) + "," + tp("shift", hd) + "," +
           tview("out", o) + "," + ti("Fdim", Fd) + "," + tp("lens", l0) + "}");
    return o;
}

// TSTP over the last feature map + the segment layer(s) (resnet.py:187-204; the same tail closes Res2Net / ERes2Net,
// res2net.py:186-199, eres2net.py:379-391, Gemini DF-ResNet and XVEC)
// two_layers: embed_b = seg_2(seg_bn_1(relu(seg_1(stats)))) (two_emb_layer), else embed_a = seg_1(stats)
// lvl: stride level of `cur` in length-masked plans (three stride-2 layers in ResNet / Res2Net, one in Gemini DF-ResNet)
bool resnet_tail(Builder& b, const View& cur, bool two_layers, int lvl = 3) {
    const int B = b.p.B, E = b.e.embed_dim;
    const int sd = cur.C * cur.F;  // stats_dim
    float* stats = b.f32((size_t)B * 2 * sd);
    b.tstats(cur, nullptr, nullptr, stats, 2 * sd, sd, lvl);  // TSTP, index c*F' + f (pooling_layers.py:78-85)
    const HostT* w1 = b.w.get("seg_1.weight");
    if (!w1) return false;
    if ((int)w1->shape[1] != 2 * sd || (int)w1->shape[0] != E) { set_err("seg_1.weight shape mismatch"); return false; }
    if (two_layers) {
        // seg_bn_1 (affine=False) folded into seg_2 (resnet.py:196-200)
        float* ea = b.f32((size_t)B * E);
        std::vector<float> s, h;
        const HostT* w2 = b.w.get("seg_2.weight");
        const HostT* b2 = b.w.get("seg_2.bias");
        if (!w2 || !b2 || !b.w.bn("seg_bn_1", false, s, h)) return false;
        std::vector<float> wf((size_t)E * E), bf(E);
        for (int o = 0; o < E; ++o) {
            double acc = b2->v[o];
            for (int i = 0; i < E; ++i) {
                wf[(size_t)o * E + i] = w2->v[(size_t)o * E + i] * s[i];
                acc += (double)w2->v[(size_t)o * E + i] * h[i];
            }
            bf[o] = (float)acc;
        }
        b.linear(stats, 2 * sd, nullptr, 0, 1, b.w.vec("seg_1.weight"), b.w.vec("seg_1.bias"), ea, E, B, 2 * sd, E, WS_ACT_RELU);
        b.linear(ea, E, nullptr, 0, 1, b.w.f32("w:seg_2.folded", wf), b.w.f32("b:seg_2.folded", bf), b.p.emb, E, B, E, E, WS_ACT_NONE);
    } else {
        b.linear(stats, 2 * sd, nullptr, 0, 1, b.w.vec("seg_1.weight"), b.w.vec("seg_1.bias"), b.p.emb, E, B, 2 * sd, E, WS_ACT_NONE);
    }
    return b.good();
}


// resnet.py:110-204
bool build_resnet(Builder& b) {
    ws_engine& e = b.e;
    const int B = b.p.B, T = b.p.T, Fd = e.feat_dim, m = 32;
    // largest activation map: the layer-1 output (m channels, x4 with Bottleneck blocks) at full (F, T)
    const std::vector<View> bufs = b.ring(e.bottleneck ? 4 : 3, (size_t)B * Fd * T * m * (e.bottleneck ? 4 : 1));
    if (!b.good()) return false;
    View cur = stem(b, "conv1.weight", "bn1", bufs[0]);
    int ci = 0;
    for (int li = 1; li <= 4 && b.good(); ++li) {
        const int cout = m << (li - 1);
        for (int bi = 0; bi < e.num_blocks[li - 1] && b.good(); ++bi) {
            const int s = (bi == 0 && li > 1) ? 2 : 1;
            const std::string p = "layer" + std::to_string(li) + "." + std::to_string(bi);
            const int lvl = li - 1, lvl_in = (s == 2) ? li - 2 : li - 1;   // stride level = number of stride-2 layers passed
            if (e.bottleneck) {   // x lives in bufs[ci]; the two intermediates and the output rotate through the other three
                View o = bottleneck_block(b, p, cur, cout, s, bufs[(ci + 1) % 4], bufs[(ci + 2) % 4], bufs[(ci + 3) % 4], lvl_in, lvl);
                ci = (ci + 3) % 4;
                cur = o;
                continue;
            }
            View o = basic_block(b, p, cur, cout, s, s, bufs[(ci + 1) % 3], bufs[(ci + 2) % 3], lvl);
            ci = (ci + 2) % 3;
            cur = o;
        }
    }
    if (!b.good()) return false;
    return resnet_tail(b, cur, e.opt("two_emb_layer", 0) != 0);
}

// ----------------------------------------------------------------------------------------------- Res2Net / ERes2Net
// res2net.py:34-199 (BasicBlockRes2Net), eres2net.py:43-391 (Hardtanh(0,20) "ReLU", AFF, BasicBlockERes2Net in layers 1-2,
// BasicBlockERes2Net_diff_AFF in layers 3-4, stride-2 3x3 downsampling + AFF bottom-up fusion of the four stage outputs).
//
// Channel padding: the split width w = floor(planes * baseWidth / 64) is 16 (or 24, 48, 96, 192 in ERes2Net34_aug); every
// width-w tensor is carried as wp = max(32, next power of two >= w) channels whose extra channels are exact zeros (zero weight
// rows and zero bias give Hardtanh(0) = 0 / SiLU(0) = 0, consumers have zero weight columns there), so every conv runs on the
// 32 / 64 / 128-channel kernels.  torch.split / torch.cat are channel slices of two buffers: conv1 writes all `scale` chunks
// into A, chain conv i writes chunk i of the concat buffer, conv3 reads the concat buffer (plus, in Res2Net, the last chunk of
// A) as K ranges.  "sp + spx[i]" ahead of a chain conv is the same conv over two sources with the weights repeated (the sum
// happens in the fp32 accumulator); BN is folded into the conv weights everywhere (conv -> BN -> Hardtanh order).
struct Res2Cfg {
    int m = 32, base_width = 32, scale = 2, expansion = 2;
    bool fuse = false;
};

static int res2_pad(int w) {
    int p = 32;
    while (p < w) p <<= 1;
    return p;
}

// rows [chunk c][j < w] of a [nchunk * w][K] matrix -> rows [c * wp + j] of a zero-initialised [nchunk * wp][K] matrix
static std::vector<float> pad_rows(const std::vector<float>& m, int nchunk, int w, int wp, int K) {
    std::vector<float> o((size_t)nchunk * wp * K, 0.f);
    for (int c = 0; c < nchunk; ++c)
        for (int j = 0; j < w; ++j)
            memcpy(&o[((size_t)c * wp + j) * K], &m[((size_t)c * w + j) * K], (size_t)K * 4);
    return o;
}
// columns [block g][chunk c][j < w] of a [R][G * nchunk * w] matrix -> columns [g][c * wp + j] of [R][G * nchunk * wp]
static std::vector<float> pad_cols(const std::vector<float>& m, int R, int G, int nchunk, int w, int wp) {
    const int Kin = G * nchunk * w, Kout = G * nchunk * wp;
    std::vector<float> o((size_t)R * Kout, 0.f);
    for (int r = 0; r < R; ++r)
        for (int g = 0; g < G; ++g)
            for (int c = 0; c < nchunk; ++c)
                memcpy(&o[(size_t)r * Kout + ((size_t)g * nchunk + c) * wp], &m[(size_t)r * Kin + ((size_t)g * nchunk + c) * w], (size_t)w * 4);
    return o;
}

// AFF (eres2net.py:75-102): out = x * att + y * (2 - att), att = 1 + tanh(BN(conv1x1(SiLU(BN(conv1x1([x | y]))))))
// x, y: views of Cp channels of which the first Cr are real (the rest zero); hid / att: scratch buffers of >= the positions.
static bool aff(Builder& b, const std::string& p, const View& x, const View& y, int Cr, View hidbuf, View attbuf, const View& out) {
    const int Cp = x.C, inter = Cr / 4, ip = std::max(32, (inter + 31) / 32 * 32);
    std::vector<float> sa, ha, sb, hb, wa, wb;
    const HostT* ba = b.w.get(p + ".local_att.0.bias");
    const HostT* bb = b.w.get(p + ".local_att.3.bias");
    if (!ba || !bb || !b.w.bn(p + ".local_att.1", true, sa, ha) || !b.w.bn(p + ".local_att.4", true, sb, hb) ||
        !b.w.pack_conv(p + ".local_att.0.weight", &sa, wa) || !b.w.pack_conv(p + ".local_att.3.weight", &sb, wb))
        return false;
    if ((int)wa.size() != inter * 2 * Cr || (int)wb.size() != Cr * inter || y.C != Cp || Cr > Cp) { set_err(p + ": AFF weight shape mismatch"); b.ok = false; return false; }
    // conv a: rows inter -> ip, columns [x: Cr -> Cp | y: Cr -> Cp]
    std::vector<float> wap = pad_rows(pad_cols(wa, inter, 2, 1, Cr, Cp), 1, inter, ip, 2 * Cp), bap(ip, 0.f);
    for (int i = 0; i < inter; ++i) bap[i] = sa[i] * ba->v[i] + ha[i];
    const View hid = hidbuf.shaped(x.B, x.F, x.T, ip);
    {
        ConvSpec cs;
        cs.dt = b.e.act_dt;
        int Fo, To;
        const int K1 = add_conv_taps(cs, x, 1, 1, 1, 1, 0, 0, 1, 1, 0, &Fo, &To);
        const int K2 = add_conv_taps(cs, y, 1, 1, 1, 1, 0, 0, 1, 1, K1, &Fo, &To);
        if (K1 != Cp || K2 != Cp || y.B != x.B || y.F != x.F || y.T != x.T) { set_err(p + ": AFF operand shape mismatch"); b.ok = false; return false; }
        cs.W = b.w.act("w:" + p + ".att0", wap); cs.Ktot = 2 * Cp; cs.Cout = ip; cs.B = x.B; cs.F = x.F; cs.T = x.T;
        cs.dense_pointwise = true;
        cs.epi.bias = b.w.f32("b:" + p + ".att0", bap);
        cs.epi.act1 = WS_ACT_SILU;
        fill_epi_out(cs.epi, hid);
        b.conv(cs);
    }
    // conv b: rows Cr -> Cp, columns inter -> ip; tanh in the epilogue
    std::vector<float> wbp = pad_rows(pad_cols(wb, Cr, 1, 1, inter, ip), 1, Cr, Cp, ip), bbp(Cp, 0.f);
    for (int i = 0; i < Cr; ++i) bbp[i] = sb[i] * bb->v[i] + hb[i];
    const View att = attbuf.shaped(x.B, x.F, x.T, Cp);
    WsEpi eb{};
    eb.bias = b.w.f32("b:" + p + ".att3", bbp);
    eb.act1 = WS_ACT_TANH;
    b.conv_simple(hid, att, b.w.act("w:" + p + ".att3", wbp), 1, 1, 1, 1, 0, 0, 1, 1, eb);
    if (!b.good()) return false;
    const View xv = x, yv = y, av = att, ov = out;
    const int dt = b.e.act_dt;
    const long long npos = x.npos();
    b.push([=](cudaStream_t s) {
        return ws_launch_aff_combine(xv.p, xv.ld, yv.p, yv.ld, av.p, av.ld, ov.p, (float*)ov.plo, ov.ld, dt, npos, Cp, s);
    }, "aff_combine", "{\"kind\":\"aff_combine\"," + ti("es", ws_esize(dt)) + "," + tview("x", xv) + "," + tview("y", yv) + "," + tview("t", av) + "," +
                      tview("out", ov) + "}");
    return b.good();
}

// 3x3 pad-1 conv (+ folded BN shift) -> act over `in` (Builder::conv3x3), or, when in2 != nullptr, over in + in2 with the
// weights repeated (the conv-GEMM).  act: WS_ACT_RELU20, WS_ACT_RELU or WS_ACT_NONE.  stride_t: the time stride when it
// differs from the frequency stride `stride` (0: the same)
static bool res2_conv3x3(Builder& b, const std::string& id, const View& in, const View* in2, const View& out, const std::vector<float>& w9,
                         const std::vector<float>& bias, int act, int stride, int lvl, int stride_t = 0) {   // lvl: stride level of `out` (length-masked plans)
    const int Cin = in.C, Cout = out.C, sf = stride, st = stride_t > 0 ? stride_t : stride;
    if ((int)w9.size() != Cout * 9 * Cin || (int)bias.size() != Cout) { set_err(id + ": 3x3 weight shape mismatch"); b.ok = false; return false; }
    const float* bd = b.w.f32("b:" + id, bias);
    if (in2 == nullptr) return b.conv3x3(in, out, b.w.act("w:" + id, w9), bd, act, sf, st, lvl);
    // two summed inputs: K = [9 taps over in | 9 taps over in2], weight rows repeated
    std::vector<float> w2((size_t)Cout * 18 * Cin);
    for (int o = 0; o < Cout; ++o) {
        memcpy(&w2[(size_t)o * 18 * Cin], &w9[(size_t)o * 9 * Cin], (size_t)9 * Cin * 4);
        memcpy(&w2[(size_t)o * 18 * Cin + 9 * Cin], &w9[(size_t)o * 9 * Cin], (size_t)9 * Cin * 4);
    }
    ConvSpec cs;
    cs.dt = b.e.act_dt;
    int Fo, To, F2, T2;
    const int K1 = add_conv_taps(cs, in, 3, 3, 1, 1, 1, 1, sf, st, 0, &Fo, &To);
    const int K2 = K1 < 0 ? -1 : add_conv_taps(cs, *in2, 3, 3, 1, 1, 1, 1, sf, st, K1, &F2, &T2);
    if (K1 != 9 * Cin || K2 != 9 * Cin || Fo != out.F || To != out.T || F2 != Fo || T2 != To) { set_err(id + ": summed-input conv shape mismatch"); b.ok = false; return false; }
    cs.W = b.w.act("w:" + id + ".x2", w2); cs.Ktot = 18 * Cin; cs.Cout = Cout; cs.B = out.B; cs.F = Fo; cs.T = To;
    cs.epi.bias = bd;
    cs.epi.act1 = act;
    fill_epi_out(cs.epi, out);
    b.conv(cs);
    b.zero_tail(out, lvl);
    return b.good();
}

struct Res2Bufs {   // per-stage scratch, sized for the stage's largest tensor of each kind
    View A, cat, fz, hid, att, xo[2];
};

// one residual block; kind 0 = BasicBlockRes2Net, 1 = BasicBlockERes2Net, 2 = BasicBlockERes2Net_diff_AFF
// Length-masked plans (lvl = stride level of the block's output): the rows behind an utterance's end are zeroed wherever a
// 3x3 conv is about to read across time (A after conv1, every chain output, and the stage outputs that ERes2Net's bottom-up
// fusion reads through stride-2 3x3 convs); the 1x1 convs and AFF never mix time, and AFF of two zero rows is zero.
static View res2_block(Builder& b, const Res2Cfg& c, const std::string& p, const View& x, int planes, int stride, int kind, Res2Bufs& bf, View obuf,
                       int lvl, bool zero_out_tail) {
    View none;
    const int w = (int)std::floor(planes * (c.base_width / 64.0)), wp = res2_pad(w), s = c.scale, cout = planes * c.expansion, cin = x.C;
    const int nconv = kind == 0 ? s - 1 : s;            // chain convs
    const int ncat = kind == 0 ? s - 1 : s;             // chunks of the concat buffer (Res2Net's last chunk stays in A)
    const int Fo = (x.F - 1) / stride + 1, To = (x.T - 1) / stride + 1;
    std::vector<float> s1, h1, s3, h3, w1, w3;
    if (!b.w.bn(p + ".bn1", true, s1, h1) || !b.w.bn(p + ".bn3", true, s3, h3) || !b.w.pack_conv(p + ".conv1.weight", &s1, w1) ||
        !b.w.pack_conv(p + ".conv3.weight", &s3, w3))
        return none;
    if ((int)w1.size() != s * w * cin || (int)w3.size() != cout * s * w) { set_err(p + ": conv1 / conv3 weight shape mismatch"); b.ok = false; return none; }
    const View A = bf.A.shaped(x.B, Fo, To, s * wp), cat = bf.cat.shaped(x.B, Fo, To, ncat * wp), o = obuf.shaped(x.B, Fo, To, cout);
    {   // conv1 (1x1, stride) + bn1 + Hardtanh -> the `scale` chunks of A
        std::vector<float> w1p = pad_rows(w1, s, w, wp, cin), b1p((size_t)s * wp, 0.f);
        for (int k = 0; k < s; ++k)
            for (int j = 0; j < w; ++j) b1p[(size_t)k * wp + j] = h1[(size_t)k * w + j];
        WsEpi e1{};
        e1.bias = b.w.f32("b:" + p + ".bn1", b1p);
        e1.act1 = WS_ACT_RELU20;
        b.conv_simple(x, A, b.w.act("w:" + p + ".conv1", w1p), 1, 1, 1, 1, 0, 0, stride, stride, e1);
        b.zero_tail(A, lvl);
        if (!b.good()) return none;
    }
    for (int i = 0; i < nconv; ++i) {
        const std::string ck = (kind == 2) ? (i == 0 ? p + ".conv2_1" : p + ".convs." + std::to_string(i - 1))
                                           : p + ".convs." + std::to_string(i);
        const std::string bk = (kind == 2) ? (i == 0 ? p + ".bn2_1" : p + ".bns." + std::to_string(i - 1))
                                           : p + ".bns." + std::to_string(i);
        std::vector<float> sc, sh, wc;
        int co, ci, nt;
        if (!b.w.bn(bk, true, sc, sh) || !b.w.pack_conv(ck + ".weight", &sc, wc, &co, &ci, &nt)) return none;
        if (co != w || ci != w || nt != 9) { set_err(ck + ".weight: expected (w, w, 3, 3)"); b.ok = false; return none; }
        // [w][9][w] -> [wp][9][wp]
        std::vector<float> wcp = pad_rows(pad_cols(wc, w, 9, 1, w, wp), 1, w, wp, 9 * wp), bcp(wp, 0.f);
        for (int j = 0; j < w; ++j) bcp[j] = sh[j];
        const View dst = cat.ch(i * wp, wp), spx = A.ch(i * wp, wp);
        if (i == 0) {
            if (!res2_conv3x3(b, ck, spx, nullptr, dst, wcp, bcp, WS_ACT_RELU20, 1, lvl)) return none;
        } else if (kind == 2) {
            const View fz = bf.fz.shaped(x.B, Fo, To, wp);
            if (!aff(b, p + ".fuse_models." + std::to_string(i - 1), cat.ch((i - 1) * wp, wp), spx, w, bf.hid, bf.att, fz)) return none;
            if (!res2_conv3x3(b, ck, fz, nullptr, dst, wcp, bcp, WS_ACT_RELU20, 1, lvl)) return none;
        } else {
            const View prev = cat.ch((i - 1) * wp, wp);
            if (!res2_conv3x3(b, ck, prev, &spx, dst, wcp, bcp, WS_ACT_RELU20, 1, lvl)) return none;
        }
    }
    // conv3 (1x1) + bn3 over [concat chunks | (Res2Net) last chunk of A] (+ the strided 1x1 shortcut conv as one more K range,
    // or the identity shortcut as the epilogue's residual), Hardtanh
    ConvSpec cs;
    cs.dt = b.e.act_dt;
    int F3, T3;
    int K = add_conv_taps(cs, cat, 1, 1, 1, 1, 0, 0, 1, 1, 0, &F3, &T3);
    if (kind == 0 && K >= 0) {
        const int K1 = add_conv_taps(cs, A.ch(ncat * wp, wp), 1, 1, 1, 1, 0, 0, 1, 1, K, &F3, &T3);
        K = K1 < 0 ? -1 : K + K1;
    }
    if (K != s * wp) { set_err(p + ": conv3 operand mismatch"); b.ok = false; return none; }
    std::vector<float> w3p = pad_cols(w3, cout, 1, s, w, wp), bias3 = h3;
    const bool has_sc = b.e.sd.count(p + ".shortcut.0.weight") != 0;
    if (has_sc) {
        if (!b.merge_shortcut(cs, p, x, stride, stride, o, w3p, K, bias3)) return none;
    } else {
        if (cin != cout || stride != 1) { set_err(p + ": identity shortcut with a shape change"); b.ok = false; return none; }
        cs.epi.res = x.p;
        cs.epi.res_ld = x.ld;
        cs.dense_pointwise = true;
    }
    cs.W = b.w.act("w:" + p + ".conv3m", w3p); cs.Ktot = K; cs.Cout = cout; cs.B = x.B; cs.F = Fo; cs.T = To;
    cs.epi.bias = b.w.f32("b:" + p + ".bn3m", bias3);
    cs.epi.act2 = WS_ACT_RELU20;
    fill_epi_out(cs.epi, o);
    b.conv(cs);
    if (zero_out_tail) b.zero_tail(o, lvl);   // a stage output the fusion path's stride-2 3x3 conv / AFF will read
    return b.good() ? o : none;
}

bool build_res2net(Builder& b, const Res2Cfg& c) {
    ws_engine& e = b.e;
    const int B = b.p.B, T = b.p.T, Fd = e.feat_dim, m = c.m;
    if (m != 32 && m != 64) { set_err("Res2Net / ERes2Net: m_channels must be 32 or 64"); return false; }
    View stem_buf = b.act(B, Fd, T, m);
    if (!b.good()) return false;
    View cur = stem(b, "conv1.weight", "bn1", stem_buf);   // plain ReLU (res2net.py:158, eres2net.py:358)
    if (!b.good() || cur.p == nullptr) return false;
    View stage[4];
    int stage_real[4];
    for (int li = 1; li <= 4 && b.good(); ++li) {
        const int planes = m << (li - 1), cout = planes * c.expansion;
        const int w = (int)std::floor(planes * (c.base_width / 64.0)), wp = res2_pad(w);
        const int stride = li == 1 ? 1 : 2;
        const int Fo = (cur.F - 1) / stride + 1, To = (cur.T - 1) / stride + 1;
        const int kind = !c.fuse ? 0 : (li >= 3 ? 2 : 1);
        // conv1 of the first block runs at the output resolution already (the stride is on conv1), so every scratch tensor of
        // the stage has Fo x To positions
        Res2Bufs bf;
        bf.A = b.act(B, Fo, To, c.scale * wp);
        bf.cat = b.act(B, Fo, To, c.scale * wp);
        if (kind == 2) {
            bf.fz = b.act(B, Fo, To, wp);
            bf.hid = b.act(B, Fo, To, std::max(32, (w / 4 + 31) / 32 * 32));
            bf.att = b.act(B, Fo, To, wp);
        }
        bf.xo[0] = b.act(B, Fo, To, cout);
        bf.xo[1] = b.act(B, Fo, To, cout);
        if (!b.good()) return false;
        for (int bi = 0; bi < e.num_blocks[li - 1] && b.good(); ++bi) {
            const std::string p = "layer" + std::to_string(li) + "." + std::to_string(bi);
            View o = res2_block(b, c, p, cur, planes, bi == 0 ? stride : 1, kind, bf, bf.xo[bi & 1], li - 1,
                                c.fuse && bi == e.num_blocks[li - 1] - 1);
            if (!b.good() || o.p == nullptr) return false;
            cur = o;
        }
        stage[li - 1] = cur;
        stage_real[li - 1] = cout;
    }
    if (!b.good()) return false;
    if (c.fuse) {
        // bottom-up fusion (eres2net.py:359-369): f = AFF(stage[k + 1], conv3x3_stride2(f)), f starting at stage 0
        View f = stage[0];
        const char* names[3] = {"fuse_mode12", "fuse_mode123", "fuse_mode1234"};
        for (int k = 0; k < 3 && b.good(); ++k) {
            const View& nx = stage[k + 1];
            const int C2 = stage_real[k + 1];
            const std::string dk = "layer" + std::to_string(k + 1) + "_downsample";
            std::vector<float> wd;
            int co, ci, nt;
            if (!b.w.pack_conv(dk + ".weight", nullptr, wd, &co, &ci, &nt)) return false;
            if (co != C2 || ci != f.C || nt != 9) { set_err(dk + ".weight shape mismatch"); return false; }
            View d = b.act(B, nx.F, nx.T, C2), hid = b.act(B, nx.F, nx.T, std::max(32, (C2 / 4 + 31) / 32 * 32)), att = b.act(B, nx.F, nx.T, C2),
                 fo = b.act(B, nx.F, nx.T, C2);
            if (!b.good()) return false;
            if (!res2_conv3x3(b, dk, f, nullptr, d, wd, std::vector<float>((size_t)C2, 0.f), WS_ACT_NONE, 2, k + 1)) return false;
            if (!aff(b, names[k], nx, d, C2, hid, att, fo)) return false;
            f = fo;
        }
        cur = f;
    }
    if (!b.good()) return false;
    return resnet_tail(b, cur, e.opt("two_emb_layer", 0) != 0);
}

// ----------------------------------------------------------------------------------------------- SimAM-ResNet + ASP
// samresnet.py:21-167 (SimAMBasicBlock; the ResNet trunk under `front.`), pooling_layers.py:151-204 (ASP).  A block is conv1
// (+bn1, ReLU) and conv2 (+bn2) on res2_conv3x3, the 1x1 strided downsample conv (+BN) written into the block's output
// buffer, then the SimAM statistics op and the apply op, which adds the shortcut (in place over the downsample output) and
// applies the ReLU.  The last block writes ASP's pooled frame [B][1][T'][F'*C] (feature f*C + c) directly; the ASP and
// bottleneck weights are permuted on the host from the reference's feature order c*F' + f (x.reshape(B, C*F', T')).
constexpr float kSimamLambda = 1e-4f;   // samresnet.py:65

// out = relu(SimAM(y) + res), out at element b*os.b + f*os.f + t*os.t + c (y's extents); lvl: stride level of y
static bool simam(Builder& b, const View& y, const View& res, const View& out, WsMapStrides os, float* partial, float* stats, int lvl) {
    const View yv = y, rv = res;
    void* op_ = out.p;
    float* olo = (float*)out.plo;
    const WsMapStrides rs{(long long)res.F * res.T * res.ld, (long long)res.T * res.ld, res.ld};
    const int* l = b.lens(lvl);
    const int dt = b.e.act_dt;
    b.push([=](cudaStream_t s) { return ws_launch_simam_stats(yv.p, dt, yv.B, yv.F, yv.T, yv.C, yv.ld, partial, stats, s, l); }, "simam_stats",
           "{\"kind\":\"simam_stats\"," + ti("es", ws_esize(dt)) + "," + tview("x", yv) + "," + tp("stats", stats) + "," + tp("lens", l) + tplo("partial", partial) + "}");
    b.p.extra_launches += 1;   // partials + merge
    b.push([=](cudaStream_t s) {
        return ws_launch_simam_apply(yv.p, yv.ld, stats, kSimamLambda, rv.p, rs, op_, olo, os, dt, yv.B, yv.F, yv.T, yv.C, s, l);
    }, "simam_apply", "{\"kind\":\"simam_apply\"," + ti("es", ws_esize(dt)) + "," + tview("y", yv) + "," + tp("stats", stats) + "," +
                      tview("res", rv) + "," + tp("out", op_) + "," + ti("out_sb", os.b) + "," + ti("out_sf", os.f) + "," +
                      ti("out_st", os.t) + "," + tp("lens", l) + ",\"lambda\":1e-4}");
    return b.good();
}

// one SimAMBasicBlock (samresnet.py:57-63); x lives in none of hbuf / ybuf / obuf.  frame != nullptr: the trunk's last block,
// whose output is the pooled frame (B,1,T',F'*C).  lvl: stride level of the block's output
static View simam_block(Builder& b, const std::string& p, const View& x, int cout, int s, View hbuf, View ybuf, View obuf, int lvl,
                        float* partial, float* stats, const View* frame) {
    View none;
    std::vector<float> s1, h1, s2, h2, w1, w2;
    if (!b.w.bn(p + ".bn1", true, s1, h1) || !b.w.bn(p + ".bn2", true, s2, h2) || !b.w.pack_conv(p + ".conv1.weight", &s1, w1) ||
        !b.w.pack_conv(p + ".conv2.weight", &s2, w2))
        return none;
    const int Fo = (x.F - 1) / s + 1, To = (x.T - 1) / s + 1;
    const View h = hbuf.shaped(x.B, Fo, To, cout), y = ybuf.shaped(x.B, Fo, To, cout), o = obuf.shaped(x.B, Fo, To, cout);
    if (!res2_conv3x3(b, p + ".conv1", x, nullptr, h, w1, h1, WS_ACT_RELU, s, lvl) || !res2_conv3x3(b, p + ".conv2", h, nullptr, y, w2, h2, WS_ACT_NONE, 1, lvl))
        return none;
    const bool has_ds = b.e.sd.count(p + ".downsample.0.weight") != 0;
    if (has_ds) {
        std::vector<float> ss, hs, wsv;
        int co, ci, nt;
        if (!b.w.bn(p + ".downsample.1", true, ss, hs) || !b.w.pack_conv(p + ".downsample.0.weight", &ss, wsv, &co, &ci, &nt)) return none;
        if (co != cout || ci != x.C || nt != 1) { set_err(p + ".downsample.0.weight: shape mismatch"); b.ok = false; return none; }
        WsEpi es{};
        es.bias = b.w.f32("bnh:" + p + ".downsample", hs);
        b.conv_simple(x, o, b.w.act("w:" + p + ".downsample", wsv), 1, 1, 1, 1, 0, 0, s, s, es);
        if (!b.good()) return none;
    } else if (x.C != cout || s != 1) {
        set_err(p + ": identity shortcut with a shape change"); b.ok = false; return none;
    }
    View dst = o;
    WsMapStrides os{(long long)Fo * To * cout, (long long)To * cout, cout};
    if (frame != nullptr) {
        if (frame->T != To || frame->C != Fo * cout) { set_err("internal: pooled frame shape mismatch"); b.ok = false; return none; }
        dst = *frame;
        os = WsMapStrides{(long long)To * Fo * cout, cout, (long long)Fo * cout};
    }
    if (!simam(b, y, has_ds ? o : x, dst, os, partial, stats, lvl)) return none;
    return dst;
}

bool build_simam_resnet(Builder& b) {
    ws_engine& e = b.e;
    const int B = b.p.B, T = b.p.T, Fd = e.feat_dim, E = e.embed_dim;
    const HostT* c1 = b.w.get("front.conv1.weight");
    if (c1 == nullptr) return false;
    const int m = (int)c1->shape[0];   // in_planes
    if (m != 32 && m != 64) { set_err("SimAM-ResNet: in_planes (the rows of front.conv1.weight) must be 32 or 64"); return false; }
    // every map has F * C = feat_dim * in_planes (the stride-2 layers halve F and double C): a layer-1 tensor is the largest
    const std::vector<View> bufs = b.ring(4, (size_t)B * Fd * T * m);
    int F4 = Fd, T4 = T;
    for (int i = 0; i < 3; ++i) { F4 = (F4 - 1) / 2 + 1; T4 = (T4 - 1) / 2 + 1; }
    const int C4 = 8 * m, D = F4 * C4;   // ASP feature_dim = in_planes * 8 * (acoustic_dim / 8) (pooling_layers.py:167-170)
    View frame = b.act(B, 1, T4, D);
    float* partial = b.f32((size_t)B * Fd * m * 2);
    float* sstats = b.f32((size_t)B * 2 * C4);
    if (!b.good()) return false;
    View cur = stem(b, "front.conv1.weight", "front.bn1", bufs[0]);
    if (!b.good() || cur.p == nullptr) return false;
    int ci = 0;
    for (int li = 1; li <= 4; ++li)
        for (int bi = 0; bi < e.num_blocks[li - 1]; ++bi) {
            const bool last = li == 4 && bi == e.num_blocks[3] - 1;
            View o = simam_block(b, "front.layer" + std::to_string(li) + "." + std::to_string(bi), cur, m << (li - 1), (bi == 0 && li > 1) ? 2 : 1,
                                 bufs[(ci + 1) % 4], bufs[(ci + 2) % 4], bufs[(ci + 3) % 4], li - 1, partial, sstats, last ? &frame : nullptr);
            if (!b.good() || o.p == nullptr) return false;
            ci = (ci + 3) % 4;
            cur = o;
        }
    // ASP (pooling_layers.py:180-204): attention.0 (Conv1d D -> 128, bias) -> ReLU -> attention.2 (BN) -> attention.3 (Conv1d
    // 128 -> D) -> softmax over T; mean / sqrt(clamp(var, 1e-5)); then the bottleneck Linear(2D -> E)
    const HostT* a0 = b.w.get("pooling.attention.0.weight");
    const HostT* a3 = b.w.get("pooling.attention.3.weight");
    const HostT* a3b = b.w.get("pooling.attention.3.bias");
    const HostT* bw = b.w.get("bottleneck.weight");
    std::vector<float> sa, ha;
    if (!a0 || !a3 || !a3b || !bw || !b.w.bn("pooling.attention.2", true, sa, ha)) return false;
    if (a0->numel() != 128LL * D || a3->numel() != 128LL * D || a3b->numel() != D || bw->shape.size() != 2 || (int)bw->shape[0] != E ||
        bw->shape[1] != 2LL * D) {
        set_err("SimAM-ResNet: pooling.attention / bottleneck shapes do not match in_planes * 8 * (feat_dim / 8) features");
        return false;
    }
    auto ref_of = [&](int j) { return (j % C4) * F4 + j / C4; };   // pooled feature j = f*C4 + c -> reference feature c*F4 + f
    std::vector<float> w0((size_t)128 * D), w3((size_t)D * 128), b3(D), wb((size_t)E * 2 * D);
    for (int o = 0; o < 128; ++o)
        for (int j = 0; j < D; ++j) w0[(size_t)o * D + j] = a0->v[(size_t)o * D + ref_of(j)];
    for (int j = 0; j < D; ++j) {
        memcpy(&w3[(size_t)j * 128], &a3->v[(size_t)ref_of(j) * 128], 128 * 4);
        b3[j] = a3b->v[ref_of(j)];
    }
    for (int o = 0; o < E; ++o)
        for (int j = 0; j < D; ++j) {
            wb[(size_t)o * 2 * D + j] = bw->v[(size_t)o * 2 * D + ref_of(j)];
            wb[(size_t)o * 2 * D + D + j] = bw->v[(size_t)o * 2 * D + D + ref_of(j)];
        }
    View hid = b.act(B, 1, T4, 128);
    float* stats = b.f32((size_t)B * 2 * D);
    if (!b.good()) return false;
    WsEpi ep{};   // ECAPA's conv -> relu -> bn epilogue
    ep.bias = b.w.vec("pooling.attention.0.bias");
    ep.act1 = WS_ACT_RELU;
    ep.scale = b.w.f32("bns:pooling.attention.2", sa);
    ep.shift = b.w.f32("bnh:pooling.attention.2", ha);
    b.conv_simple(frame, hid, b.w.act("w:pooling.attention.0", w0), 1, 1, 1, 1, 0, 0, 1, 1, ep);
    if (!b.astp_tail(frame, hid, b.w.act("w:pooling.attention.3", w3), b.w.f32("b:pooling.attention.3", b3), stats, 1e-5, 3)) return false;
    b.linear(stats, 2 * D, nullptr, 0, 1, b.w.f32("w:bottleneck.pooled", wb), b.w.vec("bottleneck.bias"), b.p.emb, E, B, 2 * D, E, WS_ACT_NONE);
    return b.good();
}

// ----------------------------------------------------------------------------------------------- Gemini DF-ResNet
// gemini_dfresnet.py:30-176: the stem (downsample_layers.0: 3x3 conv + BN + ReLU), four 3x3 downsample convs + BN (no ReLU)
// with frequency stride 2 and time strides (1, 2, 1, 1), each followed by a stage of inverted bottlenecks (1x1 expand to
// 4 dim + BN + ReLU, depthwise 3x3 + BN + ReLU, 1x1 project + BN, + x, ReLU), TSTP and the segment layer(s) of ResNet.
// Every BN is folded into its conv.  The expand and project convs are 1x1 conv-GEMMs (the residual and the final ReLU in
// the project conv's epilogue), the depthwise conv is its own bandwidth kernel (ws_dwconv.cu) and the downsample convs
// run on res2_conv3x3 (the halo-resident kernel where the channels allow, else the conv-GEMM).
constexpr int kGeminiStrideT[4] = {1, 2, 1, 1};   // gemini_dfresnet.py:74-75 (the frequency stride is 2 in all four)

// out = relu(depthwise 3x3(x, w9) + shift); rows behind an utterance's end read and written as zeros.  lvl: stride level of x
static bool dwconv3x3(Builder& b, const std::string& id, const View& x, const View& out, const float* w9, const float* shift, int lvl) {
    const int V = x.dt == WS_F32 ? 4 : 8;
    if (x.C % V != 0 || x.ld % V != 0 || out.ld % V != 0 || out.C != x.C || out.B != x.B || out.F != x.F || out.T != x.T) {
        set_err(id + ": the depthwise conv needs a channel count that is a multiple of " + std::to_string(V) + " (got " + std::to_string(x.C) + ")");
        b.ok = false;
        return false;
    }
    const View xv = x, ov = out;
    const int* l = b.lens(lvl);
    b.push([=](cudaStream_t s) {
        return ws_launch_dwconv3x3(xv.p, xv.ld, w9, shift, ov.p, (float*)ov.plo, ov.ld, xv.dt, xv.B, xv.F, xv.T, xv.C, s, l);
    }, "dwconv3x3", "{\"kind\":\"dwconv3x3\"," + ti("es", ws_esize(xv.dt)) + "," + tview("x", xv) + "," + tview("out", ov) + "," +
                    tp("w", w9) + "," + tp("shift", shift) + "," + tp("lens", l) + "}");
    return b.good();
}

// one Inverted_Bottleneck (gemini_dfresnet.py:30-48); x lives in none of hbuf / dbuf / obuf.  lvl: stride level of x
static View gemini_block(Builder& b, const std::string& p, const View& x, View hbuf, View dbuf, View obuf, int lvl) {
    View none;
    std::vector<float> s1, h1, s2, h2, s3, h3, w1, w3;
    int co1, ci1, nt1, co3, ci3, nt3;
    if (!b.w.bn(p + ".bn1", true, s1, h1) || !b.w.bn(p + ".bn2", true, s2, h2) || !b.w.bn(p + ".bn3", true, s3, h3) ||
        !b.w.pack_conv(p + ".conv1.weight", &s1, w1, &co1, &ci1, &nt1) || !b.w.pack_conv(p + ".conv3.weight", &s3, w3, &co3, &ci3, &nt3))
        return none;
    const HostT* c2 = b.w.get(p + ".conv2.weight");
    if (c2 == nullptr) return none;
    const int C4 = 4 * x.C;
    if (co1 != C4 || ci1 != x.C || nt1 != 1 || co3 != x.C || ci3 != C4 || nt3 != 1 || c2->shape.size() != 4 || c2->shape[0] != C4 ||
        c2->shape[1] != 1 || c2->numel() != 9LL * C4 || (int)s2.size() != C4) {
        set_err(p + ": inverted bottleneck weights do not match dim " + std::to_string(x.C));
        b.ok = false;
        return none;
    }
    std::vector<float> w2((size_t)C4 * 9);   // [C4][3][3] with bn2's scale folded in
    for (int c = 0; c < C4; ++c)
        for (int k = 0; k < 9; ++k) w2[(size_t)c * 9 + k] = c2->v[(size_t)c * 9 + k] * s2[c];
    const View h = hbuf.shaped(x.B, x.F, x.T, C4), d = dbuf.shaped(x.B, x.F, x.T, C4), o = obuf.shaped(x.B, x.F, x.T, x.C);
    WsEpi e1{};
    e1.bias = b.w.f32("bnh:" + p + ".bn1", h1);
    e1.act1 = WS_ACT_RELU;
    b.conv_simple(x, h, b.w.act("w:" + p + ".conv1", w1), 1, 1, 1, 1, 0, 0, 1, 1, e1);
    if (!b.good() || !dwconv3x3(b, p + ".conv2", h, d, b.w.f32("w:" + p + ".conv2", w2), b.w.f32("bnh:" + p + ".bn2", h2), lvl)) return none;
    WsEpi e3{};
    e3.bias = b.w.f32("bnh:" + p + ".bn3", h3);
    e3.res = x.p;
    e3.res_ld = x.ld;
    e3.act2 = WS_ACT_RELU;
    b.conv_simple(d, o, b.w.act("w:" + p + ".conv3", w3), 1, 1, 1, 1, 0, 0, 1, 1, e3);
    if (!b.good()) return none;
    return o;
}

bool build_gemini(Builder& b) {
    ws_engine& e = b.e;
    const int B = b.p.B, T = b.p.T, Fd = e.feat_dim;
    int dims[5], Fs[5], Ts[5];
    Fs[0] = Fd; Ts[0] = T;
    for (int i = 0; i < 5; ++i) {
        const std::string key = "downsample_layers." + std::to_string(i) + ".0.weight";
        const HostT* w = b.w.get(key);
        if (w == nullptr) return false;
        if (w->shape.size() != 4 || w->shape[2] != 3 || w->shape[3] != 3 || w->shape[1] != (i == 0 ? 1 : dims[i - 1])) {
            set_err(key + ": expected a (dim, previous dim, 3, 3) conv");
            return false;
        }
        dims[i] = (int)w->shape[0];
        if (i > 0) { Fs[i] = (Fs[i - 1] - 1) / 2 + 1; Ts[i] = (Ts[i - 1] - 1) / kGeminiStrideT[i - 1] + 1; }
    }
    // the reference sizes TSTP and seg_1 for stats_dim = int(feat_dim / 8 / 2) * dims[4] (gemini_dfresnet.py:62)
    if (Fs[4] != Fd / 16) {
        set_err("Gemini_DF_ResNet: feat_dim " + std::to_string(Fd) + " leaves " + std::to_string(Fs[4]) +
                " frequency rows after the four stride-2 convs, but the reference's stats_dim = int(feat_dim / 16) * " + std::to_string(dims[4]) +
                " expects " + std::to_string(Fd / 16));
        return false;
    }
    // the largest map: the stem output or a stage's 4x-expanded tensor
    size_t big = (size_t)Fd * T * dims[0];
    for (int i = 1; i <= 4; ++i) big = std::max(big, (size_t)Fs[i] * Ts[i] * 4 * dims[i]);
    const std::vector<View> bufs = b.ring(4, big * B);
    if (!b.good()) return false;
    View cur = stem(b, "downsample_layers.0.0.weight", "downsample_layers.0.1", bufs[0]);
    if (!b.good() || cur.p == nullptr) return false;
    int ci = 0;
    for (int i = 1; i <= 4; ++i) {
        const std::string p = "downsample_layers." + std::to_string(i);
        std::vector<float> s, h, w;
        if (!b.w.bn(p + ".1", true, s, h) || !b.w.pack_conv(p + ".0.weight", &s, w)) return false;
        // stride levels of length-masked plans: 0 up to downsample_layers.2 (the only time stride), 1 behind it
        const int lvl_in = i >= 3 ? 1 : 0, lvl = i >= 2 ? 1 : 0;
        if (i >= 2) b.zero_tail(cur, lvl_in);   // (masked plans) a stage output, read across time by the 3x3 conv
        const View o = bufs[(ci + 1) % 4].shaped(B, Fs[i], Ts[i], dims[i]);
        if (!res2_conv3x3(b, p + ".0", cur, nullptr, o, w, h, WS_ACT_NONE, 2, lvl, kGeminiStrideT[i - 1])) return false;
        ci = (ci + 1) % 4;
        cur = o;
        for (int j = 0; j < e.num_blocks[i - 1]; ++j) {
            View nx = gemini_block(b, "stages." + std::to_string(i - 1) + "." + std::to_string(j), cur, bufs[(ci + 1) % 4], bufs[(ci + 2) % 4],
                                   bufs[(ci + 3) % 4], lvl);
            if (!b.good() || nx.p == nullptr) return false;
            ci = (ci + 3) % 4;
            cur = nx;
        }
    }
    return resnet_tail(b, cur, e.opt("two_emb_layer", 0) != 0, 1);
}

// ----------------------------------------------------------------------------------------------- XVEC
// tdnn.py:23-117: five TdnnLayers BN(ReLU(Conv1d(x) + b)) WITHOUT padding (the sequence shrinks by 4 + 4 + 6 frames) and
// BatchNorm affine=False, TSTP, seg_1 -> ReLU -> seg_bn_1 -> seg_2; callers take the last element (embed_b).
bool build_xvec(Builder& b) {
    ws_engine& e = b.e;
    const int B = b.p.B, T = b.p.T, Fd = e.feat_dim;
    if (T < 15) { set_err("XVEC needs at least 15 frames (valid convolutions of context 5, 3x2, 3x3)"); return false; }
    if (b.p.masked) { set_err("length-masked batches are not implemented for XVEC (its valid convolutions shrink every utterance differently)"); return false; }
    const HostT* w5 = b.w.get("frame_5.conv_1d.weight");
    if (!w5) return false;
    const int sdim = (int)w5->shape[0];
    const int sdim_pad = (sdim + 31) / 32 * 32;          // tensor-core tiles want Cout % 32 == 0: zero rows behind the 1500
    View x0 = b.act(B, 1, T, Fd);
    b.convert_input(x0);
    const int ks[5] = {5, 3, 3, 1, 1}, dils[5] = {1, 2, 3, 1, 1};
    View cur = x0;
    for (int i = 1; i <= 5 && b.good(); ++i) {
        const std::string p = "frame_" + std::to_string(i);
        std::vector<float> wp, s, h;
        int co, ci, nt;
        const HostT* bias = b.w.get(p + ".conv_1d.bias");
        if (!bias || !b.w.pack_conv(p + ".conv_1d.weight", nullptr, wp, &co, &ci, &nt) || !b.w.bn(p + ".bn", false, s, h)) return false;
        const int cop = i == 5 ? sdim_pad : co;
        std::vector<float> bv(bias->v);
        if (cop != co) {   // padded output channels: zero weights, zero bias, BN scale / shift 0 -> exact zeros
            wp.resize((size_t)cop * nt * ci, 0.f);
            bv.resize(cop, 0.f); s.resize(cop, 0.f); h.resize(cop, 0.f);
        }
        const int To = cur.T - dils[i - 1] * (ks[i - 1] - 1);
        View out = b.act(B, 1, To, cop);
        WsEpi ep{};
        ep.bias = b.w.f32("b:" + p, bv);
        ep.act1 = WS_ACT_RELU;
        ep.scale = b.w.f32("bns:" + p, s);
        ep.shift = b.w.f32("bnh:" + p, h);
        b.conv_simple(cur, out, b.w.act("w:" + p, wp), 1, ks[i - 1], 1, dils[i - 1], 0, 0, 1, 1, ep);
        cur = out;
    }
    if (!b.good()) return false;
    View sv = cur; sv.C = sdim;                           // statistics over the real 1500 channels only
    return resnet_tail(b, sv, true, 0);
}

// ----------------------------------------------------------------------------------------------- CAM++
// campplus.py:282-413
bool build_campplus(Builder& b) {
    ws_engine& e = b.e;
    const int B = b.p.B, T = b.p.T, Fd = e.feat_dim, E = e.embed_dim, m = 32;
    const std::vector<View> bufs = b.ring(3, (size_t)B * Fd * T * m);
    if (!b.good()) return false;
    // FCM head (campplus.py:282-330): frequency-only striding
    View cur = stem(b, "head.conv1.weight", "head.bn1", bufs[0]);
    int ci = 0;
    for (int li = 1; li <= 2 && b.good(); ++li)
        for (int bi = 0; bi < 2 && b.good(); ++bi) {
            const std::string p = "head.layer" + std::to_string(li) + "." + std::to_string(bi);
            View o = basic_block(b, p, cur, m, bi == 0 ? 2 : 1, 1, bufs[(ci + 1) % 3], bufs[(ci + 2) % 3], 0);
            ci = (ci + 2) % 3;
            cur = o;
        }
    if (!b.good()) return false;
    const View y = bufs[(ci + 1) % 3].shaped(B, (cur.F + 2 - 3) / 2 + 1, cur.T, m);
    {
        std::vector<float> s, h, wp;
        if (!b.w.bn("head.bn2", true, s, h) || !b.w.pack_conv("head.conv2.weight", &s, wp)) return false;
        if (!b.conv3x3(cur, y, b.w.act("w:head.conv2", wp), b.w.f32("bnh:head.bn2", h), WS_ACT_RELU, 2, 1, 0)) return false;
    }
    // xvector.tdnn: Conv1d(C*F -> 128, k5, stride 2, pad 2) on the (B, C*F, T) reshape (channel = c*F + f),
    // + BN + ReLU (campplus.py:345-355).  The frequency index becomes a tap dimension (df = f), stride 2 uses
    // the two time-parity planes.
    const int Fh = y.F, Tp = (T + 4 - 5) / 2 + 1;
    const int growth = 32, bnc = 128;
    const int nl[3] = {12, 24, 16}, dil[3] = {1, 2, 2};
    int c0[3], cmax[3];
    c0[0] = 128;
    for (int i = 0; i < 3; ++i) { cmax[i] = c0[i] + nl[i] * growth; if (i < 2) c0[i + 1] = cmax[i] / 2; }
    View X[3];
    for (int i = 0; i < 3; ++i) X[i] = b.act(B, 1, Tp, cmax[i]);
    View Xf = b.act(B, 1, Tp, cmax[2] / 2);
    View scratch = b.act(B, 1, Tp, cmax[2]);
    View hid = b.act(B, 1, Tp, bnc);
    const int nseg = (Tp + 99) / 100;
    float* cmean = b.f32((size_t)B * bnc);
    float* csegm = b.f32((size_t)B * nseg * bnc);
    float* chid = b.f32((size_t)B * nseg * (bnc / 2));
    float* cgate = b.f32((size_t)B * nseg * growth);
    if (!b.good()) return false;
    {
        const HostT* tw = b.w.get("xvector.tdnn.linear.weight");
        std::vector<float> s, h;
        if (!tw || !b.w.bn("xvector.tdnn.nonlinear.batchnorm", true, s, h)) return false;
        const int co = (int)tw->shape[0], cin = (int)tw->shape[1];
        if (cin != m * Fh || tw->shape[2] != 5) { set_err("xvector.tdnn.linear.weight shape mismatch"); return false; }
        ConvSpec cs;
        cs.dt = e.act_dt;
        std::vector<float> wp((size_t)co * 5 * Fh * m);
        int tapi = 0;
        for (int kt = 0; kt < 5; ++kt) {
            const int off = kt - 2;
            const int pt = ((off % 2) + 2) % 2;
            WsSrc v = Builder::src_of(y);
            v.ptr = (const char*)y.p + (size_t)pt * y.ld * ws_esize(e.act_dt);
            if (y.plo) v.ptr_lo = (const char*)y.plo + (size_t)pt * y.ld * ws_esize(e.act_dt);
            v.T = (y.T - pt + 1) / 2;
            v.sT = y.ld * 2;
            int si = -1;
            for (int i = 0; i < cs.nsrc; ++i) if (cs.src[i].ptr == v.ptr) si = i;
            if (si < 0) { si = cs.nsrc; cs.src[cs.nsrc++] = v; }
            const int dtp = (off - pt) / 2;
            for (int f = 0; f < Fh; ++f, ++tapi) {
                cs.taps.push_back(WsTap{si, 0, dtp, f, tapi * m, m});
                for (int o = 0; o < co; ++o)
                    for (int c = 0; c < m; ++c)
                        wp[((size_t)o * 5 * Fh + tapi) * m + c] = tw->v[((size_t)o * cin + (c * Fh + f)) * 5 + kt] * s[o];
            }
        }
        cs.W = b.w.act("w:xvector.tdnn", wp); cs.Ktot = 5 * Fh * m; cs.Cout = co; cs.B = B; cs.F = 1; cs.T = Tp;
        cs.epi.bias = b.w.f32("bnh:xvector.tdnn", h);
        cs.epi.act1 = WS_ACT_RELU;
        fill_epi_out(cs.epi, X[0].ch(0, co));
        b.conv(cs);
    }
    const int dt = e.act_dt;
    // Fused dense layers (ws_cam_dense.cu): one launch per CAMDenseTDNNLayer (or per block with cam_block = 1) instead of four
    const bool cam_fused = e.use_tc >= 2 && e.act_dt != WS_F32 && e.opt("cam_fused", 1) != 0 && Tp <= 512;
    for (int bl = 0; bl < 3 && b.good(); ++bl) {
        bool fused_done = false;
        if (cam_fused) {
            std::vector<WsCamLayer> hl((size_t)nl[bl]);
            std::vector<std::string> hl_trace((size_t)nl[bl]);   // plan-check engines: what each layer descriptor points at
            bool okl = true;
            for (int j = 1; j <= nl[bl] && okl; ++j) {
                const std::string p = "xvector.block" + std::to_string(bl + 1) + ".tdnnd" + std::to_string(j);
                const int cin = c0[bl] + (j - 1) * growth;
                std::vector<float> s1, h1, s2, h2, w1, wl;
                const HostT* c1w = b.w.get(p + ".cam_layer.linear1.weight");
                const HostT* c2w = b.w.get(p + ".cam_layer.linear2.weight");
                okl = c1w && c2w && b.w.bn(p + ".nonlinear1.batchnorm", true, s1, h1) && b.w.bn(p + ".nonlinear2.batchnorm", true, s2, h2) &&
                      b.w.pack_conv(p + ".linear1.weight", &s2, w1) && b.w.pack_conv(p + ".cam_layer.linear_local.weight", nullptr, wl);
                if (!okl) break;
                std::vector<float> w1ct((size_t)bnc * (bnc / 2)), w2ct((size_t)(bnc / 2) * growth);
                for (int o = 0; o < bnc / 2; ++o)
                    for (int c = 0; c < bnc; ++c) w1ct[(size_t)c * (bnc / 2) + o] = c1w->v[(size_t)o * bnc + c];
                for (int g = 0; g < growth; ++g)
                    for (int o = 0; o < bnc / 2; ++o) w2ct[(size_t)o * growth + g] = c2w->v[(size_t)g * (bnc / 2) + o];
                const void* W1d = b.w.act("w:" + p + ".linear1", w1);
                const void* Wld = b.w.act("w:" + p + ".local", wl);
                const float* s1d = b.w.f32("bns:" + p + ".n1", s1);
                const float* h1d = b.w.f32("bnh:" + p + ".n1", h1);
                const float* h2d = b.w.f32("bnh:" + p + ".n2", h2);
                const float* w1cd = b.w.f32("w1ct:" + p, w1ct);
                const float* b1cd = b.w.vec(p + ".cam_layer.linear1.bias");
                const float* w2cd = b.w.f32("w2ct:" + p, w2ct);
                const float* b2cd = b.w.vec(p + ".cam_layer.linear2.bias");
                okl = cam_layer_fill(&hl[(size_t)j - 1], e.act_dt, W1d, Wld, s1d, h1d, h2d, w1cd, b1cd, w2cd, b2cd, cin, dil[bl]);
                if (plan_trace_mode())
                    hl_trace[(size_t)j - 1] = "{" + tp("W1", W1d) + "," + tp("Wl", Wld) + "," + tp("bn1_scale", s1d) + "," + tp("bn1_shift", h1d) +
                                              "," + tp("bias2", h2d) + "," + tp("w1c_t", w1cd) + "," + tp("b1c", b1cd) + "," + tp("w2c_t", w2cd) + "," +
                                              tp("b2c", b2cd) + "," + ti("cin", cin) + "," + ti("dil", dil[bl]) + "}";
            }
            if (!okl || !b.good()) { b.ok = false; break; }
            const WsCamLayer* ldev = (const WsCamLayer*)b.w.upload("camlayers:" + std::to_string(bl), hl.data(), hl.size() * sizeof(WsCamLayer));
            if (!b.good()) break;
            const bool whole = e.opt("cam_block", 1) != 0;
            fused_done = true;
            for (int j = 0; j < nl[bl]; j += whole ? nl[bl] : 1) {
                const int j1 = whole ? nl[bl] : j + 1;
                PlanOp op;
                bool unsupported = false;
                if (make_cam_dense_op(X[bl], ldev, j, j1, &op, &unsupported, b.lens(1))) {
                    if (plan_trace_mode()) {   // semantic description of the fused launch: layers [j, j1) over the concat buffer
                        op.trace = "{\"kind\":\"cam_dense\"," + ti("es", ws_esize(e.act_dt)) + "," + tview("X", X[bl]) + "," + tp("lens", b.lens(1)) + "," +
                                   ti("seg_len", 100) + ",\"layers\":[";
                        for (int k = j; k < j1; ++k) op.trace += std::string(k > j ? "," : "") + hl_trace[(size_t)k];
                        op.trace += "]}";
                    }
                    b.push(std::move(op));
                }
                else if (unsupported && j == 0) { fused_done = false; break; }
                else { b.ok = false; break; }
            }
            if (!b.good()) break;
        }
        if (!fused_done && b.p.masked) { set_err("length-masked CAM++ plans need the fused dense-layer kernel (16-bit precision, T' <= 512)"); return false; }
        for (int j = 1; j <= nl[bl] && b.good() && !fused_done; ++j) {
            const std::string p = "xvector.block" + std::to_string(bl + 1) + ".tdnnd" + std::to_string(j);
            const int cin = c0[bl] + (j - 1) * growth;
            std::vector<float> s1, h1, s2, h2, w1, wl;
            if (!b.w.bn(p + ".nonlinear1.batchnorm", true, s1, h1) || !b.w.bn(p + ".nonlinear2.batchnorm", true, s2, h2) ||
                !b.w.pack_conv(p + ".linear1.weight", &s2, w1) || !b.w.pack_conv(p + ".cam_layer.linear_local.weight", nullptr, wl))
                break;
            // nonlinear1 (BN-ReLU on the growing concat) -> scratch
            const View sv = scratch.shaped(B, 1, Tp, cin);
            b.bnrelu(X[bl].ch(0, cin), b.w.f32("bns:" + p + ".n1", s1), b.w.f32("bnh:" + p + ".n1", h1), sv);
            // linear1 (1x1, no bias) + nonlinear2 (BN folded) + ReLU -> hid
            WsEpi e1{};
            e1.bias = b.w.f32("bnh:" + p + ".n2", h2);
            e1.act1 = WS_ACT_RELU;
            b.conv_simple(sv, hid, b.w.act("w:" + p + ".linear1", w1), 1, 1, 1, 1, 0, 0, 1, 1, e1);
            // CAM context mask (campplus.py:108-115): sigmoid(W2 relu(W1 (mean_T + segmean_100)))
            View hv = hid;
            {
                const float* w1c = b.w.vec(p + ".cam_layer.linear1.weight");
                const float* b1c = b.w.vec(p + ".cam_layer.linear1.bias");
                const float* w2c = b.w.vec(p + ".cam_layer.linear2.weight");
                const float* b2c = b.w.vec(p + ".cam_layer.linear2.bias");
                const size_t cam_smem = (size_t)((bnc / 2) * bnc + nseg * bnc + 16 * bnc + nseg * (bnc / 2) + bnc) * 4;
                if (cam_smem <= 48 * 1024) {
                    b.push([=](cudaStream_t st) {
                        return ws_launch_cam_gate(hv.p, dt, B, Tp, bnc, hv.ld, 100, w1c, b1c, w2c, b2c, bnc / 2, growth, cgate, st);
                    }, "cam_gate", "{\"kind\":\"cam_gate\"," + ti("es", ws_esize(dt)) + "," + tview("x", hv) + "," + ti("seg_len", 100) + "," + tp("W1", w1c) + "," +
                                   tp("b1", b1c) + "," + tp("W2", w2c) + "," + tp("b2", b2c) + "," + ti("H", bnc / 2) + "," + ti("G", growth) + "," +
                                   tp("gate", cgate) + "}");
                } else {  // very long utterances: unfused path
                    b.push([=](cudaStream_t st) { return ws_launch_seg_means(hv.p, dt, B, Tp, bnc, hv.ld, 100, cmean, csegm, st); }, "seg_means",
                           "{\"kind\":\"seg_means\"," + ti("es", ws_esize(dt)) + "," + tview("x", hv) + "," + ti("seg_len", 100) + "," + tp("mean", cmean) + "," +
                           tp("segmean", csegm) + "}");
                    b.linear(csegm, bnc, cmean, bnc, nseg, w1c, b1c, chid, bnc / 2, B * nseg, bnc, bnc / 2, WS_ACT_RELU);
                    b.linear(chid, bnc / 2, nullptr, 0, 1, w2c, b2c, cgate, growth, B * nseg, bnc / 2, growth, WS_ACT_SIGMOID);
                }
            }
            // linear_local (k3, dilated, no bias) * mask -> appended to the concat buffer
            WsEpi e2{};
            e2.gate = cgate; e2.gate_ld = growth; e2.gate_seg = 100; e2.gate_nseg = nseg;
            b.conv_simple(hid, X[bl].ch(cin, growth), b.w.act("w:" + p + ".local", wl), 1, 3, 1, dil[bl], 0, dil[bl], 1, 1, e2);
        }
        if (!b.good()) break;
        // TransitLayer (campplus.py:204-218): BN-ReLU-Conv1x1 (no bias)
        const std::string tk = "xvector.transit" + std::to_string(bl + 1);
        std::vector<float> s, h, wt;
        if (!b.w.bn(tk + ".nonlinear.batchnorm", true, s, h) || !b.w.pack_conv(tk + ".linear.weight", nullptr, wt)) break;
        const View sv = scratch.shaped(B, 1, Tp, cmax[bl]);
        b.bnrelu(X[bl], b.w.f32("bns:" + tk, s), b.w.f32("bnh:" + tk, h), sv);
        WsEpi et{};
        View dst = (bl < 2) ? X[bl + 1].ch(0, cmax[bl] / 2) : Xf;
        b.conv_simple(sv, dst, b.w.act("w:" + tk, wt), 1, 1, 1, 1, 0, 0, 1, 1, et);
    }
    if (!b.good()) return false;
    {   // out_nonlinear (BN-ReLU) fused into TSTP; dense (1024 -> E, no bias) + BN(affine=False) folded
        std::vector<float> s, h, sdn, hdn;
        const int cf = Xf.C;
        if (!b.w.bn("xvector.out_nonlinear.batchnorm", true, s, h) || !b.w.bn("xvector.dense.nonlinear.batchnorm", false, sdn, hdn)) return false;
        float* stats = b.f32((size_t)B * 2 * cf);
        b.tstats(Xf, b.w.f32("bns:out_nl", s), b.w.f32("bnh:out_nl", h), stats, 2 * cf, cf, 1);
        const HostT* dw = b.w.get("xvector.dense.linear.weight");
        if (!dw) return false;
        if ((int)dw->shape[0] != E || (int)dw->shape[1] != 2 * cf) { set_err("xvector.dense.linear.weight shape mismatch"); return false; }
        std::vector<float> wf((size_t)E * 2 * cf);
        for (int o = 0; o < E; ++o)
            for (int i = 0; i < 2 * cf; ++i) wf[(size_t)o * 2 * cf + i] = dw->v[(size_t)o * 2 * cf + i] * sdn[o];
        b.linear(stats, 2 * cf, nullptr, 0, 1, b.w.f32("w:dense.folded", wf), b.w.f32("b:dense.folded", hdn), b.p.emb, E, B, 2 * cf, E, WS_ACT_NONE);
    }
    return b.good();
}

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
    PlanTraceScope trace_scope(e->plan_check || e->opt("plan_trace", 0) != 0);
    Builder b(*e, *p);
    if (masked) {
        p->lens = (int*)b.raw((size_t)4 * B * sizeof(int));
        int* l = p->lens;
        if (b.good()) {
            b.push([=](cudaStream_t s) { return ws_launch_lens_derive(l, B, T, 4, s); }, "lens_derive",
                   "{\"kind\":\"lens_derive\"," + tp("lens", l) + "," + ti("B", B) + "," + ti("T", T) + "," + ti("levels", 4) + "}");
        }
    }
    p->feats_in = b.f32((size_t)B * T * e->feat_dim);
    p->emb = b.f32((size_t)B * e->embed_dim);
    bool ok = b.good();
    if (ok) {
        if (e->model.rfind("ECAPA", 0) == 0) ok = build_ecapa(b);
        else if (e->model.rfind("ResNet", 0) == 0) ok = build_resnet(b);
        else if (e->model == "XVEC") ok = build_xvec(b);
        else if (e->model.rfind("SimAM_ResNet", 0) == 0) ok = build_simam_resnet(b);
        else if (e->model.rfind("Gemini_DF_ResNet", 0) == 0) ok = build_gemini(b);
        else if (e->r2_m != 0) {
            Res2Cfg c;
            c.m = e->r2_m; c.base_width = e->r2_base_width; c.scale = e->r2_scale; c.expansion = e->r2_expansion; c.fuse = e->r2_fuse;
            ok = build_res2net(b, c);
        }
        else ok = build_campplus(b);
    }
    if (!ok) return nullptr;
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
    p->lane = e->opt("plan_lanes", 1) ? (e->next_lane++ % ws_engine::kLanes) : 0;
    if (!e->plan_check && cudaEventCreateWithFlags(&p->done, cudaEventDisableTiming) != cudaSuccess) { set_err("plan event creation failed"); return nullptr; }
    Plan* raw = p.get();
    e->plans[key] = std::move(p);
    return raw;
}

int run_plan(ws_engine* e, Plan* p, cudaStream_t s) {
    const bool want_graph = e->opt("cuda_graph", 1) != 0 && !p->graph_failed;
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
    e->last_launches = (long long)p->ops.size() + p->extra_launches;
    return 0;
}

const FbankTables* fbank_tables(ws_engine* e, const char* window_type) {
    const std::string wt = window_type ? window_type : "hamming";
    auto it = e->fb.find(wt);
    if (it != e->fb.end()) return &it->second;
    std::vector<float> win(400);
    for (int j = 0; j < 400; ++j) {
        const double c = std::cos(2.0 * M_PI * j / 399.0);
        if (wt == "hamming") win[j] = (float)(0.54 - 0.46 * c);
        else if (wt == "povey") win[j] = (float)std::pow(0.5 - 0.5 * c, 0.85);
        else if (wt == "hanning") win[j] = (float)(0.5 - 0.5 * c);
        else if (wt == "rectangular") win[j] = 1.f;
        else { set_err("unknown window_type " + wt); return nullptr; }
    }
    // torchaudio kaldi.py get_mel_banks (80 bins, 20 Hz .. Nyquist, padded 512) in float32 like the reference
    const int nb = 80, nfft = 256;
    const double mel_low = 1127.0 * std::log(1.0 + 20.0 / 700.0), mel_high = 1127.0 * std::log(1.0 + 8000.0 / 700.0);
    const float delta = (float)((mel_high - mel_low) / (nb + 1)), lowf = (float)mel_low;
    std::vector<std::vector<float>> rows(nb, std::vector<float>(nfft, 0.f));
    std::vector<int> start(nb, 0), len(nb, 0);
    int maxlen = 1;
    for (int m = 0; m < nb; ++m) {
        const float left = lowf + (float)m * delta, center = lowf + ((float)m + 1.0f) * delta, right = lowf + ((float)m + 2.0f) * delta;
        int first = -1, last = -1;
        for (int k = 0; k < nfft; ++k) {
            const float mel = 1127.0f * std::log(1.0f + (31.25f * (float)k) / 700.0f);
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
    t.maxlen = maxlen;
    if (cudaMalloc(&t.window, 400 * 4) != cudaSuccess || cudaMalloc(&t.melw, melw.size() * 4) != cudaSuccess ||
        cudaMalloc(&t.melstart, nb * 4) != cudaSuccess || cudaMalloc(&t.mellen, nb * 4) != cudaSuccess) {
        set_err("fbank tables: cudaMalloc failed");
        return nullptr;
    }
    cudaMemcpy(t.window, win.data(), 400 * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(t.melw, melw.data(), melw.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(t.melstart, start.data(), nb * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(t.mellen, len.data(), nb * 4, cudaMemcpyHostToDevice);
    e->fb[wt] = t;
    return &e->fb[wt];
}

// engine-less fbank tables for ws_fbank()
ws_engine* fbank_holder(int device) {
    static std::map<int, ws_engine*> holders;
    auto it = holders.find(device);
    if (it != holders.end()) return it->second;
    ws_engine* h = new ws_engine();
    h->device = device;
    holders[device] = h;
    return h;
}

cudaStream_t lane_stream(ws_engine* e, const Plan* p) { return e->lanes[p->lane] ? e->lanes[p->lane] : e->st; }
// the plan's buffers were last used on some stream: order this use behind it, and the user's stream in front
int enter_stream(ws_engine* e, Plan* p, cudaStream_t work, cudaStream_t user) {
    WS_CK(cudaEventRecord(e->ev_in, user));
    WS_CK(cudaStreamWaitEvent(work, e->ev_in, 0));
    WS_CK(cudaStreamWaitEvent(work, p->done, 0));
    return 0;
}
int leave_stream(ws_engine* e, Plan* p, cudaStream_t work, cudaStream_t user) {
    WS_CK(cudaEventRecord(p->done, work));
    WS_CK(cudaStreamWaitEvent(user, p->done, 0));
    return 0;
}
int host_path_enter(ws_engine* e, Plan* p) { WS_CK(cudaStreamWaitEvent(e->st, p->done, 0)); return 0; }
int host_path_leave(ws_engine* e, Plan* p) { WS_CK(cudaEventRecord(p->done, e->st)); return 0; }

}  // namespace

// ================================================================================================= C ABI
// why a compute entry point cannot run on this engine (nullptr = it can)
static const char* not_runnable(const ws_engine* e) {
    if (e->plan_check) return " on a plan-check engine (it builds launch plans without a device and never computes)";
    if (!e->finalized) return " before ws_engine_finalize";
    return nullptr;
}

extern "C" {

// model name + precision -> engine configuration (shared by ws_engine_create and ws_engine_create_plan_check)
static int configure_engine(ws_engine* e, const char* model_name, const char* precision, int feat_dim, int embed_dim, int device) {
    e->model = model_name; e->prec = precision; e->feat_dim = feat_dim; e->embed_dim = embed_dim; e->device = device;
    const std::string m = e->model;
    if (m == "ECAPA_TDNN_c512") { e->channels = 512; e->glob = false; }
    else if (m == "ECAPA_TDNN_GLOB_c512") { e->channels = 512; e->glob = true; }
    else if (m == "ECAPA_TDNN_c1024") { e->channels = 1024; e->glob = false; }
    else if (m == "ECAPA_TDNN_GLOB_c1024") { e->channels = 1024; e->glob = true; }
    else if (m == "ResNet18") e->num_blocks = {2, 2, 2, 2};
    else if (m == "ResNet34") e->num_blocks = {3, 4, 6, 3};
    else if (m == "ResNet50") { e->num_blocks = {3, 4, 6, 3}; e->bottleneck = true; }
    else if (m == "ResNet101") { e->num_blocks = {3, 4, 23, 3}; e->bottleneck = true; }
    else if (m == "ResNet152") { e->num_blocks = {3, 8, 36, 3}; e->bottleneck = true; }
    else if (m == "ResNet221") { e->num_blocks = {6, 16, 48, 3}; e->bottleneck = true; }
    else if (m == "ResNet293") { e->num_blocks = {10, 20, 64, 3}; e->bottleneck = true; }
    else if (m == "XVEC") {}
    else if (m == "Res2Net34_Base") { e->num_blocks = {3, 4, 6, 3}; e->r2_m = 32; }
    else if (m == "Res2Net34_Large") { e->num_blocks = {3, 4, 6, 3}; e->r2_m = 64; }
    else if (m == "ERes2Net34_Base") { e->num_blocks = {3, 4, 6, 3}; e->r2_m = 32; e->r2_fuse = true; }
    else if (m == "ERes2Net34_Large") { e->num_blocks = {3, 4, 6, 3}; e->r2_m = 64; e->r2_fuse = true; }
    else if (m == "ERes2Net34_aug") { e->num_blocks = {3, 4, 6, 3}; e->r2_m = 64; e->r2_fuse = true; e->r2_base_width = 24; e->r2_scale = 3; e->r2_expansion = 4; }
    else if (m == "CAMPPlus") {}
    else if (m == "SimAM_ResNet34_ASP") e->num_blocks = {3, 4, 6, 3};
    else if (m == "SimAM_ResNet100_ASP") e->num_blocks = {6, 16, 24, 3};
    else if (m == "Gemini_DF_ResNet60") e->num_blocks = {3, 3, 9, 3};
    else if (m == "Gemini_DF_ResNet114") e->num_blocks = {3, 3, 27, 3};
    else if (m == "Gemini_DF_ResNet183") e->num_blocks = {3, 8, 45, 3};
    else if (m == "Gemini_DF_ResNet237") e->num_blocks = {3, 8, 63, 3};
    else { set_err("unknown / out-of-scope model name: " + m); return 1; }
    const std::string p = e->prec;
    if (p == "fp32") { e->act_dt = WS_F32; e->use_tc = 0; }
    else if (p == "tf32") { e->act_dt = WS_F32; e->use_tc = 3; }
    else if (p == "tf32x3") { e->act_dt = WS_F32; e->use_tc = 3; e->split = true; }
    else if (p == "bf16") { e->act_dt = WS_BF16; e->use_tc = 3; }
    else if (p == "fp16") { e->act_dt = WS_F16; e->use_tc = 3; }
    else { set_err("unknown precision (fp32|tf32x3|tf32|bf16|fp16): " + p); return 1; }
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
    std::unique_ptr<ws_engine> e(new ws_engine());
    if (configure_engine(e.get(), model_name, precision, feat_dim, embed_dim, device)) return 1;
    WS_CKS(ws_tc2_init());
    WS_CKS(ws_res2_init());
    WS_CKS(ws_astp_init());
    WS_CKS(ws_tc3_init());
    WS_CKS(ws_c3_init());
    WS_CKS(ws_cam_init());
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
    const std::string k = key;
    if (k == "force_simt") { if (value) e->use_tc = 0; }
    else if (k == "tc_version") {
        if (value != 2 && value != 3) {
            set_err("tc_version must be 2 (persistent tensor-core kernel) or 3 (+ weight-sharing clusters); 1, the one-tile-per-CTA "
                    "kernel, was removed");
            return 1;
        }
        if (e->use_tc) e->use_tc = (int)value;
    }
    else if (k != "two_emb_layer" && k != "emb_bn" && k != "cuda_graph" && k != "res2_fused" && k != "se_fused" && k != "se_colsum" && k != "conv3x3" && k != "cam_fused" && k != "cam_block" && k != "plan_lanes" && k != "conv3x3_strided" && k != "astp_fused" && k != "plan_trace") { set_err("unknown option " + k); return 1; }
    e->opts[k] = value;
    e->plans.clear();
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
    if (!e->plan_check) WS_CK(cudaSetDevice(e->device));
    // Build (and drop) a nominal plan: this packs/folds/uploads every weight and reports missing keys.
    Plan* p = get_plan(e, 1, 200);
    if (p == nullptr) return 1;
    e->plans.clear();
    e->finalized = true;
    return 0;
}

int ws_engine_embed_dim(const ws_engine* e) { return e ? e->embed_dim : -1; }
long long ws_engine_last_launches(const ws_engine* e) { return e ? e->last_launches : -1; }

static int forward_impl(ws_engine* e, const float* feats_dev, int B, int T, float* embs_dev, void* stream, bool join);
int ws_engine_forward(ws_engine* e, const float* feats_dev, int B, int T, float* embs_dev, void* stream) {
    return forward_impl(e, feats_dev, B, T, embs_dev, stream, true);
}
int ws_engine_forward_async(ws_engine* e, const float* feats_dev, int B, int T, float* embs_dev, void* stream) {
    return forward_impl(e, feats_dev, B, T, embs_dev, stream, false);
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
static int forward_impl(ws_engine* e, const float* feats_dev, int B, int T, float* embs_dev, void* stream, bool join) {
    if (!e || !feats_dev || !embs_dev) { set_err("ws_engine_forward: null argument"); return 1; }
    if (const char* nr = not_runnable(e)) { set_err(std::string("ws_engine_forward") + nr); return 1; }
    WS_CK(cudaSetDevice(e->device));
    Plan* p = get_plan(e, B, T);
    if (!p) return 1;
    cudaStream_t us = (cudaStream_t)stream, ws = lane_stream(e, p);
    if (enter_stream(e, p, ws, us)) return 1;
    WS_CK(cudaMemcpyAsync(p->feats_in, feats_dev, (size_t)B * T * e->feat_dim * 4, cudaMemcpyDeviceToDevice, ws));
    if (run_plan(e, p, ws)) return 1;
    WS_CK(cudaMemcpyAsync(embs_dev, p->emb, (size_t)B * e->embed_dim * 4, cudaMemcpyDeviceToDevice, ws));
    if (!join) { WS_CK(cudaEventRecord(p->done, ws)); return 0; }
    return leave_stream(e, p, ws, us);
}

// Length-masked batches: utterances of different lengths padded to a common T run as ONE batch and produce what each
// utterance produces alone (the reference has no masking, extract_vox.sh:31 runs test sets at batch 1): rows behind an
// utterance's end are kept zero wherever a convolution reads across time, and SE / ASTP / TSTP / CAM++ context statistics
// use the utterance's own frame count.  n_frames_dev: int32[B] on the device; feats rows t >= n_frames[b] are ignored.
int ws_engine_forward_masked(ws_engine* e, const float* feats_dev, const int* n_frames_dev, int B, int T, float* embs_dev,
                             void* stream) {
    if (!e || !feats_dev || !n_frames_dev || !embs_dev) { set_err("ws_engine_forward_masked: null argument"); return 1; }
    if (const char* nr = not_runnable(e)) { set_err(std::string("ws_engine_forward_masked") + nr); return 1; }
    WS_CK(cudaSetDevice(e->device));
    Plan* p = get_plan(e, B, T, true);
    if (!p) return 1;
    cudaStream_t us = (cudaStream_t)stream, ws = lane_stream(e, p);
    if (enter_stream(e, p, ws, us)) return 1;
    WS_CK(cudaMemcpyAsync(p->lens, n_frames_dev, (size_t)B * sizeof(int), cudaMemcpyDeviceToDevice, ws));
    WS_CK(cudaMemcpyAsync(p->feats_in, feats_dev, (size_t)B * T * e->feat_dim * 4, cudaMemcpyDeviceToDevice, ws));
    if (run_plan(e, p, ws)) return 1;
    WS_CK(cudaMemcpyAsync(embs_dev, p->emb, (size_t)B * e->embed_dim * 4, cudaMemcpyDeviceToDevice, ws));
    return leave_stream(e, p, ws, us);
}

// Same from padded waveforms: wav_dev [B][wav_ld] with n_samples_dev[b] valid samples each (max_samples = the longest);
// fbank of the padded rows, CMN over each utterance's own frames, masked forward.
// Length-masked extraction from waveforms.  Rectangular layout: utterance b at wav + b * wav_ld (offsets_dev == nullptr);
// ragged layout: utterance b at wav + offsets_dev[b] samples (concatenated PCM, no padding copies).  Frames behind an
// utterance's end are neither read nor computed.
static int extract_wav_masked_impl(ws_engine* e, const void* wav_dev, int wav_is_i16, long long wav_ld, const long long* offsets_dev,
                                   const int* n_samples_dev, int max_samples, int B, const char* window_type, float* embs_dev,
                                   void* stream, bool join, const char* who) {
    if (!e || !wav_dev || !n_samples_dev || !embs_dev) { set_err(std::string(who) + ": null argument"); return 1; }
    if (const char* nr = not_runnable(e)) { set_err(std::string(who) + nr); return 1; }
    if (e->feat_dim != 80) { set_err(std::string(who) + ": the fbank frontend produces 80 bins"); return 1; }
    WS_CK(cudaSetDevice(e->device));
    const int T = ws_fbank_num_frames(max_samples);
    if (T <= 0) { set_err(std::string(who) + ": waveforms shorter than one 25 ms frame"); return 1; }
    Plan* p = get_plan(e, B, T, true);
    if (!p) return 1;
    const FbankTables* t = fbank_tables(e, window_type);
    if (!t) return 1;
    cudaStream_t us = (cudaStream_t)stream, ws = lane_stream(e, p);
    if (enter_stream(e, p, ws, us)) return 1;
    WS_CKS(ws_launch_frames_from_samples(n_samples_dev, p->lens, B, T, ws));
    WS_CKS(ws_launch_fbank(wav_dev, wav_is_i16, wav_ld, max_samples, B, T, t->window, t->melw, t->melstart, t->mellen, t->maxlen,
                           p->feats_in, ws, offsets_dev, p->lens));
    WS_CKS(ws_launch_cmn(p->feats_in, B, T, 80, ws, p->lens));
    if (run_plan(e, p, ws)) return 1;
    e->last_launches += 3;
    WS_CK(cudaMemcpyAsync(embs_dev, p->emb, (size_t)B * e->embed_dim * 4, cudaMemcpyDeviceToDevice, ws));
    if (!join) { WS_CK(cudaEventRecord(p->done, ws)); return 0; }
    return leave_stream(e, p, ws, us);
}
int ws_engine_extract_wav_masked(ws_engine* e, const void* wav_dev, int wav_is_i16, long long wav_ld, const int* n_samples_dev,
                                 int max_samples, int B, const char* window_type, float* embs_dev, void* stream) {
    return extract_wav_masked_impl(e, wav_dev, wav_is_i16, wav_ld, nullptr, n_samples_dev, max_samples, B, window_type, embs_dev,
                                   stream, true, "ws_engine_extract_wav_masked");
}
int ws_engine_extract_wav_ragged(ws_engine* e, const void* wav_dev, int wav_is_i16, const long long* offsets_dev,
                                 const int* n_samples_dev, int max_samples, int B, const char* window_type, float* embs_dev,
                                 void* stream) {
    if (!offsets_dev) { set_err("ws_engine_extract_wav_ragged: null argument"); return 1; }
    return extract_wav_masked_impl(e, wav_dev, wav_is_i16, 0, offsets_dev, n_samples_dev, max_samples, B, window_type, embs_dev,
                                   stream, true, "ws_engine_extract_wav_ragged");
}
int ws_engine_extract_wav_ragged_async(ws_engine* e, const void* wav_dev, int wav_is_i16, const long long* offsets_dev,
                                       const int* n_samples_dev, int max_samples, int B, const char* window_type,
                                       float* embs_dev, void* stream) {
    if (!offsets_dev) { set_err("ws_engine_extract_wav_ragged_async: null argument"); return 1; }
    return extract_wav_masked_impl(e, wav_dev, wav_is_i16, 0, offsets_dev, n_samples_dev, max_samples, B, window_type, embs_dev,
                                   stream, false, "ws_engine_extract_wav_ragged_async");
}

int ws_engine_forward_host(ws_engine* e, const float* feats_host, int B, int T, float* embs_host) {
    if (!e || !feats_host || !embs_host) { set_err("ws_engine_forward_host: null argument"); return 1; }
    if (const char* nr = not_runnable(e)) { set_err(std::string("ws_engine_forward_host") + nr); return 1; }
    WS_CK(cudaSetDevice(e->device));
    Plan* p = get_plan(e, B, T);
    if (!p) return 1;
    if (host_path_enter(e, p)) return 1;
    WS_CK(cudaMemcpyAsync(p->feats_in, feats_host, (size_t)B * T * e->feat_dim * 4, cudaMemcpyHostToDevice, e->st));
    if (run_plan(e, p, e->st)) return 1;
    WS_CK(cudaMemcpyAsync(embs_host, p->emb, (size_t)B * e->embed_dim * 4, cudaMemcpyDeviceToHost, e->st));
    if (host_path_leave(e, p)) return 1;
    WS_CK(cudaStreamSynchronize(e->st));
    return 0;
}

int ws_fbank_num_frames(int nsamples) { return nsamples < 400 ? 0 : 1 + (nsamples - 400) / 160; }

static int fbank_into(ws_engine* e, const void* wav_dev, int is_i16, long long wav_ld, int nsamples, int B,
                      const char* window_type, int apply_cmn, float* feats, cudaStream_t s) {
    const FbankTables* t = fbank_tables(e, window_type);
    if (!t) return 1;
    const int T = ws_fbank_num_frames(nsamples);
    WS_CKS(ws_launch_fbank(wav_dev, is_i16, wav_ld, nsamples, B, T, t->window, t->melw, t->melstart, t->mellen, t->maxlen, feats, s));
    if (apply_cmn) WS_CKS(ws_launch_cmn(feats, B, T, 80, s));
    return 0;
}

int ws_fbank(const void* wav_dev, int wav_is_i16, long long wav_ld, int nsamples, int B, const char* window_type,
             int apply_cmn, float* feats_dev, void* stream) {
    if (!wav_dev || !feats_dev) { set_err("ws_fbank: null argument"); return 1; }
    int dev = 0;
    WS_CK(cudaGetDevice(&dev));
    return fbank_into(fbank_holder(dev), wav_dev, wav_is_i16, wav_ld, nsamples, B, window_type, apply_cmn, feats_dev,
                      (cudaStream_t)stream);
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
                            const char* window_type, float* embs_dev, float* feats_out_dev, void* stream, bool join);
int ws_engine_extract_wav(ws_engine* e, const void* wav_dev, int wav_is_i16, long long wav_ld, int nsamples, int B,
                          const char* window_type, float* embs_dev, float* feats_out_dev, void* stream) {
    return extract_wav_impl(e, wav_dev, wav_is_i16, wav_ld, nsamples, B, window_type, embs_dev, feats_out_dev, stream, true);
}
int ws_engine_extract_wav_async(ws_engine* e, const void* wav_dev, int wav_is_i16, long long wav_ld, int nsamples, int B,
                                const char* window_type, float* embs_dev, void* stream) {
    return extract_wav_impl(e, wav_dev, wav_is_i16, wav_ld, nsamples, B, window_type, embs_dev, nullptr, stream, false);
}
static int extract_wav_impl(ws_engine* e, const void* wav_dev, int wav_is_i16, long long wav_ld, int nsamples, int B,
                            const char* window_type, float* embs_dev, float* feats_out_dev, void* stream, bool join) {
    if (!e || !wav_dev || !embs_dev) { set_err("ws_engine_extract_wav: null argument"); return 1; }
    if (const char* nr = not_runnable(e)) { set_err(std::string("ws_engine_extract_wav") + nr); return 1; }
    if (e->feat_dim != 80) { set_err("ws_engine_extract_wav: the fbank frontend produces 80 bins"); return 1; }
    WS_CK(cudaSetDevice(e->device));
    const int T = ws_fbank_num_frames(nsamples);
    if (T <= 0) { set_err("ws_engine_extract_wav: waveform shorter than one 25 ms frame"); return 1; }
    Plan* p = get_plan(e, B, T);
    if (!p) return 1;
    cudaStream_t us = (cudaStream_t)stream, ws = lane_stream(e, p);
    if (fbank_tables(e, window_type) == nullptr) return 1;   // table upload (first use) before any lane work is enqueued
    if (enter_stream(e, p, ws, us)) return 1;
    if (fbank_into(e, wav_dev, wav_is_i16, wav_ld, nsamples, B, window_type, 1, p->feats_in, ws)) return 1;
    if (feats_out_dev)
        WS_CK(cudaMemcpyAsync(feats_out_dev, p->feats_in, (size_t)B * T * 80 * 4, cudaMemcpyDeviceToDevice, ws));
    if (run_plan(e, p, ws)) return 1;
    e->last_launches += 2;
    WS_CK(cudaMemcpyAsync(embs_dev, p->emb, (size_t)B * e->embed_dim * 4, cudaMemcpyDeviceToDevice, ws));
    if (!join) { WS_CK(cudaEventRecord(p->done, ws)); return 0; }
    return leave_stream(e, p, ws, us);
}

int ws_engine_extract_wav_host(ws_engine* e, const void* wav_host, int wav_is_i16, int nsamples, int B,
                               const char* window_type, float* embs_host) {
    if (!e || !wav_host || !embs_host) { set_err("ws_engine_extract_wav_host: null argument"); return 1; }
    if (const char* nr = not_runnable(e)) { set_err(std::string("ws_engine_extract_wav_host") + nr); return 1; }
    WS_CK(cudaSetDevice(e->device));
    const int T = ws_fbank_num_frames(nsamples);
    if (T <= 0) { set_err("ws_engine_extract_wav_host: waveform shorter than one 25 ms frame"); return 1; }
    const size_t bytes = (size_t)B * nsamples * (wav_is_i16 ? 2 : 4);
    if (bytes > e->wav_bytes) {
        if (e->wav_dev) cudaFree(e->wav_dev);
        e->wav_dev = nullptr; e->wav_bytes = 0;
        WS_CK(cudaMalloc(&e->wav_dev, bytes));
        e->wav_bytes = bytes;
    }
    Plan* p = get_plan(e, B, T);
    if (!p) return 1;
    if (host_path_enter(e, p)) return 1;
    WS_CK(cudaMemcpyAsync(e->wav_dev, wav_host, bytes, cudaMemcpyHostToDevice, e->st));
    if (fbank_into(e, e->wav_dev, wav_is_i16, nsamples, nsamples, B, window_type, 1, p->feats_in, e->st)) return 1;
    if (run_plan(e, p, e->st)) return 1;
    e->last_launches += 2;
    WS_CK(cudaMemcpyAsync(embs_host, p->emb, (size_t)B * e->embed_dim * 4, cudaMemcpyDeviceToHost, e->st));
    if (host_path_leave(e, p)) return 1;
    WS_CK(cudaStreamSynchronize(e->st));
    return 0;
}

// Pipelined host path: submit() enqueues H2D of batch i on a copy stream and the fbank+CMN+forward+D2H on the compute
// stream behind it, then returns immediately; collect() blocks until that slot's embeddings are in embs_host.  With two
// slots the H2D copy of batch i+1 overlaps the kernels of batch i (the reference overlaps with DataLoader workers and
// prefetch_factor=4, extract.py:99-103).
int ws_engine_submit_wav_host(ws_engine* e, int slot, const void* wav_host, int wav_is_i16, int nsamples, int B,
                              const char* window_type, float* embs_host) {
    if (!e || !wav_host || !embs_host || slot < 0 || slot >= ws_engine::kSlots) { set_err("ws_engine_submit_wav_host: bad argument"); return 1; }
    if (const char* nr = not_runnable(e)) { set_err(std::string("ws_engine_submit_wav_host") + nr); return 1; }
    WS_CK(cudaSetDevice(e->device));
    const int T = ws_fbank_num_frames(nsamples);
    if (T <= 0) { set_err("ws_engine_submit_wav_host: waveform shorter than one 25 ms frame"); return 1; }
    if (e->copy_st == nullptr) {
        WS_CK(cudaStreamCreateWithFlags(&e->copy_st, cudaStreamNonBlocking));
        for (int i = 0; i < ws_engine::kSlots; ++i) {
            WS_CK(cudaEventCreateWithFlags(&e->slot_copied[i], cudaEventDisableTiming));
            WS_CK(cudaEventCreateWithFlags(&e->slot_done[i], cudaEventDisableTiming));
        }
    }
    const size_t bytes = (size_t)B * nsamples * (wav_is_i16 ? 2 : 4);
    if (bytes > e->slot_bytes[slot]) {
        WS_CK(cudaStreamSynchronize(e->st));
        if (e->slot_wav[slot]) cudaFree(e->slot_wav[slot]);
        e->slot_wav[slot] = nullptr; e->slot_bytes[slot] = 0;
        WS_CK(cudaMalloc(&e->slot_wav[slot], bytes));
        e->slot_bytes[slot] = bytes;
    }
    Plan* p = get_plan(e, B, T);
    if (!p) return 1;
    // the slot's staging buffer is free once the previous job that used it finished its fbank (slot_done covers it)
    WS_CK(cudaStreamWaitEvent(e->copy_st, e->slot_done[slot], 0));
    WS_CK(cudaMemcpyAsync(e->slot_wav[slot], wav_host, bytes, cudaMemcpyHostToDevice, e->copy_st));
    WS_CK(cudaEventRecord(e->slot_copied[slot], e->copy_st));
    WS_CK(cudaStreamWaitEvent(e->st, e->slot_copied[slot], 0));
    if (host_path_enter(e, p)) return 1;
    if (fbank_into(e, e->slot_wav[slot], wav_is_i16, nsamples, nsamples, B, window_type, 1, p->feats_in, e->st)) return 1;
    if (run_plan(e, p, e->st)) return 1;
    e->last_launches += 2;
    WS_CK(cudaMemcpyAsync(embs_host, p->emb, (size_t)B * e->embed_dim * 4, cudaMemcpyDeviceToHost, e->st));
    if (host_path_leave(e, p)) return 1;
    WS_CK(cudaEventRecord(e->slot_done[slot], e->st));
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
    if (!e || !ms_out || !e->finalized || e->plan_check) { set_err("ws_engine_profile_ops: bad argument"); return -1; }
    if (cudaSetDevice(e->device) != cudaSuccess) return -1;
    Plan* p = get_plan(e, B, T);
    if (!p) return -1;
    const int n = (int)p->ops.size();
    if (n > max_ops) { set_err("ws_engine_profile_ops: output array too small"); return -1; }
    std::vector<cudaEvent_t> ev(n + 1);
    for (auto& x : ev) cudaEventCreate(&x);
    std::vector<double> acc(n, 0.0);
    for (int it = 0; it < iters + 1; ++it) {
        cudaEventRecord(ev[0], e->st);
        for (int i = 0; i < n; ++i) {
            const char* m = p->ops[i].run(e->st);
            if (m) { set_err(std::string("profile_ops launch: ") + m); return -1; }
            cudaEventRecord(ev[i + 1], e->st);
        }
        if (cudaStreamSynchronize(e->st) != cudaSuccess) { set_err("profile_ops: sync failed"); return -1; }
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
    if (!e || !e->finalized || (!e->plan_check && cudaSetDevice(e->device) != cudaSuccess)) return nullptr;
    Plan* p = get_plan(e, B, T);
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
    if (!e->finalized || (!e->plan_check && e->opt("plan_trace", 0) == 0)) {
        set_err("ws_engine_plan_trace: needs a finalized plan-check engine, or a finalized engine with the option plan_trace = 1");
        return 1;
    }
    if (!e->plan_check && cudaSetDevice(e->device) != cudaSuccess) { set_err("ws_engine_plan_trace: cudaSetDevice failed"); return 1; }
    Plan* p = get_plan(e, B, T, masked != 0);
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
        j += std::string(i ? "," : "") + "{\"label\":\"" + lab + "\",\"trace\":" + (p->ops[i].trace.empty() ? std::string("null") : p->ops[i].trace) + "}";
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
    WS_CK(cudaSetDevice(e->device));
    Plan* p = get_plan(e, B, T, masked != 0);
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
