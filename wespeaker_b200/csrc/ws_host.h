// Host-side plumbing shared by the engine translation units: error reporting, activation views, the conv
// operator builder (wgmma/TMA or FFMA), device allocation tracking.
#pragma once
#include <array>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "ws_kernels.cuh"

namespace ws {

void set_err(const std::string& msg);
const std::string& get_err();

#define WS_CK(call)                                                                               \
    do {                                                                                          \
        cudaError_t e__ = (call);                                                                 \
        if (e__ != cudaSuccess) {                                                                 \
            ws::set_err(std::string(#call) + ": " + cudaGetErrorString(e__));                     \
            return 1;                                                                             \
        }                                                                                         \
    } while (0)
#define WS_CKS(expr)                                                                              \
    do {                                                                                          \
        const char* m__ = (expr);                                                                 \
        if (m__ != nullptr) {                                                                     \
            ws::set_err(std::string(#expr) + ": " + m__);                                         \
            return 1;                                                                             \
        }                                                                                         \
    } while (0)

// Plan-check mode (ws_engine_create_plan_check): launch plans are built without a device - buffers and weights get
// placeholder addresses (never dereferenced), tensor maps are validated against the cuTensorMapEncodeTiled rules instead of
// being encoded, nothing is launched.  Thread-local, set for the duration of a plan build.
bool plan_check_mode();
struct PlanCheckScope {
    bool prev;
    explicit PlanCheckScope(bool on);
    ~PlanCheckScope();
};
void* plan_check_alloc(size_t bytes);   // 256-byte aligned placeholder address
using View = WsView;   // ws_kernels.cuh

// one fused conv/GEMM launch
struct ConvSpec {
    WsSrc src[WS_MAX_SRC];
    int nsrc = 0;
    std::vector<WsTap> taps;
    const void* W = nullptr;  // [Cout][Ktot] in activation dtype
    const void* W_lo = nullptr;  // 3xTF32: W - tf32_trunc(W)
    bool split = false;          // 3xTF32 error-compensated GEMM (fp32 activations with lo twins)
    int Ktot = 0, Cout = 0;
    int B = 0, F = 1, T = 0;  // output extents
    int dt = WS_F32;
    WsEpi epi{};
    bool dense_pointwise = false;  // every tap has dt=df=0 on a dense src with the output's extents -> flatten positions
    bool epi_generic = false;      // tensor-core kernels: run the generic epilogue even where the lean one applies (test reference)
};

// Append the taps of a (kf x kt) conv over `x` to `spec` (weights columns start at wk0, tap-major then channel).
// Strided convs are expressed with parity-plane source views so every tap is unit-stride (TMA-friendly).
// Returns the number of K columns consumed (kf*kt*x.C) and sets Fo/To.
int add_conv_taps(ConvSpec& spec, const View& x, int kf, int kt, int dil_f, int dil_t, int pad_f, int pad_t,
                  int stride_f, int stride_t, int wk0, int* Fo, int* To);

using Op = std::function<const char*(cudaStream_t)>;
// One op of a launch plan: the launch closure, a label and FLOPs (tuning aid, ws_engine_profile_ops; FLOPs 0 = not GEMM-like)
// and a JSON description of the op (operands as addresses, shapes, strides, epilogue), made when ws_engine_plan_trace asks
// for it, so that a test can re-evaluate the plan's arithmetic on the host against the oracle, or check what each kernel of
// a real engine wrote.
struct PlanOp {
    Op run;
    std::string label;
    double flops = 0;
    std::function<std::string()> trace;
};

// Plan-trace JSON fields: "name":address, "name":integer, "name":float (%.9g), "name":{view}.  Optional buffers - a 3xTF32
// lo twin, a split-K or partial-sum workspace - are named only where there is one (tplo: ",\"name\":address" or nothing).
inline std::string tp(const char* n, const void* q) { char b[96]; snprintf(b, sizeof b, "\"%s\":%llu", n, (unsigned long long)q); return b; }
inline std::string ti(const char* n, long long v) { char b[96]; snprintf(b, sizeof b, "\"%s\":%lld", n, v); return b; }
inline std::string tf(const char* n, double v) { char b[96]; snprintf(b, sizeof b, "\"%s\":%.9g", n, v); return b; }
// a float operand of a kernel, in the fewest digits that read back as the same float (1e-4f -> 0.0001)
inline std::string tff(const char* n, float v) {
    char b[96];
    for (int d = 1; d <= 9; ++d)
        if (snprintf(b, sizeof b, "\"%s\":%.*g", n, d, (double)v) > 0 && strtof(strchr(b, ':') + 1, nullptr) == v) break;
    return b;
}
inline std::string tplo(const char* n, const void* q) { return q ? "," + tp(n, q) : std::string(); }
inline std::string tview(const char* n, const View& v) {
    return std::string("\"") + n + "\":{" + tp("p", v.p) + tplo("plo", v.plo) + "," + ti("B", v.B) + "," + ti("F", v.F) + "," + ti("T", v.T) + "," + ti("C", v.C) + "," + ti("ld", v.ld) + "}";
}
inline std::string tes(int dt) { return ti("es", ws_esize(dt)); }
// the kernel a bandwidth op takes (tstats, linear, astp_stats): in "launch", like every host choice, and at the top level,
// where earlier traces named it
inline std::string tkernel(const char* k) { return std::string(",\"kernel\":\"") + k + "\",\"launch\":{\"kernel\":\"" + k + "\"}"; }

// The plan trace of each bandwidth op, from the record its launcher takes (ws_kernels.cuh)
inline std::string trace_of(const WsConvert& a) { return "{\"kind\":\"convert\"," + tes(a.dt) + "," + tp("in", a.in) + "," + tp("out", a.out) + "," + ti("n", a.n) + tplo("out_lo", a.lo) + "}"; }
inline std::string trace_of(const WsTstats& a) {
    static const char* kern[] = {"scalar", "tmean8", "tstats8"};
    return "{\"kind\":\"tstats\"," + tes(a.x.dt) + "," + tview("x", a.x) + "," + tp("pre_scale", a.pre_scale) + "," + tp("pre_shift", a.pre_shift) + "," + tp("out", a.out) + "," +
           ti("out_es", ws_esize(a.odt)) + "," + ti("out_ld", a.out_ld) + "," + ti("std_off", a.std_off) + "," + tff("eps", a.eps) + "," + tp("lens", a.lens) + tkernel(kern[a.kernel]) + "}";
}
inline std::string trace_of(const WsZeroTail& a) { return "{\"kind\":\"zero_tail\"," + tes(a.x.dt) + "," + tview("x", a.x) + "," + tp("lens", a.lens) + "}"; }
inline std::string trace_of(const WsLensDerive& a) { return "{\"kind\":\"lens_derive\"," + tp("lens", a.lens) + "," + ti("B", a.B) + "," + ti("T", a.T) + "," + ti("levels", a.levels) + "}"; }
inline std::string trace_of(const WsLinear& a) {
    return "{\"kind\":\"linear\"," + tp("in", a.in) + "," + ti("in_ld", a.in_ld) + "," + tp("in2", a.in2) + "," + ti("in2_ld", a.in2_ld) + "," + ti("rows_per_b", a.rows_per_b) + "," + tp("W", a.W) +
           "," + tp("bias", a.bias) + "," + tp("out", a.out) + "," + ti("out_ld", a.out_ld) + "," + ti("R", a.R) + "," + ti("I", a.I) + "," + ti("O", a.O) + "," + ti("act", a.act) + tplo("wsp", a.wsp) +
           tkernel(a.kernel == WS_LINEAR_ROWS64 ? "rows64" : "rows16") + "}";
}
inline std::string trace_of(const WsScaleResidual& a) {
    return "{\"kind\":\"scale_residual\"," + tes(a.x.dt) + "," + tview("x", a.x) + "," + tp("gate", a.gate) + "," + tview("res", a.res) + "," + tview("out", a.out) + "}";
}
inline std::string trace_of(const WsAffCombine& a) {
    return "{\"kind\":\"aff_combine\"," + tes(a.x.dt) + "," + tview("x", a.x) + "," + tview("y", a.y) + "," + tview("t", a.t) + "," + tview("out", a.out) + "}";
}
inline std::string trace_of(const WsAstpStats& a) {
    return "{\"kind\":\"astp_stats\"," + tes(a.x.dt) + "," + tview("x", a.x) + "," + tview("logits", a.logits) + "," + tp("stats", a.stats) + "," + tp("lens", a.lens) + "," + tff("eps", a.var_floor) +
           tkernel(a.kernel == WS_ASTP_STATS4 ? "stats4" : "scalar") + "}";
}
inline std::string trace_of(const WsSimamStats& a) {
    return "{\"kind\":\"simam_stats\"," + tes(a.y.dt) + "," + tview("x", a.y) + "," + tp("stats", a.stats) + "," + tp("lens", a.lens) + tplo("partial", a.partial) + "}";
}
inline std::string trace_of(const WsSimamApply& a) {
    View res = a.y;   // res has y's extents, at res's own row pitch
    res.p = const_cast<void*>(a.res); res.plo = nullptr; res.ld = a.rs.t;
    return "{\"kind\":\"simam_apply\"," + tes(a.y.dt) + "," + tview("y", a.y) + "," + tp("stats", a.stats) + "," + tview("res", res) + "," + tp("out", a.out) + "," + ti("out_sb", a.os.b) + "," +
           ti("out_sf", a.os.f) + "," + ti("out_st", a.os.t) + "," + tp("lens", a.lens) + "," + tff("lambda", a.lambda) + "}";
}
inline std::string trace_of(const WsDwconv3x3& a) {
    return "{\"kind\":\"dwconv3x3\"," + tes(a.x.dt) + "," + tview("x", a.x) + "," + tview("out", a.out) + "," + tp("w", a.w) + "," + tp("shift", a.shift) + "," + tp("lens", a.lens) + "}";
}
inline std::string trace_of(const WsBnRelu& a) {
    return "{\"kind\":\"bnrelu\"," + tes(a.x.dt) + "," + tview("x", a.x) + "," + tp("scale", a.scale) + "," + tp("shift", a.shift) + "," + tview("out", a.out) + "," + ti("C", a.x.C) + "}";
}
inline std::string trace_of(const WsStem& a) {
    return "{\"kind\":\"stem\"," + tes(a.out.dt) + "," + tp("feats", a.feats) + "," + tp("w9", a.w9) + "," + tp("shift", a.shift) + "," + tview("out", a.out) + "," + ti("Fdim", a.out.F) + "," +
           tp("lens", a.lens) + "}";
}
inline std::string trace_of(const WsSegMeans& a) {
    return "{\"kind\":\"seg_means\"," + tes(a.x.dt) + "," + tview("x", a.x) + "," + ti("seg_len", a.seg_len) + "," + tp("mean", a.mean) + "," + tp("segmean", a.segmean) + "}";
}
inline std::string trace_of(const WsSeGate& a) {
    return "{\"kind\":\"se_gate\"," + tes(a.x.dt) + "," + tview("x", a.x) + "," + tp("W1", a.W1) + "," + tp("b1", a.b1) + "," + tp("W2t", a.W2t) + "," + tp("b2", a.b2) + "," + ti("H", a.H) + "," +
           tp("gate", a.gate) + "," + tp("lens", a.lens) + "," + tp("colsum", a.colsum) + "}";
}
inline std::string trace_of(const WsCamGate& a) {
    return "{\"kind\":\"cam_gate\"," + tes(a.x.dt) + "," + tview("x", a.x) + "," + ti("seg_len", a.seg_len) + "," + tp("W1", a.W1) + "," + tp("b1", a.b1) + "," + tp("W2", a.W2) + "," + tp("b2", a.b2) +
           "," + ti("H", a.H) + "," + ti("G", a.G) + "," + tp("gate", a.gate) + "}";
}

// The tensor-core ops, one record each: the parameter block its launcher reads, and the operands its tensor maps were encoded
// from (a CUtensorMap cannot be read back).  trace_of writes the op's contract - every scalar the kernel reads taken from the
// parameter block - plus a "launch" object with the kernel and geometry the host chose, which may depend on the device (SM
// count, co-resident clusters); label_of writes the op's label.
struct ConvRec {                               // the conv-GEMM: tc (tc3 when tc->cl > 1, else tc2) or simt
    ConvSpec spec;                             // source views, taps and weights
    std::shared_ptr<const WsTc2Params> tc;
    std::shared_ptr<const WsSimtParams> simt;
};
struct Conv3x3Rec {
    std::shared_ptr<const WsC3Params> q;
    View x, out, res;                          // res: meaningful where q->res is set
    const void* W;
};
struct Res2Rec {
    std::shared_ptr<const WsRes2Params> q;
    View x, out;
    const void* W7;
};
struct AstpRec {
    std::shared_ptr<const WsAstpParams> q;
    View x, h;
    const void* W2;
};
struct CamRec {
    std::shared_ptr<const WsCamParams> q;
    View X;
    std::vector<WsCamLayer> layers;                      // host copies of the descriptors of layers [q->l0, q->l1)
    std::vector<std::array<const void*, 2>> weights;     // the (W1, Wl) each one's tensor maps were encoded from
};
std::string trace_of(const ConvRec& r);
std::string trace_of(const Conv3x3Rec& r);
std::string trace_of(const Res2Rec& r);
std::string trace_of(const AstpRec& r);
std::string trace_of(const CamRec& r);
std::string label_of(const ConvRec& r);
std::string label_of(const Conv3x3Rec& r);
std::string label_of(const Res2Rec& r);
std::string label_of(const AstpRec& r);
std::string label_of(const CamRec& r);

// A plan op launched and traced from one record: launch(rec, stream) runs it, trace_of(rec) describes it
template <class Rec, class Launch>
PlanOp plan_op(const Rec& rec, Launch launch, std::string label, double flops = 0) {
    return PlanOp{[rec, launch](cudaStream_t s) { return launch(rec, s); }, std::move(label), flops, [rec] { return trace_of(rec); }};
}

// Build a launch closure for `spec`; use_tc selects a tensor-core kernel (needs dt-aligned shapes) else FFMA.
// Returns false and sets the error string if the spec cannot be mapped.
bool make_conv_op(const ConvSpec& spec, int use_tc, PlanOp* out);  // 0 FFMA, 2 persistent tensor-core kernel, 3 the same with clusters on large layers

void fill_epi_out(WsEpi& e, const View& out);

// What a fused-op constructor made of a request: the op (built); nothing, because the shape is outside its kernel's envelope
// (outside: no error is set, the caller builds the layer another way); or nothing, because of an error (set_err says which).
enum class OpBuild { built, outside, error };

// Fused Res2 chain over a whole SE_Res2Block stage (7 dilated k=3 convs on w8-channel groups, ecapa_tdnn.py:29-78).
// x: block input (B,1,T,8*w8), out: block output buffer (groups 0..6 are written).  W7: [7*w8][3*w8] packed weights in
// the activation dtype; bias/scale/shift: [7][w8] fp32.  Outside the fused kernel's envelope: fp32 activations, w8 not in
// {64,128}, dilation > 4 with T > 256.
OpBuild make_res2_op(const View& x, const View& out, const void* W7, const float* bias, const float* scale,
                     const float* shift, int w8, int dil, PlanOp* op, const int* lens = nullptr);

// Fused ASTP tail (ws_astp_fused.cu): x = frame-level features (B,1,T,C), h = the attention's hidden layer (B,1,T,128), W2 =
// linear2 weight [C][128] in the activation dtype, stats = fp32 [B][2C] (weighted mean, std = sqrt(max(var, var_floor))).
// linear2's bias cancels in the softmax over time and is not needed.  Outside the envelope: fp32 activations, C % 128,
// hidden width != 128.
OpBuild make_astp_op(const View& x, const View& h, const void* W2, float* stats, float var_floor, PlanOp* op,
                     const int* lens = nullptr);

// Halo-resident 3x3 pad-1 conv (ws_conv3x3.cu), strides 1 or 2 per axis: out = act(conv(x, W) + bias [+ res]).  x/out/res:
// channels-last 16-bit views (out / res with the strided extents); W: [Cout][9*Cin] tap-major in the activation dtype; relu: 0 none,
// 1 ReLU, 2 Hardtanh(0, 20).  Outside the kernel's envelope, the caller uses make_conv_op.
OpBuild make_conv3x3_op(const View& x, const View& out, const void* W, const float* bias, const View* res, int relu,
                        PlanOp* op, int stride_f = 1, int stride_t = 1, const int* lens = nullptr);

// Fused CAM++ dense layers (ws_cam_dense.cu).  cam_layer_fill builds one host-side layer descriptor (weights are device
// pointers in the activation dtype: W1 [128][cin] with BN2 folded, Wl [32][3*128] tap-major; everything else fp32 device
// arrays).  make_cam_dense_op launches layers [l0, l1) of a device-resident descriptor array over the concat buffer X
// (B,1,T,Cmax); layers / weights: the same descriptors on the host and the (W1, Wl) each one's tensor maps were encoded
// from, for the plan trace.  Outside the kernel's envelope: T > 512, fp32 activations.
constexpr int kCamSegLen = 100;   // CAM++ context segments (campplus.py:108-135: seg_len)
bool cam_layer_fill(WsCamLayer* L, int dt, const void* W1, const void* Wl, const float* bn1_scale, const float* bn1_shift,
                    const float* bias2, const float* w1c_t, const float* b1c, const float* w2c_t, const float* b2c, int cin,
                    int dil);
OpBuild make_cam_dense_op(const View& X, const WsCamLayer* layers_dev, const std::vector<WsCamLayer>& layers,
                          const std::vector<std::array<const void*, 2>>& weights, int l0, int l1, PlanOp* op, const int* lens = nullptr);

}  // namespace ws
