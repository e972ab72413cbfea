// Host side of the fused conv operator: tap generation (incl. parity planes for strided convs), TMA tensor-map
// construction, tile-shape selection and the launch closures for the tensor-core (wgmma) and FFMA kernels.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include <memory>
#include <mutex>

#include "../../include/wespeaker_b200.h"
#include "ws_host.h"
#include "ws_tc_common.cuh"   // ws_tc_lean_kind: which epilogue a layer takes decides whether it may use 256-wide tiles

namespace ws {

static thread_local std::string g_err;
void set_err(const std::string& msg) { g_err = msg; }
const std::string& get_err() { return g_err; }

static thread_local bool g_plan_check = false;
bool plan_check_mode() { return g_plan_check; }
PlanCheckScope::PlanCheckScope(bool on) : prev(g_plan_check) { g_plan_check = on; }
PlanCheckScope::~PlanCheckScope() { g_plan_check = prev; }
std::string trace_of(const ConvRec& r) {
    const ConvSpec& s = r.spec;
    std::string j = "{\"kind\":\"conv\"," + ti("es", ws_esize(s.dt)) + ",\"src\":[";
    for (int i = 0; i < s.nsrc; ++i) {
        const WsSrc& v = s.src[i];
        j += std::string(i ? "," : "") + "{" + tp("p", v.ptr) + (s.split ? tplo("p_lo", v.ptr_lo) : std::string()) + "," + ti("B", v.B) + "," + ti("F", v.F) + "," + ti("T", v.T) + "," + ti("C", v.C) + "," +
             ti("sB", v.sB) + "," + ti("sF", v.sF) + "," + ti("sT", v.sT) + "}";
    }
    j += "],\"taps\":[";
    for (size_t i = 0; i < s.taps.size(); ++i) {
        const WsTap& t = s.taps[i];
        j += std::string(i ? "," : "") + "[" + std::to_string(t.src) + "," + std::to_string(t.c0) + "," + std::to_string(t.dt) + "," + std::to_string(t.df) + "," +
             std::to_string(t.wk) + "," + std::to_string(t.nch) + "]";
    }
    const WsEpi& e = r.tc ? r.tc->epi : r.simt->epi;
    j += "]," + tp("W", s.W) + "," + ti("Ktot", s.Ktot) + "," + ti("Cout", s.Cout) + "," + ti("B", s.B) + "," + ti("F", s.F) + "," + ti("T", s.T) +
         "," + tp("bias", e.bias) + "," + tp("rowbias", e.rowbias) + "," + ti("rowbias_ld", e.rowbias_ld) + "," + ti("act1", e.act1) + "," + tp("scale", e.scale) +
         "," + tp("shift", e.shift) + "," + tp("gate", e.gate) + "," + ti("gate_ld", e.gate_ld) + "," + ti("gate_seg", e.gate_seg) + "," + ti("gate_nseg", e.gate_nseg) + "," + tp("res", e.res) + "," + ti("res_ld", e.res_ld) + "," + ti("act2", e.act2) + "," + tp("out", e.out) +
         "," + ti("out_ld", e.out_ld) + "," + tp("out2", e.out2) + "," + ti("out2_ld", e.out2_ld) + "," + tp("add2", e.add2) + "," + ti("add2_ld", e.add2_ld) +
         "," + tp("colsum", e.colsum) + (s.split ? tplo("W_lo", s.W_lo) + tplo("out_lo", e.out_lo) + tplo("out2_lo", e.out2_lo) : std::string());
    if (!r.tc) return j + ",\"launch\":{\"kernel\":\"simt\"}}";
    const WsTc2Params& q = *r.tc;
    return j + ",\"launch\":{\"kernel\":\"" + (q.cl > 1 ? "tc3" : "tc2") + "\"," + ti("cl", q.cl) + "," + ti("bn", q.bn) + "," + ti("nstages", q.nstages) + "," +
           ti("bk_bytes", q.bk_bytes) + ",\"tile\":[" + std::to_string(1 << q.bt_log2) + "," + std::to_string(1 << q.bf_log2) + "," + std::to_string(1 << q.bb_log2) + "]," +
           ti("grid", q.grid) + "}}";
}

std::string label_of(const ConvRec& r) {
    const ConvSpec& s = r.spec;
    char kern[64] = "conv_simt", buf[160];
    if (r.tc && r.tc->cl > 1) snprintf(kern, sizeof kern, "conv_tc3 cl=%d grid=%d bn=%d st=%d", r.tc->cl, r.tc->grid, r.tc->bn, r.tc->nstages);
    else if (r.tc) snprintf(kern, sizeof kern, "conv_tc2");
    snprintf(buf, sizeof buf, "%s pos=%lld K=%d N=%d", kern, (long long)((double)s.B * s.F * s.T), s.Ktot, s.Cout);
    return buf;
}

void* plan_check_alloc(size_t bytes) {
    static thread_local unsigned long long next = 0x7000000000ull;   // far from anything a host allocator returns
    void* p = (void*)next;
    next += (bytes + 255) & ~255ull;
    if (bytes == 0) next += 256;
    return p;
}

void fill_epi_out(WsEpi& e, const View& out) {
    e.out = out.p;
    e.out_lo = out.plo;
    e.out_ld = out.ld;
    e.dtype = out.dt;
    e.FT = out.F * out.T;
    e.T = out.T;
}

static int find_or_add_src(ConvSpec& s, const WsSrc& v) {
    for (int i = 0; i < s.nsrc; ++i)
        if (s.src[i].ptr == v.ptr && s.src[i].sT == v.sT && s.src[i].sF == v.sF && s.src[i].T == v.T &&
            s.src[i].F == v.F && s.src[i].C == v.C)
            return i;
    if (s.nsrc >= WS_MAX_SRC) return -1;
    s.src[s.nsrc] = v;
    return s.nsrc++;
}

static inline int floordiv(int a, int b) { return (a >= 0) ? a / b : -((-a + b - 1) / b); }

int add_conv_taps(ConvSpec& spec, const View& x, int kf, int kt, int dil_f, int dil_t, int pad_f, int pad_t,
                  int stride_f, int stride_t, int wk0, int* Fo, int* To) {
    const int es = ws_esize(x.dt);
    *Fo = (x.F + 2 * pad_f - dil_f * (kf - 1) - 1) / stride_f + 1;
    *To = (x.T + 2 * pad_t - dil_t * (kt - 1) - 1) / stride_t + 1;
    const long long sT = x.ld, sF = (long long)x.T * x.ld, sB = (long long)x.F * x.T * x.ld;
    for (int jf = 0; jf < kf; ++jf)
        for (int jt = 0; jt < kt; ++jt) {
            const int offf = jf * dil_f - pad_f, offt = jt * dil_t - pad_t;
            const int pf = ((offf % stride_f) + stride_f) % stride_f, pt = ((offt % stride_t) + stride_t) % stride_t;
            WsSrc v;
            v.ptr = (const char*)x.p + ((size_t)pf * sF + (size_t)pt * sT) * es;
            v.ptr_lo = x.plo ? (const char*)x.plo + ((size_t)pf * sF + (size_t)pt * sT) * es : nullptr;
            v.B = x.B;
            v.F = (x.F - pf + stride_f - 1) / stride_f;
            v.T = (x.T - pt + stride_t - 1) / stride_t;
            v.C = x.C;
            // a parity plane with no rows (the odd plane of a 1-frame or 1-row input): its taps only read padding, and a
            // zero-extent tensor map cannot be encoded
            if (v.F < 1 || v.T < 1) continue;
            v.sB = sB;
            v.sF = sF * stride_f;
            v.sT = sT * stride_t;
            const int si = find_or_add_src(spec, v);
            if (si < 0) return -1;
            WsTap tap;
            tap.src = si;
            tap.c0 = 0;
            tap.df = floordiv(offf - pf, stride_f);
            tap.dt = floordiv(offt - pt, stride_t);
            tap.wk = wk0 + (jf * kt + jt) * x.C;
            tap.nch = x.C;
            spec.taps.push_back(tap);
        }
    return kf * kt * x.C;
}

// ------------------------------------------------------------------------------------------------ TMA maps
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    });
    return fn;
}

static bool encode_map(CUtensorMap* m, int dt, const void* ptr, int rank, const cuuint64_t* dims,
                       const cuuint64_t* strides_bytes, const cuuint32_t* box, int swizzle_bytes) {
    if (plan_check_mode()) {
        // no driver: check what cuTensorMapEncodeTiled would check (CUDA driver API, tensor map object management)
        const int es = ws_esize(dt);
        char buf[200];
        const char* why = nullptr;
        if (((unsigned long long)ptr & 15ull) != 0) why = "global address not 16-byte aligned";
        if (rank < 1 || rank > 5) why = "rank outside 1..5";
        for (int i = 0; i < rank && !why; ++i) {
            if (dims[i] < 1 || dims[i] > (1ull << 32)) why = "dimension outside 1..2^32";
            else if (box[i] < 1 || box[i] > 256) why = "box extent outside 1..256";
            else if (i + 1 < rank && (strides_bytes[i] % 16 != 0 || strides_bytes[i] >= (1ull << 40))) why = "stride not a multiple of 16 bytes (or >= 2^40)";
        }
        if (!why) {
            const unsigned inner = box[0] * (unsigned)es;
            if (swizzle_bytes != 0 && inner > (unsigned)swizzle_bytes) why = "inner box extent exceeds the swizzle span";
            else if (inner % 16 != 0) why = "inner box extent not a multiple of 16 bytes";
        }
        if (why) {
            snprintf(buf, sizeof buf, "tensor map check failed: %s (rank %d dims [%llu %llu ..] box [%u %u ..] sw %d)", why, rank,
                     (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0), box[0], rank > 1 ? box[1] : 0, swizzle_bytes);
            set_err(buf);
            return false;
        }
        memset(m, 0, sizeof(*m));
        return true;
    }
    EncodeTiledFn fn = get_encode();
    if (fn == nullptr) {
        set_err("cuTensorMapEncodeTiled driver entry point unavailable (no CUDA driver?)");
        return false;
    }
    const CUtensorMapDataType t = dt == WS_F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                               : (dt == WS_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                                                : CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
    const CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                  : (swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                     : (swizzle_bytes == 0 ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_32B));
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = fn(m, t, (cuuint32_t)rank, const_cast<void*>(ptr), dims, strides_bytes, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        char buf[256];
        snprintf(buf, sizeof buf,
                 "cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu %llu %llu %llu] box [%u %u %u %u] sw %d", (int)r,
                 rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
                 (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0), box[0],
                 rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0, swizzle_bytes);
        set_err(buf);
        return false;
    }
    return true;
}

// A tensor map from its extents, strides in elements (the innermost stride is 1) and box, all innermost first; the rank is
// the number of extents.
static bool encode_strided(CUtensorMap* m, int dt, const void* ptr, std::initializer_list<long long> dims,
                           std::initializer_list<long long> strides, std::initializer_list<int> box, int swizzle_bytes) {
    const int rank = (int)dims.size();
    if (rank < 1 || rank > 5 || (int)strides.size() != rank - 1 || (int)box.size() != rank) {
        set_err("tensor map: extents, strides and box disagree in rank");
        return false;
    }
    cuuint64_t d[5], s[4];
    cuuint32_t b[5];
    for (int i = 0; i < rank; ++i) { d[i] = (cuuint64_t)dims.begin()[i]; b[i] = (cuuint32_t)box.begin()[i]; }
    for (int i = 0; i + 1 < rank; ++i) s[i] = (cuuint64_t)strides.begin()[i] * ws_esize(dt);
    return encode_map(m, dt, ptr, rank, d, s, b, swizzle_bytes);
}

// A channels-last view: rank 4 over (C, T, F, B), or rank 3 over (C, T, B) for a view with F == 1, as the box's rank says
static bool encode_view(CUtensorMap* m, const View& v, std::initializer_list<int> box, int swizzle_bytes) {
    if (box.size() == 4)
        return encode_strided(m, v.dt, v.p, {v.C, v.T, v.F, v.B}, {v.ld, v.T * v.ld, (long long)v.F * v.T * v.ld}, box, swizzle_bytes);
    if (v.F != 1) { set_err("tensor map: a rank-3 view map needs F == 1"); return false; }
    return encode_strided(m, v.dt, v.p, {v.C, v.T, v.B}, {v.ld, v.T * v.ld}, box, swizzle_bytes);
}

// A row-major rows x cols matrix (row pitch cols), such as a [Cout][K] weight
static bool encode_matrix(CUtensorMap* m, int dt, const void* ptr, long long cols, long long rows, std::initializer_list<int> box,
                          int swizzle_bytes) {
    return encode_strided(m, dt, ptr, {cols, rows}, {cols}, box, swizzle_bytes);
}

static int ilog2(int v) {
    int l = 0;
    while ((1 << l) < v) ++l;
    return l;
}

// Operand side of the tensor-core conv: the k-block size, the taps in k-blocks, the output tile of 128 positions and the
// activation maps (with their 3xTF32 low twins).  The N tile is chosen by build_tc2.
static bool tc2_geometry(const ConvSpec& s, WsTc2Params* q) {
    const int es = ws_esize(s.dt);
    q->kind = s.dt == WS_F32 ? 0 : 1;
    if ((int)s.taps.size() > WS_MAX_TAPS) { set_err("tc conv: too many taps"); return false; }
    int minb = 1 << 30;
    for (const WsTap& t : s.taps) minb = std::min(minb, t.nch * es);
    if (minb < 32) { set_err("tc conv: fewer than 32 bytes of channels per tap"); return false; }
    q->bk_bytes = minb >= 128 ? 128 : (minb >= 64 ? 64 : 32);   // k-block row bytes == TMA / wgmma swizzle span
    const int bk_elems = q->bk_bytes / es;
    q->ntaps = (int)s.taps.size();
    for (int i = 0; i < q->ntaps; ++i) {
        const WsTap& t = s.taps[i];
        if (t.nch % bk_elems != 0 && t.c0 + t.nch != s.src[t.src].C) {
            set_err("tc conv: ragged k-block needs the tap to end at the source view's last channel");
            return false;
        }
        q->taps[i] = WsTcTap{t.src, t.c0, t.dt, t.df, t.wk, (t.nch + bk_elems - 1) / bk_elems};
        q->nk_total += q->taps[i].nkb;
    }
    // ---- output tile: 128 positions, flat over (B, F, T) for a dense 1x1 conv, else the 2^bt x 2^bf x 2^bb box that pads least
    int B = s.B, F = s.F, T = s.T;
    const bool flat = s.dense_pointwise;
    int bt = 128, bf = 1, bb = 1;
    if (flat) {
        T = s.B * s.F * s.T; F = 1; B = 1;
    } else {
        long long best = -1;
        for (int t = 1; t <= 128; t <<= 1)
            for (int f = 1; t * f <= 128; f <<= 1) {
                const int b = 128 / (t * f);
                if (F == 1 && f != 1) continue;
                const long long cost = (long long)((T + t - 1) / t) * t * ((F + f - 1) / f) * f * ((B + b - 1) / b) * b;
                if (best < 0 || cost < best || (cost == best && t > bt)) { best = cost; bt = t; bf = f; bb = b; }
            }
    }
    q->bt_log2 = ilog2(bt); q->bf_log2 = ilog2(bf); q->bb_log2 = ilog2(bb);
    q->tiles_t = (T + bt - 1) / bt; q->tiles_f = (F + bf - 1) / bf; q->tiles_b = (B + bb - 1) / bb;
    q->B = B; q->F = F; q->T = T;
    // ---- activation maps, one per source view (unused slots repeat the first)
    for (int i = 0; i < s.nsrc; ++i) {
        WsSrc v = s.src[i];
        if (flat) { v.B = 1; v.F = 1; v.T = T; v.sF = v.sB = T * v.sT; }   // all positions as one row
        auto enc = [&](CUtensorMap* m, const void* p) {
            return encode_strided(m, s.dt, p, {v.C, v.T, v.F, v.B}, {v.sT, v.sF, v.sB}, {bk_elems, bt, bf, bb}, q->bk_bytes);
        };
        if (!enc(&q->amap[i], v.ptr)) return false;
        q->amap_lo[i] = q->amap[i];
        if (s.split && !enc(&q->amap_lo[i], v.ptr_lo)) return false;
    }
    for (int i = s.nsrc; i < WS_MAX_SRC; ++i) { q->amap[i] = q->amap[0]; q->amap_lo[i] = q->amap_lo[0]; }
    return true;
}

// ---- the persistent tensor-core kernel (ws_gemm_tc2.cu).  cl: CTAs per cluster sharing the weight tile (1, or 2 / 4:
// ws_tc3_launch).  Outside when no N tile suits a cluster of cl >= 2 CTAs (the caller then builds the layer with cl = 1);
// every other refusal is an error that names the reason.
static OpBuild build_tc2(const ConvSpec& s, WsTc2Params* q, int cl = 1) {
    const bool pair = cl >= 2;
    const WsEpi& e = s.epi;
    if (s.Cout % 32 != 0) { set_err("tc conv: Cout must be a multiple of 32 (the narrowest N tile)"); return OpBuild::error; }
    if (e.res != nullptr && e.out2 != nullptr) { set_err("tc conv: a residual and a second output (out2) cannot be combined"); return OpBuild::error; }
    memset(q, 0, sizeof(*q));
    const int es = ws_esize(s.dt);
    q->has_out2 = e.out2 != nullptr;
    q->has_epin = (e.res != nullptr) || (e.out2 != nullptr);
    q->nsplit = s.split ? 3 : 1;
    if (s.split) {
        if (s.dt != WS_F32 || s.W_lo == nullptr || e.out_lo == nullptr || (q->has_out2 && e.out2_lo == nullptr)) {
            set_err("tc conv: 3xTF32 needs fp32 activations with lo twins for W / out / out2"); return OpBuild::error;
        }
        for (int i = 0; i < s.nsrc; ++i)
            if (s.src[i].ptr_lo == nullptr) { set_err("tc conv: 3xTF32 source without a lo twin"); return OpBuild::error; }
    }
    if (!tc2_geometry(s, q)) return OpBuild::error;
    q->nout = (s.split ? 2 : 1) * (q->has_out2 ? 2 : 1);
    const int nstage_bufs = q->nout + (q->has_epin ? 1 : 0);
    const int budget = kMaxDynSmem2 - 1024;
    q->epi_generic = s.epi_generic;
    const int mtiles = q->tiles_t * q->tiles_f * q->tiles_b;
    const int g_num_sms = ws_num_sms();
    int ncl = g_num_sms;                       // clusters (or CTAs) resident at once
    if (pair) {
        ncl = ws_tc3_max_clusters(cl);
        if (ncl <= 0) ncl = g_num_sms / cl;
    }
    // rounds of the persistent schedule: tiles of bn columns over ncl clusters
    auto rounds = [&](int c) { return ((long long)(s.Cout / c) * ((mtiles + cl - 1) / cl) + ncl - 1) / ncl; };
    // 256-wide tiles (16-bit, lean epilogue without row bias, no epilogue-input tile, 128-byte k-blocks) halve the
    // A-operand reads and the epilogue passes per FLOP, but a tile is twice the work: taken when the schedule then needs
    // at most 10 % more time than with 128-wide tiles, counted in 128-wide rounds (20 r256 <= 11 r128)
    q->epi = e; q->bn = 256; q->panel_bytes = 128;
    const bool wide_ok = s.Cout % 256 == 0 && q->kind == 1 && !q->has_epin && q->bk_bytes == 128 && !q->epi_generic &&
                         ws_tc_lean_kind(q) == s.dt + 1 && e.rowbias == nullptr && 20 * rounds(256) <= 11 * rounds(128);
    // staging + per-channel parameters (+ the row-wise epilogue's scratch): the 256-wide tile stages its whole output
    // tile at once and double-buffers its parameters, and its epilogue works in fragment layout without scratch
    auto staging_bytes = [&](int c) {
        return c == 256 ? 128 * c * es + 2 * 3 * c * 4 : nstage_bufs * 128 * c * es + 3 * c * 4 + WS_TC_EPI_SCRATCH;
    };
    // widest N tile whose staging + >=3 ring stages fit (>=2 accepted as a last resort, never for 256)
    int bn = 0, nst = 0;
    const int cands[4] = {256, 128, 64, 32};
    const char* env_bn = getenv("WS_TC2_MAX_BN");
    const int max_bn = env_bn ? atoi(env_bn) : 256;
    for (int pass = 0; pass < 2 && bn == 0; ++pass)
        for (int ci = 0; ci < 4; ++ci) {
            const int c = cands[ci];
            if (s.Cout % c != 0 || c > max_bn || (c == 256 && (!wide_ok || pass == 1))) continue;
            const int wrows = c / cl;            // clusters: each CTA fetches (and multicasts) bn / cl weight rows
            if ((wrows * q->bk_bytes) % 1024 != 0) continue;   // ... a whole number of 1024-B swizzle atoms
            const int staging = staging_bytes(c);
            const int stage_bytes = (128 + c) * q->bk_bytes;
            const int n = (budget - staging) / stage_bytes;
            if (n >= (pass == 0 ? 3 : 2)) { bn = c; nst = n > WS_TC_MAX_STAGES ? WS_TC_MAX_STAGES : n; break; }
        }
    if (bn == 0) {
        if (pair) return OpBuild::outside;
        set_err("tc conv: no N tile fits in shared memory beside the epilogue staging");
        return OpBuild::error;
    }
    q->bn = bn; q->nstages = nst;
    q->tiles_n = s.Cout / bn;
    q->num_tiles = q->tiles_n * ((mtiles + cl - 1) / cl);
    q->panel_bytes = bn * es >= 128 ? 128 : bn * es;
    const int panel_cols = q->panel_bytes / es;
    const int bk_elems = q->bk_bytes / es;
    // weights map with the chosen N tile: box of the rows ONE CTA loads per k-block
    if (!encode_matrix(&q->wmap, s.dt, s.W, s.Ktot, s.Cout, {bk_elems, bn / cl}, q->bk_bytes)) return OpBuild::error;
    q->wmap_lo = q->wmap;
    if (s.split && !encode_matrix(&q->wmap_lo, s.dt, s.W_lo, s.Ktot, s.Cout, {bk_elems, bn / cl}, q->bk_bytes)) return OpBuild::error;
    // output / epilogue-input maps: same tile geometry as the A maps over the output positions (q's extents: one row of
    // all positions for a dense 1x1 conv)
    auto out_map = [&](CUtensorMap* m, const void* ptr, long long ld) {
        const View o{const_cast<void*>(ptr), nullptr, q->B, q->F, q->T, s.Cout, ld, s.dt};
        return encode_view(m, o, {panel_cols, 1 << q->bt_log2, 1 << q->bf_log2, 1 << q->bb_log2}, q->panel_bytes);
    };
    int oi = 0;
    if (!out_map(&q->omap[oi++], e.out, e.out_ld)) return OpBuild::error;
    if (s.split && !out_map(&q->omap[oi++], e.out_lo, e.out_ld)) return OpBuild::error;
    if (q->has_out2) {
        if (!out_map(&q->omap[oi++], e.out2, e.out2_ld)) return OpBuild::error;
        if (s.split && !out_map(&q->omap[oi++], e.out2_lo, e.out2_ld)) return OpBuild::error;
        if (!out_map(&q->imap, e.add2, e.add2_ld)) return OpBuild::error;
    } else if (q->has_epin) {
        if (!out_map(&q->imap, e.res, e.res_ld)) return OpBuild::error;
    }
    for (; oi < 4; ++oi) q->omap[oi] = q->omap[0];
    if (!q->has_epin) q->imap = q->omap[0];
    q->cl = cl;
    if (pair) q->grid = cl * (q->num_tiles < ncl ? q->num_tiles : ncl);
    else q->grid = q->num_tiles < g_num_sms ? q->num_tiles : g_num_sms;
    q->smem_bytes = nst * (128 + bn) * q->bk_bytes + staging_bytes(bn) + 1024;
    return OpBuild::built;
}

static bool build_simt(const ConvSpec& s, WsSimtParams* p) {
    memset(p, 0, sizeof(*p));
    if ((int)s.taps.size() > WS_MAX_TAPS) { set_err("conv: too many taps"); return false; }
    if (s.Cout % 4 != 0) { set_err("conv: Cout must be a multiple of 4"); return false; }
    for (int i = 0; i < s.nsrc; ++i) p->src[i] = s.src[i];
    p->ntaps = (int)s.taps.size();
    for (int i = 0; i < p->ntaps; ++i) p->taps[i] = s.taps[i];
    p->W = s.W; p->Ktot = s.Ktot; p->Cout = s.Cout;
    p->B = s.B; p->F = s.F; p->T = s.T;
    p->dtype = s.dt;
    p->epi = s.epi;
    return true;
}

static const char* launch_conv(const ConvRec& r, cudaStream_t s) {
    if (r.simt) return ws_simt_launch(r.simt.get(), s);
    return r.tc->cl > 1 ? ws_tc3_launch(r.tc.get(), s) : ws_tc2_launch(r.tc.get(), s);
}

bool make_conv_op(const ConvSpec& spec, int use_tc, PlanOp* out) {
    ConvRec rec{spec};
    const long long pos = (long long)spec.B * spec.F * spec.T;
    const char* env_mp = getenv("WS_TC3_MIN_POS");
    const long long min_pos = env_mp ? atoll(env_mp) : 132LL * 128;   // one wave of 128-row tiles on an H100
    if (use_tc >= 3 && pos >= min_pos) {
        // big layers: clusters of CTAs on adjacent position tiles share the weight tile by TMA multicast
        auto q = std::make_shared<WsTc2Params>();
        // (two CTAs per cluster; WS_TC3_CL=4 takes four on the largest layers)
        const char* env_cl = getenv("WS_TC3_CL");
        const int cl = (env_cl && atoi(env_cl) == 4 && pos >= 2LL * min_pos) ? 4 : 2;
        const OpBuild r = build_tc2(spec, q.get(), cl);
        if (r == OpBuild::error) return false;
        if (r == OpBuild::built) rec.tc = q;
    }
    if (!rec.tc && use_tc >= 2) {
        auto q = std::make_shared<WsTc2Params>();
        if (build_tc2(spec, q.get()) != OpBuild::built) return false;
        rec.tc = q;
    }
    if (!rec.tc) {
        if (spec.epi.colsum != nullptr) { set_err("conv colsum: only the persistent tensor-core kernels (use_tc >= 2) produce column sums"); return false; }
        auto p = std::make_shared<WsSimtParams>();
        if (!build_simt(spec, p.get())) return false;
        rec.simt = p;
    }
    *out = plan_op(rec, launch_conv, label_of(rec), 2.0 * (double)pos * spec.Ktot * spec.Cout);
    return true;
}

OpBuild make_res2_op(const View& x, const View& out, const void* W7, const float* bias, const float* scale,
                     const float* shift, int w8, int dil, PlanOp* op, const int* lens) {
    // T > 256: time tiles with a 32-row halo per side cover the chain's receptive field (7 * dil rows) up to dilation 4
    if (x.dt == WS_F32 || out.dt != x.dt || (w8 != 64 && w8 != 128) || (x.T > 256 && dil > 4) || x.F != 1 || dil < 1 || dil > 7)
        return OpBuild::outside;
    auto q = std::make_shared<WsRes2Params>();
    memset(q.get(), 0, sizeof(WsRes2Params));
    if (!encode_view(&q->xmap, x, {64, 128, 1}, 128) || !encode_view(&q->omap, out, {64, 128, 1}, 128) ||
        !encode_view(&q->omap64, out, {64, 64, 1}, 128) || !encode_matrix(&q->wmap, x.dt, W7, 3 * w8, 7 * w8, {64, w8}, 128))
        return OpBuild::error;
    q->ntile = x.T <= 256 ? 1 : (x.T + 191) / 192;
    q->x = x.p; q->ld = x.ld; q->bias = bias; q->scale = scale; q->shift = shift; q->lens = lens;
    q->B = x.B; q->T = x.T; q->w8 = w8; q->dil = dil; q->dtype = x.dt;
    const int npan = w8 / 64;
    q->smem_bytes = npan * 272 * 128 + 4 * w8 * 128 + npan * 256 * 128 + 1024;
    const long long units = (long long)x.B * q->ntile;
    q->grid = (int)(units < ws_num_sms() ? units : ws_num_sms());
    const Res2Rec rec{q, x, out, W7};
    *op = plan_op(rec, [](const Res2Rec& r, cudaStream_t s) { return ws_res2_launch(r.q.get(), s); }, label_of(rec),
                  2.0 * x.B * x.T * 7.0 * 3.0 * (x.C / 8.0) * (x.C / 8.0));
    return OpBuild::built;
}

std::string trace_of(const Res2Rec& r) {
    const WsRes2Params& q = *r.q;
    return "{\"kind\":\"res2_fused\",\"es\":2," + tview("x", r.x) + "," + tview("out", r.out) + "," + tp("W7", r.W7) + "," + tp("bias", q.bias) + "," +
           tp("scale", q.scale) + "," + tp("shift", q.shift) + "," + ti("w8", q.w8) + "," + ti("dil", q.dil) + "," + tp("lens", q.lens) + ",\"launch\":{" +
           ti("ntile", q.ntile) + "," + ti("grid", q.grid) + "}}";
}

std::string label_of(const Res2Rec& r) {
    char buf[160];
    snprintf(buf, sizeof buf, "res2_fused B=%d T=%d C=%d", r.x.B, r.x.T, r.x.C);
    return buf;
}

OpBuild make_astp_op(const View& x, const View& h, const void* W2, float* stats, float var_floor, PlanOp* op, const int* lens) {
    if (x.dt == WS_F32 || h.dt != x.dt || x.C % 128 != 0 || h.C != 128 || h.ld != 128 || x.F != 1 || h.F != 1 || h.T != x.T ||
        h.B != x.B)
        return OpBuild::outside;
    auto q = std::make_shared<WsAstpParams>();
    memset(q.get(), 0, sizeof(WsAstpParams));
    if (!encode_view(&q->hmap, h, {64, 256, 1}, 128) || !encode_matrix(&q->wmap, x.dt, W2, 128, x.C, {64, 128}, 128) ||
        !encode_view(&q->xmap, x, {128, 128, 1}, 0))
        return OpBuild::error;
    q->x = x.p; q->x_ld = x.ld; q->out = stats; q->B = x.B; q->T = x.T; q->C = x.C; q->dtype = x.dt; q->lens = lens;
    q->var_floor = var_floor;
    // channel blocks per unit: the largest g whose static round-robin over the SMs stays within 8 % of the best balance
    const int nblk = x.C / 128, sms = ws_num_sms();
    double best = 0.0;
    int cand[6] = {12, 6, 4, 3, 2, 1};
    auto eff = [&](int g) {
        const long long units = (long long)x.B * (nblk / g);
        const long long grid = units < sms ? units : sms;
        return (double)units / (double)(((units + grid - 1) / grid) * grid);
    };
    for (int g : cand) if (nblk % g == 0 && eff(g) > best) best = eff(g);
    q->g = 1;
    for (int g : cand) if (nblk % g == 0 && eff(g) >= 0.92 * best) { q->g = g; break; }
    const long long units = (long long)x.B * (nblk / q->g);
    q->grid = (int)(units < sms ? units : sms);
    const AstpRec rec{q, x, h, W2};
    *op = plan_op(rec, [](const AstpRec& r, cudaStream_t s) { return ws_astp_launch(r.q.get(), s); }, label_of(rec),
                  2.0 * x.B * x.T * 128.0 * x.C);
    return OpBuild::built;
}

std::string trace_of(const AstpRec& r) {
    const WsAstpParams& q = *r.q;
    return "{\"kind\":\"astp_fused\",\"es\":2," + tview("x", r.x) + "," + tview("h", r.h) + "," + tp("W2", r.W2) + "," + tp("stats", q.out) + "," +
           tp("lens", q.lens) + "," + tf("eps", q.var_floor) + ",\"launch\":{" + ti("g", q.g) + "," + ti("grid", q.grid) + "}}";
}

std::string label_of(const AstpRec& r) {
    char buf[160];
    snprintf(buf, sizeof buf, "astp_fused B=%d T=%d C=%d g=%d grid=%d", r.q->B, r.q->T, r.q->C, r.q->g, r.q->grid);
    return buf;
}

OpBuild make_conv3x3_op(const View& x, const View& out, const void* W, const float* bias, const View* res, int relu,
                        PlanOp* op, int stride_f, int stride_t, const int* lens) {
    const int Cin = x.C, Cout = out.C, Tin = x.T, Fin = x.F, B = x.B, es = ws_esize(x.dt);
    const int F = (Fin + 2 - 3) / stride_f + 1, T = (Tin + 2 - 3) / stride_t + 1;   // output extents
    auto chan_ok = [](int c) { return c == 32 || c == 64 || c == 128; };
    if (x.dt == WS_F32 || out.dt != x.dt || (res && res->dt != x.dt) || !chan_ok(Cin) || !chan_ok(Cout) || out.B != B || out.F != F || out.T != T ||
        (stride_f != 1 && stride_f != 2) || (stride_t != 1 && stride_t != 2) || T < 1 || F < 1 || (x.ld * es) % 16 != 0 || (out.ld * es) % 16 != 0 || (res && (res->ld * es) % 16 != 0))
        return OpBuild::outside;
    auto q = std::make_shared<WsC3Params>();
    memset(q.get(), 0, sizeof(WsC3Params));
    q->B = B; q->F = F; q->T = T; q->Cin = Cin; q->Cout = Cout; q->dtype = x.dt;
    q->sf = stride_f; q->st = stride_t;
    q->row_bytes = Cin * es >= 128 ? 128 : Cin * es;
    q->kc = q->row_bytes / es;
    q->npan = Cin / q->kc;
    q->N = Cout; q->n_nt = 1;
    // ---- geometry of one ring slot / one step: first candidate whose ring (>= 4 slots) fits in shared memory
    const int budget = kC3MaxSmem;
    auto try_geom = [&](bool case_b, int tb, int n_mt) -> bool {
        q->case_b = case_b ? 1 : 0;
        q->tb = tb; q->n_mt = n_mt;
        q->n_tt = (T + tb - 1) / tb;
        q->P = tb + 2;
        if (case_b) {             // several short utterances side by side in one M tile (pitch P = T + 2)
            q->nb = std::min(B, 130 / q->P);   // nb * P - 2 <= 128
            q->single_box = 1;
            q->rows_loaded = q->nb * q->P;
        } else {                  // one utterance per slot, 1-2 M tiles along t
            q->nb = 1;
            q->single_box = q->P <= 256;
            q->rows_loaded = q->single_box ? q->P : 128 * n_mt + 2;
        }
        q->n_bg = (B + q->nb - 1) / q->nb;
        q->slot_rows = (std::max(q->rows_loaded, 128 * n_mt + 2) + 7) & ~7;
        q->sub_rows = 0;
        if (stride_t == 2) {      // even plane (tb rows) + shifted odd plane (tb + 1 rows), each in its own sub-slot
            if (case_b || n_mt != 1) return false;
            q->single_box = 1;
            q->sub_rows = (128 + 1 + 7) & ~7;
            q->slot_rows = 2 * q->sub_rows;
            q->rows_loaded = tb + (tb + 1);
        }
        if (n_mt * q->N > 256) return false;   // register accumulator of a consumer warpgroup: 64 rows x n_mt x N fp32
        // output panels (= TMA store units): 64 columns, or 32 when that is what it takes to give each of the two epilogue
        // warp sets its own unit
        q->panel_cols = std::min(64, q->N);
        if (q->panel_cols == 64 && n_mt * (q->N / 64) < 2) q->panel_cols = 32;
        q->panel_bytes = q->panel_cols * es;
        q->stg_rows = case_b ? 136 : 128;
        const int slot_bytes = q->npan * q->slot_rows * q->row_bytes;
        const int wblk = q->N * q->row_bytes, nwblk = 9 * q->npan;
        const int stg_bytes = n_mt * (q->N / q->panel_cols) * q->stg_rows * q->panel_bytes;
        // three output staging buffers with a residual (its TMA load then leads its use by a full step), two without (stores
        // are never waited for), as long as a ring of >= 5 slots still fits beside them; else one
        for (int bufs = res != nullptr ? 3 : 2; bufs >= 1; --bufs) {
            const int fixed = bufs * stg_bytes + q->N * 4 + 2048 /* alignment slack */;
            q->w_resident = (budget - fixed - nwblk * wblk) / slot_bytes >= 5;
            q->w_stages = q->w_resident ? 0 : 3;
            int R = (budget - fixed - (q->w_resident ? nwblk : q->w_stages) * wblk) / slot_bytes;
            if (R > WS_C3_MAX_RING) R = WS_C3_MAX_RING;
            if (const char* er = getenv("WS_C3_RING")) R = std::min(R, atoi(er));
            if (R < (bufs >= 2 ? 5 : 4) + (stride_f - 1)) continue;
            q->R = R;
            q->stg_bufs = bufs;
            q->smem_bytes = R * slot_bytes + (q->w_resident ? nwblk : q->w_stages) * wblk + fixed;
            return true;
        }
        return false;
    };
    bool ok = false;
    const bool strided = stride_f != 1 || stride_t != 1;
    if (T + 2 <= 66 && !strided) ok = try_geom(true, T, 1);
    if (!ok && stride_t == 2) ok = try_geom(false, std::min(T, 128), 1);
    if (!ok && stride_t == 1 && T <= 256) ok = try_geom(false, T, (T + 127) / 128);
    if (!ok && stride_t == 1) {   // t tiles of 256 (2 M tiles) or 128 (1 M tile): fewer 128-row tiles first, 256 on a tie
        const bool pref256 = 2 * ((T + 255) / 256) <= (T + 127) / 128;
        ok = pref256 ? (try_geom(false, 256, 2) || try_geom(false, 128, 1)) : (try_geom(false, 128, 1) || try_geom(false, 256, 2));
    }
    if (!ok) return OpBuild::outside;
    q->total_steps = q->n_nt * q->n_tt * q->n_bg * F;
    const int sms = ws_num_sms();
    q->grid = q->total_steps < sms ? q->total_steps : sms;
    // ---- tensor maps
    if (stride_t == 2) {   // even / odd time planes of the input as two tensors with a doubled t stride
        if (Tin < 2) return OpBuild::outside;
        const long long sF = Tin * x.ld, sB = Fin * sF;
        if (!encode_strided(&q->amap, x.dt, x.p, {Cin, (Tin + 1) / 2, Fin, B}, {2 * x.ld, sF, sB}, {q->kc, q->tb, 1, 1}, q->row_bytes) ||
            !encode_strided(&q->amap_tail, x.dt, (const char*)x.p + x.ld * es, {Cin, std::max(1, Tin / 2), Fin, B}, {2 * x.ld, sF, sB},
                            {q->kc, q->tb + 1, 1, 1}, q->row_bytes))
            return OpBuild::error;
    } else {
        if (!encode_view(&q->amap, x, {q->kc, q->single_box ? q->P : 128, 1, q->nb}, q->row_bytes) ||
            !encode_view(&q->amap_tail, x, {q->kc, 2, 1, 1}, q->row_bytes))
            return OpBuild::error;
    }
    const std::initializer_list<int> obox = {q->panel_cols, q->case_b ? q->P : 128, 1, q->case_b ? q->nb : 1};
    if (!encode_matrix(&q->wmap, x.dt, W, 9 * Cin, Cout, {q->kc, q->N}, q->row_bytes) || !encode_view(&q->omap, out, obox, q->panel_bytes))
        return OpBuild::error;
    q->rmap = q->omap;
    if (res) {   // the residual over out's extents, at its own row pitch
        View r = out;
        r.p = res->p; r.ld = res->ld;
        if (!encode_view(&q->rmap, r, obox, q->panel_bytes)) return OpBuild::error;
    }
    q->res = res ? res->p : nullptr;
    q->res_ld = res ? res->ld : 0;
    q->bias = bias;
    q->relu = relu;   // 0 none, 1 ReLU, 2 Hardtanh(0, 20)
    q->lens = lens;
    const Conv3x3Rec rec{q, x, out, res ? *res : View(), W};
    *op = plan_op(rec, [](const Conv3x3Rec& r, cudaStream_t s) { return ws_c3_launch(r.q.get(), s); }, label_of(rec),
                  2.0 * q->B * q->F * q->T * 9.0 * q->Cin * q->Cout);
    return OpBuild::built;
}

std::string trace_of(const Conv3x3Rec& r) {
    const WsC3Params& q = *r.q;
    return "{\"kind\":\"conv3x3\",\"es\":2," + tview("x", r.x) + "," + tview("out", r.out) + "," + tp("W", r.W) + "," + tp("bias", q.bias) + "," +
           (q.res ? tview("res", r.res) : std::string("\"res\":null")) + "," + ti("relu", q.relu) + "," + ti("sf", q.sf) + "," + ti("st", q.st) + "," + tp("lens", q.lens) +
           ",\"launch\":{" + ti("case_b", q.case_b) + "," + ti("nb", q.nb) + "," + ti("n_mt", q.n_mt) + "," + ti("tb", q.tb) + "," + ti("n_tt", q.n_tt) + "," + ti("R", q.R) + "," +
           ti("stg_bufs", q.stg_bufs) + "," + ti("w_resident", q.w_resident) + "," + ti("grid", q.grid) + "}}";
}

std::string label_of(const Conv3x3Rec& r) {
    const WsC3Params& q = *r.q;
    char buf[200];
    snprintf(buf, sizeof buf, "conv3x3 B=%d F=%d T=%d Cin=%d Cout=%d s=%dx%d caseB=%d nb=%d n_mt=%d R=%d res=%d", q.B, q.F, q.T, q.Cin, q.Cout, q.sf, q.st,
             q.case_b, q.nb, q.n_mt, q.R, q.res != nullptr);
    return buf;
}

extern "C" int ws_cam_smem_bytes(int nmt, int nstages);

bool cam_layer_fill(WsCamLayer* L, int dt, const void* W1, const void* Wl, const float* bn1_scale, const float* bn1_shift,
                    const float* bias2, const float* w1c_t, const float* b1c, const float* w2c_t, const float* b2c, int cin,
                    int dil) {
    memset(L, 0, sizeof(*L));
    if (cin % 32 != 0 || cin > 1024 || dil < 1 || dil > 8) { set_err("cam_dense: cin must be a multiple of 32 (<= 1024), dilation <= 8"); return false; }
    if (!encode_matrix(&L->w1map, dt, W1, cin, 128, {64, 128}, 128) || !encode_matrix(&L->wlmap, dt, Wl, 3 * 128, 32, {64, 32}, 128))
        return false;
    L->bn1_scale = bn1_scale; L->bn1_shift = bn1_shift; L->bias2 = bias2;
    L->w1c_t = w1c_t; L->b1c = b1c; L->w2c_t = w2c_t; L->b2c = b2c;
    L->cin = cin; L->dil = dil;
    return true;
}

OpBuild make_cam_dense_op(const View& X, const WsCamLayer* layers_dev, const std::vector<WsCamLayer>& layers,
                          const std::vector<std::array<const void*, 2>>& weights, int l0, int l1, PlanOp* op, const int* lens) {
    const int T = X.T, B = X.B;
    if (X.dt == WS_F32 || X.F != 1 || T < 1 || T > 512 || (X.ld * ws_esize(X.dt)) % 16 != 0)
        return OpBuild::outside;
    auto q = std::make_shared<WsCamParams>();
    memset(q.get(), 0, sizeof(WsCamParams));
    q->layers = layers_dev; q->l0 = l0; q->l1 = l1; q->lens = lens;
    q->B = B; q->T = T; q->nmt = (T + 127) / 128; q->seg_len = kCamSegLen; q->dtype = X.dt;
    q->hrows = 16 + 128 * q->nmt;
    int nst = 6;
    while (nst >= 2 && ws_cam_smem_bytes(q->nmt, nst) > kCamMaxSmem) --nst;
    if (nst < 2) return OpBuild::outside;
    q->nstages = nst;
    q->smem_bytes = ws_cam_smem_bytes(q->nmt, nst);
    q->grid = B;
    if (!encode_view(&q->xmap, X, {64, 128, 1}, 128) || !encode_view(&q->omap, X, {32, 128, 1}, 64)) return OpBuild::error;
    const CamRec rec{q, X, {layers.begin() + l0, layers.begin() + l1}, {weights.begin() + l0, weights.begin() + l1}};
    *op = plan_op(rec, [](const CamRec& r, cudaStream_t s) { return ws_cam_launch(r.q.get(), s); }, label_of(rec));
    return OpBuild::built;
}

std::string trace_of(const CamRec& r) {   // layers [l0, l1) over the concat buffer, each with what its descriptor points at
    const WsCamParams& q = *r.q;
    std::string j = "{\"kind\":\"cam_dense\"," + ti("es", ws_esize(q.dtype)) + "," + tview("X", r.X) + "," + tp("lens", q.lens) + "," + ti("seg_len", q.seg_len) +
                    ",\"layers\":[";
    for (size_t k = 0; k < r.layers.size(); ++k) {
        const WsCamLayer& L = r.layers[k];
        j += std::string(k ? "," : "") + "{" + tp("W1", r.weights[k][0]) + "," + tp("Wl", r.weights[k][1]) + "," + tp("bn1_scale", L.bn1_scale) + "," +
             tp("bn1_shift", L.bn1_shift) + "," + tp("bias2", L.bias2) + "," + tp("w1c_t", L.w1c_t) + "," + tp("b1c", L.b1c) + "," +
             tp("w2c_t", L.w2c_t) + "," + tp("b2c", L.b2c) + "," + ti("cin", L.cin) + "," + ti("dil", L.dil) + "}";
    }
    return j + "],\"launch\":{" + ti("nmt", q.nmt) + "," + ti("nstages", q.nstages) + "," + ti("grid", q.grid) + "}}";
}

std::string label_of(const CamRec& r) {
    char buf[160];
    snprintf(buf, sizeof buf, "cam_dense layers %d..%d B=%d T=%d", r.q->l0, r.q->l1 - 1, r.q->B, r.q->T);
    return buf;
}

}  // namespace ws

// ------------------------------------------------------------------------------------------------ C ABI: ws_conv
extern "C" int ws_conv(const ws_conv_desc* d, void* stream) {
    using namespace ws;
    if (d == nullptr) { set_err("ws_conv: null descriptor"); return 1; }
    if (d->use_tc < 0 || d->use_tc == 1) {
        set_err("ws_conv: use_tc must be 0 (FFMA) or 2..4 (tensor cores); 1, the one-tile-per-CTA tensor-core kernel, was removed");
        return 1;
    }
    View x;
    x.p = const_cast<void*>(d->x); x.plo = const_cast<void*>(d->x_lo); x.B = d->B; x.F = d->F; x.T = d->T; x.C = d->Cin; x.ld = d->x_ld; x.dt = d->dtype;
    ConvSpec s;
    s.dt = d->dtype;
    int Fo = 0, To = 0;
    const int K = add_conv_taps(s, x, d->kf, d->kt, d->dil_f, d->dil_t, d->pad_f, d->pad_t, d->stride_f, d->stride_t, 0,
                                &Fo, &To);
    if (K < 0) { set_err("ws_conv: too many source planes"); return 1; }
    s.W = d->w; s.Ktot = K; s.Cout = d->Cout;
    s.W_lo = d->w_lo; s.split = (d->x_lo != nullptr);
    s.B = d->B; s.F = Fo; s.T = To;
    s.dense_pointwise = (d->kf == 1 && d->kt == 1 && d->stride_f == 1 && d->stride_t == 1 && d->pad_f == 0 &&
                         d->pad_t == 0);
    View o;
    o.p = d->out; o.plo = d->out_lo; o.B = d->B; o.F = Fo; o.T = To; o.C = d->Cout; o.ld = d->out_ld; o.dt = d->dtype;
    fill_epi_out(s.epi, o);
    s.epi.bias = d->bias; s.epi.act1 = d->act1; s.epi.scale = d->scale; s.epi.shift = d->shift;
    s.epi.res = d->res; s.epi.res_ld = d->res_ld; s.epi.act2 = d->act2;
    s.epi.colsum = d->colsum; s.epi.colsum_T = d->colsum ? To : 0;
    { const char* eg = getenv("WS_EPI_GENERIC"); s.epi_generic = eg != nullptr && atoi(eg) != 0; }
    PlanOp op;
    bool done = false;
    if (d->use_tc >= 4 && d->kf == 3 && d->kt == 3 && d->dil_f == 1 && d->dil_t == 1 && d->pad_f == 1 && d->pad_t == 1 &&
        d->stride_f >= 1 && d->stride_f <= 2 && d->stride_t >= 1 && d->stride_t <= 2 && d->scale == nullptr && d->x_lo == nullptr && d->colsum == nullptr &&
        (d->act1 == 0 || d->res == nullptr) && (d->act1 <= 1 || d->act1 == WS_ACT_RELU20) && (d->act2 <= 1 || d->act2 == WS_ACT_RELU20) &&
        (d->act1 == 0 || d->act2 == 0 || d->act1 == d->act2)) {
        // halo-resident 3x3 kernel: act(conv + bias [+ res]); with a residual the activation is act2, else act1 (or act2)
        View r = o;
        r.p = const_cast<void*>(d->res); r.ld = d->res_ld;
        const int a = d->act1 | d->act2;   // one of them is set, or both to the same (idempotent) activation
        const OpBuild made = make_conv3x3_op(x, o, d->w, d->bias, d->res ? &r : nullptr, a == WS_ACT_RELU20 ? 2 : (a != 0 ? 1 : 0), &op,
                                             d->stride_f, d->stride_t);
        if (made == OpBuild::error) return 1;
        done = made == OpBuild::built;
    }
    if (!done && !make_conv_op(s, d->use_tc >= 4 ? 3 : d->use_tc, &op)) return 1;
    const char* m = op.run((cudaStream_t)stream);
    if (m != nullptr) { set_err(std::string("ws_conv launch: ") + m); return 1; }
    return 0;
}

extern "C" const char* ws_last_error(void) { return ws::get_err().c_str(); }
extern "C" int ws_version(void) { return 100; }
