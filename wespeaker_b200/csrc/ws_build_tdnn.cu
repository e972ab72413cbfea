// Launch plans of the TDNN families: XVEC (tdnn.py:23-117) and CAM++ (campplus.py:55-413) (wenet-e2e/wespeaker,
// wespeaker/models/).
#include "ws_plan.h"

namespace ws {

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
    const int nseg = (Tp + kCamSegLen - 1) / kCamSegLen;
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
    // Fused dense layers (ws_cam_dense.cu): one launch per CAMDenseTDNNLayer (or per block with cam_block = 1) instead of four
    const bool cam_fused = b.fused(e.opts.cam_fused) && Tp <= 512;
    for (int bl = 0; bl < 3 && b.good(); ++bl) {
        bool fused_done = false;
        if (cam_fused) {
            std::vector<WsCamLayer> hl((size_t)nl[bl]);
            std::vector<std::array<const void*, 2>> hw((size_t)nl[bl]);   // the (W1, Wl) each descriptor's tensor maps encode
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
                hw[(size_t)j - 1] = {W1d, Wld};
            }
            if (!okl || !b.good()) { b.ok = false; break; }
            const WsCamLayer* ldev = (const WsCamLayer*)b.w.upload("camlayers:" + std::to_string(bl), hl.data(), hl.size() * sizeof(WsCamLayer));
            if (!b.good()) break;
            const bool whole = e.opts.cam_block;
            fused_done = true;
            for (int j = 0; j < nl[bl]; j += whole ? nl[bl] : 1) {
                const int j1 = whole ? nl[bl] : j + 1;
                PlanOp op;
                const OpBuild r = make_cam_dense_op(X[bl], ldev, hl, hw, j, j1, &op, b.lens(1));
                if (r == OpBuild::built) b.push(std::move(op));
                else if (r == OpBuild::outside && j == 0) { fused_done = false; break; }
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
            b.push(WsBnRelu{X[bl].ch(0, cin), b.w.f32("bns:" + p + ".n1", s1), b.w.f32("bnh:" + p + ".n1", h1), sv}, ws_launch_bnrelu, "bnrelu");
            // linear1 (1x1, no bias) + nonlinear2 (BN folded) + ReLU -> hid
            WsEpi e1{};
            e1.bias = b.w.f32("bnh:" + p + ".n2", h2);
            e1.act1 = WS_ACT_RELU;
            b.conv_simple(sv, hid, b.w.act("w:" + p + ".linear1", w1), 1, 1, 1, 1, 0, 0, 1, 1, e1);
            // CAM context mask (campplus.py:108-115): sigmoid(W2 relu(W1 (mean_T + segmean_100)))
            {
                const float* w1c = b.w.vec(p + ".cam_layer.linear1.weight");
                const float* b1c = b.w.vec(p + ".cam_layer.linear1.bias");
                const float* w2c = b.w.vec(p + ".cam_layer.linear2.weight");
                const float* b2c = b.w.vec(p + ".cam_layer.linear2.bias");
                const size_t cam_smem = (size_t)((bnc / 2) * bnc + nseg * bnc + 16 * bnc + nseg * (bnc / 2) + bnc) * 4;
                if (cam_smem <= 48 * 1024) {
                    b.push(WsCamGate{hid, kCamSegLen, w1c, b1c, w2c, b2c, bnc / 2, growth, cgate}, ws_launch_cam_gate, "cam_gate");
                } else {  // very long utterances: unfused path
                    b.push(WsSegMeans{hid, kCamSegLen, cmean, csegm}, ws_launch_seg_means, "seg_means");
                    b.linear(csegm, bnc, cmean, bnc, nseg, w1c, b1c, chid, bnc / 2, B * nseg, bnc, bnc / 2, WS_ACT_RELU);
                    b.linear(chid, bnc / 2, nullptr, 0, 1, w2c, b2c, cgate, growth, B * nseg, bnc / 2, growth, WS_ACT_SIGMOID);
                }
            }
            // linear_local (k3, dilated, no bias) * mask -> appended to the concat buffer
            WsEpi e2{};
            e2.gate = cgate; e2.gate_ld = growth; e2.gate_seg = kCamSegLen; e2.gate_nseg = nseg;
            b.conv_simple(hid, X[bl].ch(cin, growth), b.w.act("w:" + p + ".local", wl), 1, 3, 1, dil[bl], 0, dil[bl], 1, 1, e2);
        }
        if (!b.good()) break;
        // TransitLayer (campplus.py:204-218): BN-ReLU-Conv1x1 (no bias)
        const std::string tk = "xvector.transit" + std::to_string(bl + 1);
        std::vector<float> s, h, wt;
        if (!b.w.bn(tk + ".nonlinear.batchnorm", true, s, h) || !b.w.pack_conv(tk + ".linear.weight", nullptr, wt)) break;
        const View sv = scratch.shaped(B, 1, Tp, cmax[bl]);
        b.push(WsBnRelu{X[bl], b.w.f32("bns:" + tk, s), b.w.f32("bnh:" + tk, h), sv}, ws_launch_bnrelu, "bnrelu");
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

}  // namespace ws
