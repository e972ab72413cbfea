// Launch plans of the 2-D residual families (wenet-e2e/wespeaker, wespeaker/models/): ResNet, Res2Net / ERes2Net, SimAM-ResNet
// and Gemini DF-ResNet, with the stem, blocks and TSTP tail they share.
#include "ws_plan.h"

namespace ws {

// ----------------------------------------------------------------------------------------------- 2-D residual blocks
// BasicBlock (resnet.py:35-69) / BasicResBlock (campplus.py:245-279): eval BN folded into the conv weights, the
// 1x1 strided shortcut conv is merged into conv2's GEMM as one extra K range, residual/ReLU in the epilogue.
// `lvl`: stride level of the block's OUTPUT (length-masked plans: frame counts b.lens(lvl)); the time stride st_ is 1 or 2
View basic_block(Builder& b, const std::string& p, const View& x, int cout, int sf, int st_, View hbuf, View obuf, int lvl) {
    std::vector<float> s1, h1, s2, h2, w1, w2;
    View none;
    if (!b.w.bn(p + ".bn1", true, s1, h1) || !b.w.bn(p + ".bn2", true, s2, h2) || !b.w.pack_conv(p + ".conv1.weight", &s1, w1) ||
        !b.w.pack_conv(p + ".conv2.weight", &s2, w2))
        return none;
    const int Fo = (x.F + 2 - 3) / sf + 1, To = (x.T + 2 - 3) / st_ + 1;
    const View h = hbuf.shaped(x.B, Fo, To, cout), o = obuf.shaped(x.B, Fo, To, cout);
    if (!b.conv3x3(x, h, b.w.act("w:" + p + ".conv1", w1), b.w.f32("bnh:" + p + ".bn1", h1), WS_ACT_RELU, sf, st_, lvl)) return none;
    const bool has_sc = b.e.sd.count(p + ".shortcut.0.weight") != 0;
    if (b.fused(b.e.opts.conv3x3) && (cout == 32 || cout == 64 || cout == 128)) {
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
    b.push(WsStem{b.p.feats_in, wd, b.w.f32("bnh:" + bnkey, h), o, b.lens(0)}, ws_launch_stem, "stem");
    return o;
}

// TSTP over the last feature map + the segment layer(s) (resnet.py:187-204; the same tail closes Res2Net / ERes2Net,
// res2net.py:186-199, eres2net.py:379-391, Gemini DF-ResNet and XVEC)
// two_layers: embed_b = seg_2(seg_bn_1(relu(seg_1(stats)))) (two_emb_layer), else embed_a = seg_1(stats)
// lvl: stride level of `cur` in length-masked plans (three stride-2 layers in ResNet / Res2Net, one in Gemini DF-ResNet)
bool resnet_tail(Builder& b, const View& cur, bool two_layers, int lvl) {
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
    const std::vector<View> bufs = b.ring(e.cfg.bottleneck ? 4 : 3, (size_t)B * Fd * T * m * (e.cfg.bottleneck ? 4 : 1));
    if (!b.good()) return false;
    View cur = stem(b, "conv1.weight", "bn1", bufs[0]);
    int ci = 0;
    for (int li = 1; li <= 4 && b.good(); ++li) {
        const int cout = m << (li - 1);
        for (int bi = 0; bi < e.cfg.num_blocks[li - 1] && b.good(); ++bi) {
            const int s = (bi == 0 && li > 1) ? 2 : 1;
            const std::string p = "layer" + std::to_string(li) + "." + std::to_string(bi);
            const int lvl = li - 1, lvl_in = (s == 2) ? li - 2 : li - 1;   // stride level = number of stride-2 layers passed
            if (e.cfg.bottleneck) {   // x lives in bufs[ci]; the two intermediates and the output rotate through the other three
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
    return resnet_tail(b, cur, e.opts.two_emb_layer);
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
    b.push(WsAffCombine{x, y, att, out}, ws_launch_aff_combine, "aff_combine");
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
static View res2_block(Builder& b, const ModelCfg& c, const std::string& p, const View& x, int planes, int stride, int kind, Res2Bufs& bf, View obuf,
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

bool build_res2net(Builder& b) {
    ws_engine& e = b.e;
    const ModelCfg& c = e.cfg;
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
        for (int bi = 0; bi < e.cfg.num_blocks[li - 1] && b.good(); ++bi) {
            const std::string p = "layer" + std::to_string(li) + "." + std::to_string(bi);
            View o = res2_block(b, c, p, cur, planes, bi == 0 ? stride : 1, kind, bf, bf.xo[bi & 1], li - 1,
                                c.fuse && bi == e.cfg.num_blocks[li - 1] - 1);
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
    return resnet_tail(b, cur, e.opts.two_emb_layer);
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
    const WsMapStrides rs{(long long)res.F * res.T * res.ld, (long long)res.T * res.ld, res.ld};
    const int* l = b.lens(lvl);
    b.push(WsSimamStats{y, partial, stats, l}, ws_launch_simam_stats, "simam_stats");
    b.p.extra_launches += 1;   // partials + merge
    b.push(WsSimamApply{y, stats, kSimamLambda, res.p, rs, out.p, (float*)out.plo, os, l}, ws_launch_simam_apply, "simam_apply");
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
        for (int bi = 0; bi < e.cfg.num_blocks[li - 1]; ++bi) {
            const bool last = li == 4 && bi == e.cfg.num_blocks[3] - 1;
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
    b.push(WsDwconv3x3{x, w9, shift, out, b.lens(lvl)}, ws_launch_dwconv3x3, "dwconv3x3");
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
        for (int j = 0; j < e.cfg.num_blocks[i - 1]; ++j) {
            View nx = gemini_block(b, "stages." + std::to_string(i - 1) + "." + std::to_string(j), cur, bufs[(ci + 1) % 4], bufs[(ci + 2) % 4],
                                   bufs[(ci + 3) % 4], lvl);
            if (!b.good() || nx.p == nullptr) return false;
            ci = (ci + 3) % 4;
            cur = nx;
        }
    }
    return resnet_tail(b, cur, e.opts.two_emb_layer, 1);
}

}  // namespace ws
