// ECAPA-TDNN launch plans (ecapa_tdnn.py:29-234, pooling_layers.py:67-148 in wenet-e2e/wespeaker, wespeaker/models/).
#include "ws_plan.h"

namespace ws {

// ----------------------------------------------------------------------------------------------- ECAPA-TDNN
// ecapa_tdnn.py:160-234.  Channels-last buffers; torch.cat is free (layer outputs are written into slices of one
// (B,T,3C) buffer), Res2 "sp + spx[i]" is produced by the previous conv's epilogue (out2 = out + add2).
bool build_ecapa(Builder& b) {
    ws_engine& e = b.e;
    const int B = b.p.B, T = b.p.T, C = e.cfg.channels, w8 = C / 8, Fd = e.feat_dim, E = e.embed_dim;
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
    if (b.fused(e.opts.se_fused && e.opts.se_colsum) && T >= 128 && (C == 512 || C == 1024) &&
        !b.p.masked)   // (column sums would include padding rows)
        se_colsum = b.f32((size_t)2 * (((size_t)B * T + 63) / 64) * C);
    for (int L = 2; L <= 4 && b.good(); ++L) {
        const int d = L;
        const std::string pf = "layer" + std::to_string(L) + ".se_res2block";
        conv_relu_bn(pf + ".0", xin, tA, 1, 1, 0);
        b.zero_tail(tA, 0);   // (masked plans) the dilated Res2 convs read tA across time
        // Res2Conv1dReluBn (ecapa_tdnn.py:29-78): 7 dependent dilated k=3 convs on w8-channel groups
        bool fused = false;
        if (b.fused(e.opts.res2_fused)) {
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
            const OpBuild r = make_res2_op(tA, tB, b.w.act("w7:" + pf, w7), b.w.f32("b7:" + pf, b7), b.w.f32("s7:" + pf, s7),
                                           b.w.f32("h7:" + pf, h7), w8, d, &op, b.lens(0));
            if (r == OpBuild::built) {
                b.push(std::move(op));
                fused = true;
            } else if (r == OpBuild::error) {
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
        if (e.opts.se_fused && (C == 512 || C == 1024)) {
            const int H = 128;   // SE bottleneck width
            const HostT* w2 = b.w.get(pf + ".3.linear2.weight");   // (C, H) -> transposed (H, C) for coalesced reads
            if (!w2) break;
            std::vector<float> w2t((size_t)H * C);
            for (int c = 0; c < C; ++c)
                for (int h = 0; h < H; ++h) w2t[(size_t)h * C + c] = w2->v[(size_t)c * H + h];
            const float* w1d = b.w.vec(pf + ".3.linear1.weight");
            const float* b1d = b.w.vec(pf + ".3.linear1.bias");
            const float* w2d = b.w.f32("w2t:" + pf, w2t);
            const float* b2d = b.w.vec(pf + ".3.linear2.bias");
            b.push(WsSeGate{tC, w1d, b1d, w2d, b2d, H, segate, se_colsum, b.lens(0)}, ws_launch_se_gate, "se_gate");
        } else {
            b.tstats(tC, nullptr, nullptr, semean, C, -1);
            b.linear(semean, C, nullptr, 0, 1, b.w.vec(pf + ".3.linear1.weight"), b.w.vec(pf + ".3.linear1.bias"), sehid, 128, B,
                     C, 128, WS_ACT_RELU);
            b.linear(sehid, 128, nullptr, 0, 1, b.w.vec(pf + ".3.linear2.weight"), b.w.vec(pf + ".3.linear2.bias"), segate, C,
                     B, 128, C, WS_ACT_SIGMOID);
        }
        {
            const View o = cat.ch((L - 2) * C, C);
            b.push(WsScaleResidual{tC, segate, xin, o}, ws_launch_scale_residual, "scale_residual");
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
        if (e.cfg.glob) {
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
        if (e.opts.emb_bn && !b.w.bn("bn2", true, s2, h2)) return false;
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

}  // namespace ws
