"""Edge-case launch plans for the per-op checker (tests/test_plan_ops_gpu.py) and the branch classifier that says which kernel
geometry each op of a plan takes.  The kernels pick their geometry from (B, T, frame counts) in host code: utterances side by
side in one M tile, tile counts and tails, chunk edges, fused-vs-unfused fallbacks.  Each case below is chosen to reach some
of those branches, and tests/test_plan_edges.py checks on the CPU that every branch in BRANCHES is reached by some case, so
moving a threshold names the branch that lost its coverage."""


def op_branches(op):
    """the kernel-geometry branch keys one traced op takes: the geometry the host chose (the trace's "launch"), and the
    extents where a kernel's own constants decide"""
    tr = op["trace"]
    kind, g = tr["kind"], tr.get("launch", {})
    out = set()
    masked = bool(tr.get("lens"))
    if kind == "conv3x3":       # make_conv3x3_op (ws_conv_host.cu)
        B, T = tr["out"]["B"], tr["out"]["T"]
        if g["case_b"]:
            out.add("conv3x3:caseB")
            if B % g["nb"]:
                out.add("conv3x3:caseB-ragged" + ("-masked" if masked else ""))
        elif tr["st"] == 2:
            out.add("conv3x3:stride2-ttiles=%s" % ("1" if g["n_tt"] == 1 else ">1"))
        elif g["n_tt"] == 1:
            out.add(f"conv3x3:n_mt={g['n_mt']}")
            if g["tb"] + 2 > 256:
                out.add("conv3x3:multibox")
        else:
            out.add(f"conv3x3:ttile={g['tb']}")
            if T % g["tb"] == 1:
                out.add(f"conv3x3:ttile={g['tb']}-tail=1")
        if T == 1:
            out.add("conv3x3:T=1")
    elif kind == "conv":        # make_conv_op / tc2_geometry (ws_conv_host.cu)
        pos = tr["B"] * tr["F"] * tr["T"]
        if g["kernel"] == "tc3":
            out.add("conv:cluster")
            if ((pos + 127) // 128) % 2:
                out.add("conv:cluster-odd-tiles")
            if g["bn"] == 256:      # the 256-wide N tile on clusters
                out.add("conv:bn=256")
        if g["kernel"] == "tc2" and 132 * 128 - 128 <= pos < 132 * 128:
            out.add("conv:just-below-cluster")
        flat = len(tr["taps"]) == 1 and tr["taps"][0][2] == 0 and tr["taps"][0][3] == 0
        if flat and pos % 128 == 1:
            out.add("conv:tail=1")
        if not flat and tr["F"] > 1:
            out.add("conv:nonflat")
        if sum(t[5] for t in tr["taps"]) < tr["Ktot"]:      # taps on empty parity planes dropped (1-frame inputs)
            out.add("conv:empty-plane")
        if tr.get("colsum"):
            out.add("conv:se-colsum")
    elif kind == "res2_fused":  # make_res2_op: time tiles
        out.add("res2:ntile=%d" % g["ntile"])
        if tr["x"]["T"] < 7 * tr["dil"]:
            out.add("res2:T<7dil")
    elif kind == "astp_fused":  # 256-frame online-softmax chunks
        T = tr["x"]["T"]
        n = (T + 255) // 256
        out.add(f"astp_fused:chunks={min(n, 3)}")
        if n > 1 and T % 256 == 1:
            out.add("astp_fused:tail=1")
    elif kind == "astp_stats":  # the kernel the plan chose (ws_astp_stats_kernel)
        out.add("astp_stats:" + g["kernel"])
    elif kind == "se_gate":     # two utterances per CTA
        if tr["x"]["B"] % 2:
            out.add("se_gate:odd-B")
        if tr["x"]["T"] < 128:
            out.add("se_gate:T<128")
    elif kind == "tstats":      # the kernel the plan chose (ws_tstats_kernel)
        k = g["kernel"]
        if k == "tstats8":
            T = tr["x"]["T"]    # tstats8's 4-wide loop runs while t + 48 < T, t = slice (0..15) + 64 k
            out.add("tstats8:" + ("T<=48" if T <= 48 else "49<=T<64" if T < 64 else "T>=64"))
        else:
            out.add("tmean8" if k == "tmean8" else "tstats:" + k)
    elif kind == "linear":      # the kernel the plan chose (ws_linear_rows_plan); split-K when the launch would not fill the SMs
        out.add("linear:" + g["kernel"])
        if tr.get("wsp"):
            out.add("linear:split-K")
    elif kind == "stem":        # 128-frame tiles
        T = tr["out"]["T"]
        out.add("stem:T<128" if T < 128 else "stem:ragged-tiles" if T % 128 else "stem:whole-tiles")
    elif kind == "cam_dense":   # make_cam_dense_op: M tiles of 128 frames, T' <= 512
        out.add(f"cam_dense:nmt={g['nmt']}")
        if tr["X"]["T"] % 100 == 1:
            out.add("cam_dense:seg-tail=1")
    elif kind in ("cam_gate", "seg_means"):     # the dense layers unfused (T' > 512 in 16-bit plans)
        if tr["es"] == 2:
            out.add("cam_dense:fallback")
        if tr["x"]["T"] % 100 == 1:
            out.add("cam_gate:seg-tail=1")
    elif kind == "dwconv3x3":   # <= 32-frame tiles
        T = tr["x"]["T"]
        out.add("dwconv:T=1" if T == 1 else "dwconv:T<32" if T < 32 else "dwconv:ragged-ttile" if T % 32 else "dwconv:whole-ttiles")
    elif kind == "simam_stats":     # 32 time slices
        T = tr["x"]["T"]
        out.add("simam:T=1" if T == 1 else "simam:T<32" if T < 32 else "simam:T>=32")
    if masked and kind != "lens_derive":
        out.add(f"{kind}:masked")
    return out


def case_branches(ops, n_frames):
    """every branch key the ops of a plan take, plus the frame-count edges of a masked case"""
    out = set()
    for op in ops:
        out |= op_branches(op)
    for n in n_frames or ():
        if n in (1, 2):
            out.add(f"mask:len={n}")
        if n in (128, 129, 256, 257):
            out.add("mask:tile-edge")
    return out


# branches that depend on the SM count or the number of co-resident clusters: the plan-check engine (no device) cannot
# predict them, so only the GPU test asserts them, from the real engine's traces
DEVICE_ONLY = {"conv:bn=256", "linear:split-K"}

# every branch some edge case must reach
BRANCHES = {
    "conv3x3:caseB", "conv3x3:caseB-ragged", "conv3x3:caseB-ragged-masked", "conv3x3:n_mt=1", "conv3x3:n_mt=2",
    "conv3x3:multibox", "conv3x3:ttile=128", "conv3x3:ttile=128-tail=1", "conv3x3:ttile=256", "conv3x3:stride2-ttiles=1",
    "conv3x3:stride2-ttiles=>1", "conv3x3:T=1", "conv3x3:masked",
    "conv:cluster", "conv:cluster-odd-tiles", "conv:just-below-cluster", "conv:tail=1", "conv:nonflat", "conv:empty-plane",
    "conv:se-colsum", "conv:bn=256",
    "res2:ntile=1", "res2:ntile=2", "res2:ntile=3", "res2:T<7dil", "res2_fused:masked",
    "astp_fused:chunks=1", "astp_fused:chunks=2", "astp_fused:chunks=3", "astp_fused:tail=1", "astp_fused:masked",
    "astp_stats:stats4", "astp_stats:scalar",
    "se_gate:odd-B", "se_gate:T<128", "se_gate:masked",
    "tmean8", "tstats8:T<=48", "tstats8:49<=T<64", "tstats8:T>=64", "tstats:scalar", "tstats:masked",
    "linear:rows64", "linear:rows16", "linear:split-K",
    "stem:T<128", "stem:ragged-tiles", "stem:masked",
    "cam_dense:nmt=1", "cam_dense:nmt=2", "cam_dense:nmt=3", "cam_dense:nmt=4", "cam_dense:seg-tail=1", "cam_dense:fallback",
    "cam_dense:masked",
    "dwconv:T=1", "dwconv:T<32", "dwconv:ragged-ttile", "dwconv3x3:masked",
    "simam:T=1", "simam:T<32", "simam:T>=32", "simam_stats:masked",
    "zero_tail:masked", "mask:len=1", "mask:len=2", "mask:tile-edge",
}

# (model, precision, B, T, frame counts of a masked batch or None, engine options, branches it must reach)
EDGE_CASES = {
    # ResNet34: 3x3 geometry over T (caseB up to T = 64, one or two M tiles up to 256, then 128- or 256-row time tiles)
    "r34_fp16_T1": ("ResNet34", "fp16", 44, 1, None, {}, {"conv3x3:T=1", "conv3x3:caseB-ragged", "conv:empty-plane", "tstats8:T<=48"}),
    "r34_fp16_T2": ("ResNet34", "fp16", 2, 2, None, {}, {"conv3x3:caseB", "conv:empty-plane"}),
    "r34_fp16_T9": ("ResNet34", "fp16", 12, 9, None, {}, {"conv3x3:caseB-ragged", "conv:nonflat"}),
    "r34_fp16_T129": ("ResNet34", "fp16", 1, 129, None, {}, {"conv3x3:n_mt=2", "conv3x3:stride2-ttiles=1", "stem:ragged-tiles"}),
    "r34_fp16_T255": ("ResNet34", "fp16", 1, 255, None, {}, {"conv3x3:multibox"}),
    "r34_fp16_T257": ("ResNet34", "fp16", 1, 257, None, {}, {"conv3x3:ttile=128-tail=1", "conv3x3:stride2-ttiles=>1"}),
    "r34_fp16_T512": ("ResNet34", "fp16", 1, 512, None, {}, {"conv3x3:ttile=256"}),
    "r34_fp16_T513": ("ResNet34", "fp16", 1, 513, None, {}, {"conv3x3:ttile=128", "tstats8:T>=64"}),
    "r34_fp32_T1": ("ResNet34", "fp32", 2, 1, None, {}, {"tstats:scalar"}),
    "r34_tf32x3_T1": ("ResNet34", "tf32x3", 2, 1, None, {}, {"tstats:scalar"}),
    # ECAPA-TDNN-512: Res2 time tiles, ASTP chunks, SE squeeze, conv-GEMM clusters and tails
    "ecapa512_bf16_T1": ("ECAPA_TDNN_c512", "bf16", 3, 1, None, {}, {"res2:T<7dil", "astp_fused:chunks=1", "se_gate:odd-B", "se_gate:T<128"}),
    "ecapa512_bf16_T127": ("ECAPA_TDNN_c512", "bf16", 3, 127, None, {}, {"se_gate:T<128", "se_gate:odd-B"}),
    "ecapa512_bf16_T128": ("ECAPA_TDNN_c512", "bf16", 2, 128, None, {}, {"conv:se-colsum", "res2:ntile=1"}),
    "ecapa512_bf16_T257": ("ECAPA_TDNN_c512", "bf16", 1, 257, None, {}, {"res2:ntile=2", "astp_fused:chunks=2", "astp_fused:tail=1"}),
    "ecapa512_bf16_T385": ("ECAPA_TDNN_c512", "bf16", 1, 385, None, {}, {"res2:ntile=3"}),
    "ecapa512_bf16_T513": ("ECAPA_TDNN_c512", "bf16", 1, 513, None, {}, {"astp_fused:chunks=3", "astp_fused:tail=1"}),
    "ecapa512_bf16_pos129": ("ECAPA_TDNN_c512", "bf16", 3, 43, None, {}, {"conv:tail=1", "linear:split-K"}),
    "ecapa512_bf16_pos16832": ("ECAPA_TDNN_c512", "bf16", 64, 263, None, {}, {"conv:just-below-cluster"}),
    "ecapa512_bf16_pos16896": ("ECAPA_TDNN_c512", "bf16", 64, 264, None, {}, {"conv:cluster"}),
    "ecapa512_bf16_pos17024": ("ECAPA_TDNN_c512", "bf16", 64, 266, None, {}, {"conv:cluster-odd-tiles", "conv:bn=256", "linear:rows64"}),
    "ecapa512_bf16_unfused_T256": ("ECAPA_TDNN_c512", "bf16", 1, 256, None, {"astp_fused": 0, "se_fused": 0}, {"astp_stats:stats4", "tmean8"}),
    "ecapa512_bf16_unfused_T257": ("ECAPA_TDNN_c512", "bf16", 1, 257, None, {"astp_fused": 0}, {"astp_stats:scalar"}),
    # global-context ECAPA: statistics kernels at the 4-wide loop's edges
    "glob512_fp16_T1": ("ECAPA_TDNN_GLOB_c512", "fp16", 2, 1, None, {}, {"tstats8:T<=48"}),
    "glob512_fp16_T49": ("ECAPA_TDNN_GLOB_c512", "fp16", 2, 49, None, {}, {"tstats8:49<=T<64"}),
    "glob512_fp16_T65": ("ECAPA_TDNN_GLOB_c512", "fp16", 2, 65, None, {}, {"tstats8:T>=64"}),
    "glob512_tf32x3_T1": ("ECAPA_TDNN_GLOB_c512", "tf32x3", 2, 1, None, {}, {"tstats:scalar"}),
    "glob512_tf32x3_T65": ("ECAPA_TDNN_GLOB_c512", "tf32x3", 2, 65, None, {}, {"tstats:scalar"}),
    # CAM++: dense blocks over T' = ceil(T / 2) frames, 100-frame context segments, unfused above 512
    "campplus_bf16_T201": ("CAMPPlus", "bf16", 1, 201, None, {}, {"cam_dense:nmt=1", "cam_dense:seg-tail=1"}),
    "campplus_bf16_T257": ("CAMPPlus", "bf16", 1, 257, None, {}, {"cam_dense:nmt=2"}),
    "campplus_bf16_T513": ("CAMPPlus", "bf16", 1, 513, None, {}, {"cam_dense:nmt=3"}),
    "campplus_bf16_T1024": ("CAMPPlus", "bf16", 1, 1024, None, {}, {"cam_dense:nmt=4"}),
    "campplus_bf16_T1025": ("CAMPPlus", "bf16", 1, 1025, None, {}, {"cam_dense:fallback"}),
    # depthwise 3x3 (<= 32-frame tiles) and SimAM (32 time slices)
    "gemini60_fp16_T1": ("Gemini_DF_ResNet60", "fp16", 2, 1, None, {}, {"dwconv:T=1"}),
    "gemini60_fp16_T20": ("Gemini_DF_ResNet60", "fp16", 2, 20, None, {}, {"dwconv:T<32"}),
    "gemini60_fp16_T33": ("Gemini_DF_ResNet60", "fp16", 2, 33, None, {}, {"dwconv:ragged-ttile"}),
    "simam34_bf16_T1": ("SimAM_ResNet34_ASP", "bf16", 2, 1, None, {}, {"simam:T=1"}),
    "simam34_bf16_T20": ("SimAM_ResNet34_ASP", "bf16", 2, 20, None, {}, {"simam:T<32"}),
    "simam34_bf16_T33": ("SimAM_ResNet34_ASP", "bf16", 2, 33, None, {}, {"simam:T>=32"}),
    # length masks: 1- and 2-frame utterances, tile edges, odd halving chains (17 -> 9 -> 5 -> 3), ragged caseB groups
    "r34_fp16_masked_edges": ("ResNet34", "fp16", 6, 257, [257, 256, 129, 128, 1, 2], {},
                              {"conv3x3:masked", "zero_tail:masked", "stem:masked", "tstats:masked", "mask:len=1", "mask:tile-edge"}),
    "r34_fp16_masked_caseB": ("ResNet34", "fp16", 7, 17, [17, 1, 2, 9, 16, 5, 3], {}, {"conv3x3:caseB-ragged-masked", "mask:len=2"}),
    "ecapa512_bf16_masked_edges": ("ECAPA_TDNN_c512", "bf16", 6, 257, [257, 256, 129, 128, 1, 2], {},
                                   {"res2_fused:masked", "astp_fused:masked", "se_gate:masked", "mask:len=1"}),
    "campplus_bf16_masked_edges": ("CAMPPlus", "bf16", 5, 257, [257, 1, 2, 201, 256], {}, {"cam_dense:masked", "mask:len=1"}),
    "gemini60_fp16_masked_edges": ("Gemini_DF_ResNet60", "fp16", 4, 33, [33, 1, 2, 17], {}, {"dwconv3x3:masked", "mask:len=1"}),
    "simam34_bf16_masked_edges": ("SimAM_ResNet34_ASP", "bf16", 4, 33, [33, 1, 2, 17], {}, {"simam_stats:masked", "mask:len=2"}),
    "eres2net_fp16_masked_edges": ("ERes2Net34_Base", "fp16", 4, 17, [17, 1, 2, 9], {}, {"conv3x3:masked", "mask:len=1"}),
}
