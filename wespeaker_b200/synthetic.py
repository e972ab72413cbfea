"""Deterministic synthetic checkpoints for the three model families on the hot path.

There is no network for pretrained checkpoints (SURVEY.md §8c), so parity tests,
`bench.py` and `smoke()` use random-init weights of the reference architectures.
This module restates the reference ``state_dict`` layout (key names + shapes, see
SURVEY.md Appendix C; reference modules `wespeaker/models/ecapa_tdnn.py:160-201`,
`wespeaker/models/resnet.py:110-169`, `wespeaker/models/campplus.py:333-390`) and
fills it from a platform-stable numpy generator keyed by (seed, key-name), so the
same checkpoint can be rebuilt on the GPU box without shipping 25-60 MB files.

BatchNorm statistics are randomised too (a fresh BN is the identity and would hide
BN bugs).  ``tests/golden/make_golden.py`` checks these specs against the real
reference modules with ``load_state_dict(strict=True)``.
"""
from __future__ import annotations

import zlib
from collections import OrderedDict

import numpy as np

ECAPA_NAMES = {
    "ECAPA_TDNN_c512": dict(channels=512, global_context_att=False),
    "ECAPA_TDNN_GLOB_c512": dict(channels=512, global_context_att=True),
    "ECAPA_TDNN_c1024": dict(channels=1024, global_context_att=False),
    "ECAPA_TDNN_GLOB_c1024": dict(channels=1024, global_context_att=True),
}
RESNET_NAMES = {
    "ResNet18": [2, 2, 2, 2],
    "ResNet34": [3, 4, 6, 3],
    # Bottleneck variants (`wespeaker/models/resnet.py:72-107,223-260`), SURVEY.md section 8(f) rank 4
    "ResNet50": [3, 4, 6, 3],
    "ResNet101": [3, 4, 23, 3],
    "ResNet152": [3, 8, 36, 3],
    "ResNet221": [6, 16, 48, 3],
    "ResNet293": [10, 20, 64, 3],
}
RESNET_BOTTLENECK = ("ResNet50", "ResNet101", "ResNet152", "ResNet221", "ResNet293")
CAMPP_NAMES = {"CAMPPlus": {}}
XVEC_NAMES = {"XVEC": {}}   # Kaldi-style x-vector TDNN (`wespeaker/models/tdnn.py:57-117`), section 8(f) rank 4
# Res2Net / ERes2Net (`wespeaker/models/res2net.py:202-221`, `wespeaker/models/eres2net.py:393-431`), section 8(f) rank 4.
# fuse: ERes2Net's local (AFF inside the layer-3/4 blocks) and global (bottom-up AFF over the four stages) feature fusion.
RES2NET_NAMES = {
    "Res2Net34_Base": dict(m_channels=32, num_blocks=[3, 4, 6, 3], base_width=32, scale=2, expansion=2, fuse=False),
    "Res2Net34_Large": dict(m_channels=64, num_blocks=[3, 4, 6, 3], base_width=32, scale=2, expansion=2, fuse=False),
    "ERes2Net34_Base": dict(m_channels=32, num_blocks=[3, 4, 6, 3], base_width=32, scale=2, expansion=2, fuse=True),
    "ERes2Net34_Large": dict(m_channels=64, num_blocks=[3, 4, 6, 3], base_width=32, scale=2, expansion=2, fuse=True),
    "ERes2Net34_aug": dict(m_channels=64, num_blocks=[3, 4, 6, 3], base_width=24, scale=3, expansion=4, fuse=True),
}
# SimAM-ResNet with ASP pooling, the VoxBlink2 models (`wespeaker/models/samresnet.py:126-167`): block counts
SIMAM_NAMES = {"SimAM_ResNet34_ASP": [3, 4, 6, 3], "SimAM_ResNet100_ASP": [6, 16, 24, 3]}
# Gemini DF-ResNet (`wespeaker/models/gemini_dfresnet.py:142-176`): inverted bottlenecks per stage
GEMINI_NAMES = {"Gemini_DF_ResNet60": [3, 3, 9, 3], "Gemini_DF_ResNet114": [3, 3, 27, 3],
                "Gemini_DF_ResNet183": [3, 8, 45, 3], "Gemini_DF_ResNet237": [3, 8, 63, 3]}
GEMINI_DIMS = (32, 32, 64, 128, 256)

DEFAULT_MODEL_ARGS = {
    # examples/voxceleb/v2/conf/{ecapa_tdnn,resnet,campplus}.yaml
    "ECAPA_TDNN_c512": dict(feat_dim=80, embed_dim=192, pooling_func="ASTP"),
    "ECAPA_TDNN_GLOB_c512": dict(feat_dim=80, embed_dim=192, pooling_func="ASTP"),
    "ECAPA_TDNN_c1024": dict(feat_dim=80, embed_dim=192, pooling_func="ASTP"),
    "ECAPA_TDNN_GLOB_c1024": dict(feat_dim=80, embed_dim=192, pooling_func="ASTP"),
    "ResNet18": dict(feat_dim=80, embed_dim=256, pooling_func="TSTP", two_emb_layer=False),
    "ResNet34": dict(feat_dim=80, embed_dim=256, pooling_func="TSTP", two_emb_layer=False),
    "CAMPPlus": dict(feat_dim=80, embed_dim=512, pooling_func="TSTP"),
    "ResNet50": dict(feat_dim=80, embed_dim=256, pooling_func="TSTP", two_emb_layer=False),
    "ResNet101": dict(feat_dim=80, embed_dim=256, pooling_func="TSTP", two_emb_layer=False),
    "ResNet152": dict(feat_dim=80, embed_dim=256, pooling_func="TSTP", two_emb_layer=False),
    "ResNet221": dict(feat_dim=80, embed_dim=256, pooling_func="TSTP", two_emb_layer=False),
    "ResNet293": dict(feat_dim=80, embed_dim=256, pooling_func="TSTP", two_emb_layer=False),
    "XVEC": dict(feat_dim=80, embed_dim=512, pooling_func="TSTP"),   # examples/voxceleb/v2/conf/xvec.yaml
    # examples/voxceleb/v2/conf/{res2net,eres2net}.yaml
    "Res2Net34_Base": dict(feat_dim=80, embed_dim=256, pooling_func="TSTP", two_emb_layer=False),
    "Res2Net34_Large": dict(feat_dim=80, embed_dim=256, pooling_func="TSTP", two_emb_layer=False),
    "ERes2Net34_Base": dict(feat_dim=80, embed_dim=512, pooling_func="TSTP", two_emb_layer=False),
    "ERes2Net34_Large": dict(feat_dim=80, embed_dim=512, pooling_func="TSTP", two_emb_layer=False),
    "ERes2Net34_aug": dict(feat_dim=80, embed_dim=512, pooling_func="TSTP", two_emb_layer=False),
    # the reference constructor's own arguments (samresnet.py:135): no feat_dim, the feature dimension is acoustic_dim
    "SimAM_ResNet34_ASP": dict(in_planes=64, embed_dim=256, acoustic_dim=80, dropout=0),
    "SimAM_ResNet100_ASP": dict(in_planes=64, embed_dim=256, acoustic_dim=80, dropout=0),
    # examples/voxceleb/v2/conf/gemini_dfresnet_adam.yaml
    "Gemini_DF_ResNet60": dict(feat_dim=80, embed_dim=256, pooling_func="TSTP", two_emb_layer=False),
    "Gemini_DF_ResNet114": dict(feat_dim=80, embed_dim=256, pooling_func="TSTP", two_emb_layer=False),
    "Gemini_DF_ResNet183": dict(feat_dim=80, embed_dim=256, pooling_func="TSTP", two_emb_layer=False),
    "Gemini_DF_ResNet237": dict(feat_dim=80, embed_dim=256, pooling_func="TSTP", two_emb_layer=False),
}


def _bn(spec, prefix, c, affine=True):
    if affine:
        spec[prefix + ".weight"] = (c,)
        spec[prefix + ".bias"] = (c,)
    spec[prefix + ".running_mean"] = (c,)
    spec[prefix + ".running_var"] = (c,)
    spec[prefix + ".num_batches_tracked"] = ()


def ecapa_spec(channels=512, feat_dim=80, embed_dim=192, pooling_func="ASTP",
               global_context_att=False, emb_bn=False):
    assert pooling_func == "ASTP", "only ASTP is on the hot path for ECAPA"
    C = channels
    w = C // 8
    s = OrderedDict()
    s["layer1.conv.weight"] = (C, feat_dim, 5)
    s["layer1.conv.bias"] = (C,)
    _bn(s, "layer1.bn", C)
    for L in (2, 3, 4):
        p = f"layer{L}.se_res2block"
        s[f"{p}.0.conv.weight"] = (C, C, 1)
        s[f"{p}.0.conv.bias"] = (C,)
        _bn(s, f"{p}.0.bn", C)
        for i in range(7):
            s[f"{p}.1.convs.{i}.weight"] = (w, w, 3)
            s[f"{p}.1.convs.{i}.bias"] = (w,)
        for i in range(7):
            _bn(s, f"{p}.1.bns.{i}", w)
        s[f"{p}.2.conv.weight"] = (C, C, 1)
        s[f"{p}.2.conv.bias"] = (C,)
        _bn(s, f"{p}.2.bn", C)
        s[f"{p}.3.linear1.weight"] = (128, C)
        s[f"{p}.3.linear1.bias"] = (128,)
        s[f"{p}.3.linear2.weight"] = (C, 128)
        s[f"{p}.3.linear2.bias"] = (C,)
    s["conv.weight"] = (1536, 3 * C, 1)
    s["conv.bias"] = (1536,)
    s["pool.linear1.weight"] = (128, 1536 * (3 if global_context_att else 1), 1)
    s["pool.linear1.bias"] = (128,)
    s["pool.linear2.weight"] = (1536, 128, 1)
    s["pool.linear2.bias"] = (1536,)
    _bn(s, "bn", 3072)
    s["linear.weight"] = (embed_dim, 3072)
    s["linear.bias"] = (embed_dim,)
    if emb_bn:
        _bn(s, "bn2", embed_dim)
    return s


def _basic_block(s, p, cin, cout, stride):
    s[f"{p}.conv1.weight"] = (cout, cin, 3, 3)
    _bn(s, f"{p}.bn1", cout)
    s[f"{p}.conv2.weight"] = (cout, cout, 3, 3)
    _bn(s, f"{p}.bn2", cout)
    if stride != 1 or cin != cout:
        s[f"{p}.shortcut.0.weight"] = (cout, cin, 1, 1)
        _bn(s, f"{p}.shortcut.1", cout)


def _bottleneck(s, p, cin, planes, stride):
    """`wespeaker/models/resnet.py:72-107` (expansion 4)."""
    s[f"{p}.conv1.weight"] = (planes, cin, 1, 1)
    _bn(s, f"{p}.bn1", planes)
    s[f"{p}.conv2.weight"] = (planes, planes, 3, 3)
    _bn(s, f"{p}.bn2", planes)
    s[f"{p}.conv3.weight"] = (4 * planes, planes, 1, 1)
    _bn(s, f"{p}.bn3", 4 * planes)
    if stride != 1 or cin != 4 * planes:
        s[f"{p}.shortcut.0.weight"] = (4 * planes, cin, 1, 1)
        _bn(s, f"{p}.shortcut.1", 4 * planes)


def resnet_spec(num_blocks, m_channels=32, feat_dim=80, embed_dim=256,
                pooling_func="TSTP", two_emb_layer=False, bottleneck=False):
    assert pooling_func == "TSTP", "only TSTP is on the hot path for ResNet"
    s = OrderedDict()
    s["conv1.weight"] = (m_channels, 1, 3, 3)
    _bn(s, "bn1", m_channels)
    cin = m_channels
    exp = 4 if bottleneck else 1
    for li, (nb, mult, stride) in enumerate(zip(num_blocks, (1, 2, 4, 8), (1, 2, 2, 2)), 1):
        cout = m_channels * mult
        for bi in range(nb):
            if bottleneck:
                _bottleneck(s, f"layer{li}.{bi}", cin, cout, stride if bi == 0 else 1)
            else:
                _basic_block(s, f"layer{li}.{bi}", cin, cout, stride if bi == 0 else 1)
            cin = cout * exp
    stats_dim = int(feat_dim / 8) * m_channels * 8 * exp
    s["seg_1.weight"] = (embed_dim, stats_dim * 2)
    s["seg_1.bias"] = (embed_dim,)
    if two_emb_layer:
        _bn(s, "seg_bn_1", embed_dim, affine=False)
        s["seg_2.weight"] = (embed_dim, embed_dim)
        s["seg_2.bias"] = (embed_dim,)
    return s


def campplus_spec(feat_dim=80, embed_dim=512, pooling_func="TSTP", growth_rate=32,
                  bn_size=4, init_channels=128, config_str="batchnorm-relu"):
    assert pooling_func == "TSTP" and config_str == "batchnorm-relu"
    s = OrderedDict()
    m = 32
    s["head.conv1.weight"] = (m, 1, 3, 3)
    _bn(s, "head.bn1", m)
    for li in (1, 2):
        for bi in range(2):
            _basic_block(s, f"head.layer{li}.{bi}", m, m, 2 if bi == 0 else 1)
    s["head.conv2.weight"] = (m, m, 3, 3)
    _bn(s, "head.bn2", m)
    ch = m * (feat_dim // 8)
    s["xvector.tdnn.linear.weight"] = (init_channels, ch, 5)
    _bn(s, "xvector.tdnn.nonlinear.batchnorm", init_channels)
    ch = init_channels
    bnc = bn_size * growth_rate
    for b, nl in enumerate((12, 24, 16), 1):
        for j in range(1, nl + 1):
            p = f"xvector.block{b}.tdnnd{j}"
            cin = ch + (j - 1) * growth_rate
            _bn(s, f"{p}.nonlinear1.batchnorm", cin)
            s[f"{p}.linear1.weight"] = (bnc, cin, 1)
            _bn(s, f"{p}.nonlinear2.batchnorm", bnc)
            s[f"{p}.cam_layer.linear_local.weight"] = (growth_rate, bnc, 3)
            s[f"{p}.cam_layer.linear1.weight"] = (bnc // 2, bnc, 1)
            s[f"{p}.cam_layer.linear1.bias"] = (bnc // 2,)
            s[f"{p}.cam_layer.linear2.weight"] = (growth_rate, bnc // 2, 1)
            s[f"{p}.cam_layer.linear2.bias"] = (growth_rate,)
        ch = ch + nl * growth_rate
        _bn(s, f"xvector.transit{b}.nonlinear.batchnorm", ch)
        s[f"xvector.transit{b}.linear.weight"] = (ch // 2, ch, 1)
        ch //= 2
    _bn(s, "xvector.out_nonlinear.batchnorm", ch)
    s["xvector.dense.linear.weight"] = (embed_dim, ch * 2, 1)
    _bn(s, "xvector.dense.nonlinear.batchnorm", embed_dim, affine=False)
    return s


def xvec_spec(feat_dim=80, hid_dim=512, stats_dim=1500, embed_dim=512, pooling_func="TSTP"):
    """`wespeaker/models/tdnn.py:57-86`: five TdnnLayers (Conv1d -> ReLU -> BN(affine=False)), TSTP, two segment layers."""
    assert pooling_func == "TSTP", "only TSTP is on the hot path for XVEC"
    s = OrderedDict()
    for i, (cin, cout, k) in enumerate(((feat_dim, hid_dim, 5), (hid_dim, hid_dim, 3), (hid_dim, hid_dim, 3),
                                        (hid_dim, hid_dim, 1), (hid_dim, stats_dim, 1)), 1):
        s[f"frame_{i}.conv_1d.weight"] = (cout, cin, k)
        s[f"frame_{i}.conv_1d.bias"] = (cout,)
        _bn(s, f"frame_{i}.bn", cout, affine=False)
    s["seg_1.weight"] = (embed_dim, stats_dim * 2)
    s["seg_1.bias"] = (embed_dim,)
    _bn(s, "seg_bn_1", embed_dim, affine=False)
    s["seg_2.weight"] = (embed_dim, embed_dim)
    s["seg_2.bias"] = (embed_dim,)
    return s


def _aff(s, p, channels, r=4):
    """`wespeaker/models/eres2net.py:75-102`: Conv2d(2C -> C/r, 1x1, bias) -> BN -> SiLU -> Conv2d(C/r -> C, 1x1, bias) -> BN."""
    inter = channels // r
    s[f"{p}.local_att.0.weight"] = (inter, 2 * channels, 1, 1)
    s[f"{p}.local_att.0.bias"] = (inter,)
    _bn(s, f"{p}.local_att.1", inter)
    s[f"{p}.local_att.3.weight"] = (channels, inter, 1, 1)
    s[f"{p}.local_att.3.bias"] = (channels,)
    _bn(s, f"{p}.local_att.4", channels)


def res2net_width(planes, base_width):
    return int(np.floor(planes * (base_width / 64.0)))


def res2net_spec(m_channels=32, num_blocks=(3, 4, 6, 3), base_width=32, scale=2, expansion=2, fuse=False, feat_dim=80,
                 embed_dim=256, pooling_func="TSTP", two_emb_layer=False):
    """Key order of the reference modules' ``state_dict()``: `res2net.py:34-58,98-151` (BasicBlockRes2Net: scale - 1 chain
    convs) and `eres2net.py:104-139,159-201,227-336` (BasicBlockERes2Net in layers 1-2: scale chain convs;
    BasicBlockERes2Net_diff_AFF in layers 3-4: conv2_1/bn2_1 + (scale - 1) convs, bns and AFF fuse models; three stride-2
    3x3 downsampling convs and three AFF modules for the bottom-up fusion)."""
    assert pooling_func == "TSTP", "only TSTP is on the hot path for Res2Net / ERes2Net"
    s = OrderedDict()
    s["conv1.weight"] = (m_channels, 1, 3, 3)
    _bn(s, "bn1", m_channels)
    cin = m_channels
    for li, (nb, mult, stride) in enumerate(zip(num_blocks, (1, 2, 4, 8), (1, 2, 2, 2)), 1):
        planes = m_channels * mult
        w = res2net_width(planes, base_width)
        cout = planes * expansion
        for bi in range(nb):
            p = f"layer{li}.{bi}"
            st = stride if bi == 0 else 1
            s[f"{p}.conv1.weight"] = (w * scale, cin, 1, 1)
            _bn(s, f"{p}.bn1", w * scale)
            if fuse and li >= 3:
                s[f"{p}.conv2_1.weight"] = (w, w, 3, 3)
                _bn(s, f"{p}.bn2_1", w)
                for i in range(scale - 1):
                    s[f"{p}.convs.{i}.weight"] = (w, w, 3, 3)
                for i in range(scale - 1):
                    _bn(s, f"{p}.bns.{i}", w)
                for i in range(scale - 1):
                    _aff(s, f"{p}.fuse_models.{i}", w)
            else:
                nums = scale if fuse else scale - 1
                for i in range(nums):
                    s[f"{p}.convs.{i}.weight"] = (w, w, 3, 3)
                for i in range(nums):
                    _bn(s, f"{p}.bns.{i}", w)
            s[f"{p}.conv3.weight"] = (cout, w * scale, 1, 1)
            _bn(s, f"{p}.bn3", cout)
            if st != 1 or cin != cout:
                s[f"{p}.shortcut.0.weight"] = (cout, cin, 1, 1)
                _bn(s, f"{p}.shortcut.1", cout)
            cin = cout
    if fuse:
        me = m_channels * expansion
        s["layer1_downsample.weight"] = (me * 2, me, 3, 3)
        s["layer2_downsample.weight"] = (me * 4, me * 2, 3, 3)
        s["layer3_downsample.weight"] = (me * 8, me * 4, 3, 3)
        _aff(s, "fuse_mode12", me * 2)
        _aff(s, "fuse_mode123", me * 4)
        _aff(s, "fuse_mode1234", me * 8)
    stats_dim = int(feat_dim / 8) * m_channels * 8 * expansion
    s["seg_1.weight"] = (embed_dim, stats_dim * 2)
    s["seg_1.bias"] = (embed_dim,)
    if two_emb_layer:
        _bn(s, "seg_bn_1", embed_dim, affine=False)
        s["seg_2.weight"] = (embed_dim, embed_dim)
        s["seg_2.bias"] = (embed_dim,)
    return s


def simam_spec(num_blocks, in_planes=64, embed_dim=256, acoustic_dim=80, dropout=0):
    """`wespeaker/models/samresnet.py:21-167`: the ResNet trunk under ``front.`` (SimAMBasicBlock: conv1/bn1, conv2/bn2, and a
    ``downsample`` Sequential of a strided 1x1 conv and a BN where the shape changes), ASP pooling (`pooling_layers.py:151-186`:
    Conv1d -> ReLU -> BN -> Conv1d over in_planes * 8 * int(acoustic_dim / 8) features) and the ``bottleneck`` Linear.
    ``dropout`` only acts in training."""
    s = OrderedDict()
    s["front.conv1.weight"] = (in_planes, 1, 3, 3)
    _bn(s, "front.bn1", in_planes)
    cin = in_planes
    for li, (nb, mult, stride) in enumerate(zip(num_blocks, (1, 2, 4, 8), (1, 2, 2, 2)), 1):
        planes = in_planes * mult
        for bi in range(nb):
            p = f"front.layer{li}.{bi}"
            s[f"{p}.conv1.weight"] = (planes, cin, 3, 3)
            _bn(s, f"{p}.bn1", planes)
            s[f"{p}.conv2.weight"] = (planes, planes, 3, 3)
            _bn(s, f"{p}.bn2", planes)
            if (stride if bi == 0 else 1) != 1 or cin != planes:
                s[f"{p}.downsample.0.weight"] = (planes, cin, 1, 1)
                _bn(s, f"{p}.downsample.1", planes)
            cin = planes
    feature_dim = in_planes * 8 * int(acoustic_dim / 8)
    s["pooling.attention.0.weight"] = (128, feature_dim, 1)
    s["pooling.attention.0.bias"] = (128,)
    _bn(s, "pooling.attention.2", 128)
    s["pooling.attention.3.weight"] = (feature_dim, 128, 1)
    s["pooling.attention.3.bias"] = (feature_dim,)
    s["bottleneck.weight"] = (embed_dim, 2 * feature_dim)
    s["bottleneck.bias"] = (embed_dim,)
    return s


def gemini_spec(depths, feat_dim=80, embed_dim=256, pooling_func="TSTP", two_emb_layer=False):
    """`wespeaker/models/gemini_dfresnet.py:30-136`: ``downsample_layers`` (the stem conv/BN, then four 3x3 convs + BN), the
    ``stages`` of Inverted_Bottleneck blocks (conv1/bn1 1x1 dim -> 4 dim, conv2/bn2 depthwise 3x3, conv3/bn3 1x1 4 dim -> dim),
    TSTP over stats_dim = int(feat_dim / 8 / 2) * 256 and the segment layer(s)."""
    assert pooling_func == "TSTP", "only TSTP is on the hot path for Gemini DF-ResNet"
    dims = GEMINI_DIMS
    s = OrderedDict()
    s["downsample_layers.0.0.weight"] = (dims[0], 1, 3, 3)
    _bn(s, "downsample_layers.0.1", dims[0])
    for i in range(4):
        s[f"downsample_layers.{i + 1}.0.weight"] = (dims[i + 1], dims[i], 3, 3)
        _bn(s, f"downsample_layers.{i + 1}.1", dims[i + 1])
    for i, n in enumerate(depths):
        d = dims[i + 1]
        for j in range(n):
            p = f"stages.{i}.{j}"
            s[f"{p}.conv1.weight"] = (4 * d, d, 1, 1)
            _bn(s, f"{p}.bn1", 4 * d)
            s[f"{p}.conv2.weight"] = (4 * d, 1, 3, 3)
            _bn(s, f"{p}.bn2", 4 * d)
            s[f"{p}.conv3.weight"] = (d, 4 * d, 1, 1)
            _bn(s, f"{p}.bn3", d)
    stats_dim = int(feat_dim / 8 / 2) * dims[-1]
    s["seg_1.weight"] = (embed_dim, stats_dim * 2)
    s["seg_1.bias"] = (embed_dim,)
    if two_emb_layer:
        _bn(s, "seg_bn_1", embed_dim, affine=False)
        s["seg_2.weight"] = (embed_dim, embed_dim)
        s["seg_2.bias"] = (embed_dim,)
    return s


def state_dict_spec(model_name: str, **model_args):
    """key -> shape for a reference model name (`wespeaker/models/speaker_model.py:31-62`)."""
    if model_name in ECAPA_NAMES:
        return ecapa_spec(**ECAPA_NAMES[model_name], **model_args)
    if model_name in RESNET_NAMES:
        return resnet_spec(RESNET_NAMES[model_name], bottleneck=model_name in RESNET_BOTTLENECK, **model_args)
    if model_name in XVEC_NAMES:
        return xvec_spec(**model_args)
    if model_name in RES2NET_NAMES:
        return res2net_spec(**RES2NET_NAMES[model_name], **model_args)
    if model_name in CAMPP_NAMES:
        return campplus_spec(**model_args)
    if model_name in SIMAM_NAMES:
        return simam_spec(SIMAM_NAMES[model_name], **model_args)
    if model_name in GEMINI_NAMES:
        return gemini_spec(GEMINI_NAMES[model_name], **model_args)
    raise ValueError(f"model {model_name!r} is not on the engine's hot path")


def _rng(seed: int, key: str) -> np.random.Generator:
    return np.random.Generator(np.random.PCG64([seed, zlib.crc32(key.encode())]))


def _gemini_downsample_bn(key):
    """the BN after each 3x3 conv of Gemini DF-ResNet's ``downsample_layers`` (``downsample_layers.<i>.1.*``)"""
    parts = key.split(".")
    return parts[0] == "downsample_layers" and parts[2] == "1"


def make_state_dict(model_name: str, seed: int = 0, **model_args):
    """Random checkpoint as ``OrderedDict[str, np.ndarray]`` (float32; counters int64)."""
    args = dict(DEFAULT_MODEL_ARGS.get(model_name, {}))
    args.update(model_args)
    spec = state_dict_spec(model_name, **args)
    sd = OrderedDict()
    for key, shape in spec.items():
        g = _rng(seed, key)
        if key.endswith("num_batches_tracked"):
            sd[key] = np.array(100, dtype=np.int64)
        elif key.endswith("running_mean"):
            sd[key] = (0.1 * g.standard_normal(shape)).astype(np.float32)
        elif key.endswith("running_var"):
            sd[key] = g.uniform(0.5, 1.5, shape).astype(np.float32)
        elif ".bn" in key or "batchnorm" in key or key.startswith("bn") or "shortcut.1" in key \
                or "seg_bn" in key or "local_att.1." in key or "local_att.4." in key or "downsample.1." in key \
                or "pooling.attention.2." in key or _gemini_downsample_bn(key):
            if (key.endswith(".bn2.weight") or key.endswith(".bn3.weight")) and "layer" in key \
                    or key.startswith("stages.") and key.endswith(".bn3.weight"):
                # residual-branch output BN of the 2-D BasicBlocks: keep the residual sum O(1)
                # over 16 blocks (a trained net does; fp16 range matters for config 3)
                sd[key] = g.uniform(0.2, 0.6, shape).astype(np.float32)
            elif key.endswith(".weight"):
                sd[key] = g.uniform(0.5, 1.5, shape).astype(np.float32)
            else:
                sd[key] = (0.1 * g.standard_normal(shape)).astype(np.float32)
        elif key.endswith(".bias"):
            sd[key] = (0.1 * g.standard_normal(shape)).astype(np.float32)
        else:  # conv / linear weight: variance-preserving
            fan_in = int(np.prod(shape[1:]))
            sd[key] = (g.standard_normal(shape) * np.sqrt(1.5 / fan_in)).astype(np.float32)
    return sd


def make_feats(batch: int, frames: int, feat_dim: int = 80, seed: int = 0, cmn: bool = True):
    """Synthetic fbank-like features (B,T,F) ~ N(0,1), mean-normalised over T like
    `wespeaker/dataset/dataset_utils.py:19-26` (`apply_cmvn`)."""
    g = np.random.Generator(np.random.PCG64([seed, 0xFEA7]))
    x = g.standard_normal((batch, frames, feat_dim)).astype(np.float32)
    if cmn:
        x = x - x.mean(axis=1, keepdims=True, dtype=np.float32)
    return x.astype(np.float32)


def make_wavs(batch: int, samples: int = 32000, seed: int = 0, scale: float = 3000.0):
    """Synthetic int16-range waveforms (B,N) float32, as after ``wav * (1 << 15)``
    (`wespeaker/dataset/processor.py:516`).  Values are rounded to integers so the same
    signal is representable as int16 PCM."""
    g = np.random.Generator(np.random.PCG64([seed, 0x0A7]))
    t = np.arange(samples, dtype=np.float64) / 16000.0
    out = np.empty((batch, samples), dtype=np.float32)
    for b in range(batch):
        f0 = g.uniform(80, 300)
        sig = sum(g.uniform(0.2, 1.0) * np.sin(2 * np.pi * f0 * h * t + g.uniform(0, 6.28))
                  for h in range(1, 12))
        sig = sig / np.abs(sig).max() * scale + g.standard_normal(samples) * scale * 0.3
        out[b] = np.clip(np.rint(sig), -32768, 32767).astype(np.float32)
    return out


def make_plda(dim: int = 256, seed: int = 3, normalize_length: bool = True):
    """Synthetic two-covariance PLDA model (SURVEY.md §8d config 5); fp64 numpy arrays
    with the field names of `wespeaker/utils/plda/two_cov_plda.py:311-363`."""
    g = np.random.Generator(np.random.PCG64([seed, 0x91DA]))
    transform = g.standard_normal((dim, dim)) / np.sqrt(dim)
    mu = 0.1 * g.standard_normal(dim)
    psi = np.sort(g.gamma(2.0, 2.0, dim))[::-1].copy()
    offset = -1.0 * transform @ mu
    return dict(mu=mu, transform=transform, psi=psi, offset=offset,
                normalize_length=normalize_length, subtract_train_set_mean=False, dim=dim)


def make_embeddings(n: int, dim: int = 256, seed: int = 3):
    g = np.random.Generator(np.random.PCG64([seed, 0xE3B, n]))
    return g.standard_normal((n, dim)).astype(np.float32)
