#!/usr/bin/env python
"""Goldens for Gemini DF-ResNet60 / 114 / 183 / 237 from the REAL reference module (`wespeaker/models/gemini_dfresnet.py`,
`wespeaker/models/pooling_layers.py`).  Build container only.

    PYTHONDONTWRITEBYTECODE=1 WESPEAKER_REFERENCE=<wespeaker checkout> python tests/golden/make_golden_gemini.py

Same recipe as make_golden_simam.py: namespace-bypass import, synthetic checkpoints loaded with strict=True (which pins the
key/shape spec of wespeaker_b200.synthetic.gemini_spec), outputs stored in tests/golden/models_gemini.npz; inputs are
regenerated from seeds at test time."""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = os.path.join(os.environ["WESPEAKER_REFERENCE"], "wespeaker")   # a checkout of wenet-e2e/wespeaker

# (model, seed, B, T, embed_dim, two_emb_layer); T = 99 is odd through the time stride
CASES = [("Gemini_DF_ResNet60", 0, 2, 200, 256, False), ("Gemini_DF_ResNet114", 1, 2, 99, 256, False),
         ("Gemini_DF_ResNet183", 0, 1, 120, 256, False), ("Gemini_DF_ResNet237", 0, 1, 64, 256, False),
         ("Gemini_DF_ResNet114", 2, 2, 150, 192, True)]


def case_key(name, seed, B, T, embed_dim, two_emb_layer):
    return f"{name}__s{seed}_B{B}_T{T}_e{embed_dim}_w{int(two_emb_layer)}"


def main():
    from wespeaker_b200 import synthetic as syn
    for pkg, path in [("wespeaker", REF), ("wespeaker.models", REF + "/models")]:
        m = types.ModuleType(pkg)
        m.__path__ = [path]
        sys.modules[pkg] = m
    import wespeaker.models.gemini_dfresnet as gemini
    torch.set_num_threads(8)
    out = {}
    for name, seed, B, T, embed_dim, two in CASES:
        args = dict(syn.DEFAULT_MODEL_ARGS[name], embed_dim=embed_dim, two_emb_layer=two)
        model = getattr(gemini, name)(**args)
        sd_np = syn.make_state_dict(name, seed, **args)
        sd = {k: torch.from_numpy(np.asarray(v)) for k, v in sd_np.items()}
        ref_keys = list(model.state_dict().keys())
        assert ref_keys == list(sd.keys()), (name, set(ref_keys) ^ set(sd.keys()))
        model.load_state_dict(sd, strict=True)
        model.eval()
        feats = torch.from_numpy(syn.make_feats(B, T, 80, seed=seed + 17 * T))
        with torch.no_grad():
            o = model(feats)
        assert isinstance(o, tuple) and len(o) == 2   # gemini_dfresnet.py:130-136: (tensor(0.), embed_a) or (embed_a, embed_b)
        key = case_key(name, seed, B, T, embed_dim, two)
        out[key] = o[-1].numpy().astype(np.float32)
        print(f"{key}: emb {tuple(o[-1].shape)} |e|={o[-1].norm(dim=1).mean():.4f} keys={len(ref_keys)} "
              f"params={sum(p.numel() for p in model.parameters()) / 1e6:.3f}M")
    np.savez_compressed(os.path.join(HERE, "models_gemini.npz"), **out)


if __name__ == "__main__":
    main()
