#!/usr/bin/env python
"""Goldens for SimAM-ResNet34 / 100 with ASP pooling (the VoxBlink2 models) from the REAL reference modules
(`wespeaker/models/samresnet.py`, `wespeaker/models/pooling_layers.py`).  Build container only.

    PYTHONDONTWRITEBYTECODE=1 WESPEAKER_REFERENCE=<wespeaker checkout> python tests/golden/make_golden_simam.py

Same recipe as make_golden_res2net.py: namespace-bypass import, synthetic checkpoints loaded with strict=True (which pins the
key/shape spec of wespeaker_b200.synthetic.simam_spec), outputs stored in tests/golden/models_simam.npz; inputs are
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

# (model, seed, B, T, in_planes, embed_dim)
CASES = [("SimAM_ResNet34_ASP", 0, 2, 200, 64, 256), ("SimAM_ResNet34_ASP", 1, 2, 99, 64, 256),
         ("SimAM_ResNet100_ASP", 0, 1, 120, 64, 256), ("SimAM_ResNet34_ASP", 2, 2, 150, 32, 192)]


def case_key(name, seed, B, T, in_planes, embed_dim):
    return f"{name}__s{seed}_B{B}_T{T}_p{in_planes}_e{embed_dim}"


def main():
    from wespeaker_b200 import synthetic as syn
    for pkg, path in [("wespeaker", REF), ("wespeaker.models", REF + "/models")]:
        m = types.ModuleType(pkg)
        m.__path__ = [path]
        sys.modules[pkg] = m
    import wespeaker.models.samresnet as samresnet
    torch.set_num_threads(8)
    out = {}
    for name, seed, B, T, in_planes, embed_dim in CASES:
        args = dict(syn.DEFAULT_MODEL_ARGS[name], in_planes=in_planes, embed_dim=embed_dim)
        model = getattr(samresnet, name)(**args)
        sd_np = syn.make_state_dict(name, seed, **args)
        sd = {k: torch.from_numpy(np.asarray(v)) for k, v in sd_np.items()}
        ref_keys = list(model.state_dict().keys())
        assert ref_keys == list(sd.keys()), (name, set(ref_keys) ^ set(sd.keys()))
        model.load_state_dict(sd, strict=True)
        model.eval()
        feats = torch.from_numpy(syn.make_feats(B, T, 80, seed=seed + 17 * T))
        with torch.no_grad():
            o = model(feats)
        assert torch.is_tensor(o)   # samresnet.py:142-149: a bare (B, E) tensor
        key = case_key(name, seed, B, T, in_planes, embed_dim)
        out[key] = o.numpy().astype(np.float32)
        print(f"{key}: emb {tuple(o.shape)} |e|={o.norm(dim=1).mean():.4f} keys={len(ref_keys)} "
              f"params={sum(p.numel() for p in model.parameters()) / 1e6:.2f}M")
    np.savez_compressed(os.path.join(HERE, "models_simam.npz"), **out)


if __name__ == "__main__":
    main()
