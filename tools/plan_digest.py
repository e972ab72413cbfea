#!/usr/bin/env python
"""Print a digest of the launch plans the engine builds for a fixed set of cases, on any host (plan-check engines: no
device, nothing computed).  Two builds of the library that print the same digests build the same plans: the same ops in the
same order with the same labels, kernels, launch parameters, weights and buffer wiring.  Use it to check that a change to
the plan builders leaves the plans alone:

    python tools/plan_digest.py > before.txt      # on the old tree
    python tools/plan_digest.py > after.txt       # on the new tree
    diff before.txt after.txt

The trace's placeholder addresses depend on what was allocated before, so each one is written in canonical form: an
activation address becomes "A<k>+<offset>" with allocations numbered in order of first reference (header, then ops), and a
weight address becomes "W<sha256 of its fp32 source>+<offset>".  --out DIR also writes each case's canonical plan to
DIR/<case>.json, for diffing the cases whose digests differ.  --strip-added drops the fields that later traces added before
digesting, for comparing with builds whose traces did not name them: the optional buffers (the 3xTF32 lo twins plo, p_lo,
W_lo, out_lo, out2_lo, the linear split-K workspace wsp and the SimAM partial sums), the kernel an op takes, the "launch"
object (the kernel and geometry the host chose for an op), tstats' eps and output element size, and se_gate's column sums
("kind.field": that field of that op kind only).
"""
import argparse
import bisect
import functools
import hashlib
import json
import multiprocessing
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from plan_interp import load_trace  # noqa: E402
from wespeaker_b200.models import SUPPORTED_MODELS, from_synthetic  # noqa: E402

PRECISIONS = ("fp32", "tf32", "tf32x3", "bf16", "fp16")
PLACEHOLDER = 0x7000000000   # plan_check_alloc hands out addresses from here up
ADDED_FIELDS = ("plo", "p_lo", "W_lo", "out_lo", "out2_lo", "wsp", "partial", "kernel", "launch", "tstats.eps", "tstats.out_es",
                "se_gate.colsum")


def cases():
    """(model, precision, B, T, masked, model_args, engine options)"""
    out = []
    for name in SUPPORTED_MODELS:
        for prec in PRECISIONS:
            out.append((name, prec, 2, 200, False, {}, {}))
            if name != "XVEC" and (name != "CAMPPlus" or prec in ("bf16", "fp16")):
                out.append((name, prec, 2, 200, True, {}, {}))
    for prec in ("fp32", "tf32x3", "bf16"):
        for T in (100, 300):
            out.append(("ECAPA_TDNN_c1024", prec, 2, T, False, {}, {}))
        for opt in ("res2_fused", "astp_fused", "se_fused", "se_colsum"):
            out.append(("ECAPA_TDNN_c1024", prec, 2, 200, False, {}, {opt: 0}))
    for name in ("ResNet34", "ResNet50", "ERes2Net34_Base", "SimAM_ResNet34_ASP", "Gemini_DF_ResNet60", "CAMPPlus"):
        for masked in (False, True):
            out.append((name, "fp16", 2, 200, masked, {}, {"conv3x3": 0}))
    for opt in ("cam_fused", "cam_block"):
        out.append(("CAMPPlus", "bf16", 2, 200, False, {}, {opt: 0}))
    for T in (998, 2400):
        out.append(("CAMPPlus", "fp32", 2, T, False, {}, {}))
    for name in ("ResNet34", "ERes2Net34_Base"):
        for prec in ("tf32x3", "fp16"):
            out.append((name, prec, 2, 200, False, {"two_emb_layer": True}, {}))
    for prec in ("tf32x3", "bf16"):
        out.append(("ECAPA_TDNN_c512", prec, 2, 200, False, {"emb_bn": True}, {}))
    for prec in ("tf32x3", "bf16"):
        out.append(("ResNet34", prec, 2, 200, False, {}, {"tc_version": 2}))
    return out


def case_id(c):
    name, prec, B, T, masked, args, opts = c
    tags = [f"{k}={int(v)}" for k, v in sorted({**args, **opts}.items())]
    return "_".join([name, prec, f"B{B}", f"T{T}"] + (["masked"] if masked else []) + tags)


def _strip_added(x):
    if isinstance(x, dict):
        kind = x.get("kind")
        return {k: _strip_added(v) for k, v in x.items() if k not in ADDED_FIELDS and f"{kind}.{k}" not in ADDED_FIELDS}
    if isinstance(x, list):
        return [_strip_added(v) for v in x]
    return x


def canonical(path, strip_added=False):
    meta, blob = load_trace(path)
    if strip_added:
        meta = {**meta, "ops": _strip_added(meta["ops"])}
    allocs = sorted((a, n) for a, n in meta["allocs"])
    starts = [a for a, _ in allocs]
    weights = {a: hashlib.sha256(blob[o:o + n].tobytes()).hexdigest() for a, o, n in meta["blobs"]}
    names = {}

    def addr(v):
        i = bisect.bisect_right(starts, v) - 1
        assert i >= 0, v
        base, nbytes = allocs[i]
        assert base <= v < base + max(nbytes, 1), (v, base, nbytes)
        if base in weights:
            return f"W{weights[base]}+{v - base}"
        if base not in names:
            names[base] = f"A{len(names)}[{nbytes}]"
        return f"{names[base]}+{v - base}"

    def walk(x):
        if isinstance(x, dict):
            return {k: walk(v) for k, v in x.items()}
        if isinstance(x, list):
            return [walk(v) for v in x]
        if isinstance(x, int) and not isinstance(x, bool) and x >= PLACEHOLDER:
            return addr(x)
        return x

    header = walk({k: v for k, v in meta.items() if k not in ("allocs", "blobs", "ops")})
    ops = walk(meta["ops"])
    return json.dumps({"header": header, "ops": ops}, indent=0, sort_keys=True)


def digest(c, strip_added=False):
    name, prec, B, T, masked, args, opts = c
    m = from_synthetic(name, 0, precision=prec, **args)
    for k, v in opts.items():
        m.set_option(k, v)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "plan.wspt")
        m.plan_trace(path, B, T, masked)
        text = canonical(path, strip_added)
    return case_id(c), hashlib.sha256(text.encode()).hexdigest(), text.count('"label"'), text


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", help="also write each case's canonical plan to OUT/<case>.json")
    ap.add_argument("--jobs", type=int, default=os.cpu_count())
    ap.add_argument("--strip-added", action="store_true", help="digest without the optional buffer fields")
    args = ap.parse_args()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
    cs = cases()
    with multiprocessing.get_context("spawn").Pool(args.jobs) as pool:
        for cid, h, nops, text in pool.imap(functools.partial(digest, strip_added=args.strip_added), cs):
            print(f"{cid} {nops} ops {h}", flush=True)
            if args.out:
                with open(os.path.join(args.out, cid + ".json"), "w") as f:
                    f.write(text)
    print(f"{len(cs)} cases", file=sys.stderr)


if __name__ == "__main__":
    main()
