#!/usr/bin/env python
"""Per-GEMM operand-precision study on the CPU oracle (test infrastructure; not part of the product path).

For each precision map (which Linear class runs with which operand format) the oracle forward is run with the
operands of those GEMMs rounded the way the tensor-core kernels round them, fp32 accumulation, and compared with
the plain fp32 oracle: match-index flips and max |d matching_scores|.  Decides which GEMMs need split operands
for index-exact results (SURVEY.md 7.3) -- the `mixed` precision mode of the CUDA path is built from this table.

    python tools/precision_study.py --pairs 8 --n 2048
"""
from __future__ import annotations

import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from lightglue_b200 import synth  # noqa: E402
from oracle import lightglue_oracle as oracle  # noqa: E402
from oracle.tc_emulation import emulated  # noqa: E402


MAPS2 = {
    "fp16x3 everywhere": dict(qkv="fp16x3", out="fp16x3", ffn0="fp16x3", ffn3="fp16x3", final="fp16x3", sim="fp16x3"),
    "qkv fp16 | rest fp16x3": dict(qkv="fp16", out="fp16x3", ffn0="fp16x3", ffn3="fp16x3", final="fp16x3", sim="fp16x3"),
    "out fp16 | rest fp16x3": dict(qkv="fp16x3", out="fp16", ffn0="fp16x3", ffn3="fp16x3", final="fp16x3", sim="fp16x3"),
    "MIXED: qkv,out fp16 | msg hi | rest fp16x3": dict(qkv="fp16", out="fp16", ffn0="fp16x3", ffn3="fp16x3", final="fp16x3", sim="fp16x3", msg="hi"),
    "qkv fp16 | out fp16x3, msg hi | rest fp16x3": dict(qkv="fp16", out="fp16x3", ffn0="fp16x3", ffn3="fp16x3", final="fp16x3", sim="fp16x3", msg="hi"),
}
MAPS = {
    "bf16 everywhere": dict(qkv="bf16", out="bf16", ffn0="bf16", ffn3="bf16", final="bf16", sim="bf16"),
    "bf16x3 everywhere": dict(qkv="bf16x3", out="bf16x3", ffn0="bf16x3", ffn3="bf16x3", final="bf16x3", sim="bf16x3"),
    "qkv,out bf16 | rest bf16x3": dict(qkv="bf16", out="bf16", ffn0="bf16x3", ffn3="bf16x3", final="bf16x3", sim="bf16x3"),
    "qkv bf16 | rest bf16x3": dict(qkv="bf16", out="bf16x3", ffn0="bf16x3", ffn3="bf16x3", final="bf16x3", sim="bf16x3"),
    "out bf16 | rest bf16x3": dict(qkv="bf16x3", out="bf16", ffn0="bf16x3", ffn3="bf16x3", final="bf16x3", sim="bf16x3"),
    "qkv,out fp16 | rest bf16x3": dict(qkv="fp16", out="fp16", ffn0="bf16x3", ffn3="bf16x3", final="bf16x3", sim="bf16x3"),
    "fp16 everywhere": dict(qkv="fp16", out="fp16", ffn0="fp16", ffn3="fp16", final="fp16", sim="fp16"),
    "qkv,out fp16 | rest fp16x2a": dict(qkv="fp16", out="fp16", ffn0="fp16x2a", ffn3="fp16x2a", final="fp16x2a", sim="fp16x3"),
    "qkv,out fp16 | ffn fp16x3": dict(qkv="fp16", out="fp16", ffn0="fp16x3", ffn3="fp16x3", final="fp16x3", sim="fp16x3"),
    "qkv fp16x2a,out fp16 | rest fp16x3": dict(qkv="fp16x2a", out="fp16", ffn0="fp16x3", ffn3="fp16x3", final="fp16x3", sim="fp16x3"),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=4)
    ap.add_argument("--n", type=int, default=2048)
    ap.add_argument("--only", default="")
    ap.add_argument("--set", type=int, default=1)
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    sd = synth.make_state_dict()
    pairs = [synth.make_pair(args.n, seed=1000 + i)[0] for i in range(args.pairs)]
    refs = [oracle.forward(sd, d) for d in pairs]
    print(f"# {args.pairs} pairs, N={args.n}; attention operands fp16 in every map; flips over {2 * args.n * args.pairs} indices")
    for name, pmap in (MAPS if args.set == 1 else MAPS2).items():
        if args.only and args.only not in name:
            continue
        t0 = time.time()
        flips, dmax = 0, 0.0
        with emulated(sd, pmap):
            for d, r in zip(pairs, refs):
                o = oracle.forward(sd, d)
                flips += int((o["matches0"] != r["matches0"]).sum()) + int((o["matches1"] != r["matches1"]).sum())
                dmax = max(dmax, float((o["matching_scores0"] - r["matching_scores0"]).abs().max()))
        print(f"{name:40s} flips={flips:4d}  max|dscore|={dmax:.2e}  ({time.time() - t0:.0f} s)", flush=True)


if __name__ == "__main__":
    main()
