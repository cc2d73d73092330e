"""Where the linear time of the bench workload goes: per-step device time of the QKV, ffn.0 and ffn.3 linears against
their MMA work, epilogue bytes and L2 operand bytes.

    python tools/linear_breakdown.py [--precision bf16x3] [--batch 32] [--steps 5]

Runs the forward `bench.py` times (B pairs of N = 2048, 9 layers, pruning off) with `matcher.timing = True` (CUDA events
around every kernel class inside the library) and prints one JSON line per class, then one with the card:
  ms_per_step        device time of the class per forward
  mma_tflop          tensor-core FLOP per forward, from the shapes (3 products over K in bf16x3)
  epilogue_gb        bytes the epilogues move per forward: QKV writes q, k, vT (fp16); ffn.0 writes h (hi, lo);
                     ffn.3 reads and writes x (fp32) and writes its hi / lo images
  l2_operand_gb      operand bytes the TMA ring loads per forward, from the tile shape (A rows x W rows per 64-wide K
                     block, bf16, once per pass); l2_operand_gbs: the same over ms_per_step
  frac_of_bf16_peak  achieved MMA rate over the bf16 peak
  floor_ms           the larger of mma / peak and bytes / HBM bandwidth (what the class could take if both overlapped)
The peaks come from MEASURED_PEAKS.json when present, else from the H100 SXM data sheet (labelled as such)."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import DESC, LAYERS, N_KPTS, measured_peaks  # noqa: E402
from lightglue_b200 import LightGlue, synth  # noqa: E402


TILE_M, TILE_N = 128, 256  # rows x columns of one CTA's tile, every linear (ffn.0: two CTAs per 128 x 512 LayerNorm tile)


def operand_bytes(rows: int, k: int, nout: int, passes: int) -> float:
    """Bytes the TMA ring loads for one GEMM: every tile reads TILE_M A rows and TILE_N W rows of 2-byte K."""
    return (rows / TILE_M) * (nout / TILE_N) * (TILE_M + TILE_N) * k * 2.0 * passes


def shapes(batch: int, n: int, layers: int, x3: bool) -> dict:
    """MMA FLOP, epilogue bytes and L2 operand bytes per forward of each linear class (every pair runs every layer:
    pruning is off)."""
    rows = 2 * batch * n  # S * Lp
    passes = 3 if x3 else 1
    images = 2 if x3 else 1  # bf16 hi (and lo) images
    d, ffn = 256, 512
    per_layer = {
        # self [q | k | v] (256 -> 768) + cross [qk | v] (256 -> 512); fp16 outputs
        "qkv": (2.0 * rows * d * (3 * d + 2 * d) * passes, rows * (3 * d + 2 * d) * 2,
                operand_bytes(rows, d, 3 * d, passes) + operand_bytes(rows, d, 2 * d, passes)),
        # self + cross: cat([x, ctx]) (512) -> 512, LayerNorm + GELU, bf16 images of h
        "ffn0": (2 * 2.0 * rows * (2 * d) * ffn * passes, 2 * rows * ffn * 2 * images,
                 2 * operand_bytes(rows, 2 * d, ffn, passes)),
        # self + cross: 512 -> 256 + residual: x read and written (fp32), bf16 images of x
        "ffn3": (2 * 2.0 * rows * ffn * d * passes, 2 * rows * d * (4 + 4 + 2 * images),
                 2 * operand_bytes(rows, ffn, d, passes)),
    }
    return {k: tuple(v * layers for v in vals) for k, vals in per_layer.items()}


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="bf16x3", choices=("bf16x3", "bf16"))
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("linear_breakdown: needs a CUDA device")

    torch.set_grad_enabled(False)
    m = LightGlue(features=None, depth_confidence=-1, width_confidence=-1, precision=a.precision)
    m.load_state_dict(synth.make_state_dict(), strict=False)
    m = m.eval().cuda()
    data, _ = synth.make_pair(N_KPTS, d=DESC, b=a.batch, seed=1000)
    data = {k: {kk: vv.cuda() for kk, vv in v.items()} for k, v in data.items()}
    for _ in range(3):
        m(data)
    torch.cuda.synchronize()
    m.timing = True
    for _ in range(a.steps):
        m(data)
    torch.cuda.synchronize()
    kt = m.kernel_times()

    peaks, how = measured_peaks()
    peak_tflops, hbm_gbs = peaks["bf16_tflops"], peaks["hbm_gbs"]
    for name, (flop, nbytes, l2bytes) in shapes(a.batch, N_KPTS, LAYERS, a.precision == "bf16x3").items():
        ms = kt[name][0] / a.steps
        floor_ms = max(flop / (peak_tflops * 1e12), nbytes / (hbm_gbs * 1e9)) * 1e3
        print(json.dumps({"class": name, "precision": a.precision, "ms_per_step": round(ms, 3),
                          "mma_tflop": round(flop / 1e12, 3), "epilogue_gb": round(nbytes / 1e9, 3),
                          "l2_operand_gb": round(l2bytes / 1e9, 1), "l2_operand_gbs": round(l2bytes / (ms * 1e-3) / 1e9),
                          "achieved_tflops": round(flop / (ms * 1e-3) / 1e12, 1),
                          "frac_of_bf16_peak": round(flop / (ms * 1e-3) / 1e12 / peak_tflops, 3),
                          "floor_ms": round(floor_ms, 2)}))
    other = {k: round(v[0] / a.steps, 3) for k, v in kt.items() if k in ("linear", "attention", "assign")}
    print(json.dumps({"card": card(), "peak_source": how, "bf16_tflops": peak_tflops, "hbm_gbs": hbm_gbs,
                      "ms_per_step": other}))


if __name__ == "__main__":
    main()
