"""Where the wgmma GEMM's time goes on the headline workload: large-v3, 64 windows x 30 s, 223 greedy decode steps per window, bf16,
seeded random weights (seed 1234), device PCM - the settings of `bench.py --no-cpu-baseline`.

Runs one warm-up pass and `--passes` timed passes (the TranscriptionTimings stage split of each), then one more pass under torch.profiler
(CUDA activity only).  In that pass every gemm_wgmma_kernel launch is given its role by its position in the launch order of encode_chunk
and admission: conv1, conv2, then per encoder layer QKV, out-proj + residual, FC1 + GELU, FC2 + residual, then the cross-K/V projection
of the admitted windows; everything after that is the decoder's swap-AB split-K GEMMs.  Prints one JSON line: card name and power limit
(read in this run), the median stage_ms, and per role the total kernel ms, launches and TFLOP/s computed from the shapes.

    python tools/bench_gemm_roles.py [--passes 3] [--trace out.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402  (synthetic windows and special tokens of the headline workload)
import whisperkit_b200 as wk  # noqa: E402
from whisperkit_b200._lib import check, wk_decode_result  # noqa: E402
from whisperkit_b200.api import make_batch_opts  # noqa: E402

ENC_ROLES = ("qkv", "out_proj_residual", "fc1_gelu", "fc2_residual")


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         check=True).stdout.strip()
    name, power = [s.strip() for s in out.split(",", 1)]
    return {"name": name, "power_limit": power}


def role_shapes(info, W: int) -> dict:
    """(M, N, K) of one launch of every role (encode_chunk in engine.cu, cross_kv_gemm in session.cu)."""
    d, T, L = info.d_model, info.n_audio_ctx, info.dec_layers
    M = W * T
    # conv1: 3 taps over the mel padded to 128 channels (kMelCols)
    return {"conv1": (W * 2 * T, d, 3 * 128), "conv2": (M, d, 3 * d), "qkv": (M, 3 * d, d), "out_proj_residual": (M, d, d),
            "fc1_gelu": (M, 4 * d, d), "fc2_residual": (M, d, 4 * d), "cross_kv_projection": (M, 2 * L * d, d)}


def gemm_kernels(trace_path: str) -> list:
    with open(trace_path) as f:
        ev = json.load(f)["traceEvents"]
    ks = [e for e in ev if e.get("cat") == "kernel" and "gemm_wgmma_kernel" in e.get("name", "")]
    ks.sort(key=lambda e: e["ts"])
    return ks


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--variant", default="large-v3")
    ap.add_argument("--windows", type=int, default=64)
    ap.add_argument("--sample-length", type=int, default=224)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--trace", default=None, help="keep the profiler's chrome trace at this path (default: a temporary file)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gemm_roles.py needs a CUDA device")
    W = args.windows
    info_card = card()
    pcm = torch.from_numpy(bench.synthetic_windows(0, W)).pin_memory().cuda()
    model = wk.Model(args.variant, max_batch=min(W, 64), dtype="bf16")
    model.init_random(seed=1234)
    dec = wk.TextDecoder(model, W)
    info = model.info
    st = bench.special_tokens_for(info.vocab).to_c()
    opts = wk.DecodingOptions(sampleLength=args.sample_length, firstTokenLogProbThreshold=None, temperatureFallbackCount=0)
    bo, keep = make_batch_opts(W, opts, None)
    res = (wk_decode_result * W)()
    torch.cuda.synchronize()

    def run():
        check(model.lib.wk_transcribe_windows_ex(model.handle, dec.handle, C.c_void_p(pcm.data_ptr()), W, 480000, None, C.byref(st),
                                                 C.byref(bo), res))
        torch.cuda.synchronize()

    run()   # warm-up: module load, step-graph capture
    stages = []
    for _ in range(args.passes):
        run()
        stages.append(model.last_timings())

    trace = args.trace or os.path.join(tempfile.mkdtemp(prefix="wk_gemm_roles_"), "trace.json")
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        run()
    prof.export_chrome_trace(trace)
    ks = gemm_kernels(trace)

    L = info.enc_layers
    order = ["conv1", "conv2"] + [ENC_ROLES[i % 4] for i in range(4 * L)] + ["cross_kv_projection"]
    if len(ks) < len(order):
        raise SystemExit(f"expected at least {len(order)} gemm_wgmma_kernel launches in the profiled pass, found {len(ks)}")
    shapes = role_shapes(info, W)
    roles = {}
    for e, role in zip(ks, order):
        r = roles.setdefault(role, {"ms": 0.0, "launches": 0, "kernel": e["name"]})
        r["ms"] += e["dur"] / 1000.0
        r["launches"] += 1
    for role, r in roles.items():
        M, N, K = shapes[role]
        flop = 2.0 * M * N * K * r["launches"]
        r["shape_MNK"] = [M, N, K]
        r["tflop_per_s"] = round(flop / (r["ms"] * 1e-3) / 1e12, 1)
        r["ms"] = round(r["ms"], 2)
    rest = ks[len(order):]
    roles["decoder_swap_ab"] = {"ms": round(sum(e["dur"] for e in rest) / 1000.0, 2), "launches": len(rest)}
    enc_roles = ["conv1", "conv2", *ENC_ROLES]
    out = {
        "card": info_card,
        "workload": f"{args.variant}, {W} x 30 s windows, greedy, sampleLength={args.sample_length}, bf16, seeded random init (1234), device PCM",
        "passes": args.passes,
        "stage_ms_median": {k: round(statistics.median(s[k] for s in stages), 1) for k in stages[0]},
        "stage_ms": stages,
        "gemm_roles": roles,
        "encoder_gemm_ms": round(sum(roles[r]["ms"] for r in enc_roles), 2),
    }
    dec.close()
    model.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
