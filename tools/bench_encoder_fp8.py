"""A/B of the encoder precision policy (Model(encoderDtype="fp8")) on the headline shapes: 64 windows x 30 s, the bf16 encoder against the
FP8 encoder (QKV, FC1, FC2 on E4M3 operands), in one process.

  * encoder alone (large-v3): wk_encode of the same 64-window log-mel, the two arms alternating, `--reps` timed calls each after a warm-up;
  * whole passes (large-v3 and large-v3-turbo): wk_transcribe_windows_ex, greedy, the bench.py --no-cpu-baseline settings, the two arms
    alternating, `--passes` timed passes each; the TranscriptionTimings stage split of every pass, and how many windows' greedy tokens are
    identical between the arms;
  * --profile: a separate torch.profiler run of one large-v3 encode per arm (written under --out), the kernel time of each encoder GEMM
    role summed over the 32 layers, with FLOP/s from the shapes against the data-sheet dense peak (989 TFLOP/s BF16, 1,979 FP8).

Prints one JSON line with the card name and power limit read in the same run.  Seeded random weights (no checkpoints offline).

    python tools/bench_encoder_fp8.py [--reps 5] [--passes 3] [--profile --out DIR]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402  (synthetic windows and special tokens of the headline workload)
import whisperkit_b200 as wk  # noqa: E402
from whisperkit_b200._lib import check, wk_decode_result  # noqa: E402
from whisperkit_b200.api import make_batch_opts  # noqa: E402

ARMS = (("bf16", None), ("fp8", "fp8"))
PEAK_TFLOPS = {"bf16": 989.0, "fp8": 1979.0}


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         check=True).stdout.strip()
    name, power = [s.strip() for s in out.split(",", 1)]
    return {"name": name, "power_limit": power}


def spread(v):
    return {"median": round(statistics.median(v), 2), "min": round(min(v), 2), "max": round(max(v), 2), "n": len(v)}


def make_arm(variant, W, enc_dtype, sample_length):
    model = wk.Model(variant, max_batch=W, dtype="bf16", encoderDtype=enc_dtype)
    model.init_random(seed=1234)
    dec = wk.TextDecoder(model, W)
    st = bench.special_tokens_for(model.info.vocab)
    opts = wk.DecodingOptions(sampleLength=sample_length, firstTokenLogProbThreshold=None, temperatureFallbackCount=0)
    bo, keep = make_batch_opts(W, opts, None)
    return dict(model=model, dec=dec, st=st.to_c(), bo=bo, keep=keep, res=(wk_decode_result * W)(), ms=[], stages=[])


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1000.0


def encoder_gemm_roles(trace_path, n_layers):
    """Kernel time per encoder GEMM role from a chrome trace of one encode: the GEMM kernels in launch order are conv1, conv2, then per
    layer QKV, out-projection, FC1, FC2."""
    ev = json.load(open(trace_path))["traceEvents"]
    k = sorted((e for e in ev if e.get("cat") == "kernel" and ("gemm_wgmma_kernel" in e["name"] or "gemm_fp8_kernel" in e["name"])),
               key=lambda e: e["ts"])
    if len(k) != 2 + 4 * n_layers:
        raise RuntimeError(f"expected {2 + 4 * n_layers} GEMM kernels in one encode, found {len(k)}")
    roles = {"qkv": [], "out_proj": [], "fc1": [], "fc2": []}
    for i, e in enumerate(k[2:]):
        roles[("qkv", "out_proj", "fc1", "fc2")[i % 4]].append((e["dur"], e["name"]))
    return roles


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--windows", type=int, default=64)
    ap.add_argument("--sample-length", type=int, default=224)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--variants", default="large-v3,large-v3-turbo")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None, help="directory for the --profile traces (default: a new temporary directory)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_encoder_fp8.py needs a CUDA device")
    W = args.windows
    out = {"card": card(), "windows": W, "workload": f"{W} x 30 s windows, greedy, sampleLength={args.sample_length}, bf16 weights, "
                                                     "seeded random init, device PCM", "variants": {}}
    pcm = torch.from_numpy(bench.synthetic_windows(0, W)).pin_memory().cuda()
    torch.cuda.synchronize()
    for variant in args.variants.split(","):
        arms = {name: make_arm(variant, W, ed, args.sample_length) for name, ed in ARMS}
        res_v = {}
        if variant == "large-v3":
            # encoder alone: the same log-mel through each arm's wk_encode
            enc_ms = {name: [] for name in arms}
            mels = {name: wk.FeatureExtractor(a["model"]).logMelSpectrogram(pcm.cpu().numpy()) for name, a in arms.items()}
            encs = {name: wk.AudioEncoder(a["model"]) for name, a in arms.items()}
            for name in arms:
                encs[name].encodeFeatures(mels[name])   # warm-up
            for _ in range(args.reps):
                for name in arms:
                    enc_ms[name].append(timed(lambda: encs[name].encodeFeatures(mels[name])))
            res_v["encoder_ms"] = {name: spread(v) for name, v in enc_ms.items()}
            if args.profile:
                import tempfile
                from torch.profiler import ProfilerActivity, profile
                args.out = args.out or tempfile.mkdtemp(prefix="bench_encoder_fp8_")
                os.makedirs(args.out, exist_ok=True)
                M = W * 1500
                d = arms["bf16"]["model"].info.d_model
                flops = {"qkv": 2 * M * d * 3 * d, "out_proj": 2 * M * d * d, "fc1": 2 * M * d * 4 * d, "fc2": 2 * M * 4 * d * d}
                res_v["gemm_roles"] = {}
                for name in arms:
                    with profile(activities=[ProfilerActivity.CUDA]) as prof:
                        encs[name].encodeFeatures(mels[name])
                        torch.cuda.synchronize()
                    path = os.path.join(args.out, f"encoder_trace_{name}.json")
                    prof.export_chrome_trace(path)
                    roles = encoder_gemm_roles(path, arms[name]["model"].info.enc_layers)
                    tbl = {}
                    for role, ks in roles.items():
                        us = sum(x[0] for x in ks)
                        fp8 = "gemm_fp8_kernel" in ks[0][1]
                        tflops = flops[role] * len(ks) / (us * 1e-6) / 1e12
                        peak = PEAK_TFLOPS["fp8" if fp8 else "bf16"]
                        tbl[role] = {"ms": round(us / 1000, 2), "kernel": "fp8" if fp8 else "bf16", "TFLOPs": round(tflops, 1),
                                     "share_of_datasheet_peak": round(tflops / peak, 3)}
                    res_v["gemm_roles"][name] = tbl

        def run(a):
            return timed(lambda: check(a["model"].lib.wk_transcribe_windows_ex(a["model"].handle, a["dec"].handle, C.c_void_p(pcm.data_ptr()),
                                                                               W, 480000, None, C.byref(a["st"]), C.byref(a["bo"]), a["res"])))

        for a in arms.values():
            run(a)   # warm-up: module load, step-graph capture
        for _ in range(args.passes):
            for a in arms.values():
                a["ms"].append(run(a))
                a["stages"].append(a["model"].last_timings())
        res_v["pass_ms"] = {name: spread(a["ms"]) for name, a in arms.items()}
        res_v["encoding_stage_ms"] = {name: spread([s["encoding"] for s in a["stages"]]) for name, a in arms.items()}
        res_v["stage_ms_median"] = {name: {k: round(statistics.median(s[k] for s in a["stages"]), 1) for k in a["stages"][0]}
                                    for name, a in arms.items()}
        tok = {n: [list(a["res"][i].tokens[:a["res"][i].n_tokens]) for i in range(W)] for n, a in arms.items()}
        res_v["identical_token_windows"] = sum(tok["bf16"][i] == tok["fp8"][i] for i in range(W))
        out["variants"][variant] = res_v
        for a in arms.values():
            a["dec"].close()
            a["model"].close()
        del arms
    print(json.dumps(out))


if __name__ == "__main__":
    main()
