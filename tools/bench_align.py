"""Cost of the teacher-forced alignment pass (wk_align_windows) against a greedy decode of the same windows (wk_transcribe_windows_ex):
large-v3, 64 windows x 30 s, bf16, seeded random weights, device PCM, 224-token sequences (4 prompt tokens, 219 text tokens, EOT), in one
process and one session, the two arms alternating over several passes.  The decode arm runs bench.py's settings (sampleLength 224, no
thresholds, no fallback).  Both arms include mel + encoder + cross K/V.  A last pass of the align arm runs under torch.profiler for the
per-kernel split.  Prints one JSON line: card name and power limit (read in this run), per-pass ms, medians and spreads, and the profile's
top kernels by device time.

    python tools/bench_align.py [--passes 3]
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402  (synthetic windows and special tokens of the headline workload)
import whisperkit_b200 as wk  # noqa: E402
from whisperkit_b200._lib import check, wk_decode_result  # noqa: E402
from whisperkit_b200.api import _flatten_token_lists, make_batch_opts  # noqa: E402


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         check=True).stdout.strip()
    name, power = [s.strip() for s in out.split(",", 1)]
    return {"name": name, "power_limit": power}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--variant", default="large-v3")
    ap.add_argument("--windows", type=int, default=64)
    ap.add_argument("--passes", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_align.py needs a CUDA device")
    W = args.windows
    info_card = card()
    pcm = torch.from_numpy(bench.synthetic_windows(0, W)).pin_memory().cuda()
    torch.cuda.synchronize()
    model = wk.Model(args.variant, max_batch=min(W, 64), dtype="bf16")
    model.init_random(seed=1234)
    dec = wk.TextDecoder(model, W)
    lib = model.lib
    sp = bench.special_tokens_for(model.info.vocab)
    st_c = sp.to_c()
    rng = np.random.default_rng(0)
    prompt = [sp.startOfTranscriptToken, sp.englishToken, sp.transcribeToken, sp.noTimestampsToken]
    seqs = [prompt + [int(v) for v in rng.integers(0, sp.specialTokenBegin, 219)] + [sp.endToken] for _ in range(W)]
    flat, offsets = _flatten_token_lists(seqs)
    status = (C.c_int32 * W)()
    bo, keep = make_batch_opts(W, wk.DecodingOptions(sampleLength=224, firstTokenLogProbThreshold=None, temperatureFallbackCount=0,
                                                     noSpeechThreshold=None, logProbThreshold=None, compressionRatioThreshold=None, seed=0), None)

    def run_align():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        check(lib.wk_align_windows(model.handle, dec.handle, C.c_void_p(pcm.data_ptr()), W, 480000, None, C.byref(st_c),
                                   C.c_void_p(flat.ctypes.data), C.c_void_p(offsets.ctypes.data), status))
        torch.cuda.synchronize()
        assert all(v == 0 for v in status)
        return (time.perf_counter() - t0) * 1000.0

    def run_decode():
        res = (wk_decode_result * W)()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        check(lib.wk_transcribe_windows_ex(model.handle, dec.handle, C.c_void_p(pcm.data_ptr()), W, 480000, None, C.byref(st_c), C.byref(bo), res))
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1000.0

    run_align(); run_decode()   # warm-up: module load, step-graph capture, workspace allocation
    arms = {"align": [], "decode": []}
    for _ in range(args.passes):
        arms["align"].append(run_align())
        arms["decode"].append(run_decode())
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        run_align()
    kernels = []
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = getattr(e, "cuda_time_total", 0)
        if t > 0:
            kernels.append((e.key, t / 1000.0, e.count))
    kernels.sort(key=lambda k: -k[1])
    total = sum(k[1] for k in kernels)
    out = {"card": info_card,
           "workload": f"{args.variant}, {W} x 30 s windows, bf16 weights, seeded random init, device PCM; align: 224-token sequences; "
                       f"decode: greedy, sampleLength 224, thresholds nil",
           "arms": {n: {"pass_ms": [round(v, 1) for v in ms], "pass_ms_median": round(statistics.median(ms), 1),
                        "spread_ms": round(max(ms) - min(ms), 1)} for n, ms in arms.items()},
           "profile_align_kernels_ms": [{"kernel": k[0][:90], "ms": round(k[1], 2), "launches": k[2]} for k in kernels[:12]],
           "profile_align_total_kernel_ms": round(total, 1),
           "windows": W}
    out["align_over_decode"] = round(out["arms"]["align"]["pass_ms_median"] / out["arms"]["decode"]["pass_ms_median"], 4)
    dec.close()
    model.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
