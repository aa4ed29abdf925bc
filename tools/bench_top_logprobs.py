"""Top log-probs (DecodingOptions.topLogProbs): what ranking the k best candidates costs inside the fused decode loop.

Headline workload: large-v3 with seeded random weights, 64 x 30 s windows, bf16, greedy, sampleLength 224, thresholds nil (every
window runs one rung), device-resident PCM.  Arms k = 0, 5 and 20 run alternately pass after pass in one process.  Reports the median
pass and decode-loop times with every pass, the step launches, whether the k > 0 results are byte-identical to k = 0, the card and its
power limit, and - from a separate torch.profiler pass per arm - the device time per launch of the sampler kernel (K7).

    python tools/bench_top_logprobs.py [--passes 3]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

import bench  # noqa: E402  (synthetic windows and special tokens of the headline workload)
import whisperkit_b200 as wk  # noqa: E402
from bench_cross_kv import card  # noqa: E402
from whisperkit_b200._lib import check, wk_decode_result  # noqa: E402
from whisperkit_b200.api import make_batch_opts, top_logprobs_set  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--windows", type=int, default=64)
    ap.add_argument("--sample-length", type=int, default=224)
    ap.add_argument("--passes", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_top_logprobs.py needs a CUDA device")
    W = args.windows
    model = wk.Model("large-v3", max_batch=W, dtype="bf16")
    model.init_random(seed=1234)
    stp = bench.special_tokens_for(model.info.vocab)
    st = stp.to_c()
    dec = wk.TextDecoder(model, W)
    pcm = torch.from_numpy(bench.synthetic_windows(0, W)).cuda()
    o = wk.DecodingOptions(sampleLength=args.sample_length, firstTokenLogProbThreshold=None, temperatureFallbackCount=0,
                           compressionRatioThreshold=None, logProbThreshold=None, noSpeechThreshold=None)
    arms = [dict(k=k) for k in (0, 5, 20)]
    for a in arms:
        a["bo"], a["keep"] = make_batch_opts(W, o, None)
        a["res"] = (wk_decode_result * W)()
        a["ms"], a["loop"] = [], []

    def run(a):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with top_logprobs_set(model.lib, dec.handle, a["k"]):
            check(model.lib.wk_transcribe_windows_ex(model.handle, dec.handle, C.c_void_p(pcm.data_ptr()), W, 480000, None, C.byref(st),
                                                     C.byref(a["bo"]), a["res"]))
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1000.0

    for a in arms:
        run(a)   # warm-up: module load, step-graph capture
        a["steps"] = dec.stats()["steps"]
    for _ in range(args.passes):
        for a in arms:
            a["ms"].append(run(a))
            a["loop"].append(model.last_timings()["decodingLoop"])
    # K7 per launch, one profiled pass per arm (the profiler slows the host: these passes are not timed above)
    for a in arms:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            run(a)
        ev = [e for e in prof.key_averages() if "sampler_kernel" in e.key]
        n = sum(e.count for e in ev)
        a["k7_launches"] = n
        a["k7_us"] = round(sum(e.device_time_total for e in ev) / max(n, 1), 2)
    ident = {f"k={a['k']}": all(bytes(x) == bytes(y) for x, y in zip(arms[0]["res"], a["res"])) for a in arms[1:]}
    out = {"card": card(), "workload": f"large-v3 seeded random weights, {W} x 30 s windows, bf16, sampleLength={args.sample_length}, "
                                  f"thresholds nil, device PCM", "byte_identical_to_k0": ident, "arms": []}
    loop0 = statistics.median(arms[0]["loop"])
    for a in arms:
        loop = statistics.median(a["loop"])
        row = {"k": a["k"], "pass_ms": round(statistics.median(a["ms"]), 1), "pass_ms_all": [round(v, 1) for v in a["ms"]],
               "decode_ms": round(loop, 1), "decode_ms_all": [round(v, 1) for v in a["loop"]],
               "decode_vs_k0_pct": round(100.0 * (loop / loop0 - 1.0), 2), "step_launches": a["steps"],
               "k7_us_per_launch": a["k7_us"], "k7_launches_profiled": a["k7_launches"]}
        out["arms"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(out))
    dec.close()
    model.close()


if __name__ == "__main__":
    main()
