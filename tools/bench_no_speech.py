"""Cost of DecodingOptions.computeNoSpeechProb on the headline workload: large-v3, 64 windows x 30 s, bf16, greedy, sampleLength 224
(bench.py's settings), in one process and one session, two arms alternating:
  on   computeNoSpeechProb=True with noSpeechThreshold, logProbThreshold and compressionRatioThreshold nil, so that the value changes no
       decision and the two arms decode the same tokens
  off  the same options without the value
Prints one JSON line: card name and power limit (read in this run), per-pass ms and the median of each arm, the decode steps each arm
launched (wk_session_stats[0]), the number of windows whose tokens are identical in the two arms, and the range of the values computed.

    python tools/bench_no_speech.py [--passes 3]
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
from whisperkit_b200.api import make_batch_opts, session_no_speech_probs  # noqa: E402


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         check=True).stdout.strip()
    name, power = [s.strip() for s in out.split(",", 1)]
    return {"name": name, "power_limit": power}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--variant", default="large-v3")
    ap.add_argument("--windows", type=int, default=64)
    ap.add_argument("--sample-length", type=int, default=224)
    ap.add_argument("--passes", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_no_speech.py needs a CUDA device")
    W = args.windows
    info_card = card()
    pcm = torch.from_numpy(bench.synthetic_windows(0, W)).pin_memory().cuda()
    torch.cuda.synchronize()
    model = wk.Model(args.variant, max_batch=min(W, 64), dtype="bf16")
    model.init_random(seed=1234)
    dec = wk.TextDecoder(model, W)
    lib = model.lib
    st_c = bench.special_tokens_for(model.info.vocab).to_c()
    base = dict(sampleLength=args.sample_length, firstTokenLogProbThreshold=None, temperatureFallbackCount=0, noSpeechThreshold=None,
                logProbThreshold=None, compressionRatioThreshold=None, seed=0)

    def run(bo):
        res = (wk_decode_result * W)()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        check(lib.wk_transcribe_windows_ex(model.handle, dec.handle, C.c_void_p(pcm.data_ptr()), W, 480000, None, C.byref(st_c), C.byref(bo), res))
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1000.0
        stats = (C.c_int64 * 4)()
        check(lib.wk_session_stats(dec.handle, stats))
        return ms, int(stats[0]), res

    arms = {}
    keep = []
    for name, on in (("on", True), ("off", False)):
        bo, k = make_batch_opts(W, wk.DecodingOptions(computeNoSpeechProb=on, **base), None)
        keep.append(k)
        arms[name] = dict(bo=bo, ms=[], steps=[])
        run(bo)   # warm-up: module load, step-graph capture
    probs = []
    for _ in range(args.passes):
        for name, a in arms.items():
            ms, steps, res = run(a["bo"])
            a["ms"].append(ms)
            a["steps"].append(steps)
            a["tokens"] = [list(res[i].tokens[:res[i].n_tokens]) for i in range(W)]
            if name == "on":
                probs = session_no_speech_probs(lib, dec.handle, W)
    out = {"card": info_card,
           "workload": f"{args.variant}, {W} x 30 s windows, greedy, sampleLength={args.sample_length}, bf16 weights, seeded random init, "
                       f"device PCM, thresholds nil",
           "arms": {n: {"pass_ms": [round(v, 1) for v in a["ms"]], "pass_ms_median": round(statistics.median(a["ms"]), 1),
                        "steps_launched": a["steps"]} for n, a in arms.items()},
           "identical_token_windows": sum(arms["on"]["tokens"][i] == arms["off"]["tokens"][i] for i in range(W)),
           "no_speech_prob_range": [min(probs), max(probs)],
           "windows_computed": sum(p == p for p in probs),
           "windows": W}
    out["overhead_pct"] = round(100.0 * (out["arms"]["on"]["pass_ms_median"] / out["arms"]["off"]["pass_ms_median"] - 1.0), 2)
    dec.close()
    model.close()
    print(json.dumps(out))
    if out["identical_token_windows"] != W:
        raise SystemExit("the two arms' tokens differ")


if __name__ == "__main__":
    main()
