"""Cost of DecodingOptions.bestOf on large-v3 (seeded random weights, bf16, synthetic 30 s windows, device PCM), one 64-row session:
  rung         the decode loop of a temperature 0.2 rung (temperatureFallbackCount 0, thresholds nil): 64 single-sample windows against
               12 best-of-5 windows (60 rows).  The decode-loop time (wk_last_timings) per window, and the cross-attention K/V bytes one
               step reads, computed from shapes: the 5 rows of a best-of window share one K/V block
  fallback     beamSize 5, bestOf 5 where every window falls back exactly once (logProbThreshold 0, temperatureFallbackCount 1: a beam
               rung at temperature 0, then a best-of-5 rung at 0.2) against the same call with bestOf nil (beam search, no ladder);
               12 windows, wall time of the call
Passes alternate the arms after one warm-up of each.  Prints one JSON line with the card name and power limit read in this run.

    python tools/bench_best_of.py [--passes 3] [--sample-length 224]
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

ROWS = 64


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         check=True).stdout.strip()
    name, power = [s.strip() for s in out.split(",", 1)]
    return {"name": name, "power_limit": power}


def cross_kv_bytes_per_step(info, windows: int) -> int:
    """K and V of every decoder layer for every window in flight: [2][L][windows][H][T][64] 16-bit elements, read once per step (the rows
    of a window share its block)."""
    return 2 * info.dec_layers * windows * info.d_model * info.n_audio_ctx * 2


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--variant", default="large-v3")
    ap.add_argument("--sample-length", type=int, default=224)
    ap.add_argument("--passes", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_best_of.py needs a CUDA device")
    info_card = card()
    pcm = torch.from_numpy(bench.synthetic_windows(0, ROWS)).pin_memory().cuda()
    torch.cuda.synchronize()
    model = wk.Model(args.variant, max_batch=ROWS, dtype="bf16")
    model.init_random(seed=1234)
    dec = wk.TextDecoder(model, ROWS)
    lib = model.lib
    st_c = bench.special_tokens_for(model.info.vocab).to_c()
    nil = dict(sampleLength=args.sample_length, firstTokenLogProbThreshold=None, noSpeechThreshold=None, compressionRatioThreshold=None, seed=0)

    def run(arm):
        W = arm["windows"]
        res = (wk_decode_result * W)()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        check(lib.wk_transcribe_windows_ex(model.handle, dec.handle, C.c_void_p(pcm.data_ptr()), W, 480000, None, C.byref(st_c),
                                           C.byref(arm["bo"]), res))
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1000.0
        stats = (C.c_int64 * 4)()
        check(lib.wk_session_stats(dec.handle, stats))
        return ms, model.last_timings()["decodingLoop"], [int(v) for v in stats], [round(res[i].temperature, 3) for i in range(W)]

    rung = dict(temperature=0.2, temperatureFallbackCount=0, logProbThreshold=None, **nil)
    fallback = dict(beamSize=5, temperature=0.0, temperatureFallbackCount=1, logProbThreshold=0.0, **nil)
    arms = {"single_x64": dict(windows=64, opts=wk.DecodingOptions(**rung)),
            "best_of_5_x12": dict(windows=12, opts=wk.DecodingOptions(bestOf=5, **rung)),
            "beam5_best_of_5_fallback_x12": dict(windows=12, opts=wk.DecodingOptions(bestOf=5, **fallback)),
            "beam5_no_best_of_x12": dict(windows=12, opts=wk.DecodingOptions(**fallback))}
    keep = []
    for a in arms.values():
        a["bo"], k = make_batch_opts(a["windows"], a["opts"], None)
        keep.append(k)
        a.update(wall_ms=[], loop_ms=[])
        run(a)   # warm-up: module load, step-graph capture for this row geometry
    for _ in range(args.passes):
        for a in arms.values():
            ms, loop_ms, stats, temps = run(a)
            a["wall_ms"].append(ms)
            a["loop_ms"].append(loop_ms)
            a["stats"], a["temperatures"] = stats, sorted(set(temps))
    out = {"card": info_card,
           "workload": f"{args.variant}, 30 s synthetic windows, sampleLength={args.sample_length}, bf16 weights, seeded random init, "
                       f"device PCM, a {ROWS}-row session",
           "arms": {}}
    for n, a in arms.items():
        W = a["windows"]
        med_loop = statistics.median(a["loop_ms"])
        out["arms"][n] = {"windows": W, "wall_ms": [round(v, 1) for v in a["wall_ms"]], "wall_ms_median": round(statistics.median(a["wall_ms"]), 1),
                          "decode_loop_ms": [round(v, 1) for v in a["loop_ms"]], "decode_loop_ms_median": round(med_loop, 1),
                          "decode_loop_ms_per_window": round(med_loop / W, 2), "steps_launched": a["stats"][0],
                          "row_steps": a["stats"][1], "ladder_readmissions": a["stats"][3], "temperatures": a["temperatures"]}
    info = model.info
    out["cross_kv_bytes_per_step"] = {"single_x64": cross_kv_bytes_per_step(info, 64), "best_of_5_x12": cross_kv_bytes_per_step(info, 12)}
    r = out["arms"]
    out["best_of_5_vs_single_per_window"] = round(r["best_of_5_x12"]["decode_loop_ms_per_window"] / r["single_x64"]["decode_loop_ms_per_window"], 2)
    out["beam5_fallback_vs_no_best_of_wall"] = round(r["beam5_best_of_5_fallback_x12"]["wall_ms_median"] / r["beam5_no_best_of_x12"]["wall_ms_median"], 2)
    dec.close()
    model.close()
    print(json.dumps(out))
    if r["beam5_best_of_5_fallback_x12"]["ladder_readmissions"] != 12 or r["beam5_no_best_of_x12"]["ladder_readmissions"] != 0:
        raise SystemExit("the fallback arms did not walk the ladder as set up")


if __name__ == "__main__":
    main()
