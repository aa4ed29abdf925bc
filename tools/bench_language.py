"""Cost of in-loop language detection on the headline workload: large-v3, 64 windows x 30 s, bf16, greedy, sampleLength 224
(bench.py's settings), in one process and one session, two arms alternating:
  detect    DecodingOptions(detectLanguage=True) with the 100 large-v3 language tokens: every window detects on its own step 0 and
            decodes with the prompt rebuilt around the detected <|xx|>
  explicit  each window's languageToken set up front to what the detect arm found (no detection)
Prints one JSON line: card name and power limit (read in this run), per-pass ms of each arm, the decode steps each arm launched
(wk_session_stats[0]), the detected-language histogram, and whether the two arms' tokens are identical for every window.

    python tools/bench_language.py [--passes 3]
"""
from __future__ import annotations

import argparse
import collections
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
from whisperkit_b200.api import language_tokens, make_batch_opts, session_languages  # noqa: E402


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
        raise SystemExit("bench_language.py needs a CUDA device")
    W = args.windows
    info_card = card()
    pcm = torch.from_numpy(bench.synthetic_windows(0, W)).pin_memory().cuda()
    torch.cuda.synchronize()
    model = wk.Model(args.variant, max_batch=min(W, 64), dtype="bf16")
    model.init_random(seed=1234)
    dec = wk.TextDecoder(model, W)
    lib = model.lib
    st = bench.special_tokens_for(model.info.vocab)
    st_c = st.to_c()
    langs = language_tokens(st, model.info.vocab)
    base = dict(sampleLength=args.sample_length, firstTokenLogProbThreshold=None, temperatureFallbackCount=0)

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

    det_bo, det_keep = make_batch_opts(W, wk.DecodingOptions(detectLanguage=True, allLanguageTokens=langs, **base), None)
    run(det_bo)   # warm-up: module load, step-graph capture
    detected, det_lp = session_languages(lib, dec.handle, W)
    if min(detected) < 0:
        raise SystemExit("a window did not detect a language")
    exp_bo, exp_keep = make_batch_opts(W, [wk.DecodingOptions(languageToken=t, **base) for t in detected], None)
    run(exp_bo)
    arms = {"detect": dict(bo=det_bo, ms=[], steps=[]), "explicit": dict(bo=exp_bo, ms=[], steps=[])}
    for _ in range(args.passes):
        for a in arms.values():
            ms, steps, res = run(a["bo"])
            a["ms"].append(ms)
            a["steps"].append(steps)
            a["tokens"] = [list(res[i].tokens[:res[i].n_tokens]) for i in range(W)]
            a["win_steps"] = [res[i].steps for i in range(W)]
    out ={"card": info_card,
           "workload": f"{args.variant}, {W} x 30 s windows, greedy, sampleLength={args.sample_length}, bf16 weights, seeded random init, "
                       f"device PCM, {len(langs)} language tokens",
           "arms": {n: {"pass_ms": [round(v, 1) for v in a["ms"]], "pass_ms_median": round(statistics.median(a["ms"]), 1),
                        "steps_launched": a["steps"]} for n, a in arms.items()},
           "detected_languages": dict(collections.Counter(int(t) for t in detected).most_common()),
           "identical_token_windows": sum(arms["detect"]["tokens"][i] == arms["explicit"]["tokens"][i] for i in range(W)),
           "identical_window_steps": arms["detect"]["win_steps"] == arms["explicit"]["win_steps"],
           "windows": W}
    out["overhead_pct"] = round(100.0 * (out["arms"]["detect"]["pass_ms_median"] / out["arms"]["explicit"]["pass_ms_median"] - 1.0), 2)
    dec.close()
    model.close()
    print(json.dumps(out))
    if out["identical_token_windows"] != W:
        raise SystemExit("the two arms' tokens differ")


if __name__ == "__main__":
    main()
