"""Contextual biasing (DecodingOptions.biasPhrases): what the phrase bonus costs inside the fused decode loop.

Headline workload: large-v3 with seeded random weights, 64 x 30 s windows, bf16, greedy, sampleLength 224, thresholds nil (every
window runs one rung).  Arms, run alternately pass after pass in one process: no bias; λ = 0 with 256 x 4-token phrases (the bias path
runs, every score is today's); λ = 2 with 16 phrases; λ = 2 with 256 phrases; beam 5 without and with 256 phrases.  Phrases are
random text ids, so they rarely match a random model's output: the arms measure the per-step work of the chains and the bonus pass,
not a changed decode.  Reports the median pass and decode-loop times, the step launches, the card, and whether the λ = 0 arm's results
are byte-identical to the no-bias arm's.

    python tools/bench_bias.py [--passes 3]
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402  (synthetic windows and special tokens of the headline workload)
import whisperkit_b200 as wk  # noqa: E402
from bench_cross_kv import card  # noqa: E402
from whisperkit_b200._lib import check, wk_decode_result  # noqa: E402
from whisperkit_b200.api import attached_bias, make_batch_opts  # noqa: E402


def phrases(n, length, text_tokens, seed):
    g = np.random.default_rng(seed)
    return [[int(v) for v in g.integers(0, text_tokens, length)] for _ in range(n)]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--windows", type=int, default=64)
    ap.add_argument("--sample-length", type=int, default=224)
    ap.add_argument("--passes", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bias.py needs a CUDA device")
    W = args.windows
    model = wk.Model("large-v3", max_batch=W, dtype="bf16")
    model.init_random(seed=1234)
    stp = bench.special_tokens_for(model.info.vocab)
    st = stp.to_c()
    dec = wk.TextDecoder(model, W)
    pcm = torch.from_numpy(bench.synthetic_windows(0, W)).pin_memory()
    base = dict(sampleLength=args.sample_length, firstTokenLogProbThreshold=None, temperatureFallbackCount=0, compressionRatioThreshold=None,
                logProbThreshold=None, noSpeechThreshold=None)
    stb = stp.specialTokenBegin
    arms = [dict(name="no bias", o=wk.DecodingOptions(**base)),
            dict(name="λ=0, 256 x 4", o=wk.DecodingOptions(biasPhrases=phrases(256, 4, stb, 1), biasBoost=0.0, **base)),
            dict(name="λ=2, 16 x 4", o=wk.DecodingOptions(biasPhrases=phrases(16, 4, stb, 2), biasBoost=2.0, **base)),
            dict(name="λ=2, 256 x 4", o=wk.DecodingOptions(biasPhrases=phrases(256, 4, stb, 3), biasBoost=2.0, **base)),
            dict(name="beam 5", o=wk.DecodingOptions(beamSize=5, **base)),
            dict(name="beam 5, λ=2, 256 x 4", o=wk.DecodingOptions(beamSize=5, biasPhrases=phrases(256, 4, stb, 3), biasBoost=2.0, **base))]
    for a in arms:
        a["bo"], a["keep"] = make_batch_opts(W, a["o"], None)
        a["res"] = (wk_decode_result * W)()
        a["ms"], a["loop"] = [], []

    def run(a):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with attached_bias(model.lib, dec.handle, a["o"], stp):
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
    ident = all(bytes(x) == bytes(y) for x, y in zip(arms[0]["res"], arms[1]["res"]))
    out = {"card": card(), "workload": f"large-v3 seeded random weights, {W} x 30 s windows, bf16, sampleLength={args.sample_length}, "
                                       f"thresholds nil", "lambda0_byte_identical_to_no_bias": ident, "arms": []}
    for a in arms:
        row = {"arm": a["name"], "pass_ms": round(statistics.median(a["ms"]), 1), "pass_ms_all": [round(v, 1) for v in a["ms"]],
               "decode_ms": round(statistics.median(a["loop"]), 1), "decode_ms_all": [round(v, 1) for v in a["loop"]], "step_launches": a["steps"],
               "result_tokens": sum(r.n_tokens for r in a["res"])}
        out["arms"].append(row)
        print(json.dumps(row, ensure_ascii=False), flush=True)
    print(json.dumps(out, ensure_ascii=False))
    dec.close()
    model.close()


if __name__ == "__main__":
    main()
