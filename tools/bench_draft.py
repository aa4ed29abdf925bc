"""Speculative greedy decoding (DecodingOptions.draftTokens): pass time, decode-loop time and rounds against draft acceptance.

The main model is large-v3 "collapsed": decoder layers 2..31 keep their random weights but get zero out-projections, FC2 and biases,
so they add exact zeros and the model computes what its first two layers compute, while every step still streams large-v3's weights
and cross K/V (the step time is representative; real checkpoints are not available offline).  Drafts: the exact one (the main's
first two layers: every proposal is accepted, the upper bound), an independent random one (almost nothing accepted, the overhead
floor) and the exact one with noise added (acceptance in between).  One draft per model (a draft is fixed once a session exists), so
each model runs its arms alternately, pass after pass: no draft, then k = 1, 3, 7.  Every arm's results are compared with the no-draft
arm of its model byte for byte.  The cross K/V cache is FP8 in every arm (256 decode rows of large-v3 do not fit in 16 bits).

    python tools/bench_draft.py [--slots 16] [--passes 3]
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
from whisperkit_b200.api import make_batch_opts  # noqa: E402


def first_layers(d, V, seed, std=0.02):
    """HF-named tensors of decoder layers 0 and 1, embedding, positions and final LayerNorm (numpy f32)."""
    g = np.random.default_rng(seed)
    r = lambda *s: (g.standard_normal(s) * std).astype(np.float32)   # noqa: E731
    w = {"model.decoder.embed_tokens.weight": r(V, d), "model.decoder.embed_positions.weight": r(448, d),
         "model.decoder.layer_norm.weight": 1 + r(d), "model.decoder.layer_norm.bias": r(d)}
    for i in range(2):
        p = f"model.decoder.layers.{i}."
        for a in ("self_attn", "encoder_attn"):
            for x in ("q", "k", "v", "out"):
                w[f"{p}{a}.{x}_proj.weight"] = r(d, d)
            for x in ("q", "v", "out"):
                w[f"{p}{a}.{x}_proj.bias"] = r(d)
        for n in ("self_attn_layer_norm", "encoder_attn_layer_norm", "final_layer_norm"):
            w[f"{p}{n}.weight"], w[f"{p}{n}.bias"] = 1 + r(d), r(d)
        w[f"{p}fc1.weight"], w[f"{p}fc1.bias"], w[f"{p}fc2.weight"], w[f"{p}fc2.bias"] = r(4 * d, d), r(4 * d), r(d, 4 * d), r(d)
    return w


def collapsed_model(slots, draft):
    model = wk.Model("large-v3", max_batch=slots, dtype="bf16", crossKVDtype="fp8")
    model.init_random(seed=1234)
    d, V, L = model.cfg.d_model, model.cfg.vocab, model.cfg.dec_layers
    w = first_layers(d, V, seed=7)
    for k, v in w.items():
        model.set_tensor(k, v)
    zero_sq, zero_fc2, zero_b = np.zeros((d, d), np.float32), np.zeros((d, 4 * d), np.float32), np.zeros(d, np.float32)
    for i in range(2, L):
        for n in ("self_attn.out_proj", "encoder_attn.out_proj"):
            model.set_tensor(f"model.decoder.layers.{i}.{n}.weight", zero_sq)
            model.set_tensor(f"model.decoder.layers.{i}.{n}.bias", zero_b)
        model.set_tensor(f"model.decoder.layers.{i}.fc2.weight", zero_fc2)
        model.set_tensor(f"model.decoder.layers.{i}.fc2.bias", zero_b)
    kind, arg = draft
    if kind == "independent":
        model.setDraftDecoder(2, seed=arg)
    else:
        g = np.random.default_rng(99)
        dw = {k: v + (g.standard_normal(v.shape).astype(np.float32) * arg * v.std() if arg else 0) for k, v in w.items()}
        model.setDraftDecoder(2, weights=dw)
    return model


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--slots", type=int, default=16, help="windows in flight in every arm (k = 7 takes 8 rows per window, 256 at most)")
    ap.add_argument("--windows", type=int, default=64)
    ap.add_argument("--sample-length", type=int, default=224)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--ks", default="1,3,7")
    ap.add_argument("--drafts", default="exact,noise:0.03,noise:0.1,noise:0.3,independent")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_draft.py needs a CUDA device")
    S, W = args.slots, args.windows
    ks = [int(v) for v in args.ks.split(",")]
    pcm = torch.from_numpy(bench.synthetic_windows(0, W)).pin_memory()
    out = {"card": card(), "workload": f"large-v3 collapsed to 2 decoder layers, {W} x 30 s windows, {S} in flight, greedy, "
                                       f"sampleLength={args.sample_length}, thresholds nil, FP8 cross K/V", "arms": []}
    for spec in args.drafts.split(","):
        kind, _, a = spec.partition(":")
        draft = (kind, 77 if kind == "independent" else (float(a) if a else 0.0))
        model = collapsed_model(S, draft)
        st = bench.special_tokens_for(model.info.vocab).to_c()
        o = wk.DecodingOptions(sampleLength=args.sample_length, firstTokenLogProbThreshold=None, temperatureFallbackCount=0,
                               compressionRatioThreshold=None, logProbThreshold=None, noSpeechThreshold=None)
        bo, keep = make_batch_opts(W, o, None)
        arms = [dict(k=0)] + [dict(k=k) for k in ks]
        for a in arms:
            a["dec"] = wk.TextDecoder(model, S * (a["k"] + 1))
            a["res"] = (wk_decode_result * W)()
            a["ms"], a["loop"], a["ident"] = [], [], True

        def run(a):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if a["k"]:
                check(model.lib.wk_transcribe_windows_draft(model.handle, a["dec"].handle, C.c_void_p(pcm.data_ptr()), W, 480000, None,
                                                            C.byref(st), C.byref(bo), a["k"], a["res"]))
            else:
                check(model.lib.wk_transcribe_windows_ex(model.handle, a["dec"].handle, C.c_void_p(pcm.data_ptr()), W, 480000, None,
                                                         C.byref(st), C.byref(bo), a["res"]))
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1000.0

        for a in arms:
            run(a)   # warm-up: module load, step-graph capture
        for _ in range(args.passes):
            for a in arms:
                a["ms"].append(run(a))
                a["loop"].append(model.last_timings()["decodingLoop"])
                a["ident"] &= all(bytes(x) == bytes(y) for x, y in zip(a["res"], arms[0]["res"]))
        for a in arms:
            ds = a["dec"].draftStats() if a["k"] else {"rounds": 0, "proposed": 0, "accepted": 0}
            steps = a["dec"].stats()["steps"]
            tokens = sum(r.n_tokens for r in a["res"])
            row = {"draft": spec, "k": a["k"], "pass_ms": round(statistics.median(a["ms"]), 1), "pass_ms_all": [round(v, 1) for v in a["ms"]],
                   "decode_loop_ms": round(statistics.median(a["loop"]), 1), "step_launches": steps, **ds,
                   "acceptance": round(ds["accepted"] / ds["proposed"], 3) if ds["proposed"] else None,
                   "tokens_per_verifying_round": round((ds["accepted"] + ds["rounds"]) / ds["rounds"], 2) if ds["rounds"] else None,
                   "result_tokens": tokens, "byte_identical_to_no_draft": a["ident"]}
            out["arms"].append(row)
            print(json.dumps(row), flush=True)
        for a in arms:
            a["dec"].close()
        model.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
