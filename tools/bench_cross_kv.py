"""A/B of the cross-attention K/V cache storage on the headline workload: large-v3, 64 windows x 30 s, 223 greedy decode steps per
window (bench.py --no-cpu-baseline settings), the bf16 cache against the FP8 (E4M3 + per-row scale) cache, in one process.

The two sessions run alternately, `--passes` timed passes each after one warm-up pass.  Prints one JSON line: card name and power limit
(read in this run), per-pass ms and the TranscriptionTimings stage split of each cache, wk_bench_kernel(0) (one layer of decoder
cross-attention over 64 rows) time, bytes and achieved GB/s, how many windows' greedy tokens are identical between the two caches, and
(--max-batch-probe) the device memory left after creating an FP8 large-v3 session with 256 decode slots.

    python tools/bench_cross_kv.py [--passes 3] [--max-batch-probe]
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
    ap.add_argument("--max-batch-probe", action="store_true", help="also create an FP8 session with 256 decode slots and report free memory")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cross_kv.py needs a CUDA device")
    W = args.windows
    info_card = card()
    pcm = torch.from_numpy(bench.synthetic_windows(0, W)).pin_memory().cuda()
    torch.cuda.synchronize()
    arms = {}
    for name, ckv in (("bf16", None), ("fp8", "fp8")):
        model = wk.Model(args.variant, max_batch=min(W, 64), dtype="bf16", crossKVDtype=ckv)
        model.init_random(seed=1234)
        dec = wk.TextDecoder(model, W)
        st = bench.special_tokens_for(model.info.vocab)
        opts = wk.DecodingOptions(sampleLength=args.sample_length, firstTokenLogProbThreshold=None, temperatureFallbackCount=0)
        bo, keep = make_batch_opts(W, opts, None)
        res = (wk_decode_result * W)()
        arms[name] = dict(model=model, dec=dec, st=st.to_c(), bo=bo, keep=keep, res=res, ms=[], stages=[])

    def run(a):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        check(a["model"].lib.wk_transcribe_windows_ex(a["model"].handle, a["dec"].handle, C.c_void_p(pcm.data_ptr()), W, 480000, None,
                                                      C.byref(a["st"]), C.byref(a["bo"]), a["res"]))
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1000.0

    for a in arms.values():
        run(a)   # warm-up: module load, step-graph capture
    for _ in range(args.passes):
        for a in arms.values():
            a["ms"].append(run(a))
            a["stages"].append(a["model"].last_timings())

    out = {"card": info_card, "workload": f"{args.variant}, {W} x 30 s windows, greedy, sampleLength={args.sample_length} "
                                          f"(steps per window {min(r.steps for r in arms['bf16']['res'])}..{max(r.steps for r in arms['bf16']['res'])}), "
                                          f"bf16 weights, seeded random init, device PCM", "arms": {}}
    for name, a in arms.items():
        ms, wk_ = C.c_float(), C.c_double()
        lib = a["model"].lib
        check(lib.wk_bench_kernel(a["model"].handle, a["dec"].handle, 0, W, 20, C.byref(ms), C.byref(wk_)))
        out["arms"][name] = {
            "cross_kv_dtype": a["model"].info.cross_kv_dtype,
            "pass_ms": [round(v, 1) for v in a["ms"]],
            "pass_ms_median": round(statistics.median(a["ms"]), 1),
            "stage_ms_median": {k: round(statistics.median(s[k] for s in a["stages"]), 1) for k in a["stages"][0]},
            "cross_attention_kernel": {"ms": round(ms.value, 4), "bytes": int(wk_.value), "GB_per_s": round(wk_.value / (ms.value * 1e-3) / 1e9, 1)},
        }
    tok = {n: [list(a["res"][i].tokens[:a["res"][i].n_tokens]) for i in range(W)] for n, a in arms.items()}
    out["identical_token_windows"] = sum(tok["bf16"][i] == tok["fp8"][i] for i in range(W))
    out["windows"] = W
    for a in arms.values():
        a["dec"].close()
        a["model"].close()
    del arms
    if args.max_batch_probe:
        model = wk.Model(args.variant, max_batch=64, dtype="bf16", crossKVDtype="fp8")
        model.init_random(seed=1234)
        try:
            dec = wk.TextDecoder(model, 256)
            free, total = torch.cuda.mem_get_info()
            out["fp8_session_256_slots"] = {"created": True, "free_GB": round(free / 1e9, 2), "total_GB": round(total / 1e9, 2)}
            dec.close()
        except wk.WhisperError as e:
            out["fp8_session_256_slots"] = {"created": False, "error": str(e)}
        model.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
