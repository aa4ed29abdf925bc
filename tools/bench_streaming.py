"""Live-stream capacity of AudioStreamTranscriber: N streams cut from tests/golden/jfk.wav (looped, each from its own offset) get 2 s of
new audio per round, useVAD=False so every stream transcribes every round (the worst case), a fixed sampleLength and no ladder.  After
`--warmup` rounds, `--rounds` rounds are timed with the host clock around transcribeCurrentBuffers (which ends in a device sync).

One JSON line per N: the card name and power limit (read in this run), round wall time (median, max), windows and decode steps per
round, and headroom = 2 s / median round time (>= 1: the streams are served live).  With random weights (no --model-dir) the decoded
timestamps are noise that can confirm past the end of the buffer and leave nothing to transcribe, so the random-weight run decodes
withoutTimestamps with requiredSegmentsForConfirmation=0: every round confirms its one segment and transcribes exactly the new 2 s of
every stream, one window per stream.  The stream stop rule runs with compressionRatioThreshold 2.4 (the DecodingOptions default) over
--check-window tokens, so its per-token compression check is in the timed rounds; logProbThreshold stays off, because random weights
would stop every window at its first token.  A window ends at EOT, at sampleLength, or where the rule stops it.

    python tools/bench_streaming.py [--streams 16,32,64,128,256] [--model-dir DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import wave

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import whisperkit_b200 as wk  # noqa: E402


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         check=True).stdout.strip()
    name, power = [s.strip() for s in out.split(",", 1)]
    return {"name": name, "power_limit": power}


def jfk() -> np.ndarray:
    with wave.open(os.path.join(ROOT, "tests", "golden", "jfk.wav"), "rb") as f:
        assert f.getframerate() == 16000 and f.getnchannels() == 1 and f.getsampwidth() == 2
        x = np.frombuffer(f.readframes(f.getnframes()), dtype="<i2").astype(np.float32) / 32768.0
    return x


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--variant", default="large-v3")
    ap.add_argument("--model-dir", default=None)
    ap.add_argument("--streams", default="16,32,64,128,256")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sample-length", type=int, default=64)
    ap.add_argument("--max-batch", type=int, default=128)
    ap.add_argument("--check-window", type=int, default=60)
    ap.add_argument("--compression-ratio-threshold", type=float, default=2.4)
    args = ap.parse_args()
    info = card()
    cfg = wk.WhisperKitConfig(model=args.variant, maxBatch=args.max_batch, seed=1234, modelFolder=args.model_dir)
    kit = wk.WhisperKit(cfg)
    src = np.tile(jfk(), 64)
    step = 2 * 16000
    opts = wk.DecodingOptions(sampleLength=args.sample_length, temperatureFallbackCount=0, firstTokenLogProbThreshold=None,
                              compressionRatioThreshold=args.compression_ratio_threshold, logProbThreshold=None, noSpeechThreshold=None,
                              withoutTimestamps=args.model_dir is None)
    required = 2 if args.model_dir else 0
    for n in [int(v) for v in args.streams.split(",")]:
        tr = wk.AudioStreamTranscriber(kit, opts, requiredSegmentsForConfirmation=required, compressionCheckWindow=args.check_window, useVAD=False)
        ids = [tr.addStream() for _ in range(n)]
        offsets = [(i * 7919) % (len(src) // 2) for i in range(n)]
        times, windows, steps = [], [], []
        for r in range(args.warmup + args.rounds):
            for i, o in zip(ids, offsets):
                tr.processBuffer(i, src[o + r * step:o + (r + 1) * step])
            t0 = time.perf_counter()
            done = tr.transcribeCurrentBuffers()
            dt = time.perf_counter() - t0
            assert len(done) == n
            s = kit.textDecoder.stats()
            if r >= args.warmup:
                times.append(dt)
                windows.append(s["admissions"])
                steps.append(s["steps"])
        tr.close()
        med = statistics.median(times)
        print(json.dumps({"bench": "streaming", "variant": args.variant, "streams": n, "new_audio_s_per_round": 2.0, "use_vad": False,
                          "sample_length": args.sample_length, "weights": args.model_dir or "random", "required_segments": required,
                          "compression_ratio_threshold": args.compression_ratio_threshold, "check_window": args.check_window, "logprob_threshold": None, "round_ms_median": round(med * 1e3, 2), "round_ms_max": round(max(times) * 1e3, 2),
                          "windows_per_round": statistics.median(windows), "decode_steps_per_round": statistics.median(steps),
                          "headroom": round(2.0 / med, 3), "gpu": info}), flush=True)


if __name__ == "__main__":
    main()
