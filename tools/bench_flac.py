"""Cost of loading FLAC files on the GPU (csrc/flac.cu: read + frame discovery + chain + decode, then the WAV path's mix + resample) against
the same audio as WAV, for one hour of 44.1 kHz stereo s16 and one hour of 16 kHz mono s16 built from tests/golden/jfk.wav (resampled,
tiled, gain-varied, seeded) and encoded with tests/flac_ref.py: 4096-sample blocks, the best fixed predictor per subframe, the best
stereo mode per frame, 16 Rice partitions (about what `flac -2` does).  The hour is 12 copies of a 5-minute unit whose length is a
whole number of blocks, so its frames are the unit's frames renumbered (the encoder codes a frame from its samples alone).

Per file, in one process and one session, alternating, --passes each:
  flac_load_s   AudioProcessor.loadAudioAsFloatArray of the FLAC file, end to end into host memory (ends in a device synchronise)
  wav_load_s    the same for the WAV twin (bit-identical output, checked)
  read_s        reading the FLAC file's bytes alone
  host_s        the same flac_core.cuh decode compiled -O2 (tests/hostcheck/flac_hostcheck.cpp) on one host core, to int32 samples
Then, in a separate torch.profiler run of one FLAC load, the device time per kernel.  Prints one JSON line with the card name and power
limit read in the same run, and writes it to --out.

    python tools/bench_flac.py --out /tmp/bench_flac [--passes 3] [--minutes 60]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
import wave

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import whisperkit_b200 as wk  # noqa: E402
from oracle import audio_ref as A  # noqa: E402
from tests import flac_ref as F  # noqa: E402
from whisperkit_b200.audio import AudioProcessor  # noqa: E402
from whisperkit_b200.build import build_flac_hostcheck  # noqa: E402

BLOCK = 4096


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         check=True).stdout.strip()
    name, power = [s.strip() for s in out.split(",", 1)]
    return {"name": name, "power_limit": power}


def unit(rate: int, channels: int, seed: int) -> np.ndarray:
    """5 minutes (rounded down to whole blocks) of jfk at `rate`, tiled with a seeded gain per tile; the right channel delayed and scaled."""
    from scipy.signal import resample_poly
    with wave.open(os.path.join(ROOT, "tests", "golden", "jfk.wav"), "rb") as w:
        j = np.frombuffer(w.readframes(w.getnframes()), "<i2").astype(np.float64)
    g = np.gcd(rate, 16000)
    j = resample_poly(j, rate // g, 16000 // g) if rate != 16000 else j
    n = (300 * rate) // BLOCK * BLOCK
    rng = np.random.default_rng(seed)
    reps = -(-n // len(j))
    x = np.concatenate([j * rng.uniform(0.3, 1.0) for _ in range(reps)])[:n]
    if channels == 2:
        x = np.stack([x, 0.6 * np.roll(x, 37) + 0.05 * x], axis=1)
    else:
        x = x[:, None]
    return np.clip(np.round(x), -32768, 32767).astype(np.int64)


def renumber(frame: bytes, number: int) -> bytes:
    """A fixed-blocking frame of this benchmark (block-size and rate codes without tails) with another frame number."""
    lead = frame[4]
    extra = 0 if lead < 0x80 else next(e for m, e in ((0xFC, 5), (0xF8, 4), (0xF0, 3), (0xE0, 2), (0xC0, 1)) if lead & m == m)
    h = frame[:4] + F.utf8_number(number)
    h = h + bytes([F.crc8(h)])
    body = h + frame[4 + 1 + extra + 1:-2]
    return body + F.crc16(body).to_bytes(2, "big")


def make(tmp: str, name: str, rate: int, channels: int, minutes: int, seed: int):
    x = unit(rate, channels, seed)
    frames = F.encode(x, rate, 16, block_size=BLOCK, stereo="auto", frames_only=True,
                      spec=lambda fi, c, v, sb: dict(kind="auto", partition=4))
    copies = minutes // 5
    full = np.tile(x, (copies, 1))
    si = F.streaminfo(BLOCK, BLOCK, min(map(len, frames)), max(map(len, frames)), rate, channels, 16, len(full), F.md5_of(full, 16))
    fp = os.path.join(tmp, f"{name}.flac")
    with open(fp, "wb") as f:
        f.write(b"fLaC" + F.metadata_block(0, si, True))
        k = 0
        for _ in range(copies):
            for fr in frames:
                f.write(renumber(fr, k) if k >= len(frames) else fr)
                k += 1
    wp = A.write_wav(os.path.join(tmp, f"{name}.wav"), full.astype(np.int16), rate, "s16")
    return fp, wp, full


def host_decode_s(lib, data: bytes, n: int) -> float:
    fmt, tot, off = (C.c_int32 * 4)(), C.c_int64(), C.c_int64()
    out = np.empty(n, np.int32)
    t = time.perf_counter()
    st = lib.wk_flac_host_decode(data, len(data), fmt, C.byref(tot), out.ctypes.data_as(C.POINTER(C.c_int32)), out.size, C.byref(off))
    dt = time.perf_counter() - t
    assert st == 0, (st, off.value)
    return dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--minutes", type=int, default=60)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    lib = C.CDLL(build_flac_hostcheck(out_dir=tempfile.mkdtemp()))
    lib.wk_flac_host_decode.argtypes = [C.c_char_p, C.c_int64, C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_int32),
                                        C.c_int64, C.POINTER(C.c_int64)]
    result = {"card": card(), "files": {}}
    model = wk.Model("toy", max_batch=1, dtype="bf16")
    model.init_random(1)
    session = wk.TextDecoder(model, 1)
    with tempfile.TemporaryDirectory() as tmp:
        for name, rate, ch in (("stereo44k", 44100, 2), ("mono16k", 16000, 1)):
            t0 = time.perf_counter()
            fp, wp, full = make(tmp, name, rate, ch, a.minutes, seed=ch)
            build_s = time.perf_counter() - t0
            data = open(fp, "rb").read()
            r = {"seconds": len(full) / rate, "flac_bytes": len(data), "wav_bytes": os.path.getsize(wp),
                 "ratio": len(data) / os.path.getsize(wp), "build_s": build_s}
            y_f = AudioProcessor.loadAudioAsFloatArray(fp, session=session)   # warm-up: page cache, workspace, filter table
            y_w = AudioProcessor.loadAudioAsFloatArray(wp, session=session)
            assert np.array_equal(y_f.view(np.uint32), y_w.view(np.uint32)), "FLAC and WAV loads differ"
            t = {"flac_load_s": [], "wav_load_s": [], "read_s": [], "host_s": []}
            for _ in range(a.passes):
                s = time.perf_counter(); AudioProcessor.loadAudioAsFloatArray(fp, session=session); t["flac_load_s"].append(time.perf_counter() - s)
                s = time.perf_counter(); AudioProcessor.loadAudioAsFloatArray(wp, session=session); t["wav_load_s"].append(time.perf_counter() - s)
                s = time.perf_counter()
                with open(fp, "rb") as f:
                    f.read()
                t["read_s"].append(time.perf_counter() - s)
                t["host_s"].append(host_decode_s(lib, data, full.size))
            for k, v in t.items():
                r[k] = {"median": statistics.median(v), "min": min(v), "max": max(v)}
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                AudioProcessor.loadAudioAsFloatArray(fp, session=session)
                torch.cuda.synchronize()
            ker = {}
            for e in prof.key_averages():
                if "flac_" in e.key or "audio_" in e.key:
                    us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                    ker[e.key] = {"ms": us / 1e3, "calls": e.count}
            r["kernels"] = ker
            result["files"][name] = r
            print(name, json.dumps(r), flush=True)
    line = json.dumps(result)
    print(line)
    with open(os.path.join(a.out, "bench_flac.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
