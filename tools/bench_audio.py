"""Cost of loading audio files on the GPU (wk_audio_load: WAV read + H2D of the stored s16 frames + channel mix + polyphase FIR to 16 kHz
+ D2H) against scipy.signal.resample_poly on one host core, for one hour of 44.1 kHz stereo s16 (sumChannels, the default) and one hour of
48 kHz mono s16.  Both WAV files are written (seeded) into --out and read back through the page cache.

Per file, in one process and one session, alternating passes:
  load_s        AudioProcessor.loadAudioAsFloatArray, end to end into host memory (ends in a device synchronise)
  read_s        reading the file's bytes alone (the host side's floor)
  h2d_conv_s    wk_audio_convert of the frames from pinned host memory into device memory (H2D + kernels)
  dev_conv_s    wk_audio_convert from device to device memory (kernels, table and plan upload)
  kernel_s      device time of the audio kernels alone (torch.profiler over --passes device-to-device calls), with the bytes they must move
                (stored frames read once per pass they make, f32 output written once) over that time, against 3.35 TB/s
  scipy_s       numpy mix + scipy.signal.resample_poly(x, up, down) on float64, the same audio
Prints one JSON line with the card name and power limit read in the same run.

    python tools/bench_audio.py --out /tmp/bench_audio [--passes 3] [--seconds 3600]
"""
from __future__ import annotations

import argparse
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

import whisperkit_b200 as wk  # noqa: E402
from oracle import audio_ref as A  # noqa: E402
from whisperkit_b200.audio import AudioProcessor  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         check=True).stdout.strip()
    name, power = [s.strip() for s in out.split(",", 1)]
    return {"name": name, "power_limit": power}


def make(path: str, rate: int, channels: int, seconds: int, seed: int) -> np.ndarray:
    """A 440 Hz tone plus seeded noise, s16, built a minute at a time."""
    rng = np.random.default_rng(seed)
    n = rate * seconds
    s = np.empty((n, channels), np.int16)
    for a in range(0, n, rate * 60):
        b = min(n, a + rate * 60)
        t = np.arange(a, b, dtype=np.float64) / rate
        x = 0.3 * np.sin(2 * np.pi * 440.0 * t)[:, None] + 0.05 * rng.standard_normal((b - a, channels))
        s[a:b] = np.clip(np.round(x * 32767), -32768, 32767)
    A.write_wav(path, s, rate, "s16")
    return s


def timed(fn):
    t0 = time.perf_counter()
    r = fn()
    return time.perf_counter() - t0, r


def kernel_seconds(fn, passes: int) -> float:
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(passes):
            fn()
        torch.cuda.synchronize()
    tot = 0.0
    for e in prof.key_averages():
        if "audio_" in e.key:
            tot += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
    return tot * 1e-6 / passes


def bench_file(path: str, s: np.ndarray, rate: int, session, passes: int) -> dict:
    from scipy.signal import resample_poly
    ch = s.shape[1]
    up, down = A.ratio(rate)
    host_in = torch.from_numpy(s).pin_memory()
    dev_in = host_in.cuda()
    n_out = -(-len(s) * up // down)
    dev_out = torch.empty(n_out, device="cuda")
    conv = dict(channelMode=("sum", None), session=session, out=dev_out)
    AudioProcessor.loadAudioAsFloatArray(path, session=session)                   # warm: workspace, table, pinned staging
    AudioProcessor.resampleAudio(dev_in, rate, **conv)
    rows = {k: [] for k in ("load_s", "read_s", "h2d_conv_s", "dev_conv_s")}
    for _ in range(passes):
        dt, y = timed(lambda: AudioProcessor.loadAudioAsFloatArray(path, session=session))
        rows["load_s"].append(dt)

        def read():
            with open(path, "rb") as f:
                return len(f.read())
        rows["read_s"].append(timed(read)[0])
        rows["h2d_conv_s"].append(timed(lambda: AudioProcessor.resampleAudio(host_in, rate, **conv))[0])
        rows["dev_conv_s"].append(timed(lambda: AudioProcessor.resampleAudio(dev_in, rate, **conv))[0])
    same = bool(len(y) == n_out and np.array_equal(y, dev_out.cpu().numpy()))   # file and in-memory frames give the same bits
    ks = kernel_seconds(lambda: AudioProcessor.resampleAudio(dev_in, rate, **conv), passes)
    in_bytes = s.nbytes * (2 if ch > 1 else 1)                                     # the peak pass reads the frames once more
    out_bytes = n_out * 4
    t0 = time.perf_counter()
    mono = A.mono_signal(A.to_float(s, "s16"), rate, pieceSeconds=600.0)   # convertToMono per read chunk, in numpy
    ref = resample_poly(mono.astype(np.float64), up, down)
    scipy_s = time.perf_counter() - t0
    err = float(np.abs(y - ref).max())
    med = {k: statistics.median(v) for k, v in rows.items()}
    audio_s = len(s) / rate
    return {"file": os.path.basename(path), "rate": rate, "channels": ch, "audio_s": audio_s, "file_bytes": os.path.getsize(path),
            **{k: round(v, 4) for k, v in med.items()},
            "spread_s": {k: round(max(v) - min(v), 4) for k, v in rows.items()},
            "kernel_s": round(ks, 5), "kernel_bytes": in_bytes + out_bytes,
            "kernel_bytes_per_s": round((in_bytes + out_bytes) / ks / 1e9, 1) if ks > 0 else None,
            "kernel_share_of_3.35TBps": round((in_bytes + out_bytes) / ks / HBM_BYTES_PER_S, 3) if ks > 0 else None,
            "scipy_s": round(scipy_s, 3), "load_x_realtime": round(audio_s / med["load_s"], 1), "scipy_x_realtime": round(audio_s / scipy_s, 1),
            "max_abs_diff_vs_scipy_f64": err, "file_equals_in_memory": same}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True, help="directory for the two WAV files")
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--seconds", type=int, default=3600)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_audio needs a GPU"
    os.makedirs(args.out, exist_ok=True)
    info = card()
    model = wk.Model("toy", max_batch=1, dtype="bf16")   # a session owns the stream and the staging buffers; the model is not used
    model.init_random(0)
    session = wk.TextDecoder(model, 1)
    res = []
    for rate, ch, seed in ((44100, 2, 1), (48000, 1, 2)):
        path = os.path.join(args.out, f"bench_{rate}_{ch}ch_s16.wav")
        s = make(path, rate, ch, args.seconds, seed)
        res.append(bench_file(path, s, rate, session, args.passes))
        del s
    print(json.dumps({"bench": "audio_load", "card": info, "passes": args.passes, "results": res}))


if __name__ == "__main__":
    main()
