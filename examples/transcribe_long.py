"""End-to-end example on an H100: long-form transcription of 16 kHz mono WAV files with segments, text and word timestamps.

  python examples/transcribe_long.py --weights /path/to/whisper-large-v3 audio1.wav audio2.wav [--vad] [--word-timestamps]

`--weights` is a HuggingFace checkpoint directory (config.json, *.safetensors, tokenizer.json).  Without it the model runs with seeded
random weights of the large-v3 shape (the token ids are then meaningless; useful as a smoke test of the machinery only)."""
import argparse
import os
import sys
import wave

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def read_wav(path: str) -> np.ndarray:
    with wave.open(path, "rb") as w:
        if w.getframerate() != 16000 or w.getnchannels() != 1 or w.getsampwidth() != 2:
            raise SystemExit(f"{path}: need 16 kHz mono s16 (resample first: the reference does this in AudioProcessor, out of scope here)")
        pcm = np.frombuffer(w.readframes(w.getnframes()), dtype=np.int16)
    return pcm.astype(np.float32) / 32768.0          # the reference's s16 -> f32 convention


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("audio", nargs="+")
    ap.add_argument("--weights", default=None)
    ap.add_argument("--variant", default="large-v3")
    ap.add_argument("--max-batch", type=int, default=64)
    ap.add_argument("--dtype", default="bf16", choices=["bf16", "f16"])
    ap.add_argument("--vad", action="store_true", help="chunkingStrategy .vad: split long audio at silences into independent units")
    ap.add_argument("--word-timestamps", action="store_true")
    ap.add_argument("--write", default=None, metavar="DIR", help="also write <audio>.srt / .vtt / .json there (ResultWriter.swift)")
    args = ap.parse_args()

    import whisperkit_b200 as wk
    from whisperkit_b200 import longform

    kit = wk.WhisperKit(wk.WhisperKitConfig(model=args.variant, maxBatch=args.max_batch, dtype=args.dtype, modelFolder=args.weights))
    tokenizer = kit.tokenizer
    if args.word_timestamps and tokenizer is None:
        raise SystemExit("--word-timestamps needs --weights (tokenizer.json)")
    opts = wk.DecodingOptions(wordTimestamps=args.word_timestamps)
    audio = [read_wav(p) for p in args.audio]
    results = longform.transcribe_audio(kit, audio, opts, tokenizer=tokenizer, chunkingStrategy="vad" if args.vad else None)
    for path, r in zip(args.audio, results):
        print(f"== {path}: {len(r.segments)} segments, {r.windows} windows decoded in total")
        print(r.text if tokenizer else "(no tokenizer: token ids only)")
        for g in r.segments:
            print(f"  [{g.start:7.2f} -> {g.end:7.2f}] {g.text if tokenizer else g.tokens[:12]}")
            for w in (g.words or []):
                print(f"      {w.start:7.2f} {w.end:7.2f} {w.probability:4.2f} {w.word!r}")
        if args.write:
            from whisperkit_b200 import writers
            stem = os.path.splitext(os.path.basename(path))[0]
            for cls in (writers.WriteSRT, writers.WriteVTT, writers.WriteJSON):
                print("   wrote", cls(args.write).write(r, stem))


if __name__ == "__main__":
    main()
