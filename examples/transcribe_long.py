"""End-to-end example on an H100: long-form transcription of WAV files with segments, text and word timestamps.

  python examples/transcribe_long.py --weights /path/to/whisper-large-v3 audio1.wav audio2.wav [--vad] [--word-timestamps]
                                     [--channel I | --channels I,J,...]

Files may have any sample rate (1 kHz .. 384 kHz) and channel count, in PCM u8 / s16 / s24 / s32 or float 32; AudioProcessor.loadAudio
mixes them to mono (all channels summed by default) and resamples them to 16 kHz on the GPU.  `--weights` is a HuggingFace checkpoint
directory (config.json, *.safetensors, tokenizer.json).  Without it the model runs with seeded random weights of the large-v3 shape (the
token ids are then meaningless; useful as a smoke test of the machinery only)."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


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
    mix = ap.add_mutually_exclusive_group()
    mix.add_argument("--channel", type=int, default=None, help="transcribe this channel only (ChannelMode.specificChannel)")
    mix.add_argument("--channels", default=None, help="comma-separated channels to sum (ChannelMode.sumChannels); default: all")
    args = ap.parse_args()

    import whisperkit_b200 as wk
    from whisperkit_b200 import longform

    kit = wk.WhisperKit(wk.WhisperKitConfig(model=args.variant, maxBatch=args.max_batch, dtype=args.dtype, modelFolder=args.weights))
    tokenizer = kit.tokenizer
    if args.word_timestamps and tokenizer is None:
        raise SystemExit("--word-timestamps needs --weights (tokenizer.json)")
    opts = wk.DecodingOptions(wordTimestamps=args.word_timestamps)
    if args.channel is not None:
        mode = wk.ChannelMode.specificChannel(args.channel)
    else:
        mode = wk.ChannelMode.sumChannels([int(c) for c in args.channels.split(",")] if args.channels else None)
    audio = [wk.AudioProcessor.loadAudio(p, mode, session=kit.textDecoder) for p in args.audio]
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
