"""AudioStreamTranscriber (csrc/streaming.cu) against the oracle's per-stream state machine (oracle/stream_ref.py) driving the oracle's
seek loop (oracle/seek_ref.seek_loop) over the whole, untrimmed buffer, window by window through the same GPU decode with the stop rule
applied in Python.  Toy models, random weights."""
import threading
import types

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import whisperkit_b200 as wk  # noqa: E402
from oracle import decode_ref as D  # noqa: E402
from oracle import mel_ref  # noqa: E402
from oracle import seek_ref as SK  # noqa: E402
from oracle import stream_ref as SR  # noqa: E402
from whisperkit_b200.streaming import AudioStreamTranscriber  # noqa: E402

F = np.float32


def make_kit(maxBatch=8):
    st_o = D.SpecialTokens.toy(1024)
    return st_o, wk.WhisperKit(wk.WhisperKitConfig(model="toy", maxBatch=maxBatch, seed=9, specialTokens=wk.SpecialTokens.from_any(st_o)))


def speech_with_silence(seed, seconds):
    """Synthetic speech in 3-8 s stretches separated by 1.5-4 s of digital silence."""
    rng = np.random.default_rng(seed)
    out, k = [], 0
    while sum(len(x) for x in out) < seconds * 16000:
        sp = mel_ref.synthetic_pcm(seed * 37 + k).astype(np.float32)[: int(rng.uniform(3, 8) * 16000)]
        out += [sp, np.zeros(int(rng.uniform(1.5, 4) * 16000), np.float32)]
        k += 1
    return np.concatenate(out)[: seconds * 16000]


def oracle_transcriber(kit, st_o, o, W, prompt_len, word_hooks=None, log=None):
    """transcribe(buffer, clipStart) of the oracle machine: seek_loop over kit.transcribe on one window at a time (no ladder), the stream
    stop rule cutting each window's history in Python."""
    def transcribe(buffer, clip_start):
        def decode_window(seek, size):
            w = np.zeros(480000, np.float32)
            w[:size] = buffer[seek:seek + size]
            r = kit.transcribe(w[None], o, samplesPerWindow=[size])[0]
            toks, lps = list(r.tokens), list(r.tokenLogProbs)
            assert toks[0] == st_o.startOfTranscriptToken
            if toks[-1] == st_o.endToken:
                toks, lps = toks[:-1], lps[:-1]
            t = SR.stop_index(toks, lps, prompt_len, W, o.compressionRatioThreshold, o.logProbThreshold)
            f = SR.truncate_and_finalize(toks, lps, t, st_o.startOfTranscriptToken, st_o.endToken, st_o.specialTokenBegin,
                                         o.compressionRatioThreshold, o.logProbThreshold)
            out = types.SimpleNamespace(tokens=f.tokens, tokenLogProbs=f.tokenLogProbs, avgLogProb=f.avgLogProb,
                                        compressionRatio=f.compressionRatio, temperature=r.temperature, stopped=t >= 0)
            if log is not None:
                log.append((t >= 0, len(r.tokens), len(f.tokens)))
            if word_hooks is not None:
                a = np.array(kit.textDecoder.alignmentWeights(0, min(len(f.tokens), 224)))
                if t >= 0:
                    a[t + 1:] = 0                                 # rows of steps the reference never ran
                out.alignment = a
            return out
        segs, _ = SK.seek_loop(len(buffer), decode_window, clipTimestamps=[clip_start], timeToken=st_o.timeTokenBegin,
                               noSpeechThreshold=o.noSpeechThreshold, logProbThreshold=o.logProbThreshold, wordTimestamps=word_hooks)
        return segs
    return transcribe


def _toy_split(tokens, special_begin):
    """Stand-in for the host tokenizer's splitToWordTokens on the toy vocabulary (the rule of tests/test_word_timestamps_host.py)."""
    words, groups = [], []
    for t in tokens:
        if t >= special_begin:
            words.append(f"<|{t}|>"); groups.append([t])
        elif t % 17 == 0:
            words.append(","); groups.append([t])
        elif t % 3 == 0 or not words or groups[-1][0] >= special_begin:
            words.append(" " + chr(97 + t % 26)); groups.append([t])
        else:
            words[-1] += chr(97 + t % 26); groups[-1].append(t)
    return words, groups


def assert_segments_equal(got, ref, words=False):
    assert [g.tokens for g in got] == [r.tokens for r in ref]
    assert [g.seek for g in got] == [r.seek for r in ref] and [g.id for g in got] == [r.id for r in ref]
    np.testing.assert_array_equal(F([g.start for g in got]), F([r.start for r in ref]))
    np.testing.assert_array_equal(F([g.end for g in got]), F([r.end for r in ref]))
    np.testing.assert_allclose([g.avgLogprob for g in got], [r.avgLogprob for r in ref], atol=1e-5)
    if words:
        for g, r in zip(got, ref):
            assert [w.word for w in g.words] == [w.word for w in r.words]
            np.testing.assert_array_equal(F([w.start for w in g.words]), F([w.start for w in r.words]))
            np.testing.assert_array_equal(F([w.end for w in g.words]), F([w.end for w in r.words]))


def assert_state_equal(got, machine):
    ref = machine.state
    assert got.lastBufferSize == ref.lastBufferSize
    assert F(got.lastConfirmedSegmentEndSeconds) == F(ref.lastConfirmedSegmentEndSeconds)
    assert_segments_equal(got.confirmedSegments, ref.confirmedSegments)
    assert_segments_equal(got.unconfirmedSegments, ref.unconfirmedSegments)


def test_round_parity_with_oracle_machine():
    st_o, kit = make_kit(maxBatch=8)
    o = wk.DecodingOptions(firstTokenLogProbThreshold=None, logProbThreshold=None, compressionRatioThreshold=None, sampleLength=24,
                           temperatureFallbackCount=0)
    P = len(kit.textDecoder.prefillDecoderInputs(o, kit.specialTokens))
    tr = AudioStreamTranscriber(kit, o, requiredSegmentsForConfirmation=1)
    rng = np.random.default_rng(7)
    audio = [speech_with_silence(11 + i, 90) for i in range(6)]
    mean_push = [1.2, 1.5, 2.0, 1.0, 1.4, 3.0]
    ids = [tr.addStream() for _ in audio]
    machines = [SR.StreamMachine(oracle_transcriber(kit, st_o, o, 60, P), requiredSegmentsForConfirmation=1) for _ in audio]
    pos = [0] * 6
    seen = dict(confirm=0, vad=0, short=0, long_unconfirmed=0, trimmed=0, multi=0)
    for rnd in range(30):
        for i in range(6):
            k = int(rng.uniform(0.2, 1.8) * mean_push[i] * 16000) if (rnd, i) != (0, 5) else 35 * 16000   # 35 s at once: several windows
            tr.processBuffer(ids[i], audio[i][pos[i]:pos[i] + k])
            pos[i] = min(pos[i] + k, len(audio[i]))
        done = tr.transcribeCurrentBuffers()
        for i in range(6):
            before = len(machines[i].state.confirmedSegments)
            clip = int(np.floor(F(machines[i].state.lastConfirmedSegmentEndSeconds) * F(16000) + 0.5))
            did = machines[i].round(audio[i][:pos[i]])
            assert (ids[i] in done) == did, (rnd, i)
            s = tr.state(ids[i])
            assert_state_equal(s, machines[i])
            seen["confirm"] += len(machines[i].state.confirmedSegments) > before
            if did and pos[i] - clip > 480000:
                seen["long_unconfirmed"] += 1
            seen["trimmed"] += s.heldSamples < s.pushedSamples
            assert s.pushedSamples == pos[i]
        if len(done) > 1:
            seen["multi"] += 1
    seen["vad"] = sum(m.skips["vad"] for m in machines)
    seen["short"] = sum(m.skips["short"] for m in machines)
    print("stream parity coverage:", seen, "duplicates:", [m.duplicates for m in machines])
    assert [tr.state(i).duplicateConfirmations for i in ids] == [m.duplicates for m in machines]
    assert seen["confirm"] > 0 and seen["vad"] > 0 and seen["short"] > 0 and seen["long_unconfirmed"] > 0 and seen["trimmed"] > 0
    assert seen["multi"] > 0
    tr.close()


def test_round_batches_streams():
    st_o, kit = make_kit(maxBatch=8)
    o = wk.DecodingOptions(firstTokenLogProbThreshold=None, logProbThreshold=None, compressionRatioThreshold=None, sampleLength=24,
                           temperatureFallbackCount=0)
    tr = AudioStreamTranscriber(kit, o, useVAD=False)
    ids = [tr.addStream() for _ in range(6)]
    assert tr.transcribeCurrentBuffers() == []                   # nothing ready: no GPU work
    for i in ids:
        tr.processBuffer(i, mel_ref.synthetic_pcm(500 + i)[:40000].astype(np.float32))
    done = tr.transcribeCurrentBuffers()
    assert sorted(done) == ids
    s = kit.textDecoder.stats()
    print("round stats:", s)
    assert s["admissions"] >= 6 and s["steps"] < s["row_steps"]
    tr.close()


def test_early_stop_and_ladder():
    st_o, kit = make_kit(maxBatch=8)
    # compression rule with the threshold unset: every window stops once its history passes the window
    o = wk.DecodingOptions(firstTokenLogProbThreshold=None, logProbThreshold=None, compressionRatioThreshold=None, sampleLength=40,
                           temperatureFallbackCount=0)
    P = len(kit.textDecoder.prefillDecoderInputs(o, kit.specialTokens))
    W = P + 6
    audio = [speech_with_silence(70 + i, 40) for i in range(4)]
    tr = AudioStreamTranscriber(kit, o, compressionCheckWindow=W, useVAD=False)
    ids = [tr.addStream() for _ in audio]
    machines = [SR.StreamMachine(oracle_transcriber(kit, st_o, o, W, P), useVAD=False) for _ in audio]
    for rnd in range(6):
        for i, x in enumerate(audio):
            tr.processBuffer(ids[i], x[rnd * 40000:(rnd + 1) * 40000])
        tr.transcribeCurrentBuffers()
        for i, x in enumerate(audio):
            machines[i].round(x[:(rnd + 1) * 40000])
            assert_state_equal(tr.state(ids[i]), machines[i])
    segs = [g for i in ids for g in tr.state(i).confirmedSegments + tr.state(i).unconfirmedSegments]
    assert segs and all(len(g.tokens) <= W - P + 2 for g in segs)  # cut after the token with count W + 1
    tr.close()
    # log-prob rule with the ladder: a stopped window whose fallback asks for it comes back at a higher temperature.  Without timestamps
    # every window is one segment holding its whole result, so the rule can be checked on each returned history
    o2 = wk.DecodingOptions(firstTokenLogProbThreshold=None, logProbThreshold=-0.2, compressionRatioThreshold=None, sampleLength=40,
                            temperatureFallbackCount=2, withoutTimestamps=True)
    P2 = len(kit.textDecoder.prefillDecoderInputs(o2, kit.specialTokens))
    tr = AudioStreamTranscriber(kit, o2, useVAD=False)
    ids = [tr.addStream() for _ in audio]
    for i, x in enumerate(audio):
        tr.processBuffer(ids[i], x[:80000])
    tr.transcribeCurrentBuffers()
    segs = [g for i in ids for g in tr.state(i).confirmedSegments + tr.state(i).unconfirmedSegments]
    assert len(segs) == len(audio)
    stopped_hot = 0
    for g in segs:
        assert g.tokens[-1] == st_o.endToken and g.tokens[0] == st_o.startOfTranscriptToken
        hist, lps = g.tokens[:-1], g.tokenLogProbs[:-1]
        t = SR.stop_index(hist, lps, P2, 60, None, -0.2)
        assert t in (-1, len(hist) - 1), (t, len(hist))         # only the last appended token meets the rule, if any
        stopped_hot += t == len(hist) - 1 and g.temperature > 0
        if g.avgLogprob < -0.2:                                   # a window that still asks for the ladder walked all of it
            assert g.temperature == pytest.approx(0.4, abs=1e-3)
    assert stopped_hot > 0
    tr.close()


def _uncut_histories(kit, st_o, o, chunks):
    """Each chunk decoded alone as one window without the stop rule: its history (prompt + appended tokens) and log-probs."""
    out = []
    for x in chunks:
        w = np.zeros(480000, np.float32)
        w[:len(x)] = x
        r = kit.transcribe(w[None], o, samplesPerWindow=[len(x)])[0]
        toks, lps = list(r.tokens), list(r.tokenLogProbs)
        if toks[-1] == st_o.endToken:
            toks, lps = toks[:-1], lps[:-1]
        out.append((toks, lps))
    return out


def _split_threshold(values):
    """values[w] = the rule's quantity at each appended index of window w, oriented so that the window stops at the first value > thr.
    Returns a threshold midway between two observed values at least 1e-4 apart (so f32 noise cannot move a decision) under which some
    window stops strictly inside its history - neither at its first appended token nor at its last, so the stop position depends on the
    rule's value at every token - preferring one under which some other window never stops; None if there is none.  (Random-weight toy
    decodes depend little on the audio, so windows often share one trajectory and no threshold separates them.)"""
    flat = sorted(set(v for vs in values for v in vs))
    cands = [(a + b) / 2 for a, b in zip(flat, flat[1:]) if b - a > 1e-4]
    cands.sort(key=lambda c: abs(c - float(np.median(flat))))
    inside = None
    for thr in cands:
        first = [next((k for k, v in enumerate(vs) if v > thr), None) for vs in values]
        if any(f is not None and 0 < f < len(vs) - 1 for f, vs in zip(first, values)):
            if any(f is None for f in first):
                return thr
            inside = thr if inside is None else inside
    return inside


@pytest.mark.parametrize("arm", ["compression", "logprob"])
def test_stop_rule_with_thresholds_matches_oracle(arm):
    """The stop rule with real thresholds, each arm alone, against the oracle machine after every round.  With nothing confirmed
    (requiredSegmentsForConfirmation above any segment count) every round's first window of a stream is its whole buffer so far, the first
    k + 1 chunks; the thresholds are chosen on those chunks' uncut decodes so that windows stop strictly inside their histories (and, where
    the decodes allow it, some never stop)."""
    st_o, kit = make_kit(maxBatch=8)
    base = dict(firstTokenLogProbThreshold=None, sampleLength=40, temperatureFallbackCount=0, withoutTimestamps=True)
    o0 = wk.DecodingOptions(logProbThreshold=None, compressionRatioThreshold=None, **base)
    P = len(kit.textDecoder.prefillDecoderInputs(o0, kit.specialTokens))
    C_ = 40000
    audio = [speech_with_silence(150 + i, 20) for i in range(6)]
    chunks = [x[:(k + 1) * C_] for k in range(6) for x in audio]
    hist = _uncut_histories(kit, st_o, o0, chunks)
    if arm == "compression":
        for W in (6, 8, 10, 12, 16, 20, 24, 28, 32):
            vals = [[float(F(D.compression_ratio(t[i + 1 - W:i + 1]))) if i + 1 > W else 0.0 for i in range(P, len(t))] for t, _ in hist]
            thr = _split_threshold(vals)
            if thr is not None:
                break
        assert thr is not None, "no compression threshold splits the probe windows"
        o = wk.DecodingOptions(logProbThreshold=None, compressionRatioThreshold=thr, **base)
    else:
        W = 60
        vals = []
        for t, lps in hist:
            acc, vs = F(0), []
            for i, v in enumerate(lps):
                acc = F(acc + F(v))
                if i >= P:
                    vs.append(-float(acc / F(i + 1)))             # stop when avg < thr, i.e. -avg > -thr
            vals.append(vs)
        neg = _split_threshold(vals)
        assert neg is not None, "no log-prob threshold splits the probe windows"
        thr = -neg
        o = wk.DecodingOptions(logProbThreshold=thr, compressionRatioThreshold=1e6, **base)   # a ratio no window reaches
    print(f"[{arm}] window {W}, threshold {thr:.5f}")
    tr = AudioStreamTranscriber(kit, o, requiredSegmentsForConfirmation=100, compressionCheckWindow=W, useVAD=False)
    ids = [tr.addStream() for _ in audio]
    log = []
    machines = [SR.StreamMachine(oracle_transcriber(kit, st_o, o, W, P, log=log), requiredSegmentsForConfirmation=100, useVAD=False)
                for _ in audio]
    for rnd in range(6):
        for i, x in enumerate(audio):
            tr.processBuffer(ids[i], x[rnd * C_:(rnd + 1) * C_])
        assert sorted(tr.transcribeCurrentBuffers()) == ids
        for i, x in enumerate(audio):
            machines[i].round(x[:(rnd + 1) * C_])
            assert_state_equal(tr.state(ids[i]), machines[i])
    stopped = [entry for entry in log if entry[0]]
    print(f"[{arm}] windows {len(log)}, stopped {len(stopped)}")
    assert len(log) >= 36 and stopped
    assert all(cut <= uncut for _, uncut, cut in stopped) and any(cut < uncut for _, uncut, cut in stopped)   # the stop shortened decodes
    tr.close()


def test_pushes_during_rounds():
    st_o, kit = make_kit(maxBatch=8)
    o = wk.DecodingOptions(firstTokenLogProbThreshold=None, logProbThreshold=None, compressionRatioThreshold=None, sampleLength=24,
                           temperatureFallbackCount=0)
    P = len(kit.textDecoder.prefillDecoderInputs(o, kit.specialTokens))
    audio = [speech_with_silence(90 + i, 60) for i in range(3)]
    tr = AudioStreamTranscriber(kit, o, requiredSegmentsForConfirmation=1)
    ids = [tr.addStream() for _ in audio]
    stop = threading.Event()

    pos = [0] * 3

    def pusher():
        rng = np.random.default_rng(5)
        while not stop.is_set() and min(pos) < 60 * 16000:
            for i in range(3):
                k = int(rng.integers(800, 6000))
                tr.processBuffer(ids[i], audio[i][pos[i]:pos[i] + k])
                pos[i] = min(pos[i] + k, len(audio[i]))
            stop.wait(0.002)
    th = threading.Thread(target=pusher)
    th.start()
    snaps = []
    try:
        for _ in range(20):
            stop.wait(0.05)
            tr.transcribeCurrentBuffers()
            snaps.append([tr.state(i) for i in ids])
    finally:
        stop.set()
        th.join()
    # replay: each round the oracle sees exactly the snapshot the streamer transcribed (lastBufferSize), or a skip
    machines = [SR.StreamMachine(oracle_transcriber(kit, st_o, o, 60, P), requiredSegmentsForConfirmation=1) for _ in audio]
    for states in snaps:
        for i, s in enumerate(states):
            if s.transcribed:
                assert machines[i].round(audio[i][:s.lastBufferSize])
            assert_state_equal(s, machines[i])
    assert any(s.transcribed for states in snaps for s in states)
    for i in ids:
        s = tr.state(i)
        clip = int(np.floor(F(s.lastConfirmedSegmentEndSeconds) * F(16000) + 0.5))
        assert s.pushedSamples == pos[i] and 0 <= s.pushedSamples - s.heldSamples <= clip   # held + dropped = pushed; nothing past the clip start dropped
    tr.close()


def test_word_timestamps_match_oracle():
    st_o, kit = make_kit(maxBatch=8)
    o = wk.DecodingOptions(firstTokenLogProbThreshold=None, logProbThreshold=None, compressionRatioThreshold=None, sampleLength=24,
                           temperatureFallbackCount=0, wordTimestamps=True)
    P = len(kit.textDecoder.prefillDecoderInputs(o, kit.specialTokens))
    SB = st_o.specialTokenBegin
    split = lambda t: _toy_split(t, SB)                          # noqa: E731
    dec_fn = lambda t: "".join(chr(97 + v % 26) for v in t)       # noqa: E731
    hooks = dict(alignment=lambda r: r.alignment, split=split, decode=dec_fn, specialTokenBegin=SB)
    audio = [speech_with_silence(120 + i, 40) for i in range(3)]
    tr = AudioStreamTranscriber(kit, o, requiredSegmentsForConfirmation=1, useVAD=False, split_to_word_tokens=split, decode=dec_fn)
    ids = [tr.addStream() for _ in audio]
    machines = [SR.StreamMachine(oracle_transcriber(kit, st_o, o, 60, P, word_hooks=hooks), requiredSegmentsForConfirmation=1, useVAD=False)
                for _ in audio]
    n_words = 0
    for rnd in range(5):
        for i, x in enumerate(audio):
            tr.processBuffer(ids[i], x[rnd * 64000:(rnd + 1) * 64000])
        tr.transcribeCurrentBuffers()
        for i, x in enumerate(audio):
            machines[i].round(x[:(rnd + 1) * 64000])
            s = tr.state(ids[i])
            assert_state_equal(s, machines[i])
            assert_segments_equal(s.confirmedSegments + s.unconfirmedSegments,
                                  machines[i].state.confirmedSegments + machines[i].state.unconfirmedSegments, words=True)
    n_words = sum(len(g.words or []) for i in ids for g in tr.state(i).confirmedSegments + tr.state(i).unconfirmedSegments)
    assert n_words > 5
    tr.close()


def test_rejected_input():
    st_o, kit = make_kit(maxBatch=8)
    for bad in (wk.DecodingOptions(beamSize=2), wk.DecodingOptions(bestOf=2)):
        with pytest.raises(wk.WhisperError) as e:
            AudioStreamTranscriber(kit, bad)
        assert e.value.case == "invalidArgument"
    tr = AudioStreamTranscriber(kit, wk.DecodingOptions())
    for call in (lambda: tr.processBuffer(99, np.zeros(10, np.float32)), lambda: tr.state(99), lambda: tr.removeStream(99)):
        with pytest.raises(wk.WhisperError) as e:
            call()
        assert e.value.case == "invalidArgument"
    tr.close()
