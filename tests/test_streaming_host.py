"""Stream transcription host pieces without a GPU: the library's relative energy and isVoiceDetected against oracle/stream_ref.py, and
the oracle's own confirmation and stop-rule semantics on hand-written cases (AudioStreamTranscriber.swift, AudioProcessor.swift)."""
import numpy as np
import pytest

from oracle import stream_ref as SR
from whisperkit_b200 import streaming as S

F = np.float32


def test_relative_energy_matches_oracle_on_random_pcm():
    rng = np.random.default_rng(0)
    for n in (0, 1599, 1600, 1601, 16000, 48000 + 700):
        x = (rng.standard_normal(n) * rng.uniform(0.001, 0.5)).astype(np.float32)
        x[: n // 3] *= 0.01                                       # quiet start, louder after
        got = S.relativeEnergy(x)
        ref = SR.relative_energies(x)
        assert len(got) == n // 1600                              # a trailing partial block does not count
        np.testing.assert_array_equal(got, np.float32(ref))


def test_relative_energy_hand_built_cases():
    blk = lambda v: np.full(1600, v, np.float32)                   # noqa: E731  (constant block: RMS = |v|)
    # first block: no reference (inf) -> NaN -> 0; silent blocks: log10(0) = -inf -> 0
    e = S.relativeEnergy(np.concatenate([blk(0.5), blk(0.0), blk(0.0)]))
    assert list(e) == [0.0, 0.0, 0.0]
    # the 1e-8 floor: after a silent block the reference is max(1e-8, 0) = 1e-8, i.e. -160 dB
    e = S.relativeEnergy(np.concatenate([blk(0.0), blk(1e-4)]))
    assert e[1] == SR.calculate_relative_energy(F(1e-4), F(0.0)) and abs(float(e[1]) - 0.5) < 1e-6
    # loud after quiet clamps to 1 (signal above full scale) and equal level is 0
    e = S.relativeEnergy(np.concatenate([blk(0.01), blk(2.0), blk(0.01)]))
    assert e[1] == 1.0 and e[2] == 0.0
    # the 20-block window: a quiet block 21 blocks back no longer sets the reference
    x = np.concatenate([blk(0.001)] + [blk(0.1)] * 20 + [blk(0.1)])
    e = S.relativeEnergy(x)
    np.testing.assert_array_equal(e, np.float32(SR.relative_energies(x)))
    assert e[20] > 0 and e[21] == 0.0
    # blocks are counted from the start of the stream, whatever the push sizes
    y = np.random.default_rng(1).standard_normal(20000).astype(np.float32) * 0.1
    np.testing.assert_array_equal(S.relativeEnergy(y[:17001]), S.relativeEnergy(y)[:10])


@pytest.mark.parametrize("n_values", [0, 5, 10, 19, 20, 21, 35, 80])
def test_is_voice_detected_matches_oracle(n_values):
    rng = np.random.default_rng(n_values)
    for trial in range(40):
        e = rng.uniform(0, 0.5, n_values).astype(np.float32)
        hot = rng.integers(0, max(1, n_values))
        if n_values:
            e[hot] = 0.9
        for secs in (-1.0, 0.0, 0.05, 0.3, 1.0, 1.05, 2.0, 2.5, 3.7, 10.0):
            thr = float(rng.choice([0.3, 0.6, 0.95]))
            assert S.isVoiceDetected(e, secs, thr) == SR.is_voice_detected(e, secs, thr), (n_values, trial, secs, thr)


def test_is_voice_detected_window_rules():
    loud_last = np.zeros(30, np.float32)
    loud_last[-1] = 1.0
    # 20 or more values: all but the last 10 are checked -> the last second is not
    assert not S.isVoiceDetected(loud_last, 3.0, 0.3) and not SR.is_voice_detected(loud_last, 3.0, 0.3)
    # fewer than 20: the first 10 are checked
    assert S.isVoiceDetected(loud_last, 1.0, 0.3)
    e = np.zeros(15, np.float32)
    e[-1] = 1.0
    assert not S.isVoiceDetected(e, 1.5, 0.3) and S.isVoiceDetected(e[-10:], 1.0, 0.3)
    # k > count: suffix is the whole list
    assert S.isVoiceDetected(np.float32([0.9, 0, 0]), 100.0, 0.3)
    # nextBufferSeconds <= 0: nothing to check
    assert not S.isVoiceDetected(np.ones(5, np.float32), 0.0, 0.3) and not S.isVoiceDetected(np.ones(5, np.float32), -2.0, 0.3)


class Seg:
    def __init__(self, start, end, seek=0, tokens=(1,)):
        self.start, self.end, self.seek, self.tokens, self.tokenLogProbs = start, end, seek, list(tokens), [0.0] * len(tokens)


def test_confirmation_rules():
    m = SR.StreamMachine(transcribe=None, requiredSegmentsForConfirmation=2)
    a, b = Seg(0.0, 1.0), Seg(1.0, 2.0)
    m.apply([a, b])                                               # <= R segments: all unconfirmed
    assert m.state.confirmedSegments == [] and m.state.unconfirmedSegments == [a, b] and m.state.lastConfirmedSegmentEndSeconds == 0.0
    c = Seg(2.0, 3.5, tokens=(2,))
    m.apply([a, b, c])                                            # 3 > 2: the first is confirmed
    assert m.state.confirmedSegments == [a] and m.state.unconfirmedSegments == [b, c] and m.state.lastConfirmedSegmentEndSeconds == 1.0
    # a candidate ending at or before lastConfirmed: nothing is appended, unconfirmed is still the last R
    d, e = Seg(3.5, 4.0, tokens=(3,)), Seg(4.0, 5.0, tokens=(4,))
    m.apply([Seg(0.5, 1.0), d, e])
    assert m.state.confirmedSegments == [a] and m.state.unconfirmedSegments == [d, e] and m.state.lastConfirmedSegmentEndSeconds == 1.0
    # candidates already confirmed (a contiguous equal run): lastConfirmed moves, nothing is appended, the oracle counts it
    m.state.lastConfirmedSegmentEndSeconds = 0.5
    m.apply([Seg(0.0, 1.0), d, e])
    assert m.state.confirmedSegments == [a] and m.duplicates == 1 and m.state.lastConfirmedSegmentEndSeconds == 1.0


def test_stop_rule_threshold_unset_and_prompt():
    P = 4
    toks = [50258, 50259, 50359, 50364] + list(range(10, 30))
    lps = [0.0] * P + [-0.1] * 20
    # compressionRatioThreshold unset: ratio > 0.0 always, so the window stops at the first token with count > window
    assert SR.stop_index(toks, lps, P, 6, None, None) == 6
    assert SR.stop_index(toks, lps, P, 2, None, None) == P      # prefill history (count 3 > 2 at index 2) never stops
    assert SR.stop_index(toks, lps, P, 60, None, None) == -1
    # avg log-prob includes the prompt's zeros: (-0.1 * 3) / 7 = -0.0428 < -0.04, (-0.1 * 2) / 6 = -0.033 is not
    assert SR.stop_index(toks, lps, P, 60, None, -0.04) == 6
    # a set compression threshold: repetitive history compresses well
    rep = [50258, 50259, 50359, 50364] + [7, 8] * 20
    assert SR.stop_index(rep, [0.0] * len(rep), P, 10, 2.4, None) > 0
    assert SR.stop_index(toks, lps, P, 10, 2.4, None) == -1


def test_truncate_and_finalize():
    sot, eot, sb = 50258, 50257, 50257
    toks = [sot, 50259, 50359, 50364, 11, 12, 13, 14]
    lps = [0.0] * 4 + [-1.0, -2.0, -3.0, -4.0]
    f = SR.truncate_and_finalize(toks, lps, 5, sot, eot, sb, 2.4, -1.0)
    assert f.tokens == [sot, 50259, 50359, 50364, 11, 12, eot] and f.tokenLogProbs[-1] == 0.0
    assert f.avgLogProb == pytest.approx(-3.0 / 7) and f.needsFallback is False
    f = SR.truncate_and_finalize(toks, lps, -1, sot, eot, sb, None, -1.0)
    assert len(f.tokens) == 9 and f.avgLogProb == pytest.approx(-10.0 / 9) and f.needsFallback is True
