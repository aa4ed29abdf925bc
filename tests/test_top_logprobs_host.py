"""DecodingOptions.topLogProbs on the host: the float64 rule of tests/top_logprobs_ref.py on hand-made rows (ties, -inf, short rows,
temperature, the timestamp rule), and the Python plumbing - option validation, the [n][k] arrays as per-position dicts, the long-form
segment slices and the stream refusal (no GPU needed)."""
import math
import types

import numpy as np
import pytest

import whisperkit_b200 as wk
from oracle import decode_ref as D
from tests import top_logprobs_ref as TL
from whisperkit_b200._lib import wk_segment
from whisperkit_b200.api import MAX_TOP_LOGPROBS, top_logprob_dicts, top_logprobs_of
from whisperkit_b200.longform import TranscriptionSegment, _segs

NEG = -np.inf


# ------------------------------------------------------------------------------------------------ the rule
def test_ranking_ties_go_to_the_lower_id_and_minus_inf_never_appears():
    row = np.array([1.0, 3.0, NEG, 3.0, 2.0, NEG, 2.0], np.float32)
    got = TL.top_logprobs(row, 10)
    assert [t for t, _ in got] == [1, 3, 4, 6, 0]                  # five finite entries: fewer than k
    vals = [v for _, v in got]
    assert vals[0] == vals[1] and vals[2] == vals[3] and all(a >= b for a, b in zip(vals, vals[1:]))
    x = row[np.isfinite(row)].astype(np.float64)
    lse = math.log(np.exp(x).sum())
    assert got[0][1] == pytest.approx(3.0 - lse, abs=1e-12)
    assert TL.top_logprobs(row, 2) == got[:2]
    assert TL.top_logprobs(np.full(4, NEG, np.float32), 3) == []
    assert TL.top_logprobs(row, 0) == []


def test_temperature_uses_the_tempered_softmax_of_the_whole_filtered_row():
    rng = np.random.default_rng(1)
    row = rng.normal(size=64).astype(np.float32)
    row[::5] = NEG
    t = 0.6
    got = TL.top_logprobs(row, 5, t)
    y = row.astype(np.float64) / float(np.float32(t))
    fin = np.isfinite(y)
    ref = y - (y[fin].max() + math.log(np.exp(y[fin] - y[fin].max()).sum()))
    for tok, v in got:
        assert v == pytest.approx(ref[tok], abs=1e-12)
    assert [tok for tok, _ in got] == [tok for tok, _ in TL.top_logprobs(row, 5, 0.0)]   # the ranking does not depend on t
    # probabilities of every finite candidate sum to 1: the normaliser is the whole row, not the topK cut
    assert sum(math.exp(v) for _, v in TL.top_logprobs(row, 64, t)) == pytest.approx(1.0, abs=1e-12)


def test_when_the_timestamp_rule_wins_only_timestamps_are_candidates_normalised_over_them():
    st = D.SpecialTokens.toy(1024)
    V = 1024
    logits = np.full(V, -5.0, np.float32)
    logits[st.timeTokenBegin:] = 1.0                                # timestamps carry the mass
    logits[10] = 2.0                                                # the best single token is text
    o = D.DecodingOptions()
    prompt = [st.startOfTranscriptToken, st.englishToken, st.transcribeToken]
    row = TL.filtered_row(logits, prompt, o, st, True, len(prompt))
    assert TL.timestamp_rule_won(row, st)
    got = TL.top_logprobs(row, 20)
    assert len(got) == 20 and all(t >= st.timeTokenBegin for t, _ in got)
    n_ts = int(np.isfinite(row[st.timeTokenBegin:]).sum())
    assert got[0][1] == pytest.approx(-math.log(n_ts), abs=1e-12)   # uniform over the unmasked timestamps
    assert st.noTimestampsToken not in dict(got)


def test_near_ties_may_swap_at_the_cut():
    row = np.array([5.0, 4.0, 3.0, 3.0 + 5e-7, 1.0])
    assert TL.sets_match([0, 1, 2], [0, 1, 3], row)
    assert not TL.sets_match([0, 1, 4], [0, 1, 3], row)
    assert TL.sets_match([1, 0], [0, 1], row)


# ------------------------------------------------------------------------------------------------ the Python plumbing
def test_option_validation():
    O = wk.DecodingOptions
    assert O().topLogProbs == 0
    assert top_logprobs_of(O()) == 0
    assert top_logprobs_of([O(topLogProbs=5), O(topLogProbs=5)]) == 5
    assert top_logprobs_of(O(topLogProbs=MAX_TOP_LOGPROBS)) == 20
    for bad in (-1, 21):
        with pytest.raises(wk.WhisperError) as e:
            top_logprobs_of(O(topLogProbs=bad))
        assert e.value.case == "invalidArgument"
    with pytest.raises(wk.WhisperError) as e:
        top_logprobs_of([O(topLogProbs=1), O(topLogProbs=2)])
    assert e.value.case == "invalidArgument"


def test_flat_pairs_become_one_dict_per_position():
    k = 3
    # position 0: forced (all padding); 1: three candidates; 2: two finite candidates, then padding; 3: the closing EOT (padding)
    tok = [-1, -1, -1, 7, 2, 9, 4, 5, -1, -1, -1, -1]
    lp = [NEG, NEG, NEG, -0.1, -2.5, -3.0, -0.5, -0.9, NEG, NEG, NEG, NEG]
    d = top_logprob_dicts(tok, lp, 4, k)
    assert d == [{}, {7: -0.1, 2: -2.5, 9: -3.0}, {4: -0.5, 5: -0.9}, {}]
    assert list(d[1]) == [7, 2, 9]                                  # insertion order is best first
    assert all(type(t) is int and type(v) is float for x in d for t, v in x.items())
    assert top_logprob_dicts([], [], 0, k) == []


def test_results_and_segments_default_to_empty_lists():
    r = wk.DecodingResult([1, 2], [0.0, -0.5], -0.25, 1.0, 0.0, None)
    assert r.topLogProbs == []
    g = TranscriptionSegment(0, 0, 0, 0.0, 1.0, [1], [0.0], 0.0, 0.0, 1.0, 0.0)
    assert g.topLogProbs == []


def test_long_form_segments_slice_their_pairs_like_their_log_probs():
    k = 2
    tokens = [10, 11, 12, 13, 14]
    lps = [-0.1, -0.2, -0.3, -0.4, -0.5]
    ttok = [10, 3, 11, 4, -1, -1, 13, 6, 14, -1]
    tlp = [-0.1, -1.0, -0.2, -2.0, NEG, NEG, -0.4, -4.0, -0.5, NEG]
    raw = (wk_segment * 2)()
    raw[0].token_offset, raw[0].n_tokens = 0, 2
    raw[1].token_offset, raw[1].n_tokens = 2, 3
    segs = _segs(raw, 2, tokens, lps, top=((ttok, tlp), k))
    assert [g.tokenLogProbs for g in segs] == [[-0.1, -0.2], [-0.3, -0.4, -0.5]]
    assert segs[0].topLogProbs == [{10: -0.1, 3: -1.0}, {11: -0.2, 4: -2.0}]
    assert segs[1].topLogProbs == [{}, {13: -0.4, 6: -4.0}, {14: -0.5}]
    assert all(len(g.topLogProbs) == len(g.tokenLogProbs) for g in segs)
    assert all(g.topLogProbs == [] for g in _segs(raw, 2, tokens, lps))


def test_the_stream_transcriber_refuses_the_option():
    kit = types.SimpleNamespace(resolveLanguage=lambda o: o)
    with pytest.raises(wk.WhisperError) as e:
        wk.AudioStreamTranscriber(kit, wk.DecodingOptions(topLogProbs=5))
    assert e.value.case == "invalidArgument"
