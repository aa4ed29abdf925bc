"""DecodingOptions.biasPhrases on the host: the KMP matcher of tests/bias_ref.py against brute-force suffix matching, the banked-bonus
identity, and the validation of wk_bias_create (host only, no GPU needed)."""
import ctypes as C
import random

import pytest

import whisperkit_b200 as wk
from tests import bias_ref as B
from whisperkit_b200 import _lib
from whisperkit_b200.api import bias_phrase_tokens


def brute_delta(w, history):
    """The longest k <= len(w) such that w[:k] is a suffix of history (k = len(w): a completion)."""
    for k in range(min(len(w), len(history)), 0, -1):
        if list(history[-k:]) == list(w[:k]):
            return k
    return 0


@pytest.mark.parametrize("phrase", [[1, 1, 2], [1, 2, 1, 2, 3], [4, 4, 4, 4], [5], [1, 2, 3, 1, 2, 4, 1, 2, 3, 1, 2, 3]])
def test_kmp_state_is_the_longest_phrase_prefix_ending_the_history(phrase):
    rng = random.Random(len(phrase))
    alphabet = sorted(set(phrase)) + [9]
    f = B.failure(phrase)
    for trial in range(200):
        m, since = 0, []               # since: the history after the last completion (a completion restarts from f(L))
        for _ in range(40):
            v = rng.choice(alphabet)
            since.append(v)
            k = B.delta(phrase, f, m, v)
            assert k == brute_delta(phrase, since), (phrase, since)
            if k == len(phrase):
                m = f[-1]
                since = since[len(since) - m:] if m else []
            else:
                m = k


def test_random_phrase_sets_match_brute_force_g():
    rng = random.Random(3)
    for _ in range(50):
        phrases = [[rng.randrange(4) for _ in range(rng.randint(1, 6))] for _ in range(rng.randint(1, 6))]
        s = B.BiasState(phrases, 1.0)
        hist = [[] for _ in phrases]
        for _ in range(60):
            v = rng.randrange(5)
            expect = [brute_delta(w, h + [v]) for w, h in zip(phrases, hist)]
            assert s.g(v) == max(expect)
            b = s.bonus(5)
            assert b[v] == float(max(expect) - s.G)
            s.advance(v)
            for p, (w, k) in enumerate(zip(phrases, expect)):
                hist[p] = (hist[p] + [v])
                if k == len(w):
                    keep = s.m[p]
                    hist[p] = hist[p][len(hist[p]) - keep:] if keep else []
                assert s.m[p] == brute_delta(w, hist[p]) or s.m[p] < len(w)


def test_banked_bonus_is_completed_phrases_plus_the_open_partial():
    # non-overlapping phrases: the cumulative bonus is λ·(tokens of completed phrases + the current partial match)
    phrases = [[10, 11, 12], [20, 21]]
    seq = [1, 10, 11, 12, 2, 20, 21, 10, 11, 3, 10, 11]     # completes both, breaks one partial (10 11 | 3), ends inside a partial
    s = B.BiasState(phrases, 2.0)
    acc = 0
    for i, v in enumerate(seq):
        g, G, done = s.advance(v)
        acc += g - G
        completed = sum(len(phrases[p]) for t in range(i + 1) for p in ([0] if seq[max(0, t - 2):t + 1] == [10, 11, 12] else [])) + \
            sum(2 for t in range(i + 1) if seq[max(0, t - 1):t + 1] == [20, 21])
        assert acc == completed + s.G, (i, v)
    assert acc == B.banked(phrases, 2.0, seq) == 3 + 2 + 2


def test_special_tokens_reset_every_state_and_bonus_uniform_off_chain():
    s = B.BiasState([[1, 2, 3]], 1.5)
    s.advance(1); s.advance(2)
    assert s.G == 2
    b = s.bonus(10)
    assert b[3] == 1.5 and b[1] == 1.5 * (1 - 2) and b[7] == 1.5 * -2
    s.advance(50000)
    assert s.m == [0]


def _create(tokens, lens, boost=2.0, stb=100):
    lib = _lib.load()
    h = C.c_void_p()
    t = (C.c_int32 * max(1, len(tokens)))(*tokens)
    ln = (C.c_int32 * max(1, len(lens)))(*lens)
    rc = lib.wk_bias_create(t, ln, len(lens), boost, stb, C.byref(h))
    if rc == 0:
        lib.wk_bias_free(h)
    return rc


def test_bias_create_validates_its_input():
    assert _create([1, 2, 3], [3]) == 0
    assert _create([1] * 1024, [4] * 256) == 0
    assert _create([100], [1]) == _lib.WK_ERR_INVALID_ARGUMENT            # a special token
    assert _create([-1], [1]) == _lib.WK_ERR_INVALID_ARGUMENT
    assert _create([], [0]) == _lib.WK_ERR_INVALID_ARGUMENT               # length 0
    assert _create([1] * 17, [17]) == _lib.WK_ERR_INVALID_ARGUMENT        # length 17
    assert _create([1] * 257, [1] * 257) == _lib.WK_ERR_INVALID_ARGUMENT  # more than 256 phrases
    assert _create([1] * 1040, [16] * 65) == _lib.WK_ERR_INVALID_ARGUMENT  # Σ L_p above 1024
    assert _create([1], [1], boost=-1.0) == _lib.WK_ERR_INVALID_ARGUMENT
    assert _create([1], [1], boost=float("inf")) == _lib.WK_ERR_INVALID_ARGUMENT
    lib = _lib.load()
    assert lib.wk_session_set_bias(None, None, 0) == _lib.WK_ERR_INVALID_ARGUMENT


def test_python_options_and_phrase_spellings():
    o = wk.DecodingOptions()
    assert o.biasPhrases is None and o.biasBoost == 2.0
    # the C option structs keep their layout: the set travels through wk_session_set_bias
    for s in (_lib.wk_decode_opts, _lib.wk_batch_opts):
        assert not [n for n, _ in s._fields_ if "bias" in n]

    class Tok:
        def encode(self, s):
            return [ord(ch) for ch in s]
    assert bias_phrase_tokens(["ab", [7, 8]], Tok()) == [[32, 97, 98], [97, 98], [7, 8]]
    with pytest.raises(wk.WhisperError):
        bias_phrase_tokens(["ab"], None)
