"""DecodingOptions.bestOf without a GPU: openai/whisper's per-rung decoder rule (tests/best_of_ref.py), the best-of ranker
(oracle/best_of_ref.py), and the wk_batch_opts field and entry point that carry it."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import whisperkit_b200 as wk
from oracle import best_of_ref as BR
from oracle import decode_ref as D
from tests import best_of_ref as L
from tests import language_ref
from whisperkit_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_rung_rule_beam_only_at_zero_best_of_only_above():
    assert L.rung_decoder(0.0, 5, 5) == ("beam", 5)
    assert L.rung_decoder(0.2, 5, 5) == ("best_of", 5)
    assert L.rung_decoder(0.0, 1, 5) == ("single", 1)          # greedy rung of a beam 1 / best-of 5 call: one of its five rows
    assert L.rung_decoder(0.4, 1, 5) == ("best_of", 5)
    assert L.rung_decoder(0.6, 3, 1) == ("single", 1)          # best_of 1: one sample
    assert L.rung_decoder(0.0, 1, 1) == ("single", 1)
    # bestOf None / 0: the plain rule - beam search whatever the temperature, else one row
    assert L.rung_decoder(0.6, 4, None) == ("beam", 4) and L.rung_decoder(0.6, 4, 0) == ("beam", 4)
    assert L.rung_decoder(0.6, 1, None) == ("single", 1)


def test_ladder_plan_walks_every_rung_only_with_best_of():
    o = D.DecodingOptions(temperature=0.0, temperatureFallbackCount=2)
    assert L.ladder_plan(o, 3, None) == [(0.0, "beam", 3)]     # a beam call without bestOf skips the ladder
    plan = L.ladder_plan(o, 3, 3)
    assert [k for _, k, _ in plan] == ["beam", "best_of", "best_of"]
    assert [t for t, _, _ in plan] == language_ref.rung_temperatures(o)
    assert [k for _, k, _ in L.ladder_plan(o, 1, None)] == ["single"] * 3


def test_ladder_stops_at_the_first_rung_without_fallback():
    o = D.DecodingOptions(temperature=0.0, temperatureFallbackCount=3)
    calls = []

    def rung(i, t, kind, rows):
        calls.append((i, kind, rows))
        fb = D.DecodingFallback(True, "logProbThreshold") if i < 2 else None
        return D.DecodingResult([1], [0.0], 0.0, 1.0, t, fb)
    res, i = L.decode_with_fallback_best_of(rung, o, 2, 4)
    assert i == 2 and calls == [(0, "beam", 2), (1, "best_of", 4), (2, "best_of", 4)]


def test_ranker_score_and_ties():
    P = 3
    a = [0.0, 0.0, 0.0, -1.0, -1.0]            # 2 sampled tokens: -1
    b = [0.0, 0.0, 0.0, -0.5, -1.0, -1.5]      # 3 sampled tokens: -1 (tie with a)
    c = [0.0, 0.0, 0.0, -0.25, -2.0]           # -1.125
    assert BR.best_of_score(a, P) == np.float32(-1.0)
    assert BR.rank_best_of([c, a, b], P) == 1   # ties go to the lower index
    assert BR.rank_best_of([c, b, a], P) == 1
    assert BR.rank_best_of([a, a, a], P) == 0
    # a sample with no sampled token divides by 1, not 0
    assert BR.best_of_score([0.0, 0.0, 0.0], P) == np.float32(0.0)
    assert BR.rank_best_of([a, [0.0, 0.0, 0.0]], P) == 1


def _header_fields(struct):
    src = open(os.path.join(ROOT, "include", "wkb200.h")).read()
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (struct, struct), src, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        m = re.search(r"\(\s*\*\s*(\w+)\s*\)", decl)   # function-pointer declarator
        fields += [m.group(1)] if m else [re.search(r"(\w+)\s*$", v).group(1) for v in decl.split(",")]
    return fields


def test_best_of_is_a_per_call_field_in_the_tail_padding_of_wk_batch_opts():
    f = _lib.wk_batch_opts
    names = [n for n, _ in f._fields_]
    assert names == _header_fields("wk_batch_opts")
    assert names[-2:] == ["encoder_chunk", "best_of"]
    assert f.best_of.offset == f.encoder_chunk.offset + 4
    assert C.sizeof(f) == f.encoder_chunk.offset + 8          # the struct keeps its size: zeroed callers decode as before
    assert f().best_of == 0
    # wk_decode_opts does not change
    assert [n for n, _ in _lib.wk_decode_opts._fields_] == _header_fields("wk_decode_opts")
    assert "best_of" not in _header_fields("wk_decode_opts")


def test_make_batch_opts_carries_one_best_of_per_call():
    from whisperkit_b200.api import make_batch_opts
    bo, _ = make_batch_opts(3, wk.DecodingOptions(), None)
    assert bo.best_of == 0
    bo, _ = make_batch_opts(3, wk.DecodingOptions(bestOf=5, beamSize=5), None)
    assert bo.best_of == 5
    bo, _ = make_batch_opts(2, [wk.DecodingOptions(bestOf=2), wk.DecodingOptions(bestOf=2, temperature=0.4)], None)
    assert bo.best_of == 2
    with pytest.raises(wk.WhisperError) as e:
        make_batch_opts(2, [wk.DecodingOptions(bestOf=2), wk.DecodingOptions(bestOf=3)], None)
    assert e.value.case == "invalidArgument"
    with pytest.raises(wk.WhisperError):
        make_batch_opts(2, [wk.DecodingOptions(bestOf=2), wk.DecodingOptions()], None)


def test_streams_entry_with_best_of_is_declared_and_bound():
    lib = wk.load()
    assert hasattr(lib, "wk_transcribe_streams_ex")
    proto = {n: a for n, _, a in _lib.SYMBOLS}
    assert len(proto["wk_transcribe_streams_ex"]) == len(proto["wk_transcribe_streams"]) + 1
