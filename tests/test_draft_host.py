"""DecodingOptions.draftTokens on the host: one value per call, passed as the draft_tokens argument of the draft entry points (the
batched-call struct keeps its layout, so callers built against it decode as before)."""
import ctypes as C

import pytest

import whisperkit_b200 as wk
from whisperkit_b200 import _lib
from whisperkit_b200.api import draft_tokens_of, make_batch_opts


def test_draft_tokens_default_off_and_one_value_per_call():
    assert wk.DecodingOptions().draftTokens == 0
    assert draft_tokens_of(wk.DecodingOptions()) == 0
    assert draft_tokens_of([wk.DecodingOptions(draftTokens=3)] * 4) == 3
    with pytest.raises(wk.WhisperError) as e:
        draft_tokens_of([wk.DecodingOptions(draftTokens=3), wk.DecodingOptions(draftTokens=2)])
    assert e.value.case == "invalidArgument"
    with pytest.raises(wk.WhisperError):
        make_batch_opts(2, [wk.DecodingOptions(draftTokens=1), wk.DecodingOptions()], None)
    bo, _ = make_batch_opts(2, [wk.DecodingOptions(draftTokens=5)] * 2, None)
    assert bo.n_opts == 2 and bo.best_of == 0


def test_draft_entry_points_take_the_setting_as_an_argument():
    protos = {n: (r, a) for n, r, a in _lib.SYMBOLS}
    _, a = protos["wk_transcribe_windows_draft"]
    assert a[7] is C.POINTER(_lib.wk_batch_opts) and a[8] is C.c_int32 and len(a) == 10
    _, a = protos["wk_decode_text_draft"]
    assert a[2] is C.POINTER(_lib.wk_batch_opts) and a[3] is C.c_int32 and len(a) == 5
    _, a = protos["wk_transcribe_streams_draft"]
    assert a[-3] is C.c_int32 and a[-2] is C.c_int32 and len(a) == 18    # best_of, draft_tokens
    assert "draft_tokens" not in [n for n, _ in _lib.wk_batch_opts._fields_]


def test_draft_decoder_calls_refuse_without_a_gpu():
    lib = _lib.load()
    if lib.wk_device_available():
        pytest.skip("GPU present")
    assert lib.wk_model_create_draft(None, 2) != 0
    n = C.c_int32(7)
    assert lib.wk_model_draft_layers(None, C.byref(n)) != 0
    assert lib.wk_session_draft_stats(None, (C.c_int64 * 3)()) != 0
