"""End-to-end parity of the CUDA hot path against the CPU oracle, through the protocol mirror
(FeatureExtractor -> AudioEncoder -> TextDecoder.predictLogits / decodeText -> WhisperKit.transcribe).

Tolerances (north_star): greedy token IDs bit-exact, log-mel and logits within 1e-3 (relative to the tensor's
scale) - against the oracle run under the same 16-bit storage policy (oracle/model_ref.py).  Because random
weights give near-uniform logits, token equality is asserted on every sequence whose smallest top-1 margin in
the oracle exceeds 20x the measured logit error (the statistic is printed), and unconditionally on the logits
themselves (teacher-forced on the oracle's tokens)."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import whisperkit_b200 as wk  # noqa: E402
from oracle import decode_ref as D  # noqa: E402
from oracle import mel_ref  # noqa: E402
from oracle import model_ref as M  # noqa: E402


def rel_err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-12))


def build(variant, policy, B, seed=5):
    dims = M.VARIANTS[variant]
    w = M.random_weights(dims, seed=seed, policy=policy)
    orc = M.WhisperOracle(dims, w, policy)
    model = wk.Model(variant, max_batch=B, dtype=policy)
    model.load_state_dict(w)
    return dims, orc, model


@pytest.mark.parametrize("variant,policy", [("toy", "bf16"), ("toy128", "f16"), ("toy128", "bf16"), ("toy512", "f16"), ("toy768", "f16")])
def test_encoder_and_logits_parity(variant, policy):
    B = 3
    dims, orc, model = build(variant, policy, B)
    pcm = np.stack([mel_ref.synthetic_pcm(10 + i) for i in range(B)])
    fe, enc, dec = wk.FeatureExtractor(model), wk.AudioEncoder(model), wk.TextDecoder(model, B)
    assert enc.embedSize == dims.d_model and dec.logitsSize == dims.vocab
    assert dec.kvCacheEmbedDim == dims.dec_layers * dims.d_model and dec.kvCacheMaxSequenceLength == 224
    mel_t = fe.logMelSpectrogram(pcm)
    mel_gpu = mel_t.numpy()
    mel_ref_ = np.stack([mel_ref.log_mel(x, dims.n_mels) for x in pcm])
    assert rel_err(mel_gpu, mel_ref_) <= 1e-3
    enc_t = enc.encodeFeatures(mel_t)
    enc_gpu = enc_t.numpy()  # [B, d, 1500], values rounded to the storage type
    assert enc_gpu.shape == (B, dims.d_model, 1500)
    with torch.no_grad():
        # feed the oracle the exact f16 mel the GPU produced so the comparison isolates the encoder
        enc_ref = orc.encode(torch.from_numpy(mel_gpu))
        e = rel_err(enc_gpu, M.round_to(enc_ref, policy).transpose(1, 2).numpy())
        print(f"[{variant}/{policy}] encoder rel err {e:.2e}")
        assert e <= (2e-2 if policy == "bf16" else 3e-3), e
        # decoder: teacher-forced logits, GPU vs oracle, both fed the GPU's encoder output
        enc_for_dec = torch.from_numpy(enc_gpu).transpose(1, 2).contiguous()
        cross = orc.cross_kv(enc_for_dec)
        cache = orc.new_cache(B)
        dec.bindEncoderOutput(enc_t)
        dec.prepareDecoderInputs()
        rng = np.random.default_rng(0)
        worst = 0.0
        for pos in range(6):
            toks = rng.integers(0, dims.vocab, size=B)
            lg_ref = orc.decode_step(torch.from_numpy(toks), pos, cache, cross).numpy()
            lg = dec.predictLogits(toks, [pos] * B)
            worst = max(worst, rel_err(lg, lg_ref))
        print(f"[{variant}/{policy}] logits rel err {worst:.2e}")
        assert worst <= (4e-3 if policy == "bf16" else 1e-3), worst
    dec.close()
    model.close()


def _oracle_decode(orc, enc_gpu, prompt, opts, st, multilingual, b):
    """Pure-CPU oracle: oracle decoder + oracle loop."""
    with torch.no_grad():
        enc_b = torch.from_numpy(enc_gpu[b:b + 1]).transpose(1, 2).contiguous()
        cross = orc.cross_kv(enc_b)
        cache = orc.new_cache(1)

        def predict(tok, idx):
            return orc.decode_step(torch.tensor([tok]), idx, cache, cross)[0].numpy()

        return D.decode_text(predict, prompt, opts, st, multilingual, keep_logits=True)


def _oracle_loop_on_gpu_logits(dec2, B, prompt, opts, st, multilingual, b):
    """Oracle decode loop / filters / sampler consuming the GPU decoder's own logits (predictLogits)."""
    def predict(tok, idx):
        return dec2.predictLogits([tok] * B, [idx] * B)[b]

    return D.decode_text(predict, prompt, opts, st, multilingual, keep_logits=True)


@pytest.mark.parametrize("variant,policy,without_ts", [("toy128", "f16", False), ("toy", "bf16", False), ("toy128", "bf16", True)])
def test_decode_text_token_parity(variant, policy, without_ts):
    B = 4
    dims, orc, model = build(variant, policy, B, seed=11)
    st_o = D.SpecialTokens.toy(dims.vocab)
    st = wk.SpecialTokens.from_any(st_o)
    pcm = np.stack([mel_ref.synthetic_pcm(20 + i) for i in range(B)])
    fe, enc = wk.FeatureExtractor(model), wk.AudioEncoder(model)
    dec, dec2 = wk.TextDecoder(model, B), wk.TextDecoder(model, B)
    enc_t = enc.encodeFeatures(fe.logMelSpectrogram(pcm))
    enc_gpu = enc_t.numpy()
    kw = dict(firstTokenLogProbThreshold=None, sampleLength=40, withoutTimestamps=without_ts, suppressTokens=[1, 2],
              suppressBlank=True)
    o_ref, o_gpu = D.DecodingOptions(**kw), wk.DecodingOptions(**kw)
    multilingual = True
    prompt_ref = D.prefill_prompt(o_ref, st_o, multilingual)
    prompt = dec.prefillDecoderInputs(o_gpu, st)
    assert prompt == prompt_ref
    res = dec.decodeText(enc_t, prompt, o_gpu, st)
    dec2.bindEncoderOutput(enc_t)
    P = len(prompt)
    for b in range(B):
        # (1) bit-exact: device-resident loop == reference loop semantics on identical logits
        ref_g = _oracle_loop_on_gpu_logits(dec2, B, prompt_ref, o_ref, st_o, multilingual, b)
        assert res[b].tokens == ref_g.tokens, (b, res[b].tokens, ref_g.tokens)
        assert res[b].steps == ref_g.steps and res[b].currentTokenCount == len(ref_g.currentTokens)
        np.testing.assert_allclose(res[b].tokenLogProbs, ref_g.tokenLogProbs, atol=2e-4)
        assert abs(res[b].avgLogProb - ref_g.avgLogProb) < 2e-4
        assert abs(res[b].compressionRatio - ref_g.compressionRatio) < 1e-5
        assert (res[b].fallback is None) == (ref_g.fallback is None)
        if ref_g.fallback is not None:
            assert res[b].fallback.fallbackReason == ref_g.fallback.fallbackReason
            assert res[b].fallback.needsFallback == ref_g.fallback.needsFallback
        # (2) against the pure-CPU oracle: identical until the first step whose top-1 margin is inside the
        #     logit error bound (random weights -> near-uniform logits -> near-ties exist)
        ref = _oracle_decode(orc, enc_gpu, prompt_ref, o_ref, st_o, multilingual, b)
        scale = max(float(np.abs(l).max()) for l in ref.stepLogits)
        bound = (4e-3 if policy == "bf16" else 1e-3) * scale
        first = next((i for i, (x, y) in enumerate(zip(res[b].tokens, ref.tokens)) if x != y), None)
        if first is None and len(res[b].tokens) != len(ref.tokens):
            first = min(len(res[b].tokens), len(ref.tokens))
        mm = min(ref.stepMargins)
        print(f"[{variant}/{policy}] seq {b}: oracle steps {ref.steps}, min top-1 margin {mm:.2e}, logit bound {bound:.1e}, "
              f"first divergence at token {first}")
        if first is not None:
            step = max(first - 1, 0)
            assert step >= P - 2, "prompt tokens can only differ at the model-predicted first timestamp"
            assert ref.stepMargins[min(step, len(ref.stepMargins) - 1)] <= 2 * bound, \
                (b, first, ref.stepMargins[step], bound)
    dec.close()
    dec2.close()
    model.close()


def test_first_token_threshold_and_graph_replay():
    """Library defaults (firstTokenLogProbThreshold = -1.5): random weights stop at step 0 exactly like the
    reference's decodeText would (TextDecoder.swift:662-671); then a second decode on the same session."""
    dims, orc, model = build("toy", "bf16", 2, seed=2)
    st = wk.SpecialTokens.from_any(D.SpecialTokens.toy(dims.vocab))
    kit_dec = wk.TextDecoder(model, 2)
    fe, enc = wk.FeatureExtractor(model), wk.AudioEncoder(model)
    pcm = np.stack([mel_ref.synthetic_pcm(1), mel_ref.synthetic_pcm(2)])
    enc_t = enc.encodeFeatures(fe.logMelSpectrogram(pcm))
    prompt = kit_dec.prefillDecoderInputs(wk.DecodingOptions(), st)
    r = kit_dec.decodeText(enc_t, prompt, wk.DecodingOptions(), st)
    assert all(x.steps == 1 and x.isFirstTokenLogProbTooLow and x.fallback.fallbackReason == "firstTokenLogProbThreshold" for x in r)
    o = wk.DecodingOptions(firstTokenLogProbThreshold=None, sampleLength=30)
    r1 = kit_dec.decodeText(None, prompt, o, st)
    r2 = kit_dec.decodeText(None, prompt, o, st)
    assert [x.tokens for x in r1] == [x.tokens for x in r2]  # deterministic (fixed reduction order, no atomics)
    assert all(x.steps == 30 or x.tokens[-1] == st.endToken for x in r1)
    kit_dec.close()
    model.close()


def test_whisperkit_transcribe_batch_and_chunking():
    """WhisperKit.transcribe(audioArrays:) with more windows than max_batch (chunked), host PCM in, tokens out;
    per-window results equal the same windows run alone (independence of the data-parallel units)."""
    kit = wk.WhisperKit(wk.WhisperKitConfig(model="toy", maxBatch=2, seed=4,
                                            specialTokens=wk.SpecialTokens.from_any(D.SpecialTokens.toy(1024))))
    pcm = np.stack([mel_ref.synthetic_pcm(30 + i) for i in range(5)])
    o = wk.DecodingOptions(firstTokenLogProbThreshold=None, sampleLength=20, temperatureFallbackCount=0)
    res = kit.transcribe(pcm, o)
    assert len(res) == 5
    single = kit.transcribe(pcm[3], o)
    assert single[0].tokens == res[3].tokens
    t = kit.model.last_timings()
    assert t["encoding"] > 0 and t["decodingLoop"] > 0
    # error mapping: bad prompt token -> prepareDecoderInputsFailed
    with pytest.raises(wk.WhisperError) as ei:
        kit.textDecoder.decodeText(None, [99999], o, kit.specialTokens)
    assert ei.value.case == "prepareDecoderInputsFailed"


def test_model_load_from_safetensors_checkpoint(tmp_path):
    """wk_model_load: HuggingFace-style directory (config.json + model.safetensors) == the set_tensor path, bit for bit."""
    import json
    from safetensors.torch import save_file
    dims = M.VARIANTS["toy"]
    w = M.random_weights(dims, seed=21, policy="bf16")
    sd = {k: v.contiguous() for k, v in M.to_hf_state_dict(w).items()}
    sd["proj_out.weight"] = sd["proj_out.weight"].clone()
    half = sorted(sd)[: len(sd) // 2]
    save_file({k: sd[k] for k in half}, str(tmp_path / "model-00001-of-00002.safetensors"))
    save_file({k: (sd[k].to(torch.bfloat16) if k.endswith("fc1.weight") else sd[k]) for k in sd if k not in half},
              str(tmp_path / "model-00002-of-00002.safetensors"))
    cfg = dict(num_mel_bins=dims.n_mels, d_model=dims.d_model, encoder_attention_heads=dims.n_heads, encoder_layers=dims.enc_layers,
               decoder_layers=dims.dec_layers, vocab_size=dims.vocab, max_source_positions=1500, max_target_positions=448)
    (tmp_path / "config.json").write_text(json.dumps(cfg))
    # the checkpoint's own word-timestamp heads (openai-whisper's alignment_heads, shipped by HF in generation_config.json)
    (tmp_path / "generation_config.json").write_text(json.dumps({"alignment_heads": [[1, 0], [1, 1]], "max_length": 448}))
    m1 = wk.Model.from_pretrained(str(tmp_path), max_batch=2, dtype="bf16")
    m2 = wk.Model("toy", max_batch=2, dtype="bf16")
    m2.load_state_dict(w)
    assert m1.info.d_model == dims.d_model and m1.info.vocab == dims.vocab
    assert m1.info.has_alignment_heads == 1 and m2.info.has_alignment_heads == 0     # supportsWordTimestamps (TextDecoder.swift:309-311)
    pcm = np.stack([mel_ref.synthetic_pcm(1), mel_ref.synthetic_pcm(2)])
    outs = []
    for m in (m1, m2):
        fe, enc, dec = wk.FeatureExtractor(m), wk.AudioEncoder(m), wk.TextDecoder(m, 2)
        e = enc.encodeFeatures(fe.logMelSpectrogram(pcm))
        dec.bindEncoderOutput(e)
        outs.append((e.numpy(), dec.predictLogits([5, 6], [0, 0])))
        dec.close()
    np.testing.assert_array_equal(outs[0][0], outs[1][0])
    np.testing.assert_array_equal(outs[0][1], outs[1][1])
    with pytest.raises(wk.WhisperError) as ei:
        wk.Model.from_pretrained(str(tmp_path / "missing"))
    assert ei.value.case == "modelsUnavailable"
    m1.close()
    m2.close()


def test_detect_language_matches_oracle():
    """detectLanguage: one step on [SOT], LanguageLogitsFilter, greedy (TextDecoder.swift:420-539)."""
    B = 3
    dims, orc, model = build("toy128", "f16", B, seed=13)
    st_o = D.SpecialTokens.toy(dims.vocab)
    st = wk.SpecialTokens.from_any(st_o)
    langs = list(range(st_o.englishToken, st_o.englishToken + 2)) + [7, 900, 1500]
    pcm = np.stack([mel_ref.synthetic_pcm(50 + i) for i in range(B)])
    fe, enc, dec = wk.FeatureExtractor(model), wk.AudioEncoder(model), wk.TextDecoder(model, B)
    enc_t = enc.encodeFeatures(fe.logMelSpectrogram(pcm))
    tok, lp = dec.detectLanguage(enc_t, st, langs)
    lg = dec.predictLogits([st.startOfTranscriptToken] * B, [0] * B)   # same step, explicit
    for b in range(B):
        row = D.LanguageLogitsFilter(langs, dims.vocab, 0).filterLogits(lg[b].copy(), [st.startOfTranscriptToken])
        r = D.GreedyTokenSampler(0.0, st_o.endToken, D.DecodingOptions()).update([], row, [])
        assert tok[b] == r.tokens[-1] and tok[b] in langs
        assert abs(lp[b] - r.logProbs[-1]) < 1e-4
    dec.close()
    model.close()


def test_temperature_fallback_ladder():
    """decodeWithFallback: random weights give avgLogProb far below logProbThreshold, so every window walks the whole ladder
    0.0, 0.2, ... 1.0 (TranscribeTask.swift:327-405) and ends at temperature 1.0 with reason logProbThreshold."""
    kit = wk.WhisperKit(wk.WhisperKitConfig(model="toy", maxBatch=4, seed=6,
                                            specialTokens=wk.SpecialTokens.from_any(D.SpecialTokens.toy(1024))))
    pcm = np.stack([mel_ref.synthetic_pcm(60 + i) for i in range(3)])
    o = wk.DecodingOptions(firstTokenLogProbThreshold=None, sampleLength=10, compressionRatioThreshold=None)
    res = kit.transcribe(pcm, o)
    assert all(abs(r.temperature - 1.0) < 1e-3 for r in res)
    assert all(r.fallback is not None and r.fallback.fallbackReason == "logProbThreshold" for r in res)
    o0 = wk.DecodingOptions(firstTokenLogProbThreshold=None, sampleLength=10, temperatureFallbackCount=0)
    res0 = kit.transcribe(pcm, o0)
    assert all(r.temperature == 0.0 for r in res0)
    o1 = wk.DecodingOptions(firstTokenLogProbThreshold=None, sampleLength=10, logProbThreshold=None, compressionRatioThreshold=None)
    assert all(r.fallback is None and r.temperature == 0.0 for r in kit.transcribe(pcm, o1))
    # word timestamps across the ladder: the alignment tensor handed back belongs to the decode whose result was kept
    ow = wk.DecodingOptions(firstTokenLogProbThreshold=None, sampleLength=10, compressionRatioThreshold=None, wordTimestamps=True)
    resw = kit.transcribe(pcm, ow)
    assert all(abs(r.temperature - 1.0) < 1e-3 for r in resw)
    for b in range(3):
        a = kit.textDecoder.alignmentWeights(b, 224)
        assert np.all(a[0] == 0) and abs(float(a[1].sum()) - 1.0) < 5e-3 and np.all(a[resw[b].steps + 1:] == 0)


def test_tiny_en_jfk_config0():
    """BASELINE configs[0] shapes: whisper-tiny.en (80 mels, d 384, 6 heads, 4+4 layers, vocab 51864, English-only prompt
    [SOT, <|0.00|>]) on the reference's own jfk.wav clip (11 s, zero-padded to 30 s by padOrTrim), CLI-style options
    (firstTokenLogProbThreshold nil).  Weights are seeded random (no checkpoints offline), so the check is parity with the
    oracle: HF log-mel golden, logits, and the decode loop."""
    import os
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jfk_logmel_hf.npz"))
    pcm = z["pcm16"].astype(np.float32) / 32768.0
    dims, orc, model = build("tiny.en", "f16", 1, seed=31)
    info = model.info
    assert (info.n_mels, info.d_model, info.vocab, info.is_multilingual) == (80, 384, 51864, 0)
    fe, enc, dec, dec2 = wk.FeatureExtractor(model), wk.AudioEncoder(model), wk.TextDecoder(model, 1), wk.TextDecoder(model, 1)
    mel_t = fe.logMelSpectrogram(pcm[None], samples_per_window=[len(pcm)])    # stride 176000 < 480000: padOrTrim in the kernel
    mel_gpu = mel_t.numpy()
    assert np.abs(mel_gpu[0][:, ::8] - z["mel80_sub8"]).max() <= 1e-3          # vs HF / openai-whisper golden
    enc_t = enc.encodeFeatures(mel_t)
    st_o = D.SpecialTokens.english_only()
    st = wk.SpecialTokens.from_any(st_o)
    kw = dict(firstTokenLogProbThreshold=None, sampleLength=24)
    o_ref, o_gpu = D.DecodingOptions(**kw), wk.DecodingOptions(**kw)
    prompt = dec.prefillDecoderInputs(o_gpu, st)
    assert prompt == D.prefill_prompt(o_ref, st_o, False) == [st_o.startOfTranscriptToken, st_o.timeTokenBegin]
    res = dec.decodeText(enc_t, prompt, o_gpu, st)[0]
    dec2.bindEncoderOutput(enc_t)
    ref_g = _oracle_loop_on_gpu_logits(dec2, 1, prompt, o_ref, st_o, False, 0)
    assert res.tokens == ref_g.tokens and res.steps == ref_g.steps == 24
    ref = _oracle_decode(orc, enc_t.numpy(), prompt, o_ref, st_o, False, 0)
    worst = max(rel_err(a, b) for a, b in zip(ref_g.stepLogits[:3], ref.stepLogits[:3]))
    print(f"[tiny.en/f16 jfk] first-steps logits rel err vs CPU oracle {worst:.2e}; tokens equal: {res.tokens == ref.tokens}")
    assert worst <= 1e-3
    for d_ in (dec, dec2):
        d_.close()
    model.close()


def test_ragged_and_silent_windows():
    """Edge cases the reference handles in padOrTrimAudio / the mel front end: all-zero audio, a 1-sample window, a full
    window; plus n_windows > max_batch chunking with per-window lengths."""
    dims, orc, model = build("toy", "bf16", 2, seed=3)
    fe = wk.FeatureExtractor(model)
    pcm = np.zeros((2, 480000), np.float32)
    pcm[1, 0] = 0.5
    got = fe.logMelSpectrogram(pcm, samples_per_window=[0, 1]).numpy()
    ref1 = mel_ref.log_mel(pcm[1], dims.n_mels)
    assert np.abs(got[0] - mel_ref.log_mel(pcm[0], dims.n_mels)).max() <= 1e-3 and np.abs(got[1] - ref1).max() <= 1e-3
    assert np.allclose(got[0], -1.5)   # silence: log10(1e-10) = -10 -> (-10 + 4) / 4
    with pytest.raises(wk.WhisperError) as ei:
        fe.logMelSpectrogram(np.zeros((3, 480000), np.float32))   # more windows than the model's max_batch
    assert ei.value.case == "audioProcessingFailed"
    model.close()


def test_transcribe_streams_seek_loop_matches_oracle_loop():
    """wk_transcribe_streams (batched TranscribeTask.run seek loop, csrc/longform.cu) against the oracle's loop
    (oracle/seek_ref.seek_loop) driven window by window through the same GPU decode: same windows visited, same segments, same
    timings, for streams of different lengths advancing in one batch, with clip timestamps and with the VAD chunker."""
    from oracle import seek_ref as S
    from whisperkit_b200 import longform as L
    st_o = D.SpecialTokens.toy(1024)
    kit = wk.WhisperKit(wk.WhisperKitConfig(model="toy", maxBatch=4, seed=9, specialTokens=wk.SpecialTokens.from_any(st_o)))
    o = wk.DecodingOptions(firstTokenLogProbThreshold=None, logProbThreshold=None, compressionRatioThreshold=None, sampleLength=24,
                           temperatureFallbackCount=0)
    rng = np.random.default_rng(3)
    lens = [480000 * 2 + 12345, 300000, 480000, 7000, 0, 1100000]
    streams = [np.concatenate([mel_ref.synthetic_pcm(200 + 10 * i + k) for k in range(3)])[:n].astype(np.float32) for i, n in enumerate(lens)]

    def oracle_stream(x, cts=(), base=0):
        def decode_window(seek, size):
            w = np.zeros(480000, np.float32)
            w[:size] = x[seek:seek + size]
            return kit.transcribe(w[None], o, samplesPerWindow=[size])[0]
        return S.seek_loop(len(x), decode_window, clipTimestamps=cts, timeToken=st_o.timeTokenBegin, noSpeechThreshold=o.noSpeechThreshold,
                           logProbThreshold=o.logProbThreshold)

    for cts in ((), (1.0, 20.0, 31.5)):
        got, windows = L.transcribe_streams(kit, streams, o, clipTimestamps=cts)
        total = 0
        for i, x in enumerate(streams):
            ref, wins = oracle_stream(x, cts)
            total += len(wins)
            assert [g.tokens for g in got[i]] == [r.tokens for r in ref], (i, cts)
            assert [g.seek for g in got[i]] == [r.seek for r in ref] and [g.id for g in got[i]] == [r.id for r in ref]
            np.testing.assert_array_equal(np.float32([g.start for g in got[i]]), np.float32([r.start for r in ref]))
            np.testing.assert_array_equal(np.float32([g.end for g in got[i]]), np.float32([r.end for r in ref]))
            np.testing.assert_allclose([g.avgLogprob for g in got[i]], [r.avgLogprob for r in ref], atol=1e-5)
        assert windows == total and total >= 6
    # VAD chunking: each chunk is an independent unit whose seeks/timings are shifted by the chunk offset (WhisperKit.swift:896-911)
    x = streams[5].copy()
    x[500000:520000] = 0
    got, windows = L.transcribe_streams(kit, [x], o, chunkingStrategy="vad")
    chunks = S.vad_chunk_all(x, 480000)
    assert len(chunks) >= 2
    ref_all = []
    for (a, b) in chunks:
        ref, _ = oracle_stream(x[a:b])
        for r in ref:
            r.seek += a
            r.start = float(np.float32(r.start) + np.float32(a) / np.float32(16000))
            r.end = float(np.float32(r.end) + np.float32(a) / np.float32(16000))
        ref_all += ref
    assert [g.tokens for g in got[0]] == [r.tokens for r in ref_all]
    assert [g.seek for g in got[0]] == [r.seek for r in ref_all]
    np.testing.assert_allclose([g.start for g in got[0]], [r.start for r in ref_all], atol=1e-4)
    np.testing.assert_allclose([g.end for g in got[0]], [r.end for r in ref_all], atol=1e-4)


def test_vad_strategy_on_short_audio_keeps_clip_timestamps():
    """chunkingStrategy .vad only applies to audio longer than one window (isChunkable, WhisperKit.swift:876-878): shorter audio goes through
    runTranscribeTask with the caller's options, clipTimestamps included."""
    from whisperkit_b200 import longform as L
    st_o = D.SpecialTokens.toy(1024)
    kit = wk.WhisperKit(wk.WhisperKitConfig(model="toy", maxBatch=2, seed=9, specialTokens=wk.SpecialTokens.from_any(st_o)))
    o = wk.DecodingOptions(firstTokenLogProbThreshold=None, logProbThreshold=None, compressionRatioThreshold=None, sampleLength=16,
                           temperatureFallbackCount=0)
    x = mel_ref.synthetic_pcm(321)[:400000].astype(np.float32)          # 25 s: not chunkable
    clips = (2.0, 9.0, 12.5)
    plain, w_plain = L.transcribe_streams(kit, [x], o, clipTimestamps=clips)
    vad, w_vad = L.transcribe_streams(kit, [x], o, clipTimestamps=clips, chunkingStrategy="vad")
    whole, _ = L.transcribe_streams(kit, [x], o, chunkingStrategy="vad")
    assert [(g.seek, g.tokens) for g in vad[0]] == [(g.seek, g.tokens) for g in plain[0]] and w_vad == w_plain == 2
    assert all(g.seek >= 32000 for g in vad[0]) and any(g.seek < 32000 for g in whole[0])   # the clips were honoured (and do change the result)


def _toy_split(tokens, special_begin):
    """Stand-in for the host tokenizer's splitToWordTokens on the toy vocabulary (same rule as tests/test_word_timestamps_host.py)."""
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


@pytest.mark.parametrize("policy", ["f16", "bf16"])
def test_alignment_heads_weights_parity(policy):
    """wordTimestamps: the decode loop's alignmentWeights tensor (mean cross-attention softmax row of the alignment heads, Float16, row
    tokenIndex + 1; TextDecoder.swift:272-296,709-717) against the oracle decoder teacher-forced on the GPU's tokens."""
    B = 3
    dims, orc, model = build("toy128", policy, B, seed=21)
    st_o = D.SpecialTokens.toy(dims.vocab)
    st = wk.SpecialTokens.from_any(st_o)
    pcm = np.stack([mel_ref.synthetic_pcm(300 + i) for i in range(B)])
    fe, enc, dec = wk.FeatureExtractor(model), wk.AudioEncoder(model), wk.TextDecoder(model, B)
    enc_t = enc.encodeFeatures(fe.logMelSpectrogram(pcm))
    enc_gpu = enc_t.numpy()
    for heads in ([], [(0, 1), (1, 0), (1, 3)]):
        model.setAlignmentHeads(heads)
        ref_heads = heads or [(l, h) for l in range(dims.dec_layers // 2, dims.dec_layers) for h in range(dims.n_heads)]
        o = wk.DecodingOptions(firstTokenLogProbThreshold=None, sampleLength=12, wordTimestamps=True)
        prompt = dec.prefillDecoderInputs(o, st)
        res = dec.decodeText(enc_t, prompt, o, st)
        with torch.no_grad():
            for b in range(B):
                toks = res[b].tokens
                steps = res[b].steps
                a = dec.alignmentWeights(b, 224)
                assert np.all(a[0] == 0) and np.all(a[steps + 1:] == 0)       # row 0 and unreached rows stay zero
                written = steps if a[steps].any() else steps - 1                # the completing step writes no row (TextDecoder.swift:668-674)
                cross = orc.cross_kv(torch.from_numpy(enc_gpu[b:b + 1]).transpose(1, 2).contiguous())
                cache = orc.new_cache(1)
                worst = 0.0
                assert written >= 3
                for i in range(written):
                    _, al = orc.decode_step(torch.tensor([toks[i]]), i, cache, cross, align_heads=ref_heads)
                    worst = max(worst, rel_err(a[i + 1], al[0].numpy()))
                    assert abs(float(a[i + 1].sum()) - 1.0) < 5e-3               # a mean of softmax rows
                print(f"[{policy}] alignment rows rel err {worst:.2e}")
                assert worst <= (2e-2 if policy == "bf16" else 4e-3), worst
    o0 = wk.DecodingOptions(firstTokenLogProbThreshold=None, sampleLength=12)
    dec.decodeText(enc_t, prompt, o0, st)
    with pytest.raises(wk.WhisperError):
        dec.alignmentWeights(0, 4)                                              # last decode did not ask for word timestamps
    dec.close()
    model.close()


def test_transcribe_streams_word_timestamps_match_oracle_loop():
    """wk_transcribe_streams with wordTimestamps (device alignment export -> DTW -> word timings -> segment/seek update) against the
    oracle's seek loop + oracle word timing (oracle/words_ref.py) fed the same GPU decode results and alignment tensors."""
    from oracle import seek_ref as S
    from whisperkit_b200 import longform as L
    st_o = D.SpecialTokens.toy(1024)
    kit = wk.WhisperKit(wk.WhisperKitConfig(model="toy", maxBatch=4, seed=9, specialTokens=wk.SpecialTokens.from_any(st_o)))
    o = wk.DecodingOptions(firstTokenLogProbThreshold=None, logProbThreshold=None, compressionRatioThreshold=None, sampleLength=24,
                           temperatureFallbackCount=0, wordTimestamps=True)
    SB = st_o.specialTokenBegin
    split = lambda t: _toy_split(t, SB)                                          # noqa: E731
    dec_fn = lambda t: "".join(chr(97 + v % 26) for v in t)                       # noqa: E731
    lens = [480000 + 200000, 250000, 900000]
    streams = [np.concatenate([mel_ref.synthetic_pcm(400 + 10 * i + k) for k in range(2)])[:n].astype(np.float32) for i, n in enumerate(lens)]
    got, windows = L.transcribe_streams(kit, streams, o, split_to_word_tokens=split, decode=dec_fn)
    n_words = 0
    for i, x in enumerate(streams):
        def decode_window(seek, size):
            w = np.zeros(480000, np.float32)
            w[:size] = x[seek:seek + size]
            r = kit.transcribe(w[None], o, samplesPerWindow=[size])[0]
            r.alignment = kit.textDecoder.alignmentWeights(0, min(len(r.tokens), 224))
            return r
        ref, wins = S.seek_loop(len(x), decode_window, timeToken=st_o.timeTokenBegin, noSpeechThreshold=o.noSpeechThreshold,
                                logProbThreshold=o.logProbThreshold,
                                wordTimestamps=dict(alignment=lambda r: r.alignment, split=split, decode=dec_fn, specialTokenBegin=SB))
        assert [g.tokens for g in got[i]] == [r.tokens for r in ref], i
        assert [g.seek for g in got[i]] == [r.seek for r in ref]
        np.testing.assert_array_equal(np.float32([g.start for g in got[i]]), np.float32([r.start for r in ref]))
        np.testing.assert_array_equal(np.float32([g.end for g in got[i]]), np.float32([r.end for r in ref]))
        for g, r in zip(got[i], ref):
            assert [w.word for w in g.words] == [w.word for w in r.words]
            assert [w.tokens for w in g.words] == [w.tokens for w in r.words]
            np.testing.assert_array_equal(np.float32([w.start for w in g.words]), np.float32([w.start for w in r.words]))
            np.testing.assert_array_equal(np.float32([w.end for w in g.words]), np.float32([w.end for w in r.words]))
            np.testing.assert_allclose([w.probability for w in g.words], [w.probability for w in r.words], atol=1e-6)
            n_words += len(g.words)
    assert n_words > 10
    # VAD chunking + word timestamps + maxWindowSeek: every chunk is an independent unit; segment AND word times carry the chunk offset
    x = streams[2].copy()
    x[430000:452000] = 0
    chunks = S.vad_chunk_all(x, 480000)
    assert len(chunks) >= 2
    got, _ = L.transcribe_streams(kit, [x], o, chunkingStrategy="vad", split_to_word_tokens=split, decode=dec_fn, maxWindowSeek=400000)
    ref_all = []
    for (a, b) in chunks:
        xc = x[a:b]

        def decode_chunk(seek, size, xc=xc):
            w = np.zeros(480000, np.float32)
            w[:size] = xc[seek:seek + size]
            r = kit.transcribe(w[None], o, samplesPerWindow=[size])[0]
            r.alignment = kit.textDecoder.alignmentWeights(0, min(len(r.tokens), 224))
            return r
        ref, _ = S.seek_loop(len(xc), decode_chunk, timeToken=st_o.timeTokenBegin, noSpeechThreshold=o.noSpeechThreshold,
                             logProbThreshold=o.logProbThreshold, maxWindowSeek=400000,
                             wordTimestamps=dict(alignment=lambda r: r.alignment, split=split, decode=dec_fn, specialTokenBegin=SB))
        off = np.float32(a) / np.float32(16000)
        for r in ref:
            r.seek += a
            r.start, r.end = float(np.float32(r.start) + off), float(np.float32(r.end) + off)
            for w in r.words:
                w.start, w.end = float(np.float32(w.start) + off), float(np.float32(w.end) + off)
        ref_all += ref
    assert [g.tokens for g in got[0]] == [r.tokens for r in ref_all] and [g.seek for g in got[0]] == [r.seek for r in ref_all]
    np.testing.assert_allclose([g.start for g in got[0]], [r.start for r in ref_all], atol=1e-4)
    assert sum(len(g.words) for g in got[0]) > 5
    for g, r in zip(got[0], ref_all):
        assert [w.word for w in g.words] == [w.word for w in r.words]
        np.testing.assert_allclose([w.start for w in g.words], [w.start for w in r.words], atol=1e-4)
        np.testing.assert_allclose([w.end for w in g.words], [w.end for w in r.words], atol=1e-4)


def _toy_tokenizer(vocab=1024):
    """A byte-level vocabulary for the toy model: ids 0..255 are the GPT-2 byte alphabet, 256..sb-1 two-byte merges, then the Whisper
    special tokens at the ids of D.SpecialTokens.toy(vocab) and <|t|> timestamps after them."""
    from whisperkit_b200.tokenizer import WhisperTokenizer
    bs = list(range(33, 127)) + list(range(161, 173)) + list(range(174, 256))
    cs = bs[:]
    n = 0
    for b in range(256):
        if b not in bs:
            bs.append(b); cs.append(256 + n); n += 1
    alphabet = {b: chr(c) for b, c in zip(bs, cs)}
    sb = vocab // 2
    toks, ids, flags = [], [], []
    for b in range(256):
        toks.append(alphabet[b]); ids.append(b); flags.append(0)
    letters = " etaoinshrdlu"
    for i in range(256, sb):
        a, c = letters[(i * 7) % len(letters)], letters[(i * 3 + 1) % len(letters)]
        toks.append(alphabet[ord(a)] + alphabet[ord(c)]); ids.append(i); flags.append(0)
    names = {sb: "<|endoftext|>", sb + 1: "<|startoftranscript|>", sb + 2: "<|en|>", sb + 3: "<|translate|>", sb + 4: "<|transcribe|>",
             sb + 5: "<|xx|>", sb + 6: "<|startofprev|>", sb + 7: "<|nospeech|>", sb + 8: "<|notimestamps|>"}
    for i in range(sb, vocab):
        toks.append(names.get(i, f"<|{(i - sb - 9) * 0.02:.2f}|>")); ids.append(i); flags.append(3)
    return WhisperTokenizer(tokens=toks, ids=ids, flags=flags)


def test_transcribe_audio_text_and_words_with_library_tokenizer():
    """longform.transcribe_audio: the whole long-form path with the library's own tokenizer (no host callbacks) - segments and word timings
    equal the callable-hook route (which is checked against the oracle above), texts are the tokenizer's decode of the segment tokens."""
    from whisperkit_b200 import longform as L
    tok = _toy_tokenizer(1024)
    st_o = D.SpecialTokens.toy(1024)
    st = tok.specialTokens
    assert (st.endToken, st.startOfTranscriptToken, st.timeTokenBegin, st.transcribeToken, st.noTimestampsToken) == \
        (st_o.endToken, st_o.startOfTranscriptToken, st_o.timeTokenBegin, st_o.transcribeToken, st_o.noTimestampsToken)
    kit = wk.WhisperKit(wk.WhisperKitConfig(model="toy", maxBatch=4, seed=9, specialTokens=st))
    o = wk.DecodingOptions(firstTokenLogProbThreshold=None, logProbThreshold=None, compressionRatioThreshold=None, sampleLength=24,
                           temperatureFallbackCount=0, wordTimestamps=True)
    streams = [np.concatenate([mel_ref.synthetic_pcm(500 + 10 * i + k) for k in range(2)])[:n].astype(np.float32)
               for i, n in enumerate([700000, 200000])]
    res = L.transcribe_audio(kit, streams, o, tokenizer=tok)
    ref, _ = L.transcribe_streams(kit, streams, o, split_to_word_tokens=tok.splitToWordTokens, decode=tok.decode)
    sb = st.specialTokenBegin
    n_words = 0
    for r, segs in zip(res, ref):
        assert [g.tokens for g in r.segments] == [g.tokens for g in segs]
        assert [(g.start, g.end) for g in r.segments] == [(g.start, g.end) for g in segs]
        for g, h in zip(r.segments, segs):
            assert [(w.word, w.tokens, w.start, w.end) for w in g.words] == [(w.word, w.tokens, w.start, w.end) for w in h.words]
            assert g.text == tok.decode(g.tokens) and g.text.startswith("<|")
            n_words += len(g.words)
        assert r.text == tok.decode([t for g in r.segments for t in g.tokens if t < sb]).strip()
    assert n_words >= 2          # the toy vocabulary glues most sub-words into few words
    o2 = wk.DecodingOptions(firstTokenLogProbThreshold=None, logProbThreshold=None, compressionRatioThreshold=None, sampleLength=24,
                            temperatureFallbackCount=0, skipSpecialTokens=True)
    r2 = L.transcribe_audio(kit, streams[:1], o2, tokenizer=tok)[0]
    assert all("<|" not in g.text for g in r2.segments) and all(g.words is None for g in r2.segments)
