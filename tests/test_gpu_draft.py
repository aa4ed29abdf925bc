"""Speculative greedy decoding (DecodingOptions.draftTokens) on the GPU.  The draft decoder only decides how many decoder steps run, so a
call with a draft must return byte-identical results to the same call without one on a session with as many decode slots - whatever
the draft proposes - for every window decoded at temperature 0, and for every window when the call has no more windows than slots (a
temperature > 0 draw uses its slot's Philox subsequence, and with more windows than slots the slot a window lands in follows when earlier
windows retire, which the draft changes).  A draft that equals the model's decoder (a "collapsed" main whose upper layers add exact
zeros, or the same weights loaded from a checkpoint) must have every proposal accepted; an unrelated draft few."""
import ctypes as C
import dataclasses
import json
import os
import struct

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import whisperkit_b200 as wk  # noqa: E402
from whisperkit_b200 import _lib  # noqa: E402
from whisperkit_b200.api import _DT  # noqa: E402
from oracle import decode_ref as D  # noqa: E402
from oracle import mel_ref  # noqa: E402

FORCE = dict(logProbThreshold=0.0, compressionRatioThreshold=None)   # every window walks the ladder (avgLogProb < 0)
NEVER = dict(logProbThreshold=None, compressionRatioThreshold=None)
DIMS = {"toy": (128, 2, 1024), "toy128": (256, 4, 2048)}             # d_model, heads, vocabulary


def st_of(variant):
    return D.SpecialTokens.toy(DIMS[variant][2])


def opts(**kw):
    d = dict(firstTokenLogProbThreshold=None, sampleLength=40, temperatureFallbackCount=0, **NEVER)
    d.update(kw)
    return wk.DecodingOptions(**d)


def same(a, b, where):
    assert a.tokens == b.tokens, where
    assert np.array_equal(np.asarray(a.tokenLogProbs, np.float32).view(np.uint32), np.asarray(b.tokenLogProbs, np.float32).view(np.uint32)), where
    assert np.float32(a.avgLogProb).tobytes() == np.float32(b.avgLogProb).tobytes(), where
    assert np.float32(a.compressionRatio).tobytes() == np.float32(b.compressionRatio).tobytes(), where
    assert (a.temperature, a.fallback, a.steps, a.currentTokenCount) == (b.temperature, b.fallback, b.steps, b.currentTokenCount), where
    assert (a.languageToken, a.languageLogProb) == (b.languageToken, b.languageLogProb), where
    assert np.float32(a.noSpeechProb).tobytes() == np.float32(b.noSpeechProb).tobytes(), where


def decoder_tensors(variant, layers, seed, std=0.02):
    """HF-named decoder tensors (numpy f32) of a random Whisper decoder with the variant's dimensions."""
    d, _, V = DIMS[variant]
    g = np.random.default_rng(seed)
    r = lambda *shape: (g.standard_normal(shape) * std).astype(np.float32)   # noqa: E731
    ln = lambda: (1.0 + r(d), r(d))                                          # noqa: E731
    w = {"model.decoder.embed_tokens.weight": r(V, d), "model.decoder.embed_positions.weight": r(448, d)}
    w["model.decoder.layer_norm.weight"], w["model.decoder.layer_norm.bias"] = ln()
    for i in range(layers):
        p = f"model.decoder.layers.{i}."
        for a in ("self_attn", "encoder_attn"):
            for x in ("q", "k", "v", "out"):
                w[f"{p}{a}.{x}_proj.weight"] = r(d, d)
            for x in ("q", "v", "out"):
                w[f"{p}{a}.{x}_proj.bias"] = r(d)
        for n in ("self_attn_layer_norm", "encoder_attn_layer_norm", "final_layer_norm"):
            w[f"{p}{n}.weight"], w[f"{p}{n}.bias"] = ln()
        w[f"{p}fc1.weight"], w[f"{p}fc1.bias"] = r(4 * d, d), r(4 * d)
        w[f"{p}fc2.weight"], w[f"{p}fc2.bias"] = r(d, 4 * d), r(d)
    return w


def write_checkpoint(path, variant, tensors, layers):
    """A HF checkpoint directory: config.json and one safetensors file (F32)."""
    d, heads, V = DIMS[variant]
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump({"d_model": d, "decoder_attention_heads": heads, "encoder_attention_heads": heads, "vocab_size": V,
                   "max_source_positions": 1500, "max_target_positions": 448, "decoder_layers": layers, "encoder_layers": 2}, f)
    header, blobs, off = {}, [], 0
    for k, v in tensors.items():
        b = np.ascontiguousarray(v, np.float32).tobytes()
        header[k] = {"dtype": "F32", "shape": list(v.shape), "data_offsets": [off, off + len(b)]}
        blobs.append(b)
        off += len(b)
    h = json.dumps(header).encode()
    h += b" " * (-len(h) % 8)
    with open(os.path.join(path, "model.safetensors"), "wb") as f:
        f.write(struct.pack("<Q", len(h)) + h + b"".join(blobs))
    return path


def make_kit(variant, policy, slots, draft_dir=None, **kw):
    return wk.WhisperKit(wk.WhisperKitConfig(model=variant, maxBatch=slots, seed=5, dtype=policy, draftModelFolder=draft_dir,
                                             specialTokens=wk.SpecialTokens.from_any(st_of(variant)), **kw))


def pcm_of(n, base):
    return np.stack([mel_ref.synthetic_pcm(base + i) for i in range(n)])


def option_mix(variant, n, k):
    """One option set per window: prompts and prefixes, timestamps on and off, suppression, detection and no-speech, hot rungs."""
    st = st_of(variant)
    langs = [st.englishToken] + list(range(200, 260))
    kinds = [dict(), dict(withoutTimestamps=True), dict(promptTokens=[5, 9, 33, 17]), dict(prefixTokens=[40, 41]),
             dict(suppressTokens=[3, 4, 5, 6, 7], suppressBlank=True), dict(computeNoSpeechProb=True, detectLanguage=True, allLanguageTokens=langs),
             dict(temperatureFallbackCount=2, seed=7, **FORCE), dict(sampleLength=13)]
    return [opts(draftTokens=k, **kinds[i % len(kinds)]) for i in range(n)]


def plain(o):
    return [dataclasses.replace(x, draftTokens=0) for x in o]


def same_where_promised(got, exp, n_windows, slots, where):
    """Every window when the call fits its slots; else the windows decoded at temperature 0 only (no fallback in either call)."""
    greedy = 0
    for i in range(n_windows):
        if n_windows <= slots or (got[i].temperature == 0.0 and exp[i].temperature == 0.0):
            same(got[i], exp[i], (where, i))
            greedy += 1
    assert greedy >= n_windows // 2, where


ALL_POLICIES = [("toy", "bf16"), ("toy", "f16"), ("toy128", "bf16"), ("toy128", "f16")]


@pytest.fixture(scope="module")
def draft_dir(tmp_path_factory):
    """An unrelated 2-layer draft per variant, written with encoder tensors beside its decoder (they must be ignored)."""
    out = {}
    for v in DIMS:
        t = decoder_tensors(v, 2, seed=91)
        t["model.encoder.layer_norm.weight"] = np.ones(DIMS[v][0], np.float32)
        out[v] = write_checkpoint(str(tmp_path_factory.mktemp(f"draft_{v}")), v, t, 2)
    return out


@pytest.mark.parametrize("variant,policy", ALL_POLICIES)
@pytest.mark.parametrize("k", [1, 3, 7])
def test_draft_results_are_byte_identical(variant, policy, k, draft_dir):
    slots = 3
    kit = make_kit(variant, policy, slots * (k + 1), draft_dir[variant])
    ref = make_kit(variant, policy, slots)
    n = 8                                                   # more windows than slots: admissions into freed slots
    pcm = pcm_of(n, 1200)
    spw = [480000, 200000, 480000, 90000, 300000, 480000, 480000, 150000]
    o = option_mix(variant, n, k)
    got = kit.transcribe(pcm, o, samplesPerWindow=spw)
    exp = ref.transcribe(pcm, plain(o), samplesPerWindow=spw)
    same_where_promised(got, exp, n, slots, (variant, policy, k))
    ds = kit.textDecoder.draftStats()
    print(f"[{variant}/{policy} k={k}] {ds}, steps {kit.textDecoder.stats()['steps']} vs {ref.textDecoder.stats()['steps']}")
    assert ds["rounds"] > 0 and 0 <= ds["accepted"] <= ds["proposed"]


@pytest.mark.parametrize("policy", [dict(crossKVDtype="fp8"), dict(encoderDtype="fp8")])
def test_draft_under_fp8_policies(policy, draft_dir):
    k, slots = 3, 8
    kit = make_kit("toy", "bf16", slots * (k + 1), draft_dir["toy"], **policy)
    ref = make_kit("toy", "bf16", slots, **policy)
    pcm = pcm_of(slots, 1300)
    o = option_mix("toy", slots, k)
    got, exp = kit.transcribe(pcm, o), ref.transcribe(pcm, plain(o))
    same_where_promised(got, exp, slots, slots, policy)


@pytest.mark.parametrize("variant,policy", ALL_POLICIES)
@pytest.mark.parametrize("k", [1, 3, 7])
def test_exact_checkpoint_draft_with_the_option_mix(variant, policy, k, tmp_path):
    """A draft loaded from a checkpoint (encoder tensors beside it, ignored) whose decoder is the model's own: every proposal is
    accepted - EOT inside accepted runs, prompts, prefixes, timestamp rules, suppression, detection, hot rungs and slot reuse included -
    and the results are those of the draft-less call.  A tensor the loader put in the wrong place would show as rejected proposals."""
    w = decoder_tensors(variant, 2, seed=23, std=0.05)
    folder = write_checkpoint(str(tmp_path / "exact"), variant, {**w, "model.encoder.layer_norm.bias": np.zeros(DIMS[variant][0], np.float32)}, 2)
    for slots, n in ((8, 8), (3, 9)):                       # all windows in flight; more windows than slots
        kit = make_kit(variant, policy, slots * (k + 1), folder)
        ref = make_kit(variant, policy, slots)
        for name, t in w.items():                           # the model's decoder := the draft's
            kit.model.set_tensor(name, t)
            ref.model.set_tensor(name, t)
        pcm = pcm_of(n, 1800)
        spw = [480000, 200000, 480000, 90000, 300000, 480000, 480000, 150000, 410000][:n]
        o = option_mix(variant, n, k)
        got = kit.transcribe(pcm, o, samplesPerWindow=spw)
        exp = ref.transcribe(pcm, plain(o), samplesPerWindow=spw)
        same_where_promised(got, exp, n, slots, (variant, policy, k, slots))
        ds = kit.textDecoder.draftStats()
        print(f"[{variant}/{policy} k={k} {n} windows / {slots} slots] exact checkpoint draft: {ds}")
        assert ds["rounds"] > 0 and ds["accepted"] == ds["proposed"] > 0
        for x in (kit, ref):
            x.textDecoder.close()
            x.model.close()


@pytest.mark.parametrize("variant,policy", ALL_POLICIES)
def test_appending_first_lets_a_block_attend_like_sequential_steps(variant, policy):
    """G rows at positions p0 .. p0 + G - 1 of one window in one step (wk_test_kv_append, then the ancestry self-attention) equal G
    sequential single-row steps bit for bit: outputs and cache rows."""
    d, _, _ = DIMS[variant]
    H, dm, G, p0, splits, Bp = d // 64, d, 8, 37, 3, 16
    tdt = torch.bfloat16 if policy == "bf16" else torch.float16
    wdt = _DT[policy]
    model = wk.Model(variant, max_batch=2, dtype=policy)
    lib, p = model.lib, lambda t: C.c_void_p(0 if t is None else t.data_ptr())   # noqa: E731
    g = torch.Generator(device="cuda").manual_seed(d + G)
    part = torch.randn(splits, Bp, 3 * dm, device="cuda", generator=g) * 0.5
    bq, bv = torch.randn(dm, device="cuda", generator=g) * 0.3, torch.randn(dm, device="cuda", generator=g) * 0.3
    prefix_k = torch.randn(H, p0, 64, device="cuda", generator=g).to(tdt)
    prefix_v = torch.randn(H, p0, 64, device="cuda", generator=g).to(tdt)
    # the block: G rows, row 0 holds the prefix, row j reads position p0 + i from row i
    kc = torch.zeros(G, H, 224, 64, device="cuda", dtype=tdt)
    vc = torch.zeros_like(kc)
    kc[0, :, :p0], vc[0, :, :p0] = prefix_k, prefix_v
    anc = torch.zeros(G, 224, dtype=torch.int32, device="cuda")
    for j in range(G):
        anc[j, p0:p0 + G] = torch.arange(G, dtype=torch.int32)
    pos = torch.arange(p0, p0 + G, dtype=torch.int32, device="cuda")
    out = torch.zeros(G, dm, device="cuda", dtype=tdt)
    _lib.check(lib.wk_test_kv_append(model.handle, p(part), splits, Bp, p(bv), p(kc), p(vc), p(pos), None, G, H, wdt))
    _lib.check(lib.wk_test_self_attention_splitk(model.handle, p(part), splits, Bp, p(bq), p(bv), p(kc), p(vc), p(pos), None, p(anc),
                                                 p(out), G, H, wdt))
    # sequential: one row, one position per step
    k1 = torch.zeros(1, H, 224, 64, device="cuda", dtype=tdt)
    v1 = torch.zeros_like(k1)
    k1[0, :, :p0], v1[0, :, :p0] = prefix_k, prefix_v
    for j in range(G):
        pj = torch.zeros(splits, Bp, 3 * dm, device="cuda")
        pj[:, 0] = part[:, j]
        o1 = torch.zeros(1, dm, device="cuda", dtype=tdt)
        pos1 = torch.tensor([p0 + j], dtype=torch.int32, device="cuda")
        _lib.check(lib.wk_test_self_attention_splitk(model.handle, p(pj), splits, Bp, p(bq), p(bv), p(k1), p(v1), p(pos1), None, None,
                                                     p(o1), 1, H, wdt))
        torch.cuda.synchronize()
        assert torch.equal(out[j].view(torch.int16), o1[0].view(torch.int16)), j
        assert torch.equal(kc[j, :, p0 + j].view(torch.int16), k1[0, :, p0 + j].view(torch.int16)), j
        assert torch.equal(vc[j, :, p0 + j].view(torch.int16), v1[0, :, p0 + j].view(torch.int16)), j
    model.close()


def test_draft_at_64_slots_of_256_rows(draft_dir):
    """The decoder GEMMs at 256 rows compute each row's columns as at 64: the split count depends on N, K and the SM count only."""
    kit = make_kit("toy", "bf16", 256, draft_dir["toy"])
    ref = make_kit("toy", "bf16", 64)
    pcm = pcm_of(70, 1400)
    o = opts(draftTokens=3, sampleLength=30)
    got, exp = kit.transcribe(pcm, o), ref.transcribe(pcm, plain([o])[0])
    for i in range(70):
        same(got[i], exp[i], i)


def collapsed_main(variant, policy, slots_rows, draft_seed=None):
    """A 4-layer model whose layers 2 and 3 add exact zeros (zero out-projections, FC2 and their biases) and a draft: its first two
    layers (draft_seed None, the model itself in exact arithmetic) or an unrelated one."""
    d, _, V = DIMS[variant]
    model = wk.Model(variant, max_batch=max(slots_rows), dtype=policy, config={"dec_layers": 4})
    model.init_random(3)
    w = decoder_tensors(variant, 4, seed=17, std=0.05)
    for i in (2, 3):
        for n in ("self_attn.out_proj", "encoder_attn.out_proj", "fc2"):
            w[f"model.decoder.layers.{i}.{n}.weight"][:] = 0
            w[f"model.decoder.layers.{i}.{n}.bias"][:] = 0
    for name, t in w.items():
        model.set_tensor(name, t)
    draft = {n: t for n, t in w.items() if not n.startswith(("model.decoder.layers.2.", "model.decoder.layers.3."))} if draft_seed is None \
        else decoder_tensors(variant, 2, seed=draft_seed)
    model.setDraftDecoder(2, weights=draft)
    return model


@pytest.mark.parametrize("variant,policy", ALL_POLICIES)
@pytest.mark.parametrize("k", [1, 3, 7])
def test_exact_draft_accepts_every_proposal(variant, policy, k):
    slots = 4
    st = wk.SpecialTokens.from_any(st_of(variant))
    results = {}
    for name, seed in (("exact", None), ("unrelated", 44)):
        model = collapsed_main(variant, policy, [slots, slots * (k + 1)], seed)
        fe, enc = wk.FeatureExtractor(model), wk.AudioEncoder(model)
        dec_d, dec_p = wk.TextDecoder(model, slots * (k + 1)), wk.TextDecoder(model, slots)
        e = enc.encodeFeatures(fe.logMelSpectrogram(pcm_of(slots, 1500)))
        o = opts(draftTokens=k, sampleLength=120, suppressTokens=[st.endToken])   # no EOT: long sequences, many full rounds
        prompt = dec_p.prefillDecoderInputs(o, st)
        got = dec_d.decodeText(e, prompt, o, st)
        exp = dec_p.decodeText(e, prompt, dataclasses.replace(o, draftTokens=0), st)
        for i in range(slots):
            same(got[i], exp[i], (name, i))
        results[name] = dec_d.draftStats()
        print(f"[{variant}/{policy} k={k}] {name} draft: {results[name]}")
    ex, un = results["exact"], results["unrelated"]
    assert ex["rounds"] > 0 and ex["accepted"] == ex["proposed"] > 0
    assert un["accepted"] < un["proposed"] and un["accepted"] / un["proposed"] < ex["accepted"] / ex["proposed"]


def test_long_form_with_a_draft(draft_dir):
    from whisperkit_b200 import longform as LF
    k = 2
    kit = make_kit("toy", "bf16", 3 * (k + 1), draft_dir["toy"])
    ref = make_kit("toy", "bf16", 3)
    streams = [np.concatenate([mel_ref.synthetic_pcm(1600 + 10 * i + j) for j in range(2)])[:n].astype(np.float32)
               for i, n in enumerate([480000 + 170000, 310000])]
    for chunking in (None, "vad"):
        o = opts(draftTokens=k, sampleLength=48)
        segs, windows = LF.transcribe_streams(kit, streams, o, chunkingStrategy=chunking)
        segs0, windows0 = LF.transcribe_streams(ref, streams, dataclasses.replace(o, draftTokens=0), chunkingStrategy=chunking)
        assert windows == windows0 >= 2
        for a, b in zip(segs, segs0):
            key = lambda g: (g.seek, g.start, g.end, g.tokens, g.tokenLogProbs, g.temperature, g.avgLogprob, g.compressionRatio)   # noqa: E731
            assert [key(g) for g in a] == [key(g) for g in b], chunking


def live_bytes():
    dev, pinned = C.c_int64(), C.c_int64()
    assert _lib.load().wk_debug_live_bytes(C.byref(dev), C.byref(pinned)) == 0
    return dev.value, pinned.value


def test_loading_refusals_and_buffers(draft_dir, tmp_path):
    import gc
    gc.collect()
    base = live_bytes()
    k, slots = 3, 2
    # the checkpoint (with encoder tensors) loads as the setters set it: the same proposals, so the same counters
    t = decoder_tensors("toy", 2, seed=91)
    pcm = pcm_of(3, 1700)
    o = opts(draftTokens=k)
    kit = make_kit("toy", "bf16", slots * (k + 1), draft_dir["toy"])
    assert kit.model.draftLayers == 2
    got = kit.transcribe(pcm, o)
    stats = kit.textDecoder.draftStats()
    m2 = wk.Model("toy", max_batch=slots * (k + 1), dtype="bf16")
    m2.init_random(5)
    m2.setDraftDecoder(2, weights=t)
    fe, enc, dec = wk.FeatureExtractor(m2), wk.AudioEncoder(m2), wk.TextDecoder(m2, slots * (k + 1))
    st = wk.SpecialTokens.from_any(st_of("toy"))
    e = enc.encodeFeatures(fe.logMelSpectrogram(pcm[:slots]))
    res = dec.decodeText(e, dec.prefillDecoderInputs(o, st), o, st)
    e_kit = kit.audioEncoder.encodeFeatures(kit.featureExtractor.logMelSpectrogram(pcm[:slots]))
    ref = kit.textDecoder.decodeText(e_kit, dec.prefillDecoderInputs(o, st), o, st)
    assert [r.tokens for r in res] == [r.tokens for r in ref]
    assert dec.draftStats() == kit.textDecoder.draftStats()
    assert stats["rounds"] > 0 and len(got) == 3
    # refusals: the draft is fixed once a session exists; mismatched dimensions; bad settings
    with pytest.raises(wk.WhisperError):
        m2.setDraftDecoder(2)
    m3 = wk.Model("toy", max_batch=4, dtype="bf16")
    bad = write_checkpoint(str(tmp_path / "bad"), "toy128", decoder_tensors("toy128", 1, seed=1), 1)
    with pytest.raises(wk.WhisperError) as e3:
        m3.loadDraftDecoder(bad)
    assert e3.value.case == "invalidArgument" and m3.draftLayers == 0
    m3.close()
    nodraft = make_kit("toy", "bf16", 4)
    for kk, kit_, o_ in ((2, nodraft, {}), (0, kit, dict(draftTokens=8)), (0, kit, dict(draftTokens=-1)), (0, kit, dict(draftTokens=3, beamSize=2)),
                         (0, kit, dict(draftTokens=3, bestOf=2)), (0, kit, dict(draftTokens=3, wordTimestamps=True))):
        with pytest.raises(wk.WhisperError) as ei:
            kit_.transcribe(pcm, opts(**({"draftTokens": kk} if kk else {}), **o_))
        assert ei.value.case == "invalidArgument", o_
    with pytest.raises(wk.WhisperError) as ei:
        make_kit("toy", "bf16", 3, draft_dir["toy"]).transcribe(pcm, opts(draftTokens=3))   # G = 4 > 3 rows
    assert ei.value.case == "invalidArgument"
    with pytest.raises(wk.WhisperError):
        kit.transcribe(pcm, [opts(draftTokens=3), opts(draftTokens=2), opts(draftTokens=3)])
    from whisperkit_b200.streaming import AudioStreamTranscriber
    with pytest.raises(wk.WhisperError) as ei:
        AudioStreamTranscriber(kit, opts(draftTokens=3))
    assert ei.value.case == "invalidArgument"
    for x in (dec, kit.textDecoder, nodraft.textDecoder):
        x.close()
    for x in (m2, kit.model, nodraft.model):
        x.close()
    del kit, nodraft, dec, m2, fe, enc, e, e_kit
    gc.collect()
    assert live_bytes() == base
