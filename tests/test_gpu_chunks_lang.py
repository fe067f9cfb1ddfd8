"""Language auto-detection per chunk on the batch path (WSP_TOKEN_LANGUAGE_AUTO in the prompt of wsp_run_chunks*) on an H100: each
chunk is decoded in the language detected from its own encode.

Oracle: tests/golden/chunks_lang.npz (per chunk, the reference's whisper_lang_auto_detect and then its greedy loop with that language
in the prompt, made by tests/golden/make_chunks_lang_golden.py from oracle/_ref): language ids and tokens identical, probabilities
within 2e-4 as for wsp_detect_language.  The larger models are checked against the single-clip path on the GPU: wsp_detect_language
on the chunk alone, and the chunk alone decoded with its language fixed in the prompt.
"""
import ctypes as C
import os

import numpy as np
import pytest

from tests.golden import make_chunks_lang_golden as mk
from whisper_b200 import capi, synth

pytestmark = pytest.mark.gpu

E_INVALIDARG, E_BOUNDS = -1, -7
LANG_TOL = mk.LANG_TOL

_cache = {}


def golden():
    if "g" not in _cache:
        _cache["g"] = np.load(os.path.join(os.path.dirname(__file__), "golden", "chunks_lang.npz"))
    return _cache["g"]


def engine(model):
    if ("engine", model) not in _cache:
        m = capi.Model(synth.model_path(model))
        _cache[("engine", model)] = (m, capi.Engine(m, 0))
    return _cache[("engine", model)]


def context(model, batch):
    m, e = engine(model)
    if (model, batch) not in _cache:
        _cache[(model, batch)] = capi.Context(e, batch)
    return m, _cache[(model, batch)]


class Settings:
    """a case's audio_ctx, speed-up and reference threads on a context, restored to the defaults afterwards"""

    def __init__(self, c, audio_ctx=0, speed_up=False, threads=4):
        self.c, self.a = c, (audio_ctx, speed_up, threads)

    def __enter__(self):
        a, s, t = self.a
        self.c.set_audio_ctx(a); self.c.set_speed_up(s); self.c.set_reference_threads(t)
        return self.c

    def __exit__(self, *exc):
        self.c.set_audio_ctx(0); self.c.set_speed_up(False); self.c.set_reference_threads(4)


def case(name):
    g = golden()
    pcms = [synth.synth_pcm(int(ch), int(n)) for ch, n in zip(g[name + "_chunks"], g[name + "_n_samples"])]
    return pcms, g[name + "_prompt"], dict(audio_ctx=int(g[name + "_audio_ctx"]))


def want(name, th, key="tokens", n_key="n_out"):
    g, p = golden(), "%s_t%d_" % (name, th)
    return [g[p + key][b, :int(g[p + n_key][b])].tolist() for b in range(g[p + key].shape[0])]


def cut_at_eot(row, eot):
    hits = np.flatnonzero(row == eot)
    return row[:hits[0] + 1] if hits.size else row


def launches(f):
    L = capi.lib()
    before = L.wsp_launch_count()
    r = f()
    return r, int(L.wsp_launch_count() - before)


def fixed_prompt(m, lang):
    return np.array(m.prompt_init(int(lang)), np.int32)


PARAMS = [(name, th) for name, spec in mk.CASES.items() for th in spec[0]]


@pytest.mark.parametrize("form", ["host", "resident", "run_chunks"])
@pytest.mark.parametrize("name,th", PARAMS)
def test_reference_parity(name, th, form):
    batch = mk.CASES[name][1]
    m, c = context(mk.MODEL, batch)
    pcms, prompt, kw = case(name)
    assert prompt.tolist() == m.prompt_init("auto")
    with Settings(c, threads=th, **kw):
        if form == "host":
            got, st = c.run_chunks_until_eot(pcms, prompt, mk.CAP)
        elif form == "resident":
            for b, p in enumerate(pcms):
                c.upload_pcm(b, p)
            got, st = c.run_chunks_until_eot(None, prompt, mk.CAP, batch=batch)
        else:
            full, st = c.run_chunks(pcms, prompt, mk.CAP)
            got = [cut_at_eot(r, m.special["eot"]) for r in full]
        ids, probs = c.chunk_languages(batch)
    g, p = golden(), "%s_t%d_" % (name, th)
    assert st[2] > 0
    assert ids.tolist() == g[p + "lang_id"].tolist()
    assert np.abs(probs - g[p + "lang_probs"]).max() < LANG_TOL
    assert [t.tolist() for t in got] == want(name, th)


def single_clip_agreement(model, pcms, prompt, cap, batch_ids, batch_probs, batch_toks, **kw):
    """each chunk alone: wsp_detect_language gives the batch's language (probabilities within LANG_TOL), and the chunk decoded with
    that language fixed in the prompt gives the batch row's tokens"""
    m, one = context(model, 1)
    with Settings(one, **kw):
        for b, pcm in enumerate(pcms):
            one.pcm_to_mel(0, pcm)
            lid, probs = one.detect_language(0, batch_probs.shape[1])
            assert lid == int(batch_ids[b]), "chunk %d" % b
            assert np.abs(probs - batch_probs[b]).max() < LANG_TOL, "chunk %d" % b
            got, _ = one.run_chunks_until_eot([pcm], fixed_prompt(m, lid), cap)
            assert got[0].tolist() == batch_toks[b].tolist(), "chunk %d" % b
            assert one.chunk_languages(1) is None


@pytest.mark.parametrize("name", list(mk.CASES))
def test_agrees_with_single_clip_path(name):
    batch = mk.CASES[name][1]
    _m, c = context(mk.MODEL, batch)
    pcms, prompt, kw = case(name)
    with Settings(c, **kw):
        got, _ = c.run_chunks_until_eot(pcms, prompt, mk.CAP)
        ids, probs = c.chunk_languages(batch)
    single_clip_agreement(mk.MODEL, pcms, prompt, mk.CAP, ids, probs, got, **kw)


# speed-up is context state the detection pass sees through the batch's own encode; no speed-up batch is pinned to the reference
# (tests/golden/make_chunks_lang_golden.py says why), so this one is checked against the single-clip path
SETTINGS = {"speed_up": (dict(speed_up=True), (960000, 880000, 760000, 740000))}


@pytest.mark.parametrize("name", list(SETTINGS))
def test_settings_agree_with_single_clip_path(name):
    kw, lengths = SETTINGS[name]
    m, c = context(mk.MODEL, 4)
    pcms = [synth.synth_pcm(13 + b, lengths[b]) for b in range(4)]
    prompt = np.array(m.prompt_init("auto"), np.int32)
    with Settings(c, **kw):
        got, _ = c.run_chunks_until_eot(pcms, prompt, mk.CAP)
        ids, probs = c.chunk_languages(4)
    single_clip_agreement(mk.MODEL, pcms, prompt, mk.CAP, ids, probs, got, **kw)


# the decoder-step kernel's paths beyond the micro model: bench.py's model and batch, and the widest model
LARGER = {"medium_b8": ("medium-sc", 8), "large_b2": ("large-sc", 2)}
LARGER_LENGTHS = (480000, 440000, 420000, 400000)
LARGER_CAP = 48


@pytest.mark.parametrize("name", list(LARGER))
def test_larger_shapes_agree_with_single_clip_path(name):
    model, batch = LARGER[name]
    m, c = context(model, batch)
    pcms = [synth.synth_pcm(b, LARGER_LENGTHS[b % len(LARGER_LENGTHS)]) for b in range(batch)]
    prompt = np.array(m.prompt_init("auto"), np.int32)
    got, _ = c.run_chunks_until_eot(pcms, prompt, LARGER_CAP)
    ids, probs = c.chunk_languages(batch)
    assert probs.shape == (batch, 99) and np.allclose(probs.sum(axis=1), 1.0, atol=1e-4)
    single_clip_agreement(model, pcms, prompt, LARGER_CAP, ids, probs, got)


def test_fixed_prompt_is_unchanged():
    """a fixed-prompt call after an auto call decodes bit for bit as on a fresh context, with the same launches; detection adds
    exactly one decoder step kernel, the vocabulary softmax and the language pick"""
    name = "base"
    batch = mk.CASES[name][1]
    m, e = engine(mk.MODEL)
    pcms, auto, _kw = case(name)
    fixed = fixed_prompt(m, 0)
    fresh = capi.Context(e, batch)
    try:
        fresh.run_chunks(pcms, fixed, mk.CAP)                          # warm: the step graph is captured once
        (ref_toks, _), n_fixed = launches(lambda: fresh.run_chunks(pcms, fixed, mk.CAP))
        ref_logits = fresh.logits(batch)
    finally:
        fresh.close()
    c = capi.Context(e, batch)
    try:
        assert c.chunk_languages(batch) is None                        # no call yet
        c.run_chunks(pcms, fixed, mk.CAP)
        _, n_auto = launches(lambda: c.run_chunks(pcms, auto, mk.CAP))
        assert c.chunk_languages(batch) is not None
        (toks, _), n = launches(lambda: c.run_chunks(pcms, fixed, mk.CAP))
        assert np.array_equal(toks, ref_toks) and np.array_equal(c.logits(batch), ref_logits)
        assert n == n_fixed and n_auto == n_fixed + 3
        assert c.chunk_languages(batch) is None
        # the same through the other two entry points
        for b, p in enumerate(pcms):
            c.upload_pcm(b, p)
        c.run_chunks_resident(batch, auto, 8)
        assert c.chunk_languages(batch) is not None
        c.run_chunks_until_eot(None, fixed, 8, batch=batch)
        assert c.chunk_languages(batch) is None
    finally:
        c.close()


def test_errors_launch_nothing():
    L = capi.lib()
    i = capi._i
    pcm = synth.synth_pcm(0)
    ptrs = (C.POINTER(C.c_float) * 2)(capi._f(pcm), capi._f(pcm))
    ns = np.array([pcm.size, pcm.size], np.int32)
    toks = np.zeros(2 * 8, np.int32)

    def run(c, prompt):
        pr = np.array(prompt, np.int32)
        before = L.wsp_launch_count()
        rc = L.wsp_run_chunks(c.h, ptrs, i(ns), 2, i(pr), pr.size, 8, i(toks), None)
        assert L.wsp_launch_count() == before, "nothing may be launched before the prompt is checked"
        return rc

    m_en, c_en = context("micro.en-sc", 2)
    assert run(c_en, [m_en.special["sot"], capi.TOKEN_LANGUAGE_AUTO]) == E_INVALIDARG          # not multilingual
    m, c = context(mk.MODEL, 2)
    sot, task = m.special["sot"], m.special["transcribe"]
    assert run(c, [sot, capi.TOKEN_LANGUAGE_AUTO, capi.TOKEN_LANGUAGE_AUTO, task]) == E_INVALIDARG
    assert run(c, [sot, -2, task]) == E_INVALIDARG
    assert run(c, [sot, m.n_vocab, task]) == E_INVALIDARG
    assert run(c_en, [m_en.special["sot"], m_en.n_vocab]) == E_INVALIDARG                      # fixed prompts are checked too
    # the languages of a call: bounds of wsp_get_chunk_languages
    c.run_chunks([pcm, pcm], m.prompt_init("auto"), 4)
    ids = np.zeros(3, np.int32)
    probs = np.zeros((3, 99), np.float32)
    before = L.wsp_launch_count()
    assert L.wsp_get_chunk_languages(c.h, 2, i(ids), capi._f(probs), 2 * 99 - 1) == E_BOUNDS
    assert L.wsp_get_chunk_languages(c.h, 3, i(ids), capi._f(probs), probs.size) == E_BOUNDS
    assert L.wsp_get_chunk_languages(c.h, 2, i(ids), None, 0) == 0
    assert L.wsp_launch_count() == before
    ids1, _ = c.chunk_languages(1)
    assert ids1[0] == ids[0]


def test_replicas_pass_the_sentinel_through():
    name = "base"
    batch = mk.CASES[name][1]
    m, c = context(mk.MODEL, 2)
    pcms, prompt, _kw = case(name)
    want_toks = np.concatenate([c.run_chunks(pcms[i:i + 2], prompt, mk.CAP)[0] for i in range(0, batch, 2)])
    r = capi.Replicas(m, [0, 0], 2)
    try:
        toks, stats = r.run_chunks(pcms, prompt, mk.CAP)
        assert toks.tolist() == want_toks.tolist()
        assert sum(s["chunks"] for s in stats) == batch and not any(s["failed"] for s in stats)
    finally:
        r.close()
