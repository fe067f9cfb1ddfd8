"""wsp_run_spans_window on an H100: each row of a batch decoded as the first window of whisper_full( clip of its source slot,
offset_ms, duration_ms ), several rows sharing one resident clip.

Oracle: tests/golden/chunks_spans.npz (tests/golden/make_chunks_spans_golden.py, from oracle/_ref: the window loop restated at each
span's seek over the reference's encode, decode and samplers, and checked against its whisper_full( offset_ms, duration_ms )).  Ids,
tids, results, segments, languages and token times must be identical; p and ptsum within 5e-3, as in
tests/test_gpu_chunks_window.py, and pt too wherever ptsum exceeds 5e-3.  The other checks compare the GPU with itself (spans against wsp_run_chunks_window, each row against
the row alone, launch counts) and with runFull( offset_ms, duration_ms ) of the COM layer on models without a fixture.
"""
import ctypes as C
import os

import numpy as np
import pytest

from tests import test_gpu_com as com
from tests.golden import make_chunks_spans_golden as mks
from tests.golden import make_chunks_window_golden as mkw
from whisper_b200 import capi, synth

pytestmark = pytest.mark.gpu

P_TOL = 5e-3
E_INVALIDARG, E_POINTER, E_BOUNDS = -1, -2, -7
F32 = np.float32
_cache = {}


def golden():
    if "g" not in _cache:
        _cache["g"] = np.load(os.path.join(os.path.dirname(__file__), "golden", "chunks_spans.npz"))
    return _cache["g"]


def engine(model):
    if model not in _cache:
        m = capi.Model(synth.model_path(model))
        _cache[model] = (m, capi.Engine(m, 0))
    return _cache[model]


def launches(f):
    L = capi.lib()
    before = L.wsp_launch_count()
    r = f()
    return r, int(L.wsp_launch_count() - before)


def sources_of(name):
    return [mks.source_pcm([tuple(int(x) for x in p) for p in s if p[0] >= 0]) for s in golden()[name + "_sources"]]


def upload(c, pcms):
    for slot, p in enumerate(pcms):
        c.upload_pcm(slot, p)


def assert_same(a, b, label=""):
    assert a["result"] == b["result"], label
    assert a["tokens"] == b["tokens"], label
    assert a["segments"] == b["segments"], label


def check_restated(m, out, spans, pcms, max_tokens, single, hop=160, speed_up=False):
    """every row's result is the rule restated at its seek over its own ids, and its segments the segmentation at that seek"""
    eot, beg, n_max = m.special["eot"], m.special["beg"], m.n_text_ctx // 2 - 4
    text = lambda i: m.token_text(i) or ""
    kinds = set()
    for b, (o, (slot, off, dur)) in enumerate(zip(out, spans)):
        seek, seek_end = mks.bounds(off, dur, pcms[slot].size // hop)
        r = o["result"]
        if seek_end <= seek + 100:
            assert r == dict(n_sampled=0, n_tokens=0, seek_delta=0, failed=0) and o["segments"] == [], b
            kinds.add("no_window")
            continue
        ids = [t["id"] for t in o["tokens"]]
        want, kind, used = mkw.rule(ids, eot, beg, max_tokens, single, n_max, seek, seek_end)
        assert kind is not None and used == len(ids) == r["n_sampled"], b
        assert (r["n_tokens"], r["seek_delta"], r["failed"]) == (want["result_len"], want["seek_delta"], want["failed"]), b
        assert o["segments"] == mkw.segments(o["tokens"], r, seek, eot, beg, text, single_segment=bool(single), speed_up=speed_up), b
        kinds.add(kind)
    return kinds


# ---- 1. the reference ------------------------------------------------------------------------------------------------------------
PARAMS = [(name, th, ml) for name, case in mks.CASES.items() for th in case[1] for ml in (None,) + (mks.MAX_LENS if mks.TOKEN_TIMES[name] else ())]


@pytest.mark.parametrize("name,th,ml", PARAMS)
def test_reference_parity(name, th, ml):
    """ml None: plain segments; 0 / 12: token times with max_len"""
    g = golden()
    model = mks.CASES[name][0]
    m, e = engine(model)
    pcms = sources_of(name)
    spans = [tuple(int(x) for x in s) for s in g[name + "_spans"]]
    mt, single = (int(x) for x in g[name + "_params"])
    c = capi.Context(e, len(spans))
    try:
        upload(c, pcms)
        c.set_reference_threads(th)
        c.set_token_timestamps(ml is not None)
        tt = None if ml is None else dict(max_len=ml)
        out, st = c.run_spans_window(spans, g[name + "_prompt"].tolist(), mt, single, token_times=tt)
        langs = c.chunk_languages(len(spans))
    finally:
        c.close()
    assert st[2] > 0
    p = "%s_t%d_" % (name, th)
    for b in range(len(spans)):
        o, r = out[b], g[p + "result"][b]
        assert [o["result"][k] for k in ("n_sampled", "n_tokens", "seek_delta", "failed")] == r.tolist(), "row %d" % b
        n = int(r[0])
        assert [(t["id"], t["tid"]) for t in o["tokens"]] == [tuple(x) for x in g[p + "tokens"][b, :n].tolist()], "row %d" % b
        got_p = np.array([[t["p"], t["pt"], t["ptsum"]] for t in o["tokens"]], np.float32).reshape(-1, 3)
        # pt = the best timestamp's share of ptsum: where ptsum itself is below P_TOL, it is a ratio of probabilities under the
        # tolerance, and no rule reads it (ptsum alone fails thold_ptsum), so it is compared only above
        dp = np.abs(got_p - g[p + "probs"][b, :n])
        dp[:, 1] = np.where(g[p + "probs"][b, :n, 2] > P_TOL, dp[:, 1], 0)
        assert dp.max(initial=0) <= P_TOL, ("row %d" % b, np.argwhere(dp > P_TOL).tolist())
        q = p if ml is None else "%sml%d_" % (p, ml)
        segs = g[q + "segments"][b]
        k = int((segs[:, 0] >= 0).sum())
        want = [(int(s[0]), int(s[1]), int(s[2]), int(s[3]), str(t)) for s, t in zip(segs[:k], g[q + "texts"][b, :k])]
        assert [(s["t0"], s["t1"], s["i0"], s["i1"], s["text"]) for s in o["segments"]] == want, "row %d" % b
        if ml is not None:
            nt = o["result"]["n_tokens"]
            want_t = [(int(a), int(z), float(v)) for (a, z), v in zip(g[q + "times"][b, :nt].tolist(), g[q + "vlen"][b, :nt].tolist())]
            assert [(t["t0"], t["t1"], float(F32(t["vlen"]))) for t in o["tokens"][:nt]] == want_t, "row %d" % b
    if (g[name + "_prompt"] == capi.TOKEN_LANGUAGE_AUTO).any():
        assert langs[0].tolist() == g[p + "lang"].tolist()
        assert len(set(langs[0].tolist())) >= 2
    else:
        assert langs is None


# ---- 2. spans { b, 0, 0 } are wsp_run_chunks_window ---------------------------------------------------------------------------------
@pytest.mark.parametrize("model,batch", [("micro.en-sc", 5), ("medium-sc", 8)])
@pytest.mark.parametrize("energy", [False, True])
def test_identity_spans_equal_chunks_window(model, batch, energy):
    m, e = engine(model)
    c = capi.Context(e, batch)
    try:
        upload(c, [synth.synth_pcm(b, mkw.LENGTHS[b % len(mkw.LENGTHS)]) for b in range(batch)])
        c.set_token_timestamps(energy)
        tt = dict(max_len=12) if energy else None
        (want, _), n_want = launches(lambda: c.run_chunks_window(None, m.prompt_init(), batch=batch, token_times=tt))
        (got, _), n_got = launches(lambda: c.run_spans_window([(b, 0, 0) for b in range(batch)], m.prompt_init(), token_times=tt))
    finally:
        c.close()
    assert n_got == n_want
    for b in range(batch):
        assert_same(got[b], want[b], "row %d" % b)


# ---- 3. each row is the span run alone ------------------------------------------------------------------------------------------
ALONE = {"base_en_b12": ("base.en-sc", 12), "medium_b8": ("medium-sc", 8)}


def long_sources():
    """a 75 s source, a 30 s one, an unused slot and an 18 s one"""
    return [synth.synth_pcm(3, 1200000), synth.synth_pcm(5, 480000), synth.synth_pcm(9, 160000), synth.synth_pcm(7, 288000)]


def spans_for(batch):
    base = [(0, 0, 0), (0, 30000, 0), (0, 61234, 0), (1, 0, 0), (1, 4000, 700), (3, 2000, 5000), (0, 45000, 20000), (3, 17500, 0),
            (0, 74500, 0), (1, 12345, 0), (3, 0, 0), (0, 10000, -1)]
    return base[:batch]


@pytest.mark.parametrize("name", list(ALONE))
def test_row_equals_span_alone(name):
    model, batch = ALONE[name]
    m, e = engine(model)
    c = capi.Context(e, batch)
    try:
        pcms = long_sources()
        upload(c, pcms)
        spans = spans_for(batch)
        out, _ = c.run_spans_window(spans, m.prompt_init())
        for b, sp in enumerate(spans):
            alone, _ = c.run_spans_window([sp], m.prompt_init())
            assert_same(out[b], alone[0], "row %d %s" % (b, sp))
        kinds = check_restated(m, out, spans, pcms, 0, 0)
    finally:
        c.close()
    assert "no_window" in kinds and len(kinds) >= 3, kinds


# ---- 4. runFull( offset_ms, duration_ms ) of the COM layer ---------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["tiny.en-sc", "base.en-sc"])
def test_rows_are_first_segments_of_run_full(model):
    m, e = engine(model)
    pcms = long_sources()
    spans = spans_for(12)
    c = capi.Context(e, len(spans))
    L, h = com.open_session(model)
    try:
        upload(c, pcms)
        out, _ = c.run_spans_window(spans, m.prompt_init())
        compared = 0
        for o, (slot, off, dur) in zip(out, spans):
            hr, full = com.run_full(L, h, pcms[slot], flags=2, off=off, dur=dur)
            assert hr == 0
            got = [(s["t0"], s["t1"], s["text"], [t["id"] for t in o["tokens"][s["i0"]:s["i1"]]]) for s in o["segments"]]
            want = [(s["t0"], s["t1"], s["text"], s["tokens"]) for s in full[:len(got)]]
            if o["result"]["failed"] or o["result"]["n_sampled"] == 0:
                continue
            assert got == want, (slot, off, dur)
            compared += bool(got)
    finally:
        c.close()
    assert compared >= 4


# ---- 5. a shared slot's log-mel and energy are computed once ---------------------------------------------------------------------
def test_shared_slot_adds_no_mel_or_energy_launch():
    """17 rows on one slot against the same rows on 17 copies of it: the same windows, three launches (one mel triple) fewer; slots
    no row names keep their log-mel and energy"""
    m, e = engine("micro.en-sc")
    B = 18
    c = capi.Context(e, B)
    try:
        pcm = synth.synth_pcm(3, 960000)
        for slot in range(17):
            c.upload_pcm(slot, pcm)
        c.set_token_timestamps(1)
        c.pcm_to_mel(17, synth.synth_pcm(4, 200000))
        mel17, en17 = c.get_mel(17), c.get_tensor("energy", 17)
        offs = [1000 * k for k in range(17)]
        (one, _), n_one = launches(lambda: c.run_spans_window([(0, o, 0) for o in offs], m.prompt_init(), token_times={}))
        (many, _), n_many = launches(lambda: c.run_spans_window([(k, o, 0) for k, o in enumerate(offs)], m.prompt_init(), token_times={}))
        for b in range(17):
            assert_same(one[b], many[b], "row %d" % b)
        assert n_many - n_one == 3
        assert np.array_equal(c.get_mel(17), mel17) and np.array_equal(c.get_tensor("energy", 17), en17)
    finally:
        c.close()


# ---- 6. speakers of a stereo source ----------------------------------------------------------------------------------------------
def test_speakers_of_a_stereo_source():
    from tests.test_gpu_chunks_speakers import downmix, gains_stereo
    m, e = engine("micro.en-sc")
    lr = gains_stereo(synth.synth_pcm(3, 960000))
    c = capi.Context(e, 6)
    try:
        c.upload_pcm_stereo(0, lr)
        c.upload_pcm(2, synth.synth_pcm(7, 320000))
        spans = [(0, 0, 0), (2, 3000, 0), (0, 36000, 0), (0, 12000, 9000), (2, 0, 0), (0, 41000, 0)]
        out, _ = c.run_spans_window(spans, m.prompt_init(), speakers=True)
        mono, _ = c.run_spans_window(spans, m.prompt_init())
        answers = set()
        for o, mo, (slot, _off, _dur) in zip(out, mono, spans):
            assert [(s["t0"], s["t1"]) for s in o["segments"]] == [(s["t0"], s["t1"]) for s in mo["segments"]]
            want = capi.test_speakers(lr, [(s["t0"], s["t1"]) for s in o["segments"]]) if slot == 0 else \
                [capi.SPEAKER_NO_STEREO] * len(o["segments"])
            assert [s["speaker"] for s in o["segments"]] == want, (slot, _off)
            answers |= set(want)
        np.testing.assert_array_equal(c.get_tensor("pcm", 0), downmix(lr))
    finally:
        c.close()
    assert {capi.SPEAKER_LEFT, capi.SPEAKER_RIGHT} <= answers, answers


# ---- 7, 8. speed-up and audio_ctx ------------------------------------------------------------------------------------------------
def enc_input_of(c, mel, seek, frames):
    want = np.zeros((frames, 80), np.float16)
    part = mel[:, seek:seek + frames].T if seek < mel.shape[1] else np.zeros((0, 80), F32)
    want[:part.shape[0]] = part.astype(np.float16)
    return want


def test_speed_up():
    """seek and seek_end at the vocoder's hop, segment times doubled, the encode at seek of the phase-vocoder log-mel"""
    m, e = engine("micro.en-sc")
    pcms = long_sources()
    spans = [(0, 0, 0), (0, 30000, 0), (0, 12345, 40000), (1, 7000, 0), (0, 59000, 0), (3, 1000, 600), (0, 20000, 6000)]
    c = capi.Context(e, len(spans))
    try:
        upload(c, pcms)
        c.set_speed_up(1)
        out, _ = c.run_spans_window(spans, m.prompt_init())
        for b, (slot, off, _d) in enumerate(spans):
            mel = c.get_mel(slot)
            assert mel.shape[1] == pcms[slot].size // 320
            got = c.get_tensor("enc.input", b).reshape(-1, 80)
            assert np.array_equal(got, enc_input_of(c, mel, off // 10, got.shape[0]).astype(got.dtype)), b
        kinds = check_restated(m, out, spans, pcms, 0, 0, hop=320, speed_up=True)
        for b, sp in enumerate(spans):
            alone, _ = c.run_spans_window([sp], m.prompt_init())
            assert_same(out[b], alone[0], "row %d" % b)
    finally:
        c.close()
    assert "no_window" in kinds and len(kinds) >= 3, kinds


def test_audio_ctx_750_with_offsets():
    m, e = engine("micro.en-sc")
    pcms = long_sources()
    spans = spans_for(8)
    c = capi.Context(e, len(spans))
    try:
        upload(c, pcms)
        c.set_audio_ctx(750)
        out, _ = c.run_spans_window(spans, m.prompt_init())
        for b, (slot, off, _d) in enumerate(spans):
            got = c.get_tensor("enc.input", b).reshape(-1, 80)
            assert got.shape[0] == 1500
            assert np.array_equal(got, enc_input_of(c, c.get_mel(slot), off // 10, 1500).astype(got.dtype)), b
        check_restated(m, out, spans, pcms, 0, 0)
        for b, sp in enumerate(spans):
            alone, _ = c.run_spans_window([sp], m.prompt_init())
            assert_same(out[b], alone[0], "row %d" % b)
    finally:
        c.close()


# ---- 9. errors --------------------------------------------------------------------------------------------------------------------
def test_errors_launch_nothing():
    m, e = engine("micro-sc")
    c = capi.Context(e, 4)
    L = capi.lib()
    try:
        c.upload_pcm(0, synth.synth_pcm(1, 320000))
        c.upload_pcm(1, synth.synth_pcm(2, 160000))
        prompt = m.prompt_init()
        auto = m.prompt_init("auto")
        cap = m.n_text_ctx // 2 - 4
        toks = (capi.TokenData * (4 * cap))()
        res = (capi.WindowResult * 4)()
        prm = capi.WindowParams(0, 0)

        def call(spans, pr=prompt, sp_null=False, prm_ref=C.byref(prm), r=res, p_null=False):
            sp = (capi.WindowSpan * max(len(spans), 1))(*[capi.WindowSpan(*s) for s in spans])
            a = np.ascontiguousarray(pr, np.int32)
            before = L.wsp_launch_count()
            st = L.wsp_run_spans_window(c.h, None if sp_null else sp, len(spans), None if p_null else capi._i(a), a.size, prm_ref, toks,
                                        cap, r, None)
            return st, int(L.wsp_launch_count() - before)

        for spans, want in [([], E_BOUNDS), ([(0, 0, 0)] * 5, E_BOUNDS), ([(4, 0, 0)], E_BOUNDS), ([(-1, 0, 0)], E_BOUNDS),
                            ([(2, 0, 0)], E_INVALIDARG), ([(0, -10, 0)], E_INVALIDARG), ([(0, 0, 0), (3, 0, 0)], E_INVALIDARG)]:
            assert call(spans) == (want, 0), spans
        assert call([(0, 0, 0), (1, 10000, 0)], pr=auto) == (E_INVALIDARG, 0)      # 1000 frames: at the end of slot 1
        assert call([(1, 9990, 0)], pr=auto)[0] == 0                                 # the last frame: detected
        assert call([(0, 0, 0)], sp_null=True) == (E_POINTER, 0)
        assert call([(0, 0, 0)], p_null=True) == (E_POINTER, 0)
        assert call([(0, 0, 0)], prm_ref=None) == (E_POINTER, 0)
        assert call([(0, 0, 0)], r=None) == (E_POINTER, 0)
        assert call([(0, 0, 0)], pr=[m.special["sot"], -5]) == (E_INVALIDARG, 0)
        # a negative duration is no error: no window
        out, _ = c.run_spans_window([(0, 5000, -20), (0, 0, 0)], prompt)
        assert out[0]["result"] == dict(n_sampled=0, n_tokens=0, seek_delta=0, failed=0) and out[1]["result"]["n_sampled"] > 0
    finally:
        c.close()


# ---- 10. the other calls are unchanged after a spans call ------------------------------------------------------------------------
def test_other_calls_unchanged():
    m, e = engine("micro.en-sc")
    B = 4
    c = capi.Context(e, B)
    pcms = [synth.synth_pcm(b, mkw.LENGTHS[b + 1]) for b in range(B)]
    prompt = m.prompt_init()

    def calls():
        upload(c, pcms)
        c.set_token_timestamps(1)
        w, nw = launches(lambda: c.run_chunks_window(None, prompt, batch=B, token_times=dict(max_len=12))[0])
        c.set_token_timestamps(0)
        u, nu = launches(lambda: [t.tolist() for t in c.run_chunks_until_eot(None, prompt, 100, batch=B)[0]])
        r, nr = launches(lambda: c.run_chunks(pcms, prompt, 24)[0].tolist())
        return (w, u, r), (nw, nu, nr)

    try:
        before, n_before = calls()
        c.upload_pcm(0, synth.synth_pcm(9, 900000))
        c.set_token_timestamps(1)
        c.run_spans_window([(0, 40000, 0), (0, 3000, 0), (2, 5000, 0)], prompt, token_times={})
        after, n_after = calls()
    finally:
        c.close()
    assert n_after == n_before
    assert after == before
