"""wsp_run_chunks_window on an H100: each chunk of a batch decoded as whisper_full's first window, ended by its window rule in the
sampler's epilogue, with token data and whisper_full's segments.

Oracle: tests/golden/chunks_window.npz (tests/golden/make_chunks_window_golden.py, from oracle/_ref: the window loop restated over the
reference's decode and samplers, and checked against its whisper_full).  Ids, tids, results and segments must be identical; p, pt
and ptsum within 5e-3, the probability tolerance of the end-to-end parity tests (tests/test_gpu_parity.py), since the logits
themselves carry the decoder's tolerance.  The other checks compare the GPU with itself: every window against the Python restatement
of the rule and of the segmentation over its own tokens, each chunk of a batch against the chunk run alone, and the window call
against wsp_run_chunks over the same steps.
"""
import ctypes as C
import os

import numpy as np
import pytest

from tests.golden import make_chunks_window_golden as mk
from whisper_b200 import capi, synth

pytestmark = pytest.mark.gpu

EOT_LAG = 8          # the host's block of steps (context.cu: kEotLag)
P_TOL = 5e-3
E_INVALIDARG, E_POINTER, E_BOUNDS = -1, -2, -7

_cache = {}


def golden():
    if "g" not in _cache:
        _cache["g"] = np.load(os.path.join(os.path.dirname(__file__), "golden", "chunks_window.npz"))
    return _cache["g"]


def context(model, batch, fresh=False):
    if ("engine", model) not in _cache:
        m = capi.Model(synth.model_path(model))
        _cache[("engine", model)] = (m, capi.Engine(m, 0))
    m, e = _cache[("engine", model)]
    if fresh:
        return m, capi.Context(e, batch)
    if (model, batch) not in _cache:
        _cache[(model, batch)] = capi.Context(e, batch)
    return m, _cache[(model, batch)]


# batches the GPU checks against itself only: the two-tile decoder step (B in 9..16) and bench.py's model and batch
GPU_ONLY = {"base_en_b12": ("base.en-sc", 12), "medium_b8": ("medium-sc", 8)}
GPU_ONLY_LENGTHS = (480000, 440000, 160000, 400000, 240000, 12000)


def model_of(name):
    return mk.CASES[name][0] if name in mk.CASES else GPU_ONLY[name][0]


def batch_of(name):
    return mk.CASES[name][2] if name in mk.CASES else GPU_ONLY[name][1]


def params_of(name):
    return (int(golden()[name + "_params"][0]), int(golden()[name + "_params"][1])) if name in mk.CASES else (0, 0)


def case_inputs(name):
    if name in GPU_ONLY:
        m, _c = context(model_of(name), batch_of(name))
        return [synth.synth_pcm(b, GPU_ONLY_LENGTHS[b % len(GPU_ONLY_LENGTHS)]) for b in range(batch_of(name))], m.prompt_init()
    g = golden()
    pcms = [synth.synth_pcm(int(c), int(n)) for c, n in zip(g[name + "_chunks"], g[name + "_n_samples"])]
    return pcms, g[name + "_prompt"].tolist()


def launches(f):
    L = capi.lib()
    before = L.wsp_launch_count()
    r = f()
    return r, int(L.wsp_launch_count() - before)


def check_self_consistent(m, out, pcms, max_tokens, single, hop=160, speed_up=False):
    """every window's result is the rule restated over its own ids, and its segments are the segmentation restated; returns the
    kinds of window end seen"""
    eot, beg, n_max = m.special["eot"], m.special["beg"], m.n_text_ctx // 2 - 4
    text = lambda i: m.token_text(i) or ""
    kinds = set()
    for b, (o, pcm) in enumerate(zip(out, pcms)):
        seek_end = pcm.size // hop
        r = o["result"]
        if seek_end <= 100:
            assert r == dict(n_sampled=0, n_tokens=0, seek_delta=0, failed=0) and o["segments"] == [], b
            continue
        ids = [t["id"] for t in o["tokens"]]
        want, kind, used = mk.rule(ids, eot, beg, max_tokens, single, n_max, 0, seek_end)
        assert kind is not None and used == len(ids) == r["n_sampled"], b
        assert (r["n_tokens"], r["seek_delta"], r["failed"]) == (want["result_len"], want["seek_delta"], want["failed"]), b
        assert o["segments"] == mk.segments(o["tokens"], r, 0, eot, beg, text, single_segment=bool(single), speed_up=speed_up), b
        kinds.add(kind)
    return kinds


def assert_same(a, b, p_tol=0.0, label=""):
    assert a["result"] == b["result"], label
    assert [(t["id"], t["tid"]) for t in a["tokens"]] == [(t["id"], t["tid"]) for t in b["tokens"]], label
    for x, y in zip(a["tokens"], b["tokens"]):
        for k in ("p", "pt", "ptsum"):
            assert abs(x[k] - y[k]) <= p_tol, (label, k, x, y)
    assert a["segments"] == b["segments"], label


PARAMS = [(name, th) for name, (_m, ths, *_r) in mk.CASES.items() for th in ths]


@pytest.mark.parametrize("form", ["host", "resident"])
@pytest.mark.parametrize("name,th", PARAMS)
def test_reference_parity(name, th, form):
    model, _ths, batch = mk.CASES[name][:3]
    m, c = context(model, batch)
    pcms, prompt = case_inputs(name)
    mt, single = params_of(name)
    c.set_reference_threads(th)
    try:
        if form == "host":
            out, st = c.run_chunks_window(pcms, prompt, mt, single)
        else:
            for b, p in enumerate(pcms):
                c.upload_pcm(b, p)
            out, st = c.run_chunks_window(None, prompt, mt, single, batch=batch)
    finally:
        c.set_reference_threads(4)
    assert len(out) == batch and st[2] > 0
    g, p = golden(), "%s_t%d_" % (name, th)
    for b in range(batch):
        o, r = out[b], g[p + "result"][b]
        assert [o["result"][k] for k in ("n_sampled", "n_tokens", "seek_delta", "failed")] == r.tolist(), "chunk %d" % b
        n = int(r[0])
        assert [(t["id"], t["tid"]) for t in o["tokens"]] == [tuple(x) for x in g[p + "tokens"][b, :n].tolist()], "chunk %d" % b
        got_p = np.array([[t["p"], t["pt"], t["ptsum"]] for t in o["tokens"]], np.float32).reshape(-1, 3)
        assert np.abs(got_p - g[p + "probs"][b, :n]).max(initial=0) <= P_TOL, "chunk %d" % b
        segs = g[p + "segments"][b]
        k = int((segs[:, 0] >= 0).sum())
        want = [dict(t0=int(s[0]), t1=int(s[1]), i0=int(s[2]), i1=int(s[3]), text=str(t)) for s, t in zip(segs[:k], g[p + "texts"][b, :k])]
        assert o["segments"] == want, "chunk %d" % b
    kinds = check_self_consistent(m, out, pcms, mt, single)
    if name == "micro_en":
        assert "audio_end" in kinds     # seek_end reaches the device from host and from resident PCM


@pytest.mark.parametrize("name", list(mk.CASES) + list(GPU_ONLY))
def test_batch_independence(name):
    """each chunk of the batch equals the same chunk run alone, and the window's tokens are those of wsp_run_chunks over n_max steps"""
    batch = batch_of(name)
    m, c = context(model_of(name), batch)
    pcms, prompt = case_inputs(name)
    mt, single = params_of(name)
    out, _ = c.run_chunks_window(pcms, prompt, mt, single)
    check_self_consistent(m, out, pcms, mt, single)
    full, _ = c.run_chunks(pcms, prompt, m.n_text_ctx // 2 - 4)
    for b in range(batch):
        assert [t["id"] for t in out[b]["tokens"]] == full[b, :out[b]["result"]["n_sampled"]].tolist(), "chunk %d" % b
    m1, c1 = context(model_of(name), 1)
    for b in range(batch):
        alone, _ = c1.run_chunks_window([pcms[b]], prompt, mt, single)
        assert_same(out[b], alone[0], P_TOL, "chunk %d" % b)
    if name in GPU_ONLY:
        assert any(o["result"]["n_sampled"] > 0 and not o["result"]["failed"] for o in out)


def test_language_sentinel():
    name = "micro_ml"
    batch = batch_of(name)
    m, c = context(model_of(name), batch)
    pcms, _prompt = case_inputs(name)
    mt, single = params_of(name)
    out, _ = c.run_chunks_window(pcms, m.prompt_init("auto"), mt, single)
    ids, _probs = c.chunk_languages(batch)
    for b in range(batch):
        fixed, _ = c.run_chunks_window([pcms[b]], m.prompt_init(int(ids[b])), mt, single)
        assert_same(out[b], fixed[0], P_TOL, "chunk %d" % b)


def test_audio_ctx_750():
    name = "micro_en"
    batch = batch_of(name)
    m, c = context(model_of(name), batch, fresh=True)
    try:
        pcms, prompt = case_inputs(name)
        c.set_audio_ctx(750)
        out, _ = c.run_chunks_window(pcms, prompt)
        check_self_consistent(m, out, pcms, 0, 0)
        full, _ = c.run_chunks(pcms, prompt, m.n_text_ctx // 2 - 4)
        for b in range(batch):
            assert [t["id"] for t in out[b]["tokens"]] == full[b, :out[b]["result"]["n_sampled"]].tolist(), "chunk %d" % b
    finally:
        c.close()


def test_speed_up_doubles_times():
    # 60 s clips fill one phase-vocoder window as 30 s clips fill a plain one; the rest are longer and shorter.  32640 samples are
    # 102 frames at the vocoder's hop of 320 (204 at 160): its first timestamp ends the window only if seek_end is n / 320
    pcms = [synth.synth_pcm(ch, n) for ch, n in ((0, 960000), (1, 960000), (2, 640000), (3, 1440000), (4, 320000), (5, 12000), (0, 32640))]
    m, c = context("micro.en-sc", len(pcms), fresh=True)
    prompt = m.prompt_init()
    try:
        c.set_speed_up(1)
        out, _ = c.run_chunks_window(pcms, prompt)
        assert "audio_end" in check_self_consistent(m, out, pcms, 0, 0, hop=320, speed_up=True)
        for o in out:
            plain = m.window_segments(o["tokens"], o["result"], 0, 0)
            assert [(s["t0"] * 2, s["t1"] * 2, s["i0"], s["i1"], s["text"]) for s in plain] == \
                [(s["t0"], s["t1"], s["i0"], s["i1"], s["text"]) for s in o["segments"]]
        assert any(o["segments"] for o in out)
    finally:
        c.close()


def steps_run(c, pcms, prompt, f):
    """decoder steps a call ran, from the launch count: wsp_run_chunks with n_decode = 1 and 2 give the fixed part and one step"""
    _, base = launches(lambda: c.run_chunks(pcms, prompt, 1))
    _, two = launches(lambda: c.run_chunks(pcms, prompt, 2))
    r, n = launches(f)
    per = two - base
    assert per > 0 and (n - base) % per == 0
    return r, 1 + (n - base) // per


@pytest.mark.parametrize("name", list(mk.CASES) + list(GPU_ONLY))
def test_stop_bound(name):
    batch = batch_of(name)
    m, c = context(model_of(name), batch)
    pcms, prompt = case_inputs(name)
    mt, single = params_of(name)
    n_max = m.n_text_ctx // 2 - 4
    (out, _), steps = steps_run(c, pcms, prompt, lambda: c.run_chunks_window(pcms, prompt, mt, single))
    last = max(o["result"]["n_sampled"] for o in out)
    assert max(last, 1) <= steps <= min(n_max, last + 2 * EOT_LAG + 1)
    # without the window that runs all n_max steps, the batch stops early
    rows = [b for b in range(batch) if out[b]["result"]["n_sampled"] < n_max]
    if rows:
        sub = [pcms[b] for b in rows]
        (out2, _), steps2 = steps_run(c, sub, prompt, lambda: c.run_chunks_window(sub, prompt, mt, single))
        last2 = max(o["result"]["n_sampled"] for o in out2)
        assert steps2 <= last2 + 2 * EOT_LAG + 1 and steps2 < n_max


def test_short_clips_only():
    m, c = context("micro.en-sc", 2, fresh=True)
    try:
        pcms = [synth.synth_pcm(0, 12000), synth.synth_pcm(1, 16000)]
        out, _ = c.run_chunks_window(pcms, m.prompt_init())
        assert all(o["result"] == dict(n_sampled=0, n_tokens=0, seek_delta=0, failed=0) and o["tokens"] == [] for o in out)
    finally:
        c.close()


def test_other_calls_unchanged():
    """wsp_run_chunks and wsp_run_chunks_until_eot on a fresh context, and again after window calls: bit-identical, same launches"""
    name = "micro_en"
    model, batch = model_of(name), batch_of(name)
    pcms, prompt = case_inputs(name)

    def both(c):
        (a, _), na = launches(lambda: c.run_chunks(pcms, prompt, 60))
        la = c.logits(batch)
        (e, _), ne = launches(lambda: c.run_chunks_until_eot(pcms, prompt, 100))
        return a, la, [t.tolist() for t in e], na, ne

    m, fresh = context(model, batch, fresh=True)
    try:
        ref = both(fresh)
    finally:
        fresh.close()
    m, c = context(model, batch, fresh=True)
    try:
        c.run_chunks_window(pcms, prompt)
        c.run_chunks_window(pcms[1:], prompt, 5, True)
        got = both(c)
        assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1])
        assert got[2:] == ref[2:]
        # the per-op path (no step graph) gives the same windows
        w1, _ = c.run_chunks_window(pcms, prompt)
        c.set_graph(False)
        w2, _ = c.run_chunks_window(pcms, prompt)
        c.set_graph(True)
        for a, b in zip(w1, w2):
            assert_same(a, b)
    finally:
        c.close()


def test_argument_and_bounds_errors():
    m, c = context("micro.en-sc", 2, fresh=True)
    L = capi.lib()
    pcm = synth.synth_pcm(0)
    ptrs = (C.POINTER(C.c_float) * 2)(capi._f(pcm), capi._f(pcm))
    ns = np.array([pcm.size, pcm.size], np.int32)
    neg = np.array([pcm.size, -1], np.int32)
    pr = np.array(m.prompt_init(), np.int32)
    n_max = m.n_text_ctx // 2 - 4
    toks = (capi.TokenData * (2 * n_max))()
    res = (capi.WindowResult * 2)()
    prm = capi.WindowParams(0, 0)
    i = capi._i

    def call(ctx=c.h, p=ptrs, n=i(ns), batch=2, prompt=i(pr), n_prompt=pr.size, params=C.byref(prm), out=toks, cap=n_max, results=res):
        before = L.wsp_launch_count()
        rc = L.wsp_run_chunks_window(ctx, p, n, batch, prompt, n_prompt, params, out, cap, results, None)
        assert L.wsp_launch_count() == before, "nothing may be launched before the arguments are checked"
        return rc

    try:
        assert call(ctx=None) == E_POINTER
        assert call(params=None) == E_POINTER
        assert call(results=None) == E_POINTER
        assert call(n=None) == E_POINTER
        assert call(n=i(neg)) == E_INVALIDARG
        assert call(batch=0) == E_BOUNDS
        assert call(batch=3) == E_BOUNDS
        assert call(prompt=None) == E_INVALIDARG
        assert call(n_prompt=0) == E_INVALIDARG
        assert call(cap=n_max - 1) == E_BOUNDS
        assert call(p=None) == E_INVALIDARG               # resident form: no PCM uploaded to the slots yet
        # tokens_out may be NULL
        rc = L.wsp_run_chunks_window(c.h, ptrs, i(ns), 2, i(pr), pr.size, C.byref(prm), None, n_max, res, None)
        assert rc == 0 and all(1 <= r.n_sampled <= n_max for r in res)
    finally:
        c.close()
