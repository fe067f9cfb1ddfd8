"""Token-level timestamps of wsp_run_chunks_window on an H100: each chunk's signal energy computed on the device
(signal_energy_kernel) and whisper_full's token times and max_len wrapping per window (wsp_window_token_times).

Oracle: tests/golden/chunks_token_ts.npz (tests/golden/make_chunks_token_ts_golden.py, from oracle/_ref: the first window restated
over the reference's decode and samplers, its segments and token times those of the reference's own whisper_full).  Ids, tids,
results, segments, texts, token t0 / t1 and vlen must be identical.  The token times read the probabilities only through
`pt > thold_pt && ptsum > thold_ptsum`, so every result token's pt and ptsum must lie on the reference's side of both thresholds
(the fixture keeps the reference's values more than 5e-3 away from them).  The energy must be bit-identical to the reference's f32
sum.  The other checks compare the
GPU with itself: each chunk of a batch against the chunk run alone, speed-up against the Python restatement over the GPU's own
tokens and energy, and a context with the energy off (or switched off again) against one that never had it on.
"""
import ctypes as C
import os

import numpy as np
import pytest

from tests.golden import make_chunks_token_ts_golden as mk
from whisper_b200 import capi, synth

pytestmark = pytest.mark.gpu

E_INVALIDARG, E_POINTER, E_BOUNDS = -1, -2, -7

_cache = {}


def golden():
    if "g" not in _cache:
        _cache["g"] = np.load(os.path.join(os.path.dirname(__file__), "golden", "chunks_token_ts.npz"))
    return _cache["g"]


def context(model, batch, fresh=False):
    if ("engine", model) not in _cache:
        m = capi.Model(synth.model_path(model))
        _cache[("engine", model)] = (m, capi.Engine(m, 0))
    m, e = _cache[("engine", model)]
    if fresh:
        return m, capi.Context(e, batch)
    if (model, batch) not in _cache:
        c = capi.Context(e, batch)
        c.set_token_timestamps(1)
        _cache[(model, batch)] = c
    return m, _cache[(model, batch)]


def launches(f):
    L = capi.lib()
    before = L.wsp_launch_count()
    r = f()
    return r, int(L.wsp_launch_count() - before)


def case_inputs(name):
    g = golden()
    return [synth.synth_pcm(int(c), int(n)) for c, n in zip(g[name + "_chunks"], g[name + "_n_samples"])], g[name + "_prompt"].tolist()


def energy_ref(pcm):
    """the reference's sum: the 65 shifted |x| arrays added in order in f32, then / 65"""
    return mk.signal_energy(pcm)


def restated(m, o, energy, max_len, speed_up=False):
    """what wsp_window_token_times must return for one window, from the Python restatement: (segments, times)"""
    segs, times = mk.window_token_times(o["tokens"], o["result"], m.special["eot"], m.special["beg"], m.token_bytes, energy, max_len,
                                        speed_up=speed_up)
    return ([(s["t0"], s["t1"], s["i0"], s["i1"], s["text"]) for s in segs],
            [(t[0], t[1], float(np.float32(t[2]))) for t in times])


def got_of(o):
    n = o["result"]["n_tokens"]
    return ([(s["t0"], s["t1"], s["i0"], s["i1"], s["text"]) for s in o["segments"]],
            [(t["t0"], t["t1"], float(np.float32(t["vlen"]))) for t in o["tokens"][:n]])


# ---- the energy -----------------------------------------------------------------------------------------------------------------
ENERGY_LENGTHS = (0, 1, 64, 65, 12000, 480000)
# the batch calls need one mel frame (160 samples) per chunk; shorter clips go through pcm_to_mel and the kernel alone below
BATCH_LENGTHS = (160, 161, 12000, 16160, 480000, 200)


@pytest.mark.parametrize("form", ["host", "resident"])
def test_energy_bit_identical(form):
    """one window call over a batch of mixed lengths; every chunk's energy equals the reference's bit for bit"""
    pcms = [synth.synth_pcm(b, n) for b, n in enumerate(BATCH_LENGTHS)]
    m, c = context("micro.en-sc", len(pcms))
    if form == "host":
        c.run_chunks_window(pcms, m.prompt_init())
    else:
        for b, p in enumerate(pcms):
            c.upload_pcm(b, p)
        c.run_chunks_window(None, m.prompt_init(), batch=len(pcms))
    for b, p in enumerate(pcms):
        got = c.get_tensor("energy", b)
        assert got.size == p.size and got.tobytes() == energy_ref(p).tobytes(), "chunk %d (%d samples)" % (b, p.size)


def test_energy_kernel_alone():
    pcms = [synth.synth_pcm(b, n) if n else np.zeros(0, np.float32) for b, n in enumerate(ENERGY_LENGTHS)]
    got, _ms = capi.test_signal_energy(pcms)
    assert all(x.tobytes() == energy_ref(p).tobytes() for x, p in zip(got, pcms))


@pytest.mark.parametrize("n", ENERGY_LENGTHS)
def test_energy_of_pcm_to_mel(n):
    m, c = context("micro.en-sc", 2, fresh=True)
    try:
        c.set_token_timestamps(1)
        pcm = synth.synth_pcm(3, n) if n else np.zeros(0, np.float32)
        _, k = launches(lambda: c.pcm_to_mel(1, pcm))
        assert c.get_tensor("energy", 1).tobytes() == energy_ref(pcm).tobytes()
        c.set_token_timestamps(0)
        _, k0 = launches(lambda: c.pcm_to_mel(1, pcm))
        assert k == k0 + 1
    finally:
        c.close()


# ---- reference parity -----------------------------------------------------------------------------------------------------------
PARAMS = [(name, th, ml) for name, (_m, ths, _b) in mk.CASES.items() for th in ths for ml in mk.MAX_LENS]


@pytest.mark.parametrize("form", ["host", "resident"])
@pytest.mark.parametrize("name,th,ml", PARAMS)
def test_reference_parity(name, th, ml, form):
    model, _ths, batch = mk.CASES[name]
    m, c = context(model, batch)
    pcms, prompt = case_inputs(name)
    c.set_reference_threads(th)
    try:
        if form == "host":
            out, _ = c.run_chunks_window(pcms, prompt, token_times=dict(max_len=ml))
        else:
            for b, p in enumerate(pcms):
                c.upload_pcm(b, p)
            out, _ = c.run_chunks_window(None, prompt, batch=batch, token_times=dict(max_len=ml))
    finally:
        c.set_reference_threads(4)
    g, p = golden(), "%s_t%d_" % (name, th)
    q = "%sml%d_" % (p, ml)
    for b in range(batch):
        o, r = out[b], g[p + "result"][b]
        assert [o["result"][k] for k in ("n_sampled", "n_tokens", "seek_delta", "failed")] == r.tolist(), "chunk %d" % b
        n_s, n = int(r[0]), int(r[1])
        assert [(t["id"], t["tid"]) for t in o["tokens"]] == [tuple(x) for x in g[p + "tokens"][b, :n_s].tolist()], "chunk %d" % b
        got_p = np.array([[t["pt"], t["ptsum"]] for t in o["tokens"][:n]], np.float32).reshape(-1, 2)
        want_p = g[p + "probs"][b, :n, 1:]
        thold = np.array([mk.THOLD_PT, mk.THOLD_PTSUM], np.float32)
        assert np.array_equal(got_p > thold, want_p > thold), "chunk %d" % b
        segs = g[q + "segments"][b]
        k = int((segs[:, 0] >= 0).sum())
        want_s = [(int(s[0]), int(s[1]), int(s[2]), int(s[3]), str(t)) for s, t in zip(segs[:k], g[q + "texts"][b, :k])]
        want_t = [(int(a), int(z), float(v)) for (a, z), v in zip(g[q + "times"][b, :n].tolist(), g[q + "vlen"][b, :n].tolist())]
        assert got_of(o) == (want_s, want_t), "chunk %d" % b
        assert all(seg["tokens"] == o["tokens"][seg["i0"]:seg["i1"]] for seg in o["segments"])


# ---- the GPU against itself -----------------------------------------------------------------------------------------------------
GPU_ONLY = {"base_en_b12": ("base.en-sc", 12), "medium_b8": ("medium-sc", 8)}
GPU_ONLY_LENGTHS = (480000, 440000, 160000, 400000, 240000, 12000)


def inputs_of(name):
    if name in mk.CASES:
        return mk.CASES[name][0], case_inputs(name)
    model, batch = GPU_ONLY[name]
    m, _c = context(model, batch)
    return model, ([synth.synth_pcm(b, GPU_ONLY_LENGTHS[b % len(GPU_ONLY_LENGTHS)]) for b in range(batch)], m.prompt_init())


@pytest.mark.parametrize("name", list(mk.CASES) + list(GPU_ONLY))
def test_chunk_alone(name):
    """each chunk of a batch equals the same chunk run alone, and both equal the restatement over the GPU's tokens and energy"""
    model, (pcms, prompt) = inputs_of(name)
    m, c = context(model, len(pcms))
    m1, c1 = context(model, 1)
    for ml in mk.MAX_LENS:
        out, _ = c.run_chunks_window(pcms, prompt, token_times=dict(max_len=ml))
        energies = [c.get_tensor("energy", b) for b in range(len(pcms))]
        for b, pcm in enumerate(pcms):
            alone, _ = c1.run_chunks_window([pcm], prompt, token_times=dict(max_len=ml))
            assert [(t["id"], t["tid"]) for t in alone[0]["tokens"]] == [(t["id"], t["tid"]) for t in out[b]["tokens"]], (ml, b)
            assert got_of(alone[0]) == got_of(out[b]), (ml, b)
            assert energies[b].tobytes() == energy_ref(pcm).tobytes(), b
            assert got_of(out[b]) == restated(m, out[b], energies[b], ml), (ml, b)
        if name in GPU_ONLY:
            assert any(o["segments"] for o in out)


def test_speed_up():
    """segment times doubled, timestamp-token times not, the energy of the original samples: the restatement over the GPU's own
    tokens and energy"""
    pcms = [synth.synth_pcm(ch, n) for ch, n in ((0, 960000), (1, 960000), (2, 640000), (3, 320000), (5, 12000))]
    m, c = context("micro.en-sc", len(pcms), fresh=True)
    try:
        c.set_token_timestamps(1)
        c.set_speed_up(1)
        for ml in mk.MAX_LENS:
            out, _ = c.run_chunks_window(pcms, m.prompt_init(), token_times=dict(max_len=ml))
            for b, pcm in enumerate(pcms):
                energy = c.get_tensor("energy", b)
                assert energy.tobytes() == energy_ref(pcm).tobytes()
                assert got_of(out[b]) == restated(m, out[b], energy, ml, speed_up=True), (ml, b)
            assert any(len(o["segments"]) > 0 for o in out)
    finally:
        c.close()


# ---- the energy off ---------------------------------------------------------------------------------------------------------------
def test_off_state_unchanged():
    """with the energy off, after it was never on and after it was on and off again, wsp_run_chunks_window, wsp_run_chunks and
    wsp_run_chunks_until_eot are bit-identical with the same launches; with it on, a window call adds one launch"""
    name = "micro_en"
    model, batch = mk.CASES[name][0], mk.CASES[name][2]
    pcms, prompt = case_inputs(name)

    def calls(c):
        (w, _), nw = launches(lambda: c.run_chunks_window(pcms, prompt))
        (a, _), na = launches(lambda: c.run_chunks(pcms, prompt, 60))
        la = c.logits(batch)
        (e, _), ne = launches(lambda: c.run_chunks_until_eot(pcms, prompt, 100))
        return w, a, la, [t.tolist() for t in e], (nw, na, ne)

    m, never = context(model, batch, fresh=True)
    try:
        ref = calls(never)
    finally:
        never.close()
    m, c = context(model, batch, fresh=True)
    try:
        c.set_token_timestamps(1)
        (w_on, _), n_on = launches(lambda: c.run_chunks_window(pcms, prompt, token_times={}))
        assert n_on == ref[4][0] + 1
        for a, b in zip(w_on, ref[0]):
            assert [(t["id"], t["tid"], t["p"], t["pt"], t["ptsum"]) for t in a["tokens"]] == \
                [(t["id"], t["tid"], t["p"], t["pt"], t["ptsum"]) for t in b["tokens"]] and a["result"] == b["result"]
        c.set_token_timestamps(0)
        got = calls(c)
        assert got[0] == ref[0]
        assert np.array_equal(got[1], ref[1]) and np.array_equal(got[2], ref[2]) and got[3] == ref[3]
        assert got[4] == ref[4]
    finally:
        c.close()


# ---- errors -----------------------------------------------------------------------------------------------------------------------
def test_errors_launch_nothing():
    m, c = context("micro.en-sc", 2, fresh=True)
    L = capi.lib()
    pcms = [synth.synth_pcm(0, 160000), synth.synth_pcm(1, 480000)]
    prompt = m.prompt_init()
    prm = capi.TokenTimeParams(0.01, 0.01, 0)
    segs = (capi.Segment * 64)()
    n_segs = np.zeros(1, np.int32)
    i = capi._i

    def window_data(out, b):
        toks = (capi.TokenData * max(1, len(out[b]["tokens"])))(*[capi.TokenData(t["id"], t["tid"], t["p"], t["pt"], t["ptsum"]) for t in out[b]["tokens"]])
        r = out[b]["result"]
        return toks, capi.WindowResult(r["n_sampled"], r["n_tokens"], r["seek_delta"], r["failed"]), (capi.TokenTime * max(1, r["n_tokens"]))()

    def call(ctx, chunk, toks, res, times, params=C.byref(prm), seg=segs, cap=64, n=None):
        before = L.wsp_launch_count()
        rc = L.wsp_window_token_times(ctx, chunk, toks, res, 0, params, seg, cap, i(n_segs) if n is None else n, times)
        assert L.wsp_launch_count() == before
        return rc

    try:
        out, _ = c.run_chunks_window(pcms, prompt)                  # energy off: no window call with it yet
        toks, res, times = window_data(out, 1)
        assert call(c.h, 0, toks, C.byref(res), times) == E_INVALIDARG
        c.set_token_timestamps(1)
        assert call(c.h, 0, toks, C.byref(res), times) == E_INVALIDARG    # still: the last window call ran with it off
        out, _ = c.run_chunks_window(pcms, prompt)
        toks, res, times = window_data(out, 1)
        assert res.n_tokens > 2
        assert call(None, 1, toks, C.byref(res), times) == E_POINTER
        assert call(c.h, 1, None, C.byref(res), times) == E_POINTER
        assert call(c.h, 1, toks, None, times) == E_POINTER
        assert call(c.h, 1, toks, C.byref(res), None) == E_POINTER
        assert call(c.h, 1, toks, C.byref(res), times, params=None) == E_POINTER
        assert call(c.h, 1, toks, C.byref(res), times, seg=None) == E_POINTER
        assert call(c.h, 1, toks, C.byref(res), times, n=C.cast(None, C.POINTER(C.c_int32))) == E_POINTER
        assert call(c.h, 2, toks, C.byref(res), times) == E_BOUNDS
        assert call(c.h, -1, toks, C.byref(res), times) == E_BOUNDS
        assert call(c.h, 1, toks, C.byref(res), times) == 0
        n_all = int(n_segs[0])
        assert n_all >= 1
        n_segs[0] = -1
        assert call(c.h, 1, toks, C.byref(res), times, seg=None, cap=0) == E_BOUNDS and n_segs[0] == n_all
        # a window call with the energy off again makes the times unavailable
        c.set_token_timestamps(0)
        c.run_chunks_window(pcms, prompt)
        assert call(c.h, 1, toks, C.byref(res), times) == E_INVALIDARG
    finally:
        c.close()


def test_failed_and_short_windows_have_no_segments():
    g = golden()
    name = "micro_en"
    model, _ths, batch = mk.CASES[name]
    m, c = context(model, batch)
    pcms, prompt = case_inputs(name)
    out, _ = c.run_chunks_window(pcms, prompt, token_times=dict(max_len=12))
    kinds = [set(str(k).split(",")) for k in g[name + "_branches"]]
    seen = set()
    for b, o in enumerate(out):
        if o["result"]["failed"] or pcms[b].size // 160 <= 100:
            assert o["segments"] == [], b
            seen.add("failed" if o["result"]["failed"] else "short")
    assert seen == {"failed", "short"} and any("failed" in k for k in kinds)
