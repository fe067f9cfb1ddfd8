"""wsp_run_chunks_until_eot on an H100: each chunk of a batch decoded greedily up to its first EOT, the batch stopped soon after its
last chunk has ended.

Oracle: tests/golden/chunks_eot.npz (the reference's greedy loop per chunk until EOT or the cap, made by
tests/golden/make_chunks_eot_golden.py from oracle/_ref); tokens and output lengths must be identical.  The prefix, early-stop and
context-reuse checks compare the GPU with itself, bit for bit: the end-of-text log in the sampler must not change a token, and a
context must decode exactly as before once the call is over.
"""
import ctypes as C
import os

import numpy as np
import pytest

from tests.golden import make_chunks_eot_golden as mk
from whisper_b200 import capi, synth

pytestmark = pytest.mark.gpu

EOT_LAG = 8          # the host's block of steps (context.cu: kEotLag)
E_INVALIDARG, E_POINTER, E_BOUNDS = -1, -2, -7

_cache = {}


def golden():
    if "g" not in _cache:
        _cache["g"] = np.load(os.path.join(os.path.dirname(__file__), "golden", "chunks_eot.npz"))
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


# batches the GPU checks against itself only (prefix, early stop): the two-tile path of the decoder step (B in 9..16) and bench.py's
# model and batch; 30 s clips end on their script, the zero-padded ones end elsewhere or never
GPU_ONLY = {"base_en_b12": ("base.en-sc", 12), "medium_b8": ("medium-sc", 8)}
GPU_ONLY_LENGTHS = (480000, 440000, 420000, 400000)


def model_of(name):
    return mk.CASES[name][0] if name in mk.CASES else GPU_ONLY[name][0]


def batch_of(name):
    return mk.CASES[name][2] if name in mk.CASES else GPU_ONLY[name][1]


def case_inputs(name, rows=None):
    rows = range(batch_of(name)) if rows is None else rows
    if name in GPU_ONLY:
        m, _c = context(model_of(name), batch_of(name))
        return [synth.synth_pcm(b, GPU_ONLY_LENGTHS[b % len(GPU_ONLY_LENGTHS)]) for b in rows], np.array(m.prompt_init(), np.int32)
    g = golden()
    return [synth.synth_pcm(int(g[name + "_chunks"][b]), int(g[name + "_n_samples"][b])) for b in rows], g[name + "_prompt"]


def eot_of(name):
    m, _c = context(model_of(name), batch_of(name))
    return m.special["eot"]


def want(name, th, b):
    p = "%s_t%d_" % (name, th)
    return golden()[p + "tokens"][b, :int(golden()[p + "n_out"][b])]


def cut_at_eot(row, eot):
    hits = np.flatnonzero(row == eot)
    return row[:hits[0] + 1] if hits.size else row


def launches(f):
    L = capi.lib()
    before = L.wsp_launch_count()
    r = f()
    return r, int(L.wsp_launch_count() - before)


PARAMS = [(name, th) for name, (_m, ths, _b) in mk.CASES.items() for th in ths]


@pytest.mark.parametrize("form", ["host", "resident"])
@pytest.mark.parametrize("name,th", PARAMS)
def test_reference_parity(name, th, form):
    model, _ths, batch = mk.CASES[name]
    m, c = context(model, batch)
    pcms, prompt = case_inputs(name)
    c.set_reference_threads(th)
    try:
        if form == "host":
            got, st = c.run_chunks_until_eot(pcms, prompt, mk.CAP)
        else:
            for b, p in enumerate(pcms):
                c.upload_pcm(b, p)
            got, st = c.run_chunks_until_eot(None, prompt, mk.CAP, batch=batch)
    finally:
        c.set_reference_threads(4)
    assert len(got) == batch and st[2] > 0
    for b in range(batch):
        assert got[b].tolist() == want(name, th, b).tolist(), "chunk %d" % b


@pytest.mark.parametrize("name", list(mk.CASES) + list(GPU_ONLY))
def test_prefix_of_fixed_length_run(name):
    """the same batch through wsp_run_chunks(n_decode = max_decode), cut at each row's first EOT"""
    batch = batch_of(name)
    m, c = context(model_of(name), batch)
    pcms, prompt = case_inputs(name)
    eot = eot_of(name)
    full, _ = c.run_chunks(pcms, prompt, mk.CAP)
    got, _ = c.run_chunks_until_eot(pcms, prompt, mk.CAP)
    for b in range(batch):
        assert got[b].tolist() == cut_at_eot(full[b], eot).tolist(), "chunk %d" % b
    if name in GPU_ONLY:
        # the batch ends on the script and off it
        assert any(t[-1] == eot for t in got)


def steps_run(c, pcms, prompt, f):
    """decoder steps a call ran, from the launch count: wsp_run_chunks with n_decode = 1 and 2 give the fixed part and one step"""
    _, base = launches(lambda: c.run_chunks(pcms, prompt, 1))
    _, two = launches(lambda: c.run_chunks(pcms, prompt, 2))
    r, n = launches(f)
    per = two - base
    assert per > 0 and (n - base) % per == 0
    return r, 1 + (n - base) // per


@pytest.mark.parametrize("name", list(mk.CASES) + list(GPU_ONLY))
def test_early_stop(name):
    batch = batch_of(name)
    m, c = context(model_of(name), batch)
    eot = eot_of(name)
    pcms, prompt = case_inputs(name)
    # the whole batch: it stops at the cap when one of its chunks reaches it, else within 2 blocks of its last EOT
    (got, _), steps = steps_run(c, pcms, prompt, lambda: c.run_chunks_until_eot(pcms, prompt, mk.CAP))
    ends = np.array([len(t) if t[-1] == eot else 0 for t in got])
    if (ends == 0).any():
        assert steps == mk.CAP
    else:
        assert ends.max() <= steps <= min(mk.CAP, ends.max() + 2 * EOT_LAG + 1)
    if name in mk.CASES:
        assert ends.tolist() == golden()[name + "_t4_eot_step"].tolist()
    # only the chunks that end, under a cap far above their EOT steps: the batch stops within 2 blocks of its last EOT
    rows = [b for b in range(batch) if ends[b] > 0]
    assert rows
    pcms, prompt = case_inputs(name, rows)
    cap = 200
    (got, _), steps = steps_run(c, pcms, prompt, lambda: c.run_chunks_until_eot(pcms, prompt, cap))
    last = max(len(t) for t in got)
    assert [len(t) for t in got] == [int(ends[b]) for b in rows]
    assert last <= steps <= last + 2 * EOT_LAG + 1 and steps < cap
    # afterwards the context holds the state of the last step run: the same as a fixed-length run of that many steps
    lg = c.logits(len(rows))
    sk = c.get_tensor("self_k", len(rows) - 1)
    c.run_chunks(pcms, prompt, steps)
    assert np.array_equal(lg, c.logits(len(rows)))
    assert np.array_equal(sk, c.get_tensor("self_k", len(rows) - 1))


def test_context_reuse_is_untouched():
    """wsp_run_chunks before and after wsp_run_chunks_until_eot on one context decodes exactly as a fresh context does"""
    name = "micro_en"
    model, _ths, batch = mk.CASES[name]
    pcms, prompt = case_inputs(name)
    m, fresh = context(model, batch, fresh=True)
    try:
        ref_toks, _ = fresh.run_chunks(pcms, prompt, mk.CAP)
        ref_logits = fresh.logits(batch)
    finally:
        fresh.close()
    m, c = context(model, batch, fresh=True)
    try:
        before, _ = c.run_chunks(pcms, prompt, mk.CAP)
        assert np.array_equal(before, ref_toks) and np.array_equal(c.logits(batch), ref_logits)
        c.run_chunks_until_eot(pcms, prompt, mk.CAP)
        c.run_chunks_until_eot(pcms[1:], prompt, 40)
        after, _ = c.run_chunks(pcms, prompt, mk.CAP)
        assert np.array_equal(after, ref_toks) and np.array_equal(c.logits(batch), ref_logits)
        # the per-op path (no step graph) gives the same tokens
        c.set_graph(False)
        got, _ = c.run_chunks_until_eot(pcms, prompt, mk.CAP)
        c.set_graph(True)
        got2, _ = c.run_chunks_until_eot(pcms, prompt, mk.CAP)
        assert [t.tolist() for t in got] == [t.tolist() for t in got2]
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
    toks = np.zeros(2 * 448, np.int32)
    n_out = np.zeros(2, np.int32)
    i = capi._i

    def call(ctx=c.h, p=ptrs, n=i(ns), batch=2, prompt=i(pr), n_prompt=pr.size, max_decode=8, out=i(toks), nout=i(n_out)):
        before = L.wsp_launch_count()
        rc = L.wsp_run_chunks_until_eot(ctx, p, n, batch, prompt, n_prompt, max_decode, out, nout, None)
        assert L.wsp_launch_count() == before, "nothing may be launched before the arguments are checked"
        return rc

    try:
        assert call(ctx=None) == E_POINTER
        assert call(nout=None) == E_POINTER
        assert call(n=None) == E_POINTER
        assert call(n=i(neg)) == E_INVALIDARG
        assert call(batch=0) == E_BOUNDS
        assert call(batch=3) == E_BOUNDS
        assert call(prompt=None) == E_INVALIDARG
        assert call(n_prompt=0) == E_INVALIDARG
        assert call(max_decode=0) == E_BOUNDS
        assert call(max_decode=m.n_text_ctx - pr.size + 1) == E_BOUNDS
        assert call(p=None) == E_INVALIDARG               # resident form: no PCM uploaded to the slots yet
        # the largest max_decode is accepted; tokens_out may be NULL
        rc = L.wsp_run_chunks_until_eot(c.h, ptrs, i(ns), 2, i(pr), pr.size, m.n_text_ctx - pr.size, None, i(n_out), None)
        assert rc == 0 and (n_out >= 1).all() and (n_out <= m.n_text_ctx - pr.size).all()
    finally:
        c.close()
