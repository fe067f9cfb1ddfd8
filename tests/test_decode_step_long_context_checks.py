"""Would tests/test_gpu_decode_step_long_context.py notice the mistakes the step kernel's long self-attention path invites?  (CPU)

The step's self attention is restated in numpy in decode_flow_kernel's own order of operations: K rows scored slot by slot (CR rows
per slot), then the V rows of each reference thread's key range dc = ceil(n / parts) chained in f16 round by round (RR rows of a
part per round), this step's own V row closing the chain of part pOwn = n_past / dc, and the parts summed in f32.  Unmutated it
equals the oracle's self attention bit for bit.  Each mutation below replaces the self attention of one chunk's single-token steps in
the GPU test's oracle decoder (StepDecoder's self_attn); the chunk is decoded at the GPU test's own positions and tokens
with the mutation, and the GPU test's comparisons (logits, and the self_k / self_v rows every step appends) must fail at least
once against the unmutated decoder.  Cross-K/V: the first CROSS_KEYS rows of whisper_np.encode's memories, to stay fast.

Caught on micro.en-sc (the scripted model the GPU test runs at all its thread counts): the last partial K slot dropped, K rows shifted
by one across a slot boundary, dc computed from n_past, the V rows of rounds >= 1 reused from round 0, and another chunk's cache
rows.  Two mutations are not caught on either model, because both only move one f16 rounding of the attention output, which the
kernel rounds to f16 anyway before the output projection:
- this step's own V row chained into part 0 instead of part pOwn: largest deviation 0.96 of its tolerance on micro.en-sc (9 reference
  threads; 0.49 on micro.en).  The row's product p v is still added once; only which f16 partial absorbs it changes.  At 1 thread
  pOwn is 0 and the mutation is the identity.
- this step's own V row added in f32 after the chains: largest deviation 0.89 of its tolerance on micro.en-sc (2 threads; 0.51 on
  micro.en), and exactly 0 at 1 thread, where the missing f16 rounding of the last chain step is the output's own f16 rounding.
"""
import numpy as np
import pytest

from oracle import whisper_np as wn
from tests.test_gpu_decode_step_long_context import (CALLS, MICRO_THREADS, N_TEXT_CTX, RUN_CASES, STEPS, WINDOWS, StepDecoder, boundaries,
                                                     chunk_tokens, kv_tol, logit_tol, pv_side_by_side, slot_rows, v_rounds)
from whisper_b200 import synth

F16, F32 = np.float16, np.float32
CROSS_KEYS = 64
_cache = {}


def model(name):
    """NpModel and the cross-K/V of a synthetic clip's first CROSS_KEYS audio positions"""
    if name not in _cache:
        m = wn.NpModel(synth.model_path(name))
        mel = wn.log_mel(synth.synth_pcm(70), m.filters)
        _, ck, cv = wn.encode(m, mel)
        _cache[name] = (m, ck[:, :CROSS_KEYS].copy(), cv[:, :CROSS_KEYS].copy())
    return _cache[name]


# ---- the step's self attention, restated ----------------------------------------------------------------------------------------
def chain(y, v, p):
    """one step of the reference's f16 V^T*P chain: y = f16(fma(v, p, y)) (ggml_vec_mad_f16)"""
    acc = v.astype(np.float64) * p.astype(np.float64)
    acc += y
    return acc.astype(F32).astype(F16)


def flow_self_attn(q, K, V, parts, cr, mut=None, K_other=None, V_other=None):
    """decode_flow_kernel's self attention of one query: q [H][1][64], K / V [H][n][64] (row n - 1 = this step's own) -> [H][1][64].
    mut names a mistake to make; K_other / V_other are another chunk's cache rows (mutation "slot")."""
    H, n, _ = K.shape
    n_old = n - 1
    Kc, Vc = (K_other, V_other) if mut == "slot" else (K, V)
    rows = np.arange(n_old)
    if mut == "shift":                      # slots after the first read their K rows one row early
        rows = np.where(rows >= cr, rows - 1, rows)
    S = np.einsum("hqd,hkd->hqk", q, Kc[:, rows]).astype(F32)
    if mut == "drop" and n_old > cr and n_old % cr:   # the last, partial slot is not scored
        S[:, :, n_old // cr * cr:] = -np.inf
    S = np.concatenate([S, np.einsum("hqd,hkd->hqk", q, K[:, n_old:]).astype(F32)], 2)
    P = wn.softmax_rows(S)[:, 0]            # [H][n]
    dc = -(-(n_old if mut == "dc" else n) // parts)
    rr = cr // -(-parts // min(parts, 4))
    y = np.zeros((parts, H, 64), F16)
    for pp in range(parts):
        for j in range(pp * dc, min((pp + 1) * dc, n_old)):
            i = (j - pp * dc) // rr           # the round that carries key j
            jv = j - i * rr if mut == "round0" else j
            y[pp] = chain(y[pp], Vc[:, jv], P[:, j, None])
    p_own = n_old // dc
    if mut == "own_part0":
        p_own = 0
    if p_own < parts and mut != "own_f32":
        y[p_own] = chain(y[p_own], V[:, n_old], P[:, n_old, None])
    out = y[0].astype(F32)
    for pp in range(1, parts):
        out = (out + y[pp].astype(F32)).astype(F32)
    if mut == "own_f32":                    # this step's own row added after the chains, in f32
        out = (out + V[:, n_old].astype(F32) * P[:, n_old, None]).astype(F32)
    return out[:, None, :]


MUTATIONS = {
    "drop": "the keys of the last partial K slot are dropped",
    "shift": "K rows shifted by one row across a slot boundary",
    "dc": "dc computed from n_past instead of n_past + 1",
    "round0": "the V rows of rounds >= 1 reused from round 0",
    "slot": "chunk 0's cache rows read from chunk 1's slot",
}
# below the f16 resolution of the attention output (see the module's docstring); flow_self_attn keeps them for that record
UNCAUGHT = {
    "own_part0": "this step's own V row chained into part 0 instead of part pOwn",
    "own_f32": "this step's own V row added in f32 after the chains",
}


def first_failure(name, threads, mut):
    """Decode chunks 0 and 1 of the GPU test's tokens through CALLS, chunk 0 also with the mutation; the first comparison of the GPU
    test that fails (text), or None.  Returns (failure, largest deviation of the logits and of the cache rows, each over its tolerance)."""
    m, ck, cv = model(name)
    cr = slot_rows(m.n_text_state)
    tokens = chunk_tokens(m.token_sot, m.token_eot, 2, 1000 + threads)
    ref = [StepDecoder(m, ck, cv, threads) for _ in range(2)]
    other = ref[1]

    def mutated(il, q, K, V):
        rows = [a[il, :K.shape[1]].reshape(-1, m.n_text_head, 64).transpose(1, 0, 2) for a in (other.k, other.v)]
        return flow_self_attn(q, K, V, threads, cr, mut, *rows)

    bad = StepDecoder(m, ck, cv, threads, mutated)
    worst = 0.0
    for p, n in CALLS:
        ref[1].decode(tokens[1][p:p + n], p)     # chunk 1 first: its rows [0, p] exist when chunk 0 reads them
        want = ref[0].decode(tokens[0][p:p + n], p)
        got = bad.decode(tokens[0][p:p + n], p)
        if n > 1:
            continue
        dev = [float(np.abs(got[-1] - want[-1]).max()) / logit_tol(want[-1])]
        for l in range(m.n_text_layer):
            for a, w in ((bad.k, ref[0].k), (bad.v, ref[0].v)):
                dev.append(float(np.abs(a[l, p] - w[l, p]).max()) / kv_tol(w[l, p], l))
        worst = max(worst, max(dev))
        if worst >= 1.0:
            return "n_past %d: deviation %.3g x its tolerance" % (p, worst), worst
    return None, worst


def test_side_by_side_chains_are_the_oracle():
    """the GPU test's V^T*P is wn.pv_mad_f16 bit for bit: masked (zero) probabilities, keys that leave the last thread short or
    without keys, several query rows"""
    rng = np.random.default_rng(5)
    for H, Nq, nk in ((2, 1, 1), (2, 1, 129), (2, 7, 300), (2, 3, 5), (20, 1, 100), (2, 2, 1500)):
        S = rng.standard_normal((H, Nq, nk)).astype(F32) * 3
        S[:, :, nk // 2:nk // 2 + (nk > 1)] = -np.inf       # never every key of a row: a causal row keeps its own
        P = wn.softmax_rows(S)
        V = wn.r16(rng.standard_normal((H, nk, 64)))
        for threads in (1, 2, 3, 5, 6, 9, 16):
            assert np.array_equal(pv_side_by_side(P, V, threads), wn.pv_mad_f16(P, V, threads)), (H, Nq, nk, threads)


@pytest.mark.parametrize("threads", [1, 5, 16])
def test_step_decoder_is_the_oracle(threads):
    """StepDecoder (the GPU test's oracle) computes NpDecoder's logits and cache rows bit for bit, for multi-token and single-token
    calls"""
    m, ck, cv = model("micro.en-sc")
    tokens = chunk_tokens(m.token_sot, m.token_eot, 1, 1000 + threads)[0]
    fast, slow = StepDecoder(m, ck, cv, threads), wn.NpDecoder(m, ck, cv, pv_threads=threads)
    for p, n in ((0, 20), (20, 1), (21, 1), (22, 9), (31, 1)):
        assert np.array_equal(fast.decode(tokens[p:p + n], p), slow.decode(tokens[p:p + n], p)[0]), (p, n)
    assert np.array_equal(fast.k, slow.k) and np.array_equal(fast.v, slow.v)


@pytest.mark.parametrize("threads", [1, 2, 3, 5, 16])
def test_restated_step_attention_is_the_oracle(threads):
    """unmutated, the restatement is the oracle's self attention bit for bit (the order of the chains is the reference's)"""
    rng = np.random.default_rng(threads)
    for n in (1, 129, 257, 385, 448):
        q = wn.r16(rng.standard_normal((2, 1, 64)))
        K, V = (wn.r16(rng.standard_normal((2, n, 64)) * s) for s in (0.5, 1.0))
        P = wn.softmax_rows(np.einsum("hqd,hkd->hqk", q, K).astype(F32))
        assert np.array_equal(flow_self_attn(q, K, V, threads, 128), wn.pv_mad_f16(P, V, threads)), n


@pytest.mark.parametrize("mut", list(MUTATIONS))
def test_mutation_is_caught(mut):
    """micro.en-sc at the GPU test's thread counts, in an order that reaches each mutation's case early"""
    seen = []
    for threads in MICRO_THREADS:
        found, worst = first_failure("micro.en-sc", threads, mut)
        if found:
            return
        seen.append("threads %d: %.3g" % (threads, worst))
    pytest.fail("%s: not caught (largest deviation over tolerance: %s)" % (MUTATIONS[mut], ", ".join(seen)))


# ---- the windows ----------------------------------------------------------------------------------------------------------------
# where the step's self attention changes shape, as (CR, reference threads, n_past); one row per row of DESIGN.md's table
TABLE = [
    ("K slots 1->2, 2->3, 3->4", [(128, None, 129), (128, None, 257), (128, None, 385), (160, None, 161), (160, None, 321)]),
    ("V rounds > 1, 1 thread", [(128, 1, 128), (128, 1, 256), (128, 1, 384), (160, 1, 160), (160, 1, 320)]),
    ("V rounds > 1, 2 / 3 threads", [(128, 2, 256), (128, 3, 384), (160, 2, 320)]),
    ("V rounds > 1, 5 / 6 threads", [(128, 5, 320), (128, 6, 384), (160, 5, 400)]),
    ("V rounds > 1, 9 threads", [(128, 9, 378)]),
    ("last position", [(128, None, 447), (160, None, 447)]),
]


def test_windows_cover_every_boundary():
    """CR follows decode_flow.cu's Cfg<D> for every model shape; every row of the table is a boundary of the formulas and lies inside
    a window for at least one (CR, threads) the GPU test runs; no fill between windows is a single token"""
    assert [slot_rows(d) for d in (128, 384, 512, 768, 1024, 1280)] == [128, 128, 128, 128, 128, 160]
    run = set(RUN_CASES)
    for what, cells in TABLE:
        covered = False
        for cr, parts, n_old in cells:
            assert any(lo <= n_old <= hi for lo, hi in WINDOWS), (what, n_old)
            if parts is None:
                assert n_old == N_TEXT_CTX - 1 or n_old in boundaries(cr, 1), (what, n_old)
                covered |= any(c == cr for c, _ in run)
            else:
                assert n_old in boundaries(cr, parts), (what, cr, parts, n_old)
                covered |= (cr, parts) in run
        assert covered, what
    assert all(n >= 2 for p, n in CALLS if n != 1) and all(n <= 256 for p, n in CALLS)
    assert [p for p, n in CALLS] == sorted(p for p, n in CALLS) and CALLS[-1] == (N_TEXT_CTX - 1, 1)
    assert sum(n for p, n in CALLS) == N_TEXT_CTX and set(STEPS) == {p for lo, hi in WINDOWS for p in range(lo, hi + 1)}
