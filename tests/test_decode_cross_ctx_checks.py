"""Would tests/test_gpu_decode_cross_ctx.py notice the mistakes the decoder's cross attention invites along audio_ctx?  (CPU)

The constants its boundary lists depend on are read from the kernel sources, and every T where a restated shape function changes
must lie in the run list of a case that runs its (CR, GS, reference threads).  decode_flow_kernel's cross attention is restated
in numpy in its own order (flow_cross_attn): K slots of CR rows scored in groups of GS slots in 16-row tiles, V rows chained in f16
round by round (RR rows of a part per slot, the slots of a round in group order), the parts summed in f32; kStreamScores' register
batches likewise (stream_cross_attn).  Unmutated both equal wn.pv_mad_f16 on wn.softmax_rows bit for bit.  Each mutation replaces
the cross attention of chunk 0's single-token steps in the GPU file's oracle (MutantDecoder, StepDecoder with that one step
replaced), decoded at the GPU
file's tokens and (T, threads) runs, and the GPU file's comparison against the unmutated oracle (every logit row, every self-KV
row) must fail.  Cross-K/V: rows [0, T) of one whisper_np.encode of a synthetic clip at the full 1500 positions.

Caught on micro.en-sc: the last partial K slot dropped, the group tail read as GS slots, a part's last round clipped at RR
(overlap), an empty part taking part 0's chain, dc from T - 1, and kStreamScores' refills one register batch ahead.  Not caught:
- the last slot scored as a full CR rows (the next head's rows): those rows only raise the running maximum the softmax subtracts,
  and the reference's softmax is shift-invariant up to the f16 rounding of its exponentials.  Largest deviation 0.49 of its
  tolerance at every trial (T = 129, 257, 1025, 1409 at 16 threads, 1153 at 1).

Against the six audio_ctx values of the reference fixtures (1499, 750, 129, 128, 100, 16 at 1, 4 and 16 threads), measured with the
same mutated oracle and this file's comparison of the logits alone (all of the vocabulary, where the fixtures hold a sample): every
caught mutation moves the logits there too (largest deviation over tolerance: drop 11.8, tail 105, overlap 455, empty 7.2, dc 5.9,
late 8.4), and "full" stays at 0.33.  So these seven are not what the fixture set misses; what it misses is the shapes: it never
runs 2, 3, 5 or 9 threads, a V round boundary other than 1 thread's at 129, a group of K slots (T > 1025), a kStreamScores batch
edge (385, 769, 1153) or T = 1500 itself, and it never looks at a self-KV row.
"""
import os
import re

import numpy as np
import pytest

from oracle import whisper_np as wn
from tests.test_batch_shapes_checks import FL_WARPS as NS_FL_WARPS
from tests.test_batch_shapes_checks import ncols, ring_slots
from tests.test_gpu_decode_cross_ctx import (ATTN_THREADS, ATTN_WARPS, FL_WARPS, K_BATCH, LARGE_CASES, LARGE_THREADS, MG_SMEM_A, MICRO_RUNS,
                                             MICRO_THREADS, STREAM_ROWS, T_MAX, WALK, WIDE_RUNS, WORST, changes, compare, empty_parts,
                                             part_geometry, part_shape, run_oracle, slot_shape, stream_shape)
from tests.test_gpu_decode_step_long_context import StepDecoder, chunk_tokens, pv_side_by_side, slot_rows
from whisper_b200 import synth

F16, F32 = np.float16, np.float32
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "whisper_b200", "csrc")


def source_int(fname, pattern):
    with open(os.path.join(CSRC, fname)) as f:
        m = re.search(pattern, f.read())
    assert m, (fname, pattern)
    return int(m.group(1))


# ---- constants and coverage ------------------------------------------------------------------------------------------------------
def test_constants_are_the_sources():
    assert source_int("ref_arith.cuh", r"constexpr int kKBatch = (\d+);") == K_BATCH
    assert source_int("ref_arith.cuh", r"constexpr int kAttnThreads = (\d+);") == ATTN_THREADS == ATTN_WARPS * 32
    assert re.search(r"kKStep = kAttnWarps \* 4;", open(os.path.join(CSRC, "ref_arith.cuh")).read())
    assert STREAM_ROWS == ATTN_WARPS * 4 * K_BATCH == 384
    assert source_int("decode_flow.cu", r"constexpr int FL_WARPS = (\d+);") == FL_WARPS == NS_FL_WARPS
    assert source_int("decode_mega.cu", r"constexpr int MG_SMEM_A = (\d+);") == MG_SMEM_A
    assert T_MAX * 128 == MG_SMEM_A          # the largest audio_ctx exactly fills mode 1's V tile


def gs_of(d, B):
    return min(FL_WARPS, ring_slots(d, ncols(B)))


def test_runs_cover_every_boundary():
    """every T where the K side, modes 1 / 0 or the V side of a run thread count changes shape is run, with T - 1, at that
    (CR, GS, threads); case C at large-sc's CR 160 and both its group sizes"""
    assert slot_rows(128) == 128 and slot_rows(1280) == 160
    assert gs_of(128, 3) == gs_of(128, 16) == 8 and gs_of(1280, 1) == 8 and gs_of(1280, 9) == 7
    for T in changes(lambda T: slot_shape(T, 128, 8)) | changes(stream_shape) | {1, T_MAX}:
        for t in (T - 1, T):
            if t >= 1:
                assert {1, 16} <= set(MICRO_RUNS[t]), t
    for parts in MICRO_THREADS:
        for T in changes(lambda T: part_shape(T, 128, parts)) | set(range(1, parts + 1)):
            for t in (T - 1, T):
                if t >= 1:
                    assert parts in MICRO_RUNS[t], (parts, t)
    # the values named in the file's table
    first_round = {p: min(T for T in range(1, T_MAX + 1) if part_shape(T, 128, p)[0] > 1) for p in (1, 2, 5, 9, 3, 16)}
    assert first_round == {1: 129, 2: 257, 5: 321, 9: 379, 3: 385, 16: 513}
    assert [part_geometry(p, 128)[2] for p in (1, 5, 9, 16)] == [128, 64, 42, 32]
    assert empty_parts(17, 16) == 7 and min(T for T in range(17, 300) if empty_parts(T, 16)) == 17
    assert 8 * 128 + 1 in MICRO_RUNS and 1025 in changes(lambda T: slot_shape(T, 128, 8))
    # large-sc
    for B, gs in ((1, 8), (9, 7)):
        run = {(T, t) for b, g, T, t in LARGE_CASES if b == B and g == gs}
        for T in changes(lambda T: slot_shape(T, 160, gs)):
            assert (T, 1) in run, (B, T)
        for T in (160, 161, 320, 321, gs * 160, gs * 160 + 1, 1280, 1281, T_MAX):
            assert (T, 16) in run, (B, T)
        for parts in LARGE_THREADS:
            for T in changes(lambda T: part_shape(T, 160, parts)[0]):
                assert (T, parts) in run, (B, parts, T)
    assert {T for T, _ in WIDE_RUNS} == {1, 17, 129, 1025, 1153, 1500} and set(WALK) == {1, 17, 1025, 1500}


# ---- the restatements -------------------------------------------------------------------------------------------------------------
def chain(y, v, p):
    """one step of the reference's f16 V^T*P chain: y = f16(fma(v, p, y))"""
    acc = v.astype(np.float64) * p.astype(np.float64)
    acc += y
    return acc.astype(F32).astype(F16)


def softmax_at(S, mx):
    """wn.softmax_rows with the running maximum mx of the scores the kernel wrote (their true maximum, unmutated)"""
    with np.errstate(invalid="ignore", over="ignore"):
        e = np.exp(wn.r16(S - mx[:, None]).astype(np.float64)).astype(F16).astype(F32)
    e = np.where(np.isneginf(S), 0.0, e).astype(F32)
    s = e.astype(np.float64).sum(-1, keepdims=True)
    with np.errstate(divide="ignore"):
        return (e * (1.0 / s).astype(F32)).astype(F32)


def sum_parts(y, T, dc, mut):
    parts = y.shape[0]
    if mut == "empty":                      # a part without keys takes part 0's chain
        y = np.array([y[0] if pp * dc >= T else y[pp] for pp in range(parts)])
    out = y[0].astype(F32)
    for pp in range(1, parts):
        out = (out + y[pp].astype(F32)).astype(F32)
    return out[:, None, :]


def flow_cross_attn(q, K, V, parts, cr, gs, mut=None, K_next=None):
    """decode_flow_kernel's cross attention of one query: q [H][1][64], K / V [H][T][64] -> [H][1][64].  mut names a mistake;
    K_next [H][>= CR][64]: the rows that follow each head's in memory (mutation "full")."""
    H, T, _ = K.shape
    nkc = -(-T // cr)
    S = np.einsum("hqd,hkd->hqk", q, K).astype(F32)[:, 0]
    sp = np.full((H, T), -np.inf, F32)
    mx = np.full(H, -np.inf, F32)
    groups = [(c0, min(gs, nkc - c0)) for c0 in range(0, nkc, gs)] if nkc > 1 else [(0, 1)]
    for c0, ng in groups:
        for ci in range(c0, c0 + ng):
            r0, n = ci * cr, min(cr, T - ci * cr)
            if mut == "drop" and nkc > 1 and ci == nkc - 1 and n < cr:      # the last, partial slot is not scored
                continue
            for tb in range(0, n, 16):                                          # 16-row tiles, the last one masked at n
                rows = slice(r0 + tb, r0 + min(tb + 16, n))
                sp[:, rows] = S[:, rows]
                mx = np.maximum(mx, S[:, rows].max(1))
            if mut == "full" and ci == nkc - 1 and n < cr:                     # scored as CR rows: the next head's rows too
                extra = np.einsum("hqd,hkd->hqk", q, K_next[:, :cr - n]).astype(F32)[:, 0]
                mx = np.maximum(mx, extra.max(1))
    P = softmax_at(sp, mx)
    ng_, pg, rr = part_geometry(parts, cr)
    dc = -(-((T - 1) if mut == "dc" else T) // parts)
    rounds = -(-dc // rr)

    def clip(pp, i):
        j0 = pp * dc + i * rr
        j1 = min(j0 + rr, T if mut == "overlap" else min((pp + 1) * dc, T))
        return j0, max(0, j1 - j0) if pp < parts else 0

    def slot(i, q_):
        """the producer's slot of group q_ in round i: {offset in the slot: V row}"""
        out = {}
        for k in range(pg):
            j0, n = clip(q_ * pg + k, i)
            out.update({k * rr + r: j0 + r for r in range(n)})
        return out

    seq = [(i, q_) for i in range(rounds) for q_ in range(ng_)]
    late = gs - groups[-1][1] if mut == "tail" and nkc > 1 else 0      # the tail group releases GS slots: V slots read late
    y = np.zeros((parts, H, 64), F16)
    zero = np.zeros((H, 64), F32)
    for s, (i, q_) in enumerate(seq):
        content = slot(*seq[s + late]) if s + late < len(seq) else {}
        for k in range(pg):
            pp = q_ * pg + k
            j0, n = clip(pp, i)
            for r in range(n):
                row = content.get(k * rr + r)
                y[pp] = chain(y[pp], V[:, row] if row is not None else zero, P[:, j0 + r, None])
    return sum_parts(y, T, dc, mut)


def stream_cross_attn(q, K, V, parts, mut=None):
    """modes 1 / 0: kStreamScores in register batches of STREAM_ROWS rows, softmaxRow, pvSplitF16.  mut "late": every refill loads
    one batch ahead, so batch b >= 1 scores the rows of batch b + 1 (zeros past T)."""
    H, T, _ = K.shape
    S = np.empty((H, T), F32)
    for b0 in range(0, T, STREAM_ROWS):
        rows = np.arange(b0, min(b0 + STREAM_ROWS, T))
        src = rows + STREAM_ROWS if (mut == "late" and b0 > 0) else rows
        Kb = np.where((src < T)[None, :, None], K[:, np.minimum(src, T - 1)], 0.0).astype(F32)
        S[:, rows] = np.einsum("hqd,hkd->hqk", q, Kb).astype(F32)[:, 0]
    return wn.pv_mad_f16(wn.softmax_rows(S[:, None, :]), V, parts)


def oracle_attn(q, K, V, parts):
    return wn.pv_mad_f16(wn.softmax_rows(np.einsum("hqd,hkd->hqk", q, K).astype(F32)), V, parts)


def random_qkv(T, seed):
    rng = np.random.default_rng(seed)
    q = wn.r16(rng.standard_normal((2, 1, 64)) * 0.6)
    K, V = (wn.r16(rng.standard_normal((2, T, 64)) * s) for s in (0.6, 1.0))
    return q, K, V


def test_restatements_are_the_oracle():
    """unmutated, at every (T, threads) of case A and of case B's runs, bit for bit"""
    pairs = sorted({(T, t) for T, ts in MICRO_RUNS.items() for t in ts} | set(WIDE_RUNS))
    for T, t in pairs:
        q, K, V = random_qkv(T, T * 31 + t)
        want = oracle_attn(q, K, V, t)
        assert np.array_equal(flow_cross_attn(q, K, V, t, 128, 8), want), (T, t)
        if t in (1, 16):
            assert np.array_equal(stream_cross_attn(q, K, V, t), want), (T, t)
    for T in (1, 160, 161, 1121, 1281, 1500):         # CR 160 at both group sizes
        q, K, V = random_qkv(T, T)
        for gs in (7, 8):
            assert np.array_equal(flow_cross_attn(q, K, V, 5, 160, gs), oracle_attn(q, K, V, 5)), (T, gs)


# ---- mutations ----------------------------------------------------------------------------------------------------------------------
MUTATIONS = {
    "drop": "the last partial K slot is not scored",
    "tail": "the group tail is read as GS slots, so the V slots are read that many slots late",
    "overlap": "a part's last round is clipped at RR instead of at the part's end",
    "empty": "a part without keys takes part 0's chain",
    "dc": "dc is computed from T - 1",
    "late": "kStreamScores' refills load one register batch ahead (modes 1 and 0)",
}
# below the f16 resolution of the comparison (see the module's docstring); flow_cross_attn keeps it for that record
UNCAUGHT = {"full": "the last slot is scored as a full CR rows, reading the next head's rows"}
# (T, threads) of case A in the order they are tried: the shapes where each mistake is largest first
TRIALS = {
    "drop": [(1089, 16), (193, 1), (1473, 16)],
    "tail": [(257, 16), (1089, 1), (1473, 16)],
    "overlap": [(379, 9), (385, 3), (1135, 9)],
    "empty": [(17, 16), (2, 16), (46, 16)],
    "dc": [(1, 1), (17, 16), (1025, 16)],
    "late": [(1500, 16), (769, 1)],
}
CROSS_SEED = 70
_cache = {}


def model():
    """micro.en-sc's NpModel and the cross-K/V of one clip at all 1500 positions"""
    if "m" not in _cache:
        m = wn.NpModel(synth.model_path("micro.en-sc"))
        _, ck, cv = wn.encode(m, wn.log_mel(synth.synth_pcm(CROSS_SEED), m.filters))
        _cache["m"] = (m, ck, cv)
    return _cache["m"]


class MutantDecoder(StepDecoder):
    """StepDecoder whose single-token calls take their cross attention from cross_attn(il, Qh [H][1][64], Kh, Vh [H][T][64]) ->
    [H][1][64]; multi-token calls are StepDecoder's own.  With the unmutated restatement it is StepDecoder bit for bit
    (test_mutant_decoder_unmutated_is_the_oracle)."""

    def __init__(self, m, cross_k, cross_v, pv_threads, cross_attn):
        super().__init__(m, cross_k, cross_v, pv_threads)
        self.cross_attn = cross_attn

    def decode(self, tokens, n_past):
        if len(tokens) != 1:
            return super().decode(tokens, n_past)
        m, th = self.m, self.pv_threads
        d, H = m.n_text_state, m.n_text_head
        s = F32(np.power(64.0, -0.25))
        te = m["decoder.token_embedding.weight"]
        x = te[np.asarray(tokens)] + m["decoder.positional_embedding"][n_past:n_past + 1]
        nk, Tk = n_past + 1, self.ck.shape[1]
        for il in range(m.n_text_layer):
            p = "decoder.blocks.%d." % il
            cur = wn.norm(x, m[p + "attn_ln.weight"], m[p + "attn_ln.bias"])
            Q = (wn.mul_mat(m[p + "attn.query.weight"], cur) + m[p + "attn.query.bias"]) * s
            self.k[il, n_past] = wn.r16(wn.mul_mat(m[p + "attn.key.weight"], cur) * s)[0]
            self.v[il, n_past] = wn.r16(wn.mul_mat(m[p + "attn.value.weight"], cur) + m[p + "attn.value.bias"])[0]
            Qh = wn.r16(Q).reshape(1, H, 64).transpose(1, 0, 2)
            Kh = self.k[il, :nk].reshape(nk, H, 64).transpose(1, 0, 2)
            Vh = self.v[il, :nk].reshape(nk, H, 64).transpose(1, 0, 2)
            A = pv_side_by_side(wn.softmax_rows(np.einsum("hqd,hkd->hqk", Qh, Kh).astype(F32)), Vh, th)   # one query: no mask
            x = wn.mul_mat(m[p + "attn.out.weight"], A.transpose(1, 0, 2).reshape(1, d)) + m[p + "attn.out.bias"] + x
            cur = wn.norm(x, m[p + "cross_attn_ln.weight"], m[p + "cross_attn_ln.bias"])
            Q = (wn.mul_mat(m[p + "cross_attn.query.weight"], cur) + m[p + "cross_attn.query.bias"]) * s
            Qh = wn.r16(Q).reshape(1, H, 64).transpose(1, 0, 2)
            A = self.cross_attn(il, Qh, *(a[il].reshape(Tk, H, 64).transpose(1, 0, 2) for a in (self.ck, self.cv)))
            x = wn.mul_mat(m[p + "cross_attn.out.weight"], A.transpose(1, 0, 2).reshape(1, d)) + m[p + "cross_attn.out.bias"] + x
            cur = wn.norm(x, m[p + "mlp_ln.weight"], m[p + "mlp_ln.bias"])
            cur = wn.gelu(wn.mul_mat(m[p + "mlp.0.weight"], cur) + m[p + "mlp.0.bias"])
            x = wn.mul_mat(m[p + "mlp.2.weight"], cur) + m[p + "mlp.2.bias"] + x
        return wn.mul_mat(te, wn.norm(x, m["decoder.ln.weight"], m["decoder.ln.bias"]))


def mutant(mut):
    """run_oracle's decoder with mutation mut (None: the unmutated restatement) in chunk 0's single-token cross attention"""
    return lambda m, ck, cv, threads: MutantDecoder(m, ck, cv, threads, mutated_attn(mut, threads))


def mutated_attn(mut, threads):
    def attn(il, q, K, V):
        if mut == "late":
            return stream_cross_attn(q, K, V, threads, mut)
        return flow_cross_attn(q, K, V, threads, 128, 8, mut, np.roll(K, -1, axis=0))
    return attn


def deviation(mut, T, threads):
    """(failures of the GPU file's comparison of chunk 0 against the unmutated oracle, largest err / tol)"""
    m, ck, cv = model()
    cross = {0: (ck[:, :T].copy(), cv[:, :T].copy())}
    tokens = chunk_tokens(m.token_sot, m.token_eot, 3, 3000 + T)
    want = run_oracle(m, cross, tokens, threads, [0])
    got = run_oracle(m, cross, tokens, threads, [0], mutant(mut))
    bad = compare(got, want, "%s at T %d, %d threads" % (mut, T, threads), "mutation")
    return bad, WORST.pop("mutation")


@pytest.mark.parametrize("T,threads", [(1, 16), (129, 5), (1025, 9), (1500, 1)])
def test_mutant_decoder_unmutated_is_the_oracle(T, threads):
    """MutantDecoder with the unmutated flow restatement computes StepDecoder's logits and cache rows bit for bit"""
    m, ck, cv = model()
    cross = {0: (ck[:, :T].copy(), cv[:, :T].copy())}
    tokens = chunk_tokens(m.token_sot, m.token_eot, 1, 3000 + T)
    want = run_oracle(m, cross, tokens, threads, [0])[0]
    got = run_oracle(m, cross, tokens, threads, [0], mutant(None))[0]
    assert all(np.array_equal(got[k], want[k]) for k in ("logits", "k", "v"))


@pytest.mark.parametrize("mut", list(MUTATIONS))
def test_mutation_is_caught(mut):
    seen = []
    for T, t in TRIALS[mut]:
        assert t in MICRO_RUNS[T], (T, t)
        bad, worst = deviation(mut, T, t)
        if bad:
            return
        seen.append("T %d, %d threads: %.3g" % (T, t, worst))
    pytest.fail("%s: not caught (largest deviation over tolerance: %s)" % (MUTATIONS[mut], ", ".join(seen)))
