"""The decoder's cross attention at every audio_ctx where its kernels change shape, in all three step modes, on an H100.

Cross attention runs over the T = audio_ctx rows (1..1500) of the encoder's K/V memory of each (chunk, head).  Along T:

decode_flow_kernel (step mode 2, decode_flow.cu), CR = Cfg<D>::CR rows per ring slot (128; 160 at d = 1280):
  - T <= CR: one short slot, scoreRows<1> spread over the 8 warps.  T > CR: nKc = ceil(T / CR) slots scored in groups of
    GS = min(FL_WARPS, NS) slots, one warp per slot in 64-row strides (scoreRows<4>), the last slot's last 16-row tile masked.
  - V rows come in rounds = ceil(dc / RR) rounds, dc = ceil(T / parts) keys per reference thread (part), NG = min(parts, 4) groups
    of PG = ceil(parts / NG) parts, RR = CR / PG rows of each part per slot.  Parts with pp * dc >= T own no keys.
decode_mega_kernel (mode 1) and attn_decode_kernel (mode 0, also the prompt pass), ref_arith.cuh:
  - kStreamScores: 4-row warp groups (T <= 32 leaves warps without a row), register batches of kKStep * kKBatch = 384 rows;
    softmaxRow in 256-thread strides; pvSplitF16 clipping each part at min(part * dc, T).  Mode 1 stages the whole V tile in
    MG_SMEM_A = 192000 bytes: T = 1500 fills it exactly.

The T values are derived from those formulas (boundaries below), each with its neighbours T - 1 and T + 1:

  CR 128, GS 8 (micro.en-sc, any thread count)
    path, slots, groups      128/129, 256/257, 384/385, ..., 1408/1409 (k CR + 1 for every k), 1024/1025 (GS CR + 1)
    16- and 64-row tiles      16/17, 32/33, ..., 128/129 in the short slot; CR + 16/17, CR + 64/65, GS CR + 16/17, GS CR + 64/65,
                              11 CR + 16/17, 11 CR + 64/65 (the second slot, the first of the second group, the last slot)
    kStreamScores, softmax    5, 9, ..., 29 (warps with a key row), 384k + 1, 256k + 1, 1, 1500
  reference threads (parts) of the same model, V rounds > 1 and empty parts
    1: 129, 257, 385, ...   2: 257, 513, ...   3: 385, 769, 1153   4: 513, 1025   5: 321, 641, 961, 1281 (also 1..17)
    9: 379, 757, 1135 (RR 42; also 1..65)   16: 513, 1025 (RR 32; also 1..226, where parts 9..15 own no key at T = 17)
  CR 160 (large-sc), GS 8 at B = 1 and 7 at B = 9
    160/161, 320/321, 1120/1121/1122, 1280/1281, 1500; V rounds at 1 thread (RR 160) 161, 321, ..., 1441 (every k CR + 1), at
    5 threads (RR 80) 401, 801, 1201, at 16 threads (RR 40) 641, 1281

Case A runs every T of the first two blocks on micro.en-sc, B = 3 distinct clips, at 1 and 16 reference threads and at every
thread count whose own boundary it is: an encode at T, a 5-token prompt through the per-op pass (DECODE_ALL_LOGITS: the per-op
kernel's multi-query cross attention) and 4 sampled single-token steps through the step graph, in modes 2, 1 and 0.  Every prompt
row's logits, every step's logits and the self-KV rows of every position and layer are compared in full with
tests/test_gpu_decode_step_long_context.StepDecoder on the GPU's own cross-K/V, and modes 2 and 1 with mode 0: the rows of layers
>= 1 carry the previous layer's cross-attention output at f16 resolution, where a wrong clip shows long before it shows in the
logits.  Case B runs two column tiles (B = 16), case C large-sc (modes 2 and 1 against mode 0; B = 9 gives more (chunk, head)
units than SMs), case D one context walked through several T with the step graph replayed.
tests/test_decode_cross_ctx_checks.py restates the flow kernel's cross attention and shows which mistakes these comparisons catch.
"""
import numpy as np
import pytest

from tests.test_gpu_audio_ctx import open_model
from tests.test_gpu_decode_step_long_context import STEP_LAUNCHES, StepDecoder, chunk_tokens, kv_tol, logit_tol, restore, sm_count
from whisper_b200 import capi, synth

pytestmark = pytest.mark.gpu

# ---- the kernels' shape constants (tests/test_decode_cross_ctx_checks.py reads them from the sources) ------------------------
T_MAX = 1500                      # the model's n_audio_ctx
FL_WARPS = 8                      # decode_flow.cu: consumer warps, the largest group of K slots
K_BATCH = 12                      # ref_arith.cuh kKBatch: register loads in flight per lane
ATTN_WARPS = 8                    # ref_arith.cuh kAttnWarps
ATTN_THREADS = ATTN_WARPS * 32
STREAM_ROWS = ATTN_WARPS * 4 * K_BATCH   # key rows of one register batch of kStreamScores: 384
MG_SMEM_A = 192000                # decode_mega.cu: the V tile of mode 1, T rows of 128 bytes
PROMPT_N, N_STEPS = 5, 4
NPOS = PROMPT_N + N_STEPS
MICRO_THREADS = (1, 2, 3, 4, 5, 9, 16)


def part_geometry(parts, cr):
    """(NG, PG, RR) of decode_flow_kernel's V rounds"""
    ng = min(parts, 4)
    pg = -(-parts // ng)
    return ng, pg, cr // pg


def empty_parts(T, parts):
    dc = -(-T // parts)
    return sum(pp * dc >= T for pp in range(parts))


def slot_shape(T, cr, gs):
    """the flow kernel's K side at T keys: (short path, slots nKc, groups of GS slots)"""
    nkc = -(-T // cr)
    return T <= cr, nkc, -(-nkc // gs)


def stream_shape(T):
    """modes 1 and 0: (warps with a first key row, kStreamScores register batches, softmaxRow strides, V tile fits MG_SMEM_A)"""
    return min(-(-T // 4), ATTN_WARPS), -(-T // STREAM_ROWS), -(-T // ATTN_THREADS), T * 128 <= MG_SMEM_A


def part_shape(T, cr, parts):
    """the flow kernel's V side at T keys and `parts` reference threads: (V rounds, some part owns no key)"""
    rr = part_geometry(parts, cr)[2]
    return -(-(-(-T // parts)) // rr), empty_parts(T, parts) > 0


def changes(f):
    return {T for T in range(2, T_MAX + 1) if f(T) != f(T - 1)}


def shape_boundaries(cr, gs, stream=True):
    """T where the K side (or, with stream, modes 1 / 0) changes shape, the 16- and 64-row tile edges of the short slot, of the
    second slot, of the first slot of the second group and of the last slot, and T = 1, T_MAX"""
    out = {1, T_MAX} | changes(lambda T: slot_shape(T, cr, gs))
    if stream:
        out |= changes(stream_shape)
    for k in (1, gs, (T_MAX - 1) // cr):
        for r in (16, 64):
            out |= {k * cr + r, k * cr + r + 1}
    out |= {t for r in range(16, cr + 1, 16) for t in (r, r + 1)}
    return {T for T in out if T <= T_MAX}


def part_boundaries(cr, parts):
    """T where the V side changes shape for `parts` threads, and every T <= parts (parts without keys)"""
    return set(range(1, parts + 1)) | changes(lambda T: part_shape(T, cr, parts))


def near(ts):
    return {x for T in ts for x in (T - 1, T, T + 1) if 1 <= x <= T_MAX}


def micro_runs():
    """{T: reference threads} of case A"""
    runs = {T: {1, 16} for T in near(shape_boundaries(128, FL_WARPS))}
    for parts in MICRO_THREADS:
        for T in near(part_boundaries(128, parts)):
            runs.setdefault(T, {1, 16}).add(parts)
    return {T: tuple(sorted(v)) for T, v in sorted(runs.items())}


MICRO_RUNS = micro_runs()
WIDE_RUNS = [(1, 16), (17, 16), (129, 1), (1025, 9), (1153, 5), (1500, 16)]     # case B: (T, threads)
WIDE_SLOTS = (0, 7, 8, 15)
LARGE_THREADS = (1, 5, 16)


def large_runs(gs):
    """(T, threads) of case C at group size gs: the K side at 16 threads, the V rounds at their own thread count"""
    out = {(T, 16) for T in (1, 160, 161, 320, 321, gs * 160, gs * 160 + 1, gs * 160 + 2, 1120, 1121, 1280, 1281, 1500)}
    for parts in LARGE_THREADS:
        out |= {(T, parts) for T in changes(lambda T: part_shape(T, 160, parts)[0])}
    return sorted(out)


def large_cases():
    """(B, GS, T, threads); at 1 thread the V rounds change where the K slots do, k CR + 1"""
    return [(B, gs, T, t) for B, gs in ((1, 8), (9, 7)) for T, t in large_runs(gs)]


LARGE_CASES = large_cases()
WALK = (1500, 17, 1025, 17, 1500, 1)      # case D
WALK_THREADS = 5

WORST = {}


@pytest.fixture(scope="module", autouse=True)
def report_margins():
    yield
    if WORST:
        print("\nlargest error / tolerance per case: " + ", ".join("%s %.3g" % kv for kv in WORST.items()))


# ---- the two sides -----------------------------------------------------------------------------------------------------------
def encode(c, B, T, seed=70):
    c.set_audio_ctx(T)
    for b in range(B):
        c.pcm_to_mel(b, synth.synth_pcm(seed + b))
    c.encode(B, [0] * B)


def cross_of(c, m, b):
    """slot b's cross K / V as [L][T][d] (head h in columns [64h, 64h + 64))"""
    L, H, d = m.n_text_layer, m.n_text_head, m.n_text_state
    return tuple(c.get_tensor(nm, b).reshape(L, H, -1, 64).transpose(0, 2, 1, 3).reshape(L, -1, d) for nm in ("cross_k", "cross_v"))


def kv_rows(c, m, name, b):
    """self_k / self_v of slot b at positions [0, NPOS): [L][NPOS][d]"""
    L, H = m.n_text_layer, m.n_text_head
    return c.get_tensor(name, b).reshape(L, H, m.n_text_ctx, 64)[:, :, :NPOS].transpose(0, 2, 1, 3).reshape(L, NPOS, H * 64)


def run_gpu(c, m, tokens, threads, mode, kv_slots=None):
    """the prompt through the per-op pass (all logits), then N_STEPS sampled single-token steps through the step graph.
    -> {slot: dict(logits [NPOS][vocab], k, v [L][NPOS][d])}; k / v only for kv_slots (default: every slot)"""
    B = len(tokens)
    lib = capi.lib()
    c.set_reference_threads(threads)
    c.set_step_mode(mode)
    c.decode([t[:PROMPT_N] for t in tokens], 0, B, capi.DECODE_ALL_LOGITS)
    rows = [c.logits(B * PROMPT_N).reshape(B, PROMPT_N, -1)]
    for p in range(PROMPT_N, NPOS):
        before = lib.wsp_launch_count()
        c.decode([t[p:p + 1] for t in tokens], p, B, 0)
        launches = lib.wsp_launch_count() - before
        # a step kernel that declined this shape would leave the per-op path running in its place
        assert (launches == STEP_LAUNCHES) == (mode != 0), "mode %d, %d threads, n_past %d: %d launches" % (mode, threads, p, launches)
        rows.append(c.logits(B)[:, None])
    logits = np.concatenate(rows, 1)
    out = {}
    for b in range(B):
        out[b] = dict(logits=logits[b])
        if kv_slots is None or b in kv_slots:
            out[b].update(k=kv_rows(c, m, "self_k", b), v=kv_rows(c, m, "self_v", b))
    return out


def run_oracle(npm, cross, tokens, threads, slots, decoder=StepDecoder):
    """StepDecoder of every slot on its cross-K/V, fed the same calls: the same dicts.  decoder(npm, cross_k, cross_v, threads):
    another decoder in its place (the mutations of tests/test_decode_cross_ctx_checks.py)"""
    out = {}
    for b in slots:
        dec = decoder(npm, *cross[b], threads)
        rows = [dec.decode(tokens[b][:PROMPT_N], 0)] + [dec.decode(tokens[b][p:p + 1], p) for p in range(PROMPT_N, NPOS)]
        out[b] = dict(logits=np.concatenate(rows), k=dec.k[:, :NPOS].copy(), v=dec.v[:, :NPOS].copy())
    return out


def compare(got, want, what, case):
    """every logit row and every self-KV row (where `want` has them) of every slot in `want`; the worst err / tol goes to WORST[case]"""
    bad, worst = [], WORST.get(case, 0.0)
    for b, w in want.items():
        g = got[b]
        for i in range(NPOS):
            err, tol = float(np.abs(g["logits"][i] - w["logits"][i]).max()), logit_tol(w["logits"][i])
            worst = max(worst, err / tol if err == err else np.inf)
            if not err < tol:
                bad.append("%s: chunk %d position %d: |logit error| %.4g >= %.4g" % (what, b, i, err, tol))
        for nm in ("k", "v"):
            if nm not in w:
                continue
            for l in range(w[nm].shape[0]):
                for p in range(NPOS):
                    err, tol = float(np.abs(g[nm][l, p] - w[nm][l, p]).max()), kv_tol(w[nm][l, p], l)
                    worst = max(worst, err / tol if err == err else np.inf)
                    if not err < tol:
                        bad.append("%s: chunk %d self_%s layer %d position %d: |error| %.4g >= %.4g" % (what, b, nm, l, p, err, tol))
    WORST[case] = worst
    return bad


_np_models = {}


def np_model(name):
    if name not in _np_models:
        from oracle import whisper_np as wn
        _np_models[name] = wn.NpModel(synth.model_path(name))
    return _np_models[name]


def micro(B):
    m, e, c = open_model("micro.en-sc", B)
    return m, c


def check_against_numpy(m, c, B, T, threads, modes, case, slots=None, seed=0):
    """one encode at T, then every mode at every thread count: against numpy (slots) and modes 2 / 1 against mode 0"""
    slots = list(range(B)) if slots is None else list(slots)
    tokens = chunk_tokens(m.special["sot"], m.special["eot"], B, 3000 + T + seed)
    encode(c, B, T, 70 + seed)
    cross = {b: cross_of(c, m, b) for b in slots}
    assert cross[slots[0]][0].shape[1] == T
    bad = []
    for t in threads:
        got = {mode: run_gpu(c, m, tokens, t, mode) for mode in modes}
        want = run_oracle(np_model("micro.en-sc"), cross, tokens, t, slots)
        for mode in modes:
            bad += compare(got[mode], want, "T %d, %d threads, mode %d vs numpy" % (T, t, mode), case)
            if mode != 0 and 0 in got:
                bad += compare(got[mode], got[0], "T %d, %d threads, mode %d vs mode 0" % (T, t, mode), case + " vs mode 0")
    return bad


# ---- A: micro.en-sc at every boundary ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", list(MICRO_RUNS))
def test_cross_attention_against_numpy(T):
    B = 3
    m, c = micro(B)
    try:
        c.set_graph(True)
        bad = check_against_numpy(m, c, B, T, MICRO_RUNS[T], (2, 1, 0), "A micro B3")
    finally:
        restore(c)
    assert not bad, "%d failures, first: %s" % (len(bad), "\n".join(bad[:12]))


# ---- B: two column tiles -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T,threads", WIDE_RUNS)
def test_two_column_tiles_against_numpy(T, threads):
    """B = 16: the step kernels' second 8-column tile; numpy on the first and last slot of each tile"""
    B = 16
    m, c = micro(B)
    try:
        c.set_graph(True)
        bad = check_against_numpy(m, c, B, T, (threads,), (2, 1, 0), "B micro B16", WIDE_SLOTS)
    finally:
        restore(c)
    assert not bad, "%d failures, first: %s" % (len(bad), "\n".join(bad[:12]))


# ---- C: large-sc, CR = 160 -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,gs,T,threads", LARGE_CASES)
def test_large_step_kernels_against_per_op(B, gs, T, threads):
    """modes 2 and 1 against mode 0 (pinned against numpy by case A): every chunk's logits, and the self-KV rows of the last chunk
    (at B = 9 a (chunk, head) unit that shares its CTA with another)"""
    m, e, c = open_model("large-sc", 9)
    assert m.n_text_state == 1280
    assert (B * m.n_text_head > sm_count()) == (B == 9)
    tokens = chunk_tokens(m.special["sot"], m.special["eot"], B, 4000 + T)
    try:
        c.set_graph(True)
        encode(c, B, T, 90)
        got = {mode: run_gpu(c, m, tokens, threads, mode, kv_slots=(B - 1,)) for mode in (0, 2, 1)}
    finally:
        restore(c)
    bad = []
    for mode in (2, 1):
        bad += compare(got[mode], got[0], "large B %d, T %d, %d threads, mode %d vs mode 0" % (B, T, threads, mode), "C large B%d vs mode 0" % B)
    assert not bad, "%d failures, first: %s" % (len(bad), "\n".join(bad[:12]))


# ---- D: one context through several audio_ctx settings ---------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [2, 1, 0])
def test_one_context_through_settings(mode):
    """T walks 1500 -> 17 -> 1025 -> 17 -> 1500 -> 1 in one context with the step graph on: after a larger T the memory just past
    the new T holds real rows, so a step graph captured at another T, or a read past T, moves the result"""
    B = 3
    m, c = micro(B)
    bad = []
    try:
        c.set_graph(True)
        for i, T in enumerate(WALK):
            bad += check_against_numpy(m, c, B, T, (WALK_THREADS,), (mode,), "D walk", seed=i)
    finally:
        restore(c)
    assert not bad, "%d failures, first: %s" % (len(bad), "\n".join(bad[:12]))
