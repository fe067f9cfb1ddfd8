"""The chunk path at the decoder widths and batch sizes the API accepts, on an H100.

A model loads if its decoder width is one the step kernels are instantiated for (128, 384, 512, 768, 1024, 1280), and a context
takes any max_batch from 1 to 256.  The step kernels work on 8 chunk columns up to B = 8 and on two n-tiles of 8 (ncols = 16) up
to B = 16; decode_flow_kernel's weight / K-V ring then has NS slots (Cfg<D>::SLOT bytes each, smemLayout / ringSlots):

    D                      128  384  512  768  1024  1280
    NS, B <= 8 (ncols 8)    12   12   12   12    11     9
    NS, B >  8 (ncols 16)   12   11   11   10    10     7

large at B > 8 is the one shape with NS < FL_WARPS = 8: its cross attention scores K slots in groups of GS = 7, so 1500 keys (10
slots of 160 rows) run as groups of 7 + 3 and audio_ctx 1121 (7 full slots + 1 row) as 7 + 1; at B = 1 it keeps GS = 8 (8 + 2).
Past 16 chunks neither step kernel takes the batch, and every single-token step runs the per-op kernels.

1. Step kernels at every width and both column tiles (test_step_kernels_at_batch_shape): B distinct clips, one teacher-forced prompt
   pass of PROMPT_N = 5 tokens per chunk (chunk b fills per-op columns 5b .. 5b + 4, so chunks straddle the skinny GEMM's 16-column
   tiles), then N_STEPS single-token steps through the step graph, in step modes 2, 1 and 0.  Checked:
   - every step's logits and the self-KV rows of all NPOS positions in every layer against StepDecoder on the GPU's own cross-K/V of
     the slot (every slot for d <= 512; slots {0, 7, 8, B - 1}, the edges of each n-tile, for d >= 768); for d >= 1024 at the
     first thread count only, and modes 2 and 1 against mode 0 at the second, to keep numpy's time in bounds;
   - the launch count of every step, so a step kernel that declines a shape fails instead of running mode 0 under its label;
   - bit for bit, each chunk's logits and self-KV rows when the same chunks run reversed and rotated by 8 (columns 0..7 move into
     the second tile): a column's arithmetic does not depend on its position or its neighbours;
   - bit for bit, at B = 9, slots 9..15 of the 16-slot context (self-KV and cross-K of an earlier 16-chunk run) across the whole
     case; and, at every B < 16, the case's results in a context with max_batch == B.
2. The encoder stages at d = 768 (test_encoder_stages_d768): tests/test_gpu_encoder_stages.run_case on the random-weight small model.
3. Past 16 chunks, on micro.en-sc: run_chunks at B = 17, 33 and 256 against each clip run alone in mode 0 (tokens, last logits, log-mel,
   cross-K, bit for bit), the teacher-forced harness of part 1 at B = 17 and 33, and run_chunks_until_eot at B = 17.

The small model has random weights (there is no scripted small): every check of part 1 is teacher-forced, so that is enough.
tests/test_batch_shapes_checks.py shows on the CPU that the numpy comparison catches swapped slots, a wrong token and a neighbour's
cross-K/V.  The module prints the largest error / tolerance of every case at its end.
"""
import hashlib

import numpy as np
import pytest

from oracle import whisper_np as wn
from tests.test_gpu_decode_step_long_context import STEP_LAUNCHES, StepDecoder, chunk_tokens, kv_tol, logit_tol, restore
from tests.test_gpu_encoder_stages import Check, Weights, run_case
from whisper_b200 import capi, synth

pytestmark = pytest.mark.gpu

PROMPT_N = 5                 # tokens of the prompt pass: chunk b fills per-op columns [5b, 5b + 5)
N_STEPS = 6
CALLS = [(0, PROMPT_N)] + [(PROMPT_N + i, 1) for i in range(N_STEPS)]
NPOS = PROMPT_N + N_STEPS    # self-KV positions written
FLOW_MAX_B = 16              # the step kernels' largest batch (flowSupported, megaSupported)
SKINNY_COLS = 16             # columns per pass of the per-op skinny GEMM (kernels_decode.cu SK_COLS)
PCM_SEED = 500
NUMPY_ONCE_D = 1024          # from this width on, numpy runs at the first thread count of a case only
OUTSIDE_B = 9                # a case at this B first fills slots B..15 of its 16-slot context and checks they stay untouched

# (model, B, reference threads, audio_ctx)
CASES = ([("micro.en-sc", B, (1, 4, 16), 1500) for B in (1, 8, 9, 16)]
         + [(m, 16, (4, 16), 1500) for m in ("tiny.en-sc", "base.en-sc", "medium-sc")]
         + [("small", B, (4, 16), 1500) for B in (1, 9, 16)]
         + [("large-sc", 1, (4,), 1500)]
         + [("large-sc", B, (4, 16), n) for B in (9, 16) for n in (1500, 1121)])


def per_op_launches(m):
    """a host-token step on the per-op path: n_past / flag setters, embedding, 8 per layer, logits, the sampler's two"""
    return 8 * m.n_text_layer + 6


def checked_slots(d, B):
    """the slots compared with numpy: all up to d = 512, else the first and last column of each n-tile"""
    if d <= 512:
        return list(range(B))
    return sorted({b for b in (0, 7, 8, B - 1) if b < B})


def orders(B):
    """(name, perm): column j holds chunk perm[j]"""
    out = []
    if B > 1:
        out.append(("reversed", list(range(B))[::-1]))
    if B > 8:
        out.append(("rotated by 8", [(j - 8) % B for j in range(B)]))
    return out


# ---- engines, one model at a time (large's f32 NpModel takes gigabytes of host memory) ---------------------------------------
_open = {}
_np = {}
WORST = {}
ENC_WORST = {}


def close_all():
    for m, e in _open.values():
        e.close()
        m.close()
    _open.clear()
    _np.clear()


def open_engine(name):
    if name not in _open:
        close_all()
        m = capi.Model(synth.model_path(name))
        _open[name] = (m, capi.Engine(m, 0))
    return _open[name]


def np_model(name):
    if name not in _np:
        _np[name] = wn.NpModel(synth.model_path(name))
    return _np[name]


@pytest.fixture(scope="module", autouse=True)
def report_margins():
    yield
    close_all()
    if WORST:
        print("\nlargest error / tolerance against numpy per case: " + ", ".join("%s %.3g" % kv for kv in WORST.items()))
    if ENC_WORST:
        print("small encoder stages, largest error / tolerance: " + ", ".join("%s %.3g" % kv for kv in ENC_WORST.items()))


# ---- the two sides -------------------------------------------------------------------------------------------------------------
def encode(c, seeds, audio_ctx):
    c.set_audio_ctx(audio_ctx)
    for b, s in enumerate(seeds):
        c.pcm_to_mel(b, synth.synth_pcm(s))
    c.encode(len(seeds), [0] * len(seeds))


def cross_of(c, m, b):
    """slot b's cross K / V as [L][T][d] (head h in columns [64h, 64h + 64))"""
    L, H, d = m.n_text_layer, m.n_text_head, m.n_text_state
    return tuple(c.get_tensor(nm, b).reshape(L, H, -1, 64).transpose(0, 2, 1, 3).reshape(L, -1, d) for nm in ("cross_k", "cross_v"))


def kv_rows(c, m, name, b):
    """self_k / self_v of slot b at positions [0, NPOS): [L][NPOS][d]"""
    L, H = m.n_text_layer, m.n_text_head
    t = c.get_tensor(name, b).reshape(L, H, m.n_text_ctx, 64)[:, :, :NPOS]
    return t.transpose(0, 2, 1, 3).reshape(L, NPOS, H * 64)


def run_gpu(c, m, tokens, threads, mode):
    """CALLS on the GPU in one step mode: the prompt pass without sampling, then sampled single-token steps (the step graph).
    Returns per chunk dict(logits [N_STEPS][vocab], k, v [L][NPOS][d])."""
    B = len(tokens)
    lib = capi.lib()
    c.set_reference_threads(threads)
    c.set_step_mode(mode)
    want = STEP_LAUNCHES if mode != 0 and B <= FLOW_MAX_B else per_op_launches(m)
    logits = []
    for p, n in CALLS:
        toks = [t[p:p + n] for t in tokens]
        if n > 1:
            c.decode(toks, p, B, capi.DECODE_NO_SAMPLE)
            continue
        before = lib.wsp_launch_count()
        c.decode(toks, p, B, 0)
        launches = lib.wsp_launch_count() - before
        assert launches == want, "B = %d, mode %d, n_past %d: %d launches, expected %d" % (B, mode, p, launches, want)
        logits.append(c.logits(B))
    logits = np.stack(logits, 1)
    return [dict(logits=logits[b], k=kv_rows(c, m, "self_k", b), v=kv_rows(c, m, "self_v", b)) for b in range(B)]


def run_oracle(npm, cross, tokens, threads):
    """StepDecoder of every slot in `cross` ({slot: (cross_k, cross_v)}) fed CALLS with tokens[slot]: the same per chunk dicts"""
    out = {}
    for b, (ck, cv) in cross.items():
        dec = StepDecoder(npm, ck, cv, threads)
        rows = [dec.decode(tokens[b][p:p + n], p)[-1] for p, n in CALLS]
        out[b] = dict(logits=np.array(rows[1:]), k=dec.k[:, :NPOS].copy(), v=dec.v[:, :NPOS].copy())
    return out


def compare(got, want, what):
    """one chunk: every step's logits (logit_tol) and every self-KV row of every layer (kv_tol).  -> (failures, worst err / tol)"""
    bad, worst = [], 0.0
    for i in range(N_STEPS):
        w = want["logits"][i]
        err, tol = float(np.abs(got["logits"][i] - w).max()), logit_tol(w)
        worst = max(worst, err / tol if err == err else np.inf)
        if not err < tol:
            bad.append("%s: step %d: |logit error| %.4g >= %.4g" % (what, i, err, tol))
    for nm in ("k", "v"):
        for l in range(want[nm].shape[0]):
            for p in range(NPOS):
                w = want[nm][l, p]
                err, tol = float(np.abs(got[nm][l, p] - w).max()), kv_tol(w, l)
                worst = max(worst, err / tol if err == err else np.inf)
                if not err < tol:
                    bad.append("%s: self_%s layer %d position %d: |error| %.4g >= %.4g" % (what, nm, l, p, err, tol))
    return bad, worst


def same(a, b):
    return all(np.array_equal(a[k], b[k]) for k in ("logits", "k", "v"))


def outside_snapshot(c, slots):
    """digests of the self-KV and cross-K of `slots` (large's would take gigabytes of host memory as arrays)"""
    return {(b, nm): hashlib.sha256(c.get_tensor(nm, b).tobytes()).hexdigest() for b in slots for nm in ("self_k", "self_v", "cross_k")}


# ---- 1. step kernels at every width and both column tiles ----------------------------------------------------------------------
def case_id(case):
    model, B, threads, n = case
    return "%s-B%d-ctx%d" % (model, B, n)


@pytest.mark.parametrize("model,B,threads,audio_ctx", CASES, ids=[case_id(c) for c in CASES])
def test_step_kernels_at_batch_shape(model, B, threads, audio_ctx):
    m, e = open_engine(model)
    npm = np_model(model)
    d = m.n_text_state
    seeds = [PCM_SEED + b for b in range(B)]
    tokens = [t[:NPOS] for t in chunk_tokens(m.special["sot"], m.special["eot"], B, 3000 + B)]
    slots = checked_slots(d, B)
    bad, worst, first = [], 0.0, None
    c = capi.Context(e, FLOW_MAX_B)
    try:
        outside = None
        if B == OUTSIDE_B:
            # slots B..15 hold another 16-chunk run; nothing of this case may touch them
            encode(c, [PCM_SEED + 100 + b for b in range(FLOW_MAX_B)], audio_ctx)
            run_gpu(c, m, chunk_tokens(m.special["sot"], m.special["eot"], FLOW_MAX_B, 77), threads[0], 2)
            outside = outside_snapshot(c, range(B, FLOW_MAX_B))
        encode(c, seeds, audio_ctx)
        cross = {b: cross_of(c, m, b) for b in slots}
        for th in threads:
            got = {mode: run_gpu(c, m, tokens, th, mode) for mode in (2, 1, 0)}
            if first is None:
                first = got
            # past the first thread count the widest models check modes 2 and 1 against mode 0, to keep numpy's time in bounds
            numpy = th == threads[0] or d < NUMPY_ONCE_D
            want = run_oracle(npm, cross, tokens, th) if numpy else {b: got[0][b] for b in slots}
            for mode in (2, 1, 0) if numpy else (2, 1):
                for b in slots:
                    f, w = compare(got[mode][b], want[b], "%d threads, mode %d vs %s, slot %d" % (th, mode, "numpy" if numpy else "mode 0", b))
                    bad += f
                    worst = max(worst, w)
        for name, perm in orders(B):
            encode(c, [seeds[k] for k in perm], audio_ctx)
            for mode in (2, 1, 0):
                got = run_gpu(c, m, [tokens[k] for k in perm], threads[0], mode)
                for j, k in enumerate(perm):
                    if not same(got[j], first[mode][k]):
                        bad.append("%s, mode %d: chunk %d in column %d differs from its run in column %d" % (name, mode, k, j, k))
        if outside is not None:
            after = outside_snapshot(c, range(B, FLOW_MAX_B))
            bad += ["slot %d outside the batch: %s changed" % k for k in outside if after[k] != outside[k]]
    finally:
        restore(c)
        c.close()
    if B < FLOW_MAX_B:
        # the same case in a context of exactly B slots: its [L][maxB][...] layouts change strides, not results
        cb = capi.Context(e, B)
        try:
            encode(cb, seeds, audio_ctx)
            for mode in (2, 1, 0):
                got = run_gpu(cb, m, tokens, threads[0], mode)
                for b in range(B):
                    if not same(got[b], first[mode][b]):
                        bad.append("max_batch %d, mode %d: chunk %d differs from max_batch 16" % (B, mode, b))
        finally:
            restore(cb)
            cb.close()
    WORST[case_id((model, B, threads, audio_ctx))] = worst
    assert not bad, "%d failures, first: %s" % (len(bad), "\n".join(bad[:12]))


# ---- 2. the encoder stages at d = 768 --------------------------------------------------------------------------------------------
def test_encoder_stages_d768():
    """small (random weights): the first and last layer and decoder layers 0, L/2, L - 1's cross-K/V, one slot at n = 1500, then three
    at n = 129, each equal to itself encoded alone, as test_gpu_encoder_stages.test_stages_wide_models runs the other wide models"""
    m, e = open_engine("small")
    assert m.n_text_state == m.n_audio_state == 768
    W = Weights(synth.model_path("small"))
    c, single = capi.Context(e, 4), capi.Context(e, 1)
    saved = dict(Check.worst)
    Check.worst.clear()
    try:
        layers, cross = [0, W.Le - 1], [0, W.L // 2, W.L - 1]
        run_case(W, e, c, 1500, 1, layers, cross)
        run_case(W, e, c, 129, 3, layers, cross, single)
    finally:
        ENC_WORST.update(Check.worst)
        Check.worst.clear()
        Check.worst.update(saved)
        c.close()
        single.close()


# ---- 3. past 16 chunks: the per-op path --------------------------------------------------------------------------------------------
PER_OP_MODEL = "micro.en-sc"
N_DECODE = 12
_alone = {}


def alone(e, m, seed):
    """a clip run alone in a one-slot context in mode 0: tokens, last-step logits row, log-mel and cross-K"""
    if seed not in _alone:
        c = capi.Context(e, 1)
        try:
            c.set_step_mode(0)
            toks, _ = c.run_chunks([synth.synth_pcm(seed)], m.prompt_init(), N_DECODE)
            _alone[seed] = dict(tokens=toks[0], logits=c.logits(1)[0], mel=c.get_mel(0), cross_k=c.get_tensor("cross_k", 0))
        finally:
            restore(c)
            c.close()
    return _alone[seed]


@pytest.mark.parametrize("B", [17, 33, 256])
def test_run_chunks_past_16(B):
    """run_chunks through the step graph (mode 2, which declines B > 16): every checked chunk equals its clip run alone, bit for bit.
    The log-mel covers the second and later mel launches (16 chunks each) and their maxima at melMax + slot0 + b0."""
    m, e = open_engine(PER_OP_MODEL)
    c = capi.Context(e, B)
    try:
        toks, _ = c.run_chunks([synth.synth_pcm(PCM_SEED + b) for b in range(B)], m.prompt_init(), N_DECODE)
        last = c.logits(B)
        for b in (range(B) if B < 64 else (0, 15, 16, B - 1)):
            a = alone(e, m, PCM_SEED + b)
            assert np.array_equal(toks[b], a["tokens"]), "B = %d, chunk %d: tokens %s, alone %s" % (B, b, toks[b], a["tokens"])
            assert np.array_equal(last[b], a["logits"]), "B = %d, chunk %d: last logits differ" % (B, b)
            assert np.array_equal(c.get_mel(b), a["mel"]), "B = %d, chunk %d: log-mel differs" % (B, b)
            assert np.array_equal(c.get_tensor("cross_k", b), a["cross_k"]), "B = %d, chunk %d: cross_k differs" % (B, b)
    finally:
        c.close()


@pytest.mark.parametrize("B", [17, 33])
def test_teacher_forced_past_16(B):
    """part 1's prompt pass and steps at B > 16: every step costs the per-op path's launches in all three modes (which therefore
    agree bit for bit), and slots {0, 15, 16, B - 1} match StepDecoder"""
    m, e = open_engine(PER_OP_MODEL)
    npm = np_model(PER_OP_MODEL)
    tokens = [t[:NPOS] for t in chunk_tokens(m.special["sot"], m.special["eot"], B, 4000 + B)]
    slots = [0, 15, 16, B - 1]
    c = capi.Context(e, B)
    try:
        encode(c, [PCM_SEED + b for b in range(B)], 0)
        cross = {b: cross_of(c, m, b) for b in slots}
        got = {mode: run_gpu(c, m, tokens, 4, mode) for mode in (2, 1, 0)}
    finally:
        restore(c)
        c.close()
    want = run_oracle(npm, cross, tokens, 4)
    bad, worst = [], 0.0
    for b in slots:
        f, w = compare(got[0][b], want[b], "slot %d" % b)
        bad += f
        worst = max(worst, w)
        for mode in (2, 1):
            if not same(got[mode][b], got[0][b]):
                bad.append("mode %d differs from mode 0 at slot %d" % (mode, b))
    WORST["%s-B%d-per-op" % (PER_OP_MODEL, B)] = worst
    assert not bad, "%d failures, first: %s" % (len(bad), "\n".join(bad[:12]))


def test_until_eot_past_16():
    """run_chunks_until_eot at B = 17: each chunk's tokens, up to and including its EOT, are those of the chunk alone in mode 0"""
    B, max_decode = 17, 72
    m, e = open_engine(PER_OP_MODEL)
    pcms = [synth.synth_pcm(PCM_SEED + b) for b in range(B)]
    c, single = capi.Context(e, B), capi.Context(e, 1)
    try:
        outs, _ = c.run_chunks_until_eot(pcms, m.prompt_init(), max_decode)
        single.set_step_mode(0)
        for b in range(B):
            a, _ = single.run_chunks_until_eot([pcms[b]], m.prompt_init(), max_decode)
            assert np.array_equal(outs[b], a[0]), "chunk %d: %s, alone %s" % (b, outs[b], a[0])
    finally:
        restore(single)
        c.close()
        single.close()
    assert any(len(t) and t[-1] == m.special["eot"] for t in outs), "no chunk reached its EOT within %d tokens" % max_decode
