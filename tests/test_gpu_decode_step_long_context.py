"""The single-token decoder step kernels deep into the 448-position text context, on an H100.

A step (N = 1, no all-logits request) runs decode_flow_kernel in step mode 2, decode_mega_kernel in mode 1 and the per-op kernels in
mode 0, replayed as a CUDA graph.  Self attention changes shape with the number of cached keys n_past: past CR rows the K rows of the
flow kernel come in several ring slots, and once a reference thread's key range dc = ceil((n_past + 1) / threads) exceeds RR rows
its V rows need several rounds.  The boundary windows below are derived from those formulas; the cache is filled up to each window
by one per-op call (at most 256 tokens, no sampling) and every position inside a window is one single-token step.

Oracle: oracle/whisper_np.NpDecoder on the GPU's own cross-K/V, one decoder per chunk, fed exactly the same calls (the reference
cuts its threads' key ranges from each call's n_past + N, so cache rows depend on how the calls were cut).  It runs as StepDecoder,
the same arithmetic with the reference threads' f16 chains advanced side by side and without the vocabulary softmax;
tests/test_decode_step_long_context_checks.py pins it to NpDecoder bit for bit.  At every step the
logits are compared, and so are the K/V rows that step appended to the self-KV cache in every layer and head: the rows of layers
>= 1 depend on the previous layer's self-attention output at f16 resolution, so a wrong output at one position shows in that
position's rows and not only, blurred, in the logits.  The large shapes, where numpy is too slow, compare modes 2 and 1 with
mode 0, whose per-op attention kernel tests/test_gpu_decoder_attention.py pins against numpy at 448 keys.
"""
import numpy as np
import pytest

from oracle import whisper_np as wn
from tests.test_gpu_audio_ctx import TOL_KV, TOL_LOGIT, open_model
from whisper_b200 import capi, synth

pytestmark = pytest.mark.gpu

N_TEXT_CTX = 448
HALF_WINDOW = 4          # steps on each side of a boundary
# reference threads of the numpy comparison on micro.en-sc: 3 covers the V rounds of 2 and 3 threads (n = 385 at CR 128; 2 threads
# second round at n = 257 coincides with 1 thread's third); 2 threads and the random-weight model are left out to keep the numpy
# oracle (about 20 s a case on 3 chunks x 1500 cross keys) inside the file's four-minute budget
MICRO_THREADS = (1, 3, 5, 6, 9, 16)
LARGE_THREADS = (1, 5, 16)
STEP_LAUNCHES = 5        # a step through the graph of a step kernel: n_past / flag setters + the kernel + the sampler's two


# ---- where the step kernel's self attention changes shape (decode_flow.cu, decode_flow_kernel) --------------------------------
def slot_rows(d):
    """Cfg<D>::CR: the K/V rows (128 bytes each) of one ring slot of max(8 (2 d + 64), 16384) bytes, a multiple of 8."""
    return (max(8 * (2 * d + 64), 16384) // 128) & ~7


def v_rounds(n, parts, cr):
    """Rounds of V rows for n keys: NG = min(parts, 4) groups own PG = ceil(parts / NG) parts each, a slot carries RR = CR / PG
    rows of each part, and part p owns dc = ceil(n / parts) keys."""
    ng = min(parts, 4)
    rr = cr // -(-parts // ng)
    return -(-(-(-n // parts)) // rr)


def boundaries(cr, parts):
    """n_past values where the step's self attention first needs one more K slot (of >= 2) or one more V round (of >= 2), and the
    last position."""
    out = {N_TEXT_CTX - 1}
    for n_old in range(2, N_TEXT_CTX):
        slots = -(-n_old // cr)
        if slots >= 2 and slots != -(-(n_old - 1) // cr):
            out.add(n_old)
        r = v_rounds(n_old + 1, parts, cr)
        if r >= 2 and r != v_rounds(n_old, parts, cr):
            out.add(n_old)
    return out


def windows(cases):
    """Merged [lo, hi] ranges of single-token n_past values around every boundary of (CR, threads) in `cases`; windows less than
    two positions apart are merged so that every fill between them is a multi-token (per-op) call."""
    spans = sorted((max(1, b - HALF_WINDOW), min(N_TEXT_CTX - 1, b + HALF_WINDOW)) for cr, parts in cases for b in boundaries(cr, parts))
    out = []
    for lo, hi in spans:
        if out and lo <= out[-1][1] + 2:
            out[-1][1] = max(out[-1][1], hi)
        else:
            out.append([lo, hi])
    return [tuple(w) for w in out]


RUN_CASES = [(128, t) for t in MICRO_THREADS] + [(160, t) for t in LARGE_THREADS]
WINDOWS = windows(RUN_CASES)


def schedule(wins=WINDOWS):
    """[(n_past, N)] of the decode calls: fills of at most 256 tokens up to each window, then one call per position in it."""
    calls, pos = [], 0
    for lo, hi in wins:
        while pos < lo:
            n = min(256, lo - pos)
            calls.append((pos, n))
            pos += n
        calls += [(p, 1) for p in range(lo, hi + 1)]
        pos = hi + 1
    return calls


CALLS = schedule()
STEPS = np.array([p for p, n in CALLS if n == 1])


def chunk_tokens(sot, eot, batch, seed):
    """a different random sequence of non-special tokens after sot for every chunk"""
    rng = np.random.default_rng(seed)
    return [[sot] + rng.integers(0, eot, N_TEXT_CTX - 1).tolist() for _ in range(batch)]


# ---- the oracle ----------------------------------------------------------------------------------------------------------------
F16, F32 = np.float16, np.float32


def pv_side_by_side(P, V, n_threads):
    """wn.pv_mad_f16 with the threads' chains advanced together: step j adds key ith*dc + j to chain ith.  Keys past nk are padded
    with P = V = 0, and f16(fma(0, 0, y)) = y leaves a chain as it is.  P [h][q][k], V [h][k][64] -> [h][q][64]."""
    H, Nq, nk = P.shape
    dc = -(-nk // n_threads)
    pad = n_threads * dc - nk
    Vp = np.concatenate([V.astype(np.float64), np.zeros((H, pad, V.shape[2]))], 1).reshape(H, n_threads, dc, V.shape[2])
    Pp = np.concatenate([P.astype(np.float64), np.zeros((H, Nq, pad))], 2).reshape(H, Nq, n_threads, dc)
    Vp = np.ascontiguousarray(Vp.transpose(2, 1, 0, 3))[:, :, :, None, :]     # [dc][thread][h][1][64]
    Pp = np.ascontiguousarray(Pp.transpose(3, 2, 0, 1))[..., None]            # [dc][thread][h][q][1]
    y = np.zeros((n_threads, H, Nq, V.shape[2]), F16)
    for j in range(dc):
        acc = Vp[j] * Pp[j]               # exact in float64, then one f32 rounding of the sum: the f32 fma
        acc += y
        y = acc.astype(F32).astype(F16)
    out = y[0].astype(F32)
    for ith in range(1, n_threads):
        out = (out + y[ith].astype(F32)).astype(F32)
    return out


class StepDecoder(wn.NpDecoder):
    """NpDecoder.decode (whisper.cpp:1508-1859) with pv_side_by_side for its V^T*P chains, logits only, and an optional self_attn(il,
    Qh [H][1][64], Kh, Vh [H][n_past + 1][64]) -> [H][1][64] in place of the self attention of single-token calls."""

    def __init__(self, m, cross_k, cross_v, pv_threads, self_attn=None):
        super().__init__(m, cross_k, cross_v, pv_threads)
        self.self_attn = self_attn

    def decode(self, tokens, n_past):
        m, th = self.m, self.pv_threads
        d, H = m.n_text_state, m.n_text_head
        N = len(tokens)
        s = F32(np.power(64.0, -0.25))
        te = m["decoder.token_embedding.weight"]
        x = te[np.asarray(tokens)] + m["decoder.positional_embedding"][n_past:n_past + N]
        for il in range(m.n_text_layer):
            p = "decoder.blocks.%d." % il
            cur = wn.norm(x, m[p + "attn_ln.weight"], m[p + "attn_ln.bias"])
            Q = (wn.mul_mat(m[p + "attn.query.weight"], cur) + m[p + "attn.query.bias"]) * s
            K = wn.mul_mat(m[p + "attn.key.weight"], cur) * s
            V = wn.mul_mat(m[p + "attn.value.weight"], cur) + m[p + "attn.value.bias"]
            self.k[il, n_past:n_past + N] = wn.r16(K)
            self.v[il, n_past:n_past + N] = wn.r16(V)
            nk = n_past + N
            Qh = wn.r16(Q).reshape(N, H, 64).transpose(1, 0, 2)
            Kh = self.k[il, :nk].reshape(nk, H, 64).transpose(1, 0, 2)
            Vh = self.v[il, :nk].reshape(nk, H, 64).transpose(1, 0, 2)
            if self.self_attn is not None and N == 1:
                A = self.self_attn(il, Qh, Kh, Vh)
            else:
                S = np.einsum("hqd,hkd->hqk", Qh, Kh).astype(F32)
                mask = np.arange(nk)[None, :] > (n_past + np.arange(N))[:, None]
                A = pv_side_by_side(wn.softmax_rows(np.where(mask[None], -np.inf, S).astype(F32)), Vh, th)
            x = wn.mul_mat(m[p + "attn.out.weight"], A.transpose(1, 0, 2).reshape(N, d)) + m[p + "attn.out.bias"] + x
            cur = wn.norm(x, m[p + "cross_attn_ln.weight"], m[p + "cross_attn_ln.bias"])
            Q = (wn.mul_mat(m[p + "cross_attn.query.weight"], cur) + m[p + "cross_attn.query.bias"]) * s
            Tk = self.ck.shape[1]
            Qh = wn.r16(Q).reshape(N, H, 64).transpose(1, 0, 2)
            Kh = self.ck[il].reshape(Tk, H, 64).transpose(1, 0, 2)
            Vh = self.cv[il].reshape(Tk, H, 64).transpose(1, 0, 2)
            A = pv_side_by_side(wn.softmax_rows(np.einsum("hqd,hkd->hqk", Qh, Kh).astype(F32)), Vh, th)
            x = wn.mul_mat(m[p + "cross_attn.out.weight"], A.transpose(1, 0, 2).reshape(N, d)) + m[p + "cross_attn.out.bias"] + x
            cur = wn.norm(x, m[p + "mlp_ln.weight"], m[p + "mlp_ln.bias"])
            cur = wn.gelu(wn.mul_mat(m[p + "mlp.0.weight"], cur) + m[p + "mlp.0.bias"])
            x = wn.mul_mat(m[p + "mlp.2.weight"], cur) + m[p + "mlp.2.bias"] + x
        return wn.mul_mat(te, wn.norm(x, m["decoder.ln.weight"], m["decoder.ln.bias"]))


# ---- tolerances ------------------------------------------------------------------------------------------------------------------
def logit_tol(want):
    """TOL_LOGIT, scaled with the logits' spread as in tests/test_gpu_parity.py"""
    return TOL_LOGIT * max(1.0, float(np.std(want)) / 3.0)


def kv_tol(want, layer):
    """Tolerance of cache rows `want` ([..][64] values of one layer).  A layer-0 row is f16(W f16(LN(embedding))): both sides round
    the same f16 operands and differ only in the f32 order of the LayerNorm and of the dot products, so an element lands at most one
    f16 step from the oracle's: 1.5 units in the last place of the row's largest value.  Rows of later layers also carry the difference of every
    earlier layer's attention and MLP outputs at f16 resolution: TOL_KV, scaled with the rows' rms like the logits."""
    if layer == 0:
        return 1.5 * float(np.spacing(np.float16(np.abs(want).max())))
    return TOL_KV * max(1.0, float(np.sqrt(np.mean(np.square(want)))))


def compare(got, want, what):
    """got / want: dict(logits [S][B][vocab], k, v [S][B][L][d]) at the single-token steps.  Returns the failures as text."""
    bad = []
    for i, p in enumerate(STEPS):
        for b in range(want["logits"].shape[1]):
            err, tol = float(np.abs(got["logits"][i, b] - want["logits"][i, b]).max()), logit_tol(want["logits"][i, b])
            if not err < tol:
                bad.append("%s: n_past %d chunk %d: |logit error| %.4g >= %.4g" % (what, p, b, err, tol))
            for nm in ("k", "v"):
                for l in range(want[nm].shape[2]):
                    w = want[nm][i, b, l]
                    err, tol = float(np.abs(got[nm][i, b, l] - w).max()), kv_tol(w, l)
                    if not err < tol:
                        bad.append("%s: n_past %d chunk %d: self_%s layer %d: |error| %.4g >= %.4g" % (what, p, b, nm, l, err, tol))
    return bad


# ---- the two sides ---------------------------------------------------------------------------------------------------------------
def run_oracle(npm, cross, tokens, threads):
    """the oracle decoder of every chunk fed the calls of CALLS; logits and the appended cache rows at every single-token step"""
    logits = []
    decs = [StepDecoder(npm, ck, cv, threads) for ck, cv in cross]
    for p, n in CALLS:
        rows = [dec.decode(t[p:p + n], p)[-1] for dec, t in zip(decs, tokens)]
        if n == 1:
            logits.append(rows)
    return dict(logits=np.array(logits), k=np.stack([dec.k[:, STEPS] for dec in decs], 1).transpose(2, 1, 0, 3),
                v=np.stack([dec.v[:, STEPS] for dec in decs], 1).transpose(2, 1, 0, 3))


def cache_rows(c, m, name, b):
    """self_k / self_v of slot b at the steps' positions: [S][L][d] (head h in columns [64h, 64h + 64))"""
    L, H = m.n_text_layer, m.n_text_head
    t = c.get_tensor(name, b).reshape(L, H, m.n_text_ctx, 64)[:, :, STEPS]
    return t.transpose(2, 0, 1, 3).reshape(len(STEPS), L, H * 64)


def run_gpu(c, m, tokens, threads, mode):
    """the same calls on the GPU in one step mode; single-token steps are sampled so that they replay the captured step graph"""
    B = len(tokens)
    lib = capi.lib()
    c.set_reference_threads(threads)
    c.set_step_mode(mode)
    logits = []
    for p, n in CALLS:
        toks = [t[p:p + n] for t in tokens]
        if n > 1:
            c.decode(toks, p, B, capi.DECODE_NO_SAMPLE)
            continue
        before = lib.wsp_launch_count()
        c.decode(toks, p, B, 0)
        launches = lib.wsp_launch_count() - before
        # a step kernel that declined this shape would leave the per-op path running in its place
        assert (launches == STEP_LAUNCHES) == (mode != 0), "mode %d, n_past %d: %d launches" % (mode, p, launches)
        logits.append(c.logits(B))
    k = np.stack([cache_rows(c, m, "self_k", b) for b in range(B)], 1)
    v = np.stack([cache_rows(c, m, "self_v", b) for b in range(B)], 1)
    return dict(logits=np.array(logits), k=k, v=v)


def encode_chunks(c, B, seed, audio_ctx):
    c.set_audio_ctx(audio_ctx)
    for b in range(B):
        c.pcm_to_mel(b, synth.synth_pcm(seed + b))
    c.encode(B, [0] * B)


def restore(c):
    c.set_step_mode(2)
    c.set_reference_threads(4)
    c.set_audio_ctx(0)
    c.set_graph(True)


# ---- against numpy -------------------------------------------------------------------------------------------------------------
_np_models = {}


@pytest.mark.parametrize("model,threads", [("micro.en-sc", t) for t in MICRO_THREADS])
def test_step_kernels_against_numpy(model, threads):
    """B = 3 chunks over the full 1500-key audio context; modes 2, 1 and 0 against one oracle run, and against each other."""
    B = 3
    m, e, c = open_model(model, B)
    assert m.n_text_ctx == N_TEXT_CTX and slot_rows(m.n_text_state) == 128
    if model not in _np_models:
        _np_models[model] = wn.NpModel(synth.model_path(model))
    npm = _np_models[model]
    tokens = chunk_tokens(m.special["sot"], m.special["eot"], B, 1000 + threads)
    L, H, d = m.n_text_layer, m.n_text_head, m.n_text_state
    try:
        encode_chunks(c, B, 70, 0)
        cross = [tuple(c.get_tensor(nm, b).reshape(L, H, -1, 64).transpose(0, 2, 1, 3).reshape(L, -1, d) for nm in ("cross_k", "cross_v"))
                 for b in range(B)]
        got = {mode: run_gpu(c, m, tokens, threads, mode) for mode in (2, 1, 0)}
    finally:
        restore(c)
    want = run_oracle(npm, cross, tokens, threads)
    bad = []
    for mode in (2, 1, 0):
        bad += compare(got[mode], want, "mode %d vs numpy" % mode)
    for mode in (2, 1):
        bad += compare(got[mode], got[0], "mode %d vs mode 0" % mode)
    assert not bad, "%d failures, first: %s" % (len(bad), "\n".join(bad[:12]))


# ---- large shapes: the step kernels against the per-op path ----------------------------------------------------------------
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("threads", LARGE_THREADS)
@pytest.mark.parametrize("model", ["large-sc", "medium-sc"])
def test_step_kernels_against_per_op_large_shapes(model, threads):
    """large-sc (CR = 160) with more (chunk, head) units than SMs, and medium-sc at B = 9 (two column tiles, also more units than
    SMs): one CTA runs several units' long self attention back to back.  audio_ctx 100 keeps cross attention short."""
    H, d = synth.MODELS[model[:-3]].n_text_head, synth.MODELS[model[:-3]].n_text_state
    B = 9 if model == "medium-sc" else sm_count() // H + 1
    assert B * H > sm_count()
    m, e, c = open_model(model, B)
    assert slot_rows(d) == (160 if model == "large-sc" else 128)
    tokens = chunk_tokens(m.special["sot"], m.special["eot"], B, 2000 + threads)
    try:
        encode_chunks(c, B, 90, 100)
        got = {mode: run_gpu(c, m, tokens, threads, mode) for mode in (0, 2, 1)}
    finally:
        restore(c)
    bad = []
    for mode in (2, 1):
        bad += compare(got[mode], got[0], "%s mode %d vs mode 0" % (model, mode))
    assert not bad, "%d failures, first: %s" % (len(bad), "\n".join(bad[:12]))


# ---- the measured path to the end of the text context -----------------------------------------------------------------------
def test_run_chunks_to_the_end_of_the_text_context():
    """run_chunks (tokens fed back and n_past advanced on the device, the step graph of mode 2) for len(prompt) + n_decode = 448,
    then the GPU's own tokens replayed through teacher-forced mode-0 calls: the last step's logits agree, and every sampled token is
    mode 0's choice wherever that choice is the plain argmax with a top-2 margin above 3 x TOL_LOGIT."""
    B = 2
    m, e, c = open_model("micro.en-sc", B)
    prompt = m.prompt_init()
    n_decode = N_TEXT_CTX - len(prompt)
    pcms = [synth.synth_pcm(110 + b) for b in range(B)]
    try:
        c.set_graph(True)
        c.set_step_mode(2)
        toks, _ = c.run_chunks(pcms, prompt, n_decode)
        last = c.logits(B)
        c.set_step_mode(0)
        s = c.decode([prompt] * B, 0, B, capi.DECODE_FORCE_TIMESTAMP | capi.DECODE_INITIAL)
        checked, lg = 0, None
        for i in range(n_decode):
            if i > 0:
                s = c.decode([[int(toks[b, i - 1])] for b in range(B)], len(prompt) + i - 1, B, 0)
            lg = c.logits(B)
            for b in range(B):
                top = np.sort(lg[b])[-2:]
                if s[b]["id"] == int(np.argmax(lg[b])) and top[1] - top[0] > 3 * TOL_LOGIT:
                    assert toks[b, i] == s[b]["id"], "chunk %d, token %d" % (b, i)
                    checked += 1
    finally:
        restore(c)
    assert checked > 0
    assert np.abs(last - lg).max() < logit_tol(lg)
