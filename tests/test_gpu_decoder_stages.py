"""Every op of the decoder's kernel-by-kernel pass on an H100 against a float64 numpy restatement of that op alone, fed with the GPU's own
input to it, and the vocabulary softmax bit for bit.

wsp_debug_set_decoder_stop(layer, op) ends a decoder pass after one op; a pass repeated with the same tokens and n_past rewrites the same
self-KV rows with the same values, so the snapshots after two consecutive stops are the input and the output of one op.  Each op is
compared in full (every chunk, token row and column) with the weights of oracle/whisper_np.NpModel and the primitives that
tests/test_oracle.py pins against the reference (norm, gelu, r16, softmax_rows).  Tolerances follow from the arithmetic, element by
element, as in tests/test_gpu_encoder_stages.py (whose helpers this file imports):
  * LN + GEMM: the GPU's f32 sum of K exact f16 products, plus the f16 steps where the GPU's LayerNorm may round the other way;
  * f32 epilogues (bias, scale, the in-place residual) round once each; f16 stores (K/V rows, the MLP hidden) may flip one step where
    the value lies within its bound of a rounding midpoint;
  * attention: the f32 score error moves x - max, which moves the f16-table exp where f16(x - max) or exp lies near a rounding
    midpoint; the probabilities inherit that through the sum; along each reference thread's f16 V^T·P chain the bound of a step is
    its own perturbation plus the f16 step of the chain value where that perturbation can flip its rounding, cut down to the f16
    grid both chains lie on (wn.pv_mad_f16's chain, advanced for all threads side by side), then the threads' f32 sum and the f16
    store.
tests/test_decoder_stages_checks.py shows on the CPU that a correct pass meets every one of these checks exactly and that a wrong row,
slot, band, mask, thread split or column fails the check of its op.

The vocabulary softmax (the sampler's and softmaxRows) must equal wn.softmax_rows bit for bit: its exp is an f16 table and its sum of
f16 terms in double is exact, so there is no rounding left to tolerate.
"""
import time

import numpy as np
import pytest
import torch

from oracle import whisper_np as wn
from tests.test_gpu_encoder_stages import Check, flip_step, gelu_tol, gemm, layer_norm
from whisper_b200 import capi, synth

F16, F32, F64 = np.float16, np.float32, np.float64
U = 2.0 ** -23              # per-rounding bound of an f32 operation, relative to its result
SCALE = F32(np.power(64.0, -0.25))
N_TEXT_CTX = 448


# ---------------------------------------------------------------------------------------------------------------------------------
# arithmetic helpers
def f16_out(y, err):
    """an f32 value y (bound err) stored as f16: the rounded reference and how far the GPU's store can be from it"""
    return wn.r16(y).astype(F64), err + flip_step(y, err)


def table_exp(x):
    """the reference's exp table, f16(f32(exp(f16(x)))) in double (ggml.c:1372-1383, 5075-5077)"""
    return np.exp(wn.r16(x).astype(F64)).astype(F32).astype(F16).astype(F64)


class DecWeights:
    """The decoder weights of a model file, read through NpModel."""

    def __init__(self, path):
        m = wn.NpModel(path)
        self.m = m
        self.d, self.H, self.L, self.n_vocab = m.n_text_state, m.n_text_head, m.n_text_layer, m.n_vocab

    def __getitem__(self, k):
        return self.m[k]

    def blk(self, il, leaf):
        return self.m["decoder.blocks.%d.%s" % (il, leaf)]


# ---------------------------------------------------------------------------------------------------------------------------------
# the ops: each takes the GPU's input to it ([rows][cols], rows = tokens) and returns (want, tol) of its output
def ref_embedding(W, tokens, n_past):
    """f32(te[token]) + pe[n_past + i] in f32 (whisper.cpp:1545-1548): exact"""
    x = W["decoder.token_embedding.weight"][np.asarray(tokens)] + W["decoder.positional_embedding"][n_past:n_past + len(tokens)]
    return x.astype(F32).astype(F64), np.zeros(x.shape)


def ln_gemm(x, g, b, Wm, bias):
    """LayerNorm(x) as f16 times Wm^T plus bias in f32: (y, bound)"""
    a, delta = layer_norm(x, g, b)
    y, err = gemm(wn.r16(a), Wm, flip_step(a, delta))
    y = y + bias
    return y, err + U * (np.abs(y) + np.abs(bias))


def ref_qkv(W, il, x):
    """op 0: (Q f32 scaled, K f16 scaled, V f16), each (want, tol) [rows][d] (whisper.cpp:1578-1613)"""
    d = W.d
    Wqkv = np.concatenate([W.blk(il, "attn.query.weight"), W.blk(il, "attn.key.weight"), W.blk(il, "attn.value.weight")])
    bias = np.concatenate([W.blk(il, "attn.query.bias"), np.zeros(d, F32), W.blk(il, "attn.value.bias")])
    y, err = ln_gemm(x, W.blk(il, "attn_ln.weight"), W.blk(il, "attn_ln.bias"), Wqkv, bias)
    q = y[:, :d] * SCALE
    k = y[:, d:2 * d] * SCALE
    return ((q, err[:, :d] * SCALE + U * np.abs(q)), f16_out(k, err[:, d:2 * d] * SCALE + U * np.abs(k)),
            f16_out(y[:, 2 * d:], err[:, 2 * d:]))


def ref_cross_q(W, il, x):
    """op 3: the cross-attention query (LN + GEMM + bias) * 64^-0.25 in f32 (whisper.cpp:1690-1700)"""
    y, err = ln_gemm(x, W.blk(il, "cross_attn_ln.weight"), W.blk(il, "cross_attn_ln.bias"), W.blk(il, "cross_attn.query.weight"),
                     W.blk(il, "cross_attn.query.bias"))
    q = y * SCALE
    return q, err * SCALE + U * np.abs(q)


def ref_resid(Wm, bias, x, a16):
    """ops 2, 5, 7 (SK_BIAS_RESID): x + (a16 Wm^T + bias) in place, two f32 roundings"""
    y, err = gemm(a16, Wm)
    yb = y + bias
    out = np.asarray(x, F64) + yb
    return out, err + U * (np.abs(yb) + err + np.abs(out))


def ref_fc1(W, il, x):
    """op 6: gelu(LN3(x) W1^T + b1) as f16 (whisper.cpp:1775-1790)"""
    pre, err = ln_gemm(x, W.blk(il, "mlp_ln.weight"), W.blk(il, "mlp_ln.bias"), W.blk(il, "mlp.0.weight"), W.blk(il, "mlp.0.bias"))
    h = wn.gelu(pre).astype(F64)
    return h, gelu_tol(pre, err, h)


def ref_logits(W, x):
    """final LN + tok_emb^T (whisper.cpp:1820-1840) of rows x"""
    a, delta = layer_norm(x, W["decoder.ln.weight"], W["decoder.ln.bias"])
    return gemm(wn.r16(a), W["decoder.token_embedding.weight"], flip_step(a, delta))


def ref_attention(q, K, V, nkv, n_all, threads):
    """softmax(f16(q) K^T) V over the keys [0, nkv[i]) of query row i, with the reference threads' V^T·P split of n_all keys (ggml.c
    :4680-4722: thread t chains keys [t dc, (t + 1) dc), dc = ceil(n_all / threads), in f16; masked keys add nothing).
    q [B][N][H*64] f32, K, V [B][H][keys][64] f16 values, nkv [N] -> (want, tol) [B][N][H*64]."""
    B, N = q.shape[:2]
    H = K.shape[1]
    n = max(n_all, int(np.max(nkv)))
    qf = wn.r16(q).astype(F64).reshape(B, N, H, 64).transpose(0, 2, 1, 3)   # [B][H][N][64]
    Kk, Vk = np.asarray(K[:, :, :n], F64), np.asarray(V[:, :, :n], F64)
    S = np.matmul(qf, Kk.transpose(0, 1, 3, 2))                                # [B][H][N][n], exact products
    # the GPU adds 8 products per lane, then the 8 lanes of a key in a 3-level tree: at most 11 f32 roundings on any term's path
    errS = 2.0 ** -20 * np.matmul(np.abs(qf), np.abs(Kk).transpose(0, 1, 3, 2))
    valid = np.arange(n)[None, :] < np.asarray(nkv)[:, None]                   # [N][n]
    S = np.where(valid, S, -np.inf)
    m = S.max(-1, keepdims=True)
    x = np.where(valid, S - m, 0.0)
    dx = errS + np.where(valid, errS, 0.0).max(-1, keepdims=True) + U * np.abs(x)
    t_in = dx + flip_step(x, dx)                                               # f16(x - max)
    E = np.exp(wn.r16(x).astype(F64))
    de = E * np.expm1(t_in) + 2.0 ** -21 * E * np.exp(t_in)                   # exp of the moved input, 2 f32 ulp of expf
    e = np.where(valid, table_exp(x), 0.0)
    te = np.where(valid, de + flip_step(E, de), 0.0)
    s = e.sum(-1, keepdims=True)
    inv = (1.0 / s).astype(F32).astype(F64)
    P = (e * inv).astype(F32).astype(F64)
    rel = (te.sum(-1, keepdims=True) + n * 2.0 ** -24 * s) / s + U
    tP = np.where(valid, (te * inv + e * inv * rel + U * P) * (1 + 2.0 ** -10), 0.0)
    y, tol = pv_chains(P, tP, Vk, valid, threads, -(-n_all // threads))
    return y.transpose(0, 2, 1, 3).reshape(B, N, H * 64), tol.transpose(0, 2, 1, 3).reshape(B, N, H * 64)


def pow2(e):
    """2^e for int64 tensors e (normal float64 range) by its bit pattern"""
    return ((e + 1023) << 52).view(torch.float64)


def pv_chains(P, tP, V, valid, threads, dc):
    """wn.pv_mad_f16's V^T·P with a bound carried along every thread's f16 chain: thread t adds keys [t dc, (t + 1) dc) as
    y = f16(f32(fma(V[j], P[j], y))) key by key, the threads advanced side by side, then adds the threads' rows in f32 in thread order
    and stores the sum as f16.  P, tP [B][H][N][n] (no step where valid [N][n] is False), V [B][H][n][64] -> (want, tol) [B][H][N][64].

    A step's bound is the chain's bound t plus the step's own perturbation dl = |V[j]| tP[j] + one f32 ulp of the fma, plus the f16
    step that dl can flip (flip_step).  Both chains hold f16 values, so their difference is a multiple of the f16 spacing wherever
    both lie: the bound is cut down to such a multiple.  Where the inherited t is itself a multiple of the spacing and the spacing
    is the same all over the bound's range, shifting by it commutes with the rounding and only dl can flip it (otherwise t + dl can).
    The chains run as float64 torch CPU tensors: the same IEEE arithmetic as numpy, on all cores."""
    B, H, N, n = P.shape
    n = min(n, threads * dc)
    pad = threads * dc - n
    steps = lambda a: torch.from_numpy(np.ascontiguousarray(np.moveaxis(a, -1, 0)))   # [dc][...]: one contiguous slab per step
    Pp = steps(np.concatenate([P[..., :n], np.zeros((B, H, N, pad))], 3).reshape(B, H, N, threads, dc))[..., None]
    tPp = steps(np.concatenate([tP[..., :n], np.zeros((B, H, N, pad))], 3).reshape(B, H, N, threads, dc))[..., None]
    act = np.concatenate([valid[:, :n], np.zeros((N, pad), bool)], 1).reshape(N, threads, dc)
    Vp = torch.from_numpy(np.ascontiguousarray(np.concatenate([V[:, :, :n], np.zeros((B, H, pad, 64))], 2)
                                               .reshape(B, H, threads, dc, 64).transpose(3, 0, 1, 2, 4)))[:, :, :, None]
    y = torch.zeros((B, H, N, threads, 64), dtype=torch.float64)
    t = torch.zeros_like(y)
    zero = torch.zeros((), dtype=torch.float64)
    for j in range(dc):
        vj = Vp[j]                                             # [B][H][1][threads][64]
        a = (vj * Pp[j] + y).to(torch.float32).to(torch.float64)
        q16 = a.to(torch.float16)
        yn = q16.to(torch.float64)
        bits = q16.view(torch.int16).to(torch.int64) & 0x7FFF
        ex = bits >> 10                                        # f16 exponent field: spacing 2^(max(ex, 1) - 25)
        e1 = ex.clamp(min=1)
        s = pow2(e1 - 25)
        normal = ex > 1
        ay = yn.abs()
        r = a.abs() - ay                                       # a's offset from f16(a), away from zero
        below = torch.where(normal & ((bits & 0x3FF) == 0), s / 2, s)   # the spacing just below a power of two halves
        dist = torch.minimum(s / 2 - r, below / 2 + r)         # to the nearer rounding midpoint
        dl = vj.abs() * tPp[j] + a.abs() * 2.0 ** -23
        b1 = t + dl
        b1 = b1 + torch.where(dist <= b1, s, zero)             # + flip_step(a, t + dl)
        lo = ay - b1
        base = torch.where(normal, pow2(ex - 15), zero)        # the binade of spacing s is [base, 2^(e1 - 14))
        shift = (lo >= base) & (ay + b1 < pow2(e1 - 14)) & (torch.floor(t / s) * s == t)
        g = torch.where(lo >= base, s, torch.where(lo >= base / 2, s / 2, torch.full((), 2.0 ** -24, dtype=torch.float64)))
        tn = torch.where(shift, torch.floor((t + dl + torch.where(dist <= dl, s, zero)) / s) * s, torch.floor(b1 / g) * g)
        on = act[:, :, j]
        if on.all():
            y, t = yn, tn
        else:
            on = torch.from_numpy(np.ascontiguousarray(on))[:, :, None]
            y = torch.where(on, yn, y)
            t = torch.where(on, tn, t)
    y, t = y.numpy(), t.numpy()
    out = y[..., 0, :].astype(F32)
    for k in range(1, threads):
        out = (out + y[..., k, :].astype(F32)).astype(F32)
    st = t.sum(3)
    st = np.where(st > 0, st + threads * U * np.abs(y).sum(3), 0.0)     # equal chains add up to the same f32 sum
    out = out.astype(F64)
    return wn.r16(out).astype(F64), st + flip_step(out, st)


# ---------------------------------------------------------------------------------------------------------------------------------
# checks of one decoder pass, chunk by chunk
def band(c):
    return "head %d cols %d..%d" % (c // 64, c - c % 32, c - c % 32 + 31)


def vocab_band(c):
    return "tokens %d..%d" % (c - c % 1024, c - c % 1024 + 1023)


def check_embedding(W, chk, tokens, n_past, x):
    """x [B][N][d] after the embedding of tokens [B][N]"""
    for b in range(len(tokens)):
        chk("embedding", b, x[b], *ref_embedding(W, tokens[b], n_past), band)


def kv_rows(cache, il, n_past, N):
    """rows n_past.. n_past + N - 1 of layer il of one chunk's [L][H][n_text_ctx][64] cache as [N][H*64]"""
    H = cache.shape[1]
    return cache[il, :, n_past:n_past + N].transpose(1, 0, 2).reshape(N, H * 64)


def check_layer(W, chk, t, il, prev, n_past, N):
    """Every op of decoder layer il of a B-chunk pass but the attentions (check_attention).  t: the GPU's tensors [B][N][.] — x_in
    (the layer's input), and after op k: q0, attn1, x2, q3, attn4, x5, h6, x7 — and the self-KV caches kv_before / kv_after (per
    chunk (K, V) [L][H][n_text_ctx][64]) read after op 0 of layer prev (or before the pass) and of layer il: inside layers (prev, il]
    the rows n_past.. n_past + N - 1 are this pass's, all other rows must be unchanged."""
    H, B = W.H, len(t["x_in"])
    lband = lambda c: "layer %d %s" % (il, band(c))
    rows = lambda k: np.asarray(t[k], F64).reshape(B * N, -1)             # the row-wise ops run on all chunks' rows at once
    chunks = lambda r: tuple(a.reshape(B, N, -1) for a in r)
    (q, tq), (k, tk), (v, tv) = (chunks(r) for r in ref_qkv(W, il, rows("x_in")))
    x2 = chunks(ref_resid(W.blk(il, "attn.out.weight"), W.blk(il, "attn.out.bias"), rows("x_in"), rows("attn1")))
    q3 = chunks(ref_cross_q(W, il, rows("x2")))
    x5 = chunks(ref_resid(W.blk(il, "cross_attn.out.weight"), W.blk(il, "cross_attn.out.bias"), rows("x2"), rows("attn4")))
    h6 = chunks(ref_fc1(W, il, rows("x5")))
    x7 = chunks(ref_resid(W.blk(il, "mlp.2.weight"), W.blk(il, "mlp.2.bias"), rows("x5"), rows("h6")))
    for b in range(B):
        chk("qkv", b, t["q0"][b], q[b], tq[b], lband)
        Kb, Vb = t["kv_before"][b]
        Ka, Va = t["kv_after"][b]
        chk("qkv", b, kv_rows(Ka, il, n_past, N), k[b], tk[b], lambda c: "K " + lband(c))
        chk("qkv", b, kv_rows(Va, il, n_past, N), v[b], tv[b], lambda c: "V " + lband(c))
        for nm, before, after in (("K", Kb, Ka), ("V", Vb, Va)):
            got = after.copy()
            got[prev + 1:il + 1, :, n_past:n_past + N] = before[prev + 1:il + 1, :, n_past:n_past + N]
            if not np.array_equal(got, before):
                chk("kv-cache", b, got.reshape(-1, 64), before.reshape(-1, 64), np.zeros((got.size // 64, 64)),
                    lambda c, nm=nm: "%s cache (row = (layer * %d + head) * %d + position)" % (nm, H, N_TEXT_CTX))
        chk("self-out", b, t["x2"][b], x2[0][b], x2[1][b], lband)
        chk("cross q", b, t["q3"][b], q3[0][b], q3[1][b], lband)
        chk("cross-out", b, t["x5"][b], x5[0][b], x5[1][b], lband)
        chk("fc1", b, t["h6"][b], h6[0][b], h6[1][b], lambda c: "layer %d hidden cols %d..%d" % (il, c - c % 32, c - c % 32 + 31))
        chk("fc2", b, t["x7"][b], x7[0][b], x7[1][b], lband)
    t["self_kv"] = tuple(np.stack([kv[i][il] for kv in t["kv_after"]]) for i in (0, 1))   # what check_attention reads of the caches


def check_attention(chk, layers, n_past, N, threads):
    """The self and the cross attention of several layers of a B-chunk pass at once (the reference threads' f16 chains are long and
    run in step for all of them).  layers: [(il, t, (cross K, cross V) [B][H][T][64])], t as check_layer leaves it."""
    n_all = min(n_past + N, N_TEXT_CTX)
    nkv = np.minimum(n_past + np.arange(N) + 1, N_TEXT_CTX)
    cat = lambda f: np.concatenate([f(il, t, c) for il, t, c in layers])
    sa = ref_attention(cat(lambda il, t, c: t["q0"]), cat(lambda il, t, c: t["self_kv"][0]), cat(lambda il, t, c: t["self_kv"][1]),
                       nkv, n_all, threads)
    T = layers[0][2][0].shape[2]
    ca = ref_attention(cat(lambda il, t, c: t["q3"]), cat(lambda il, t, c: c[0]), cat(lambda il, t, c: c[1]), np.full(N, T), T, threads)
    k = 0
    for il, t, _c in layers:
        for b in range(len(t["q0"])):
            lband = lambda c, il=il: "layer %d %s" % (il, band(c))
            chk("self attention", b, t["attn1"][b], sa[0][k], sa[1][k], lband)
            chk("cross attention", b, t["attn4"][b], ca[0][k], ca[1][k], lband)
            k += 1


def check_logits(W, chk, stage, x_rows, logits):
    """logits [B][rows][n_vocab] of the residual rows x_rows [B][rows][d] (the final pass's dec.x)"""
    B, R = x_rows.shape[:2]
    want, tol = (a.reshape(B, R, -1) for a in ref_logits(W, np.asarray(x_rows, F64).reshape(B * R, -1)))
    for b in range(B):
        chk(stage, b, logits[b], want[b], tol[b], vocab_band)


def check_probs(chk, logits, probs):
    """probs [rows][n] must be wn.softmax_rows of the same logits, bit for bit"""
    want = wn.softmax_rows(np.asarray(logits, F32))
    for r in range(len(probs)):
        chk("probs", r, np.asarray(probs[r:r + 1], F64), want[r:r + 1].astype(F64), np.zeros((1, want.shape[1])), vocab_band)


# ---------------------------------------------------------------------------------------------------------------------------------
# GPU runs
_open = {}


def open_model(name):
    """(DecWeights, Model, Engine) of one model at a time: the wide models' float32 weights take gigabytes of host memory"""
    if name not in _open:
        close_models()
        path = synth.model_path(name)
        m = capi.Model(path)
        _open[name] = (DecWeights(path), m, capi.Engine(m, 0))
    return _open[name]


def close_models():
    for _w, m, e in _open.values():
        e.close()
        m.close()
    _open.clear()


@pytest.fixture(scope="module", autouse=True)
def report_margins():
    others = dict(Check.worst)
    Check.worst.clear()
    yield
    close_models()
    if Check.worst:
        print("\nlargest error / tolerance per decoder stage: " + ", ".join("%s %.3g" % kv for kv in Check.worst.items()))
    Check.worst.clear()
    Check.worst.update(others)


def decode_stop(c, tokens, n_past, il, op, names):
    """one pass of tokens [B][N] at n_past that ends after op `op` of layer il; the named dec.* tensors as [B][N][.]"""
    B, N = tokens.shape
    c.set_decoder_stop(il, op)
    c.decode(tokens, n_past, B, capi.DECODE_NO_SAMPLE)
    return {nm: np.stack([c.get_tensor("dec." + nm, b) for b in range(B)]).reshape(B, N, -1) for nm in names}


def self_kv(c, W, B):
    shape = (W.L, W.H, N_TEXT_CTX, 64)
    return [(c.get_tensor("self_k", b).reshape(shape), c.get_tensor("self_v", b).reshape(shape)) for b in range(B)]


def run_case(name, B, N, n_past, threads, layers=None, audio_ctx=0, seed=0):
    """B chunks of N tokens at n_past through every stop of the listed layers (default all), each op checked; then the final LN +
    logits (last token of each chunk; all rows under DECODE_ALL_LOGITS when N <= 8) and the vocabulary softmax of the all-logits
    path and of the sampler."""
    t0 = time.time()
    W, m, e = open_model(name)
    layers = list(range(W.L)) if layers is None else layers
    c = capi.Context(e, B)
    chk = Check()
    try:
        c.set_audio_ctx(audio_ctx)
        for b in range(B):
            c.pcm_to_mel(b, synth.synth_pcm(90 + b, 480000 - 20000 * (b % 5)))
        c.encode(B)
        T = audio_ctx or m.n_audio_ctx
        cross = [(c.get_tensor("cross_k", b).reshape(W.L, W.H, T, 64), c.get_tensor("cross_v", b).reshape(W.L, W.H, T, 64)) for b in range(B)]
        rng = np.random.default_rng(seed)
        toks = rng.integers(0, m.special["eot"], (B, n_past + N)).astype(np.int32)
        c.set_step_mode(0)
        for p0 in range(0, n_past, 224):         # the cache rows before n_past: one pass per at most 224 tokens
            c.decode(toks[:, p0:min(n_past, p0 + 224)], p0, B, capi.DECODE_NO_SAMPLE)
        c.set_reference_threads(threads)
        cur = np.ascontiguousarray(toks[:, n_past:])
        kv_prev, prev, done = self_kv(c, W, B), -1, []
        x = decode_stop(c, cur, n_past, -1, 0, ["x"])["x"]
        check_embedding(W, chk, cur, n_past, x)
        for il in layers:
            t = {"x_in": x if il == 0 else decode_stop(c, cur, n_past, il - 1, 7, ["x"])["x"]}
            t["q0"] = decode_stop(c, cur, n_past, il, 0, ["q"])["q"]
            t["kv_before"], t["kv_after"] = kv_prev, self_kv(c, W, B)
            for op, nm in ((1, "attn"), (2, "x"), (3, "q"), (4, "attn"), (5, "x"), (6, "h"), (7, "x")):
                t[nm + str(op)] = decode_stop(c, cur, n_past, il, op, [nm])[nm]
            check_layer(W, chk, t, il, prev, n_past, N)
            kv_prev, prev = t.pop("kv_after"), il
            del t["kv_before"]
            done.append((il, t, tuple(np.stack([kv[i][il] for kv in cross]) for i in (0, 1))))
        del kv_prev
        check_attention(chk, done, n_past, N, threads)
        c.set_decoder_stop(-1, -1)
        c.decode(cur, n_past, B, capi.DECODE_NO_SAMPLE)
        xf = np.stack([c.get_tensor("dec.x", b) for b in range(B)]).reshape(B, N, -1)
        check_logits(W, chk, "logits", xf[:, N - 1:], c.logits(B)[:, None])
        if N <= 8:
            c.decode(cur, n_past, B, capi.DECODE_ALL_LOGITS)
            lg = c.logits(B * N)
            check_logits(W, chk, "all logits", xf, lg.reshape(B, N, -1))
            check_probs(chk, lg, c.probs(B * N))
        c.decode(cur, n_past, B)                 # sampled: the sampler's probabilities of the last tokens' logits
        check_probs(chk, c.logits(B), c.probs(B))
    finally:
        c.set_decoder_stop(-1, -1)
        c.close()
    print("\n%s B=%d N=%d n_past=%d threads=%d audio_ctx=%d layers=%s: %.1f s" % (name, B, N, n_past, threads, audio_ctx, layers,
                                                                              time.time() - t0))
    chk.done("%s: %d chunks x %d tokens at n_past %d, %d reference threads, audio_ctx %d" % (name, B, N, n_past, threads, audio_ctx))


MICRO_SHAPES = [(3, 7, 5), (2, 224, 0), (2, 8, 440), (17, 1, 20)]     # (B, N, n_past)


@pytest.mark.gpu
@pytest.mark.parametrize("threads", [1, 4, 16])
@pytest.mark.parametrize("shape", MICRO_SHAPES, ids=["B3-N7", "B2-N224", "B2-N8-past440", "B17-N1"])
def test_stages_micro(shape, threads):
    """micro.en-sc (d = 128): 21 columns (a full 16-column tile and a ragged one), the longest prompt, keys up to 448, a per-op step
    of 17 chunks"""
    B, N, n_past = shape
    run_case("micro.en-sc", B, N, n_past, threads)


@pytest.mark.gpu
def test_stages_micro_audio_ctx():
    run_case("micro.en-sc", 3, 7, 5, 4, audio_ctx=129)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny.en-sc", "base.en-sc", "small"])
def test_stages_mid_models(name):
    """d = 384, 512 and 768 (small has random weights), every layer"""
    run_case(name, 9, 3, 6, 4)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["medium-sc", "large-sc"])
def test_stages_wide_models(name):
    """d = 1024 and 1280 (the fused LayerNorm's ten registers exactly full): layers 0, L/2 and L - 1"""
    L = synth.MODELS[name[:-3]].n_text_layer
    run_case(name, 2, 4, 3, 4, layers=[0, L // 2, L - 1])


# ---------------------------------------------------------------------------------------------------------------------------------
# the vocabulary softmax, bit for bit
def table_row(n_vocab):
    """every finite f16 value <= 0 (maximum 0, so x - max is exact), padded with -65504"""
    row = np.full(n_vocab, -65504.0, F32)
    neg = np.arange(0x8000, 0xFC00, dtype=np.uint16).view(F16).astype(F32)
    row[:neg.size] = neg
    return row[None]


@pytest.mark.gpu
@pytest.mark.parametrize("n_vocab", [51864, 51865])
def test_vocab_softmax_table(n_vocab):
    """The f16-table exp at all 31 744 inputs, through the sampler's 4-CTA cluster and through softmaxRows."""
    from tests.test_gpu_sampler import BEG, NOT, SOLM, SOT
    lg = table_row(n_vocab)
    want = wn.softmax_rows(lg)
    for label, probs in (("sampler", capi.test_sample(lg, [BEG, SOT, SOLM, NOT])[0]), ("softmaxRows", capi.test_softmax_rows(lg))):
        bad = np.nonzero(probs[0] != want[0])[0]
        assert bad.size == 0, "%s: %d inputs differ, x - max = %s" % (label, bad.size, lg[0, bad[:8]].tolist())
        chk = Check(record=False)
        check_probs(chk, lg, probs)
        chk.done(label)


@pytest.mark.gpu
def test_vocab_softmax_rows():
    """The sampler's rows (random, ties, peaked; tests/test_gpu_sampler.py) and the small vocabularies, through both kernels."""
    from tests.test_gpu_sampler import BEG, NOT, SOLM, SOT, make_rows
    from tests.test_gpu_sampler_small_vocab import small_vocab_rows
    chk = Check(record=False)
    for lg, force_ts, initial, _label in make_rows():
        check_probs(chk, lg, capi.test_sample(lg, [BEG, SOT, SOLM, NOT], force_ts, initial)[0])
        check_probs(chk, lg, capi.test_softmax_rows(lg))
    for n_vocab, seed in ((1000, 3), (4095, 2), (9, 1)):
        lg, sm = small_vocab_rows(n_vocab, seed) if n_vocab > 9 else (
            (np.random.default_rng(seed).standard_normal((16, 9)) * 2.0).astype(F32), None)
        special = [sm.token_beg, sm.token_sot, sm.token_solm, sm.token_not] if sm else [5, 1, 2, 3]
        check_probs(chk, lg, capi.test_sample(lg, special)[0])
        check_probs(chk, lg, capi.test_softmax_rows(lg))
    chk.done("vocabulary softmax")
