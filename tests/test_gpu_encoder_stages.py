"""Every encoder stage on an H100 against a float64 numpy restatement of that stage alone, fed with the GPU's own input to it.

A stage is read before and after it runs with wsp_get_tensor (wsp_debug_set_encoder_layers(k) stops the encoder after layer k), its
reference is computed from the GPU's input on the same f16-rounded operands with the weights of oracle/whisper_np.NpModel and the
primitives that tests/test_oracle.py pins against the reference (conv1d, norm, gelu, r16), and the GPU's output is compared in full:
every slot of the batch, every row, every column.  Shortened audio contexts pack the chunks densely (2n + 2 rows per chunk up to
conv1, n rows after conv2), so these comparisons are what shows a row written across a chunk boundary, a stale halo or V^T pad
column, a bias on the wrong column band or a cross-K/V memory written into the wrong slot or layer.

Tolerances follow from the arithmetic, element by element:
  * an f16 x f16 product is exact in f32 and the GPU sums K of them in f32 in its own order: |error| <= K 2^-23 (|A| |W|^T);
  * a LayerNorm output rounded to f16 on both sides can round differently only where it lies within the two LayerNorms' distance of
    an f16 rounding midpoint; those elements move by one f16 step, which enters through |W| like the product bound (ln_post, whose
    f16 output is compared directly, gets one f16 ulp plus that distance);
  * an f16 output may differ by one f16 ulp more, a GELU (slope at most 1.13) passes its input's difference on, and its f16 table
    value differs by at most one ulp of the output;
  * f32 epilogue additions (bias, residual, positional embedding) round once each.
The attention keeps the 3e-3 of tests/test_gpu_kernels.py plus one f16 ulp of its output (attention over real activations reaches
|out| > 4, where the f16 store alone may cost 2e-3; the kernel test's random inputs average out to |out| < 1).  The mel window must
be bit-exact and the V^T pad columns exactly zero.
"""
import copy

import numpy as np
import pytest

from oracle import whisper_np as wn
from whisper_b200 import capi, synth

F16, F32, F64 = np.float16, np.float32, np.float64
U = 2.0 ** -23          # per-addition bound of an f32 sum (rounding or truncation), relative to the sum of |terms|
GELU_SLOPE = 1.13       # max |gelu'| over the reals
ATTN_TOL = 3e-3
SCALE_K = F32(np.power(64.0, -0.25))


# ---------------------------------------------------------------------------------------------------------------------------------
# arithmetic helpers
def ulp16(v):
    """f16 spacing at |v| (the larger one where |v| rounds up to a power of two)."""
    return np.spacing(np.abs(np.asarray(v, F64)).astype(F16)).astype(F64)


def flip_step(a, delta):
    """How far r16(a') can be from r16(a) for |a' - a| <= delta: the f16 step where a lies within delta of a rounding midpoint, else 0."""
    a = np.asarray(a, F64)
    q = a.astype(F16)
    qd = q.astype(F64)
    lo = np.nextafter(q, F16(-np.inf)).astype(F64)
    hi = np.nextafter(q, F16(np.inf)).astype(F64)
    near = np.minimum(a - (qd + lo) / 2, (qd + hi) / 2 - a) <= delta
    return np.where(near, np.maximum(qd - lo, hi - qd), 0.0)


def gemm(a16, W, extra=0.0):
    """a16 @ W^T in float64 and the bound of the GPU's f32 sum of the same products, plus `extra` (a per-input-element difference of
    the f16 operand) carried through |W|.  The bound's own matmul runs in f32 on non-negative terms: its relative error is < 2^-10."""
    W = np.asarray(W, F64)
    a16 = np.asarray(a16, F64)
    y = a16 @ W.T
    spread = (a16.shape[-1] * U) * np.abs(a16) + extra
    err = (spread.astype(F32) @ np.abs(W).astype(F32).T).astype(F64) * (1 + 2.0 ** -10)
    return y, err


def conv(x16, w, stride):
    """wn.conv1d (f32 sum of three float64 tap products) and the bound of the GPU's sum over its 3 cin products per output;
    conv1d's own three f32 roundings are inside the extra 2^-22."""
    y = wn.conv1d(np.asarray(x16, F32), w, stride).astype(F64)
    K = 3 * w.shape[1]
    err = wn.conv1d(np.abs(np.asarray(x16, F32)), np.abs(w), stride).astype(F64) * ((K * U + 2.0 ** -22) * (1 + 2.0 ** -10))
    return y, err


def layer_norm(x, g, b, dx=None):
    """wn.norm of the rows of x, and per element how far the GPU's LayerNorm of the same rows can be from it: f32 statistics and
    affine (2^-16 relative, 2^-18 of the row's max |x| for the mean), plus, when the GPU's x may differ from x by up to dx, that
    difference carried through the normalisation (shift, mean and scale, to first order)."""
    xd = np.asarray(x, F64)
    a = wn.norm(xd, g, b).astype(F64)
    mu = xd.mean(-1, keepdims=True)
    rstd = 1.0 / np.sqrt(((xd - mu) ** 2).mean(-1, keepdims=True) + 1e-5)
    xhat = np.abs((xd - mu) * rstd)
    ag = np.abs(np.asarray(g, F64))
    delta = 2.0 ** -16 * (xhat + 1.0) * ag + 2.0 ** -20 * np.abs(b) + ag * rstd * 2.0 ** -18 * np.abs(xd).max(-1, keepdims=True)
    if dx is not None:
        m = dx.max(-1, keepdims=True)
        delta = delta + ag * rstd * (dx + m + xhat * m)
    return a, delta


def gelu_tol(pre, err, out):
    """tolerance of an f16 gelu(pre) whose f32 input may be off by err"""
    step = flip_step(pre, err)
    return ulp16(out) + np.where(step > 0, GELU_SLOPE * (err + step), 0.0)


def attention_ref(Q, K, V):
    """softmax(Q K^T / 8) V per head with P rounded to f16: tests/test_gpu_kernels.attn_ref's arithmetic, through matmul"""
    Qf, Kf, Vf = (np.asarray(t, F32) for t in (Q, K, V))
    S = np.matmul(Qf, Kf.transpose(0, 2, 1)) * F32(0.125)
    P = np.exp(S - S.max(-1, keepdims=True))
    P = wn.r16(P / P.sum(-1, keepdims=True))
    return np.matmul(P, Vf)


# ---------------------------------------------------------------------------------------------------------------------------------
# the stages: each takes the GPU's input to it and returns (want, tol) in row-major [rows][cols] layout
class Weights:
    """The encoder and cross-attention weights of a model file, read through NpModel."""

    def __init__(self, path):
        m = wn.NpModel(path)
        self.d, self.H, self.Le, self.L = m.n_audio_state, m.n_audio_head, m.n_audio_layer, m.n_text_layer
        self.m = m

    def __getitem__(self, k):
        return self.m[k]

    def blk(self, il, leaf):
        return self.m["encoder.blocks.%d.%s" % (il, leaf)]


def ref_window(mel, off, n):
    w = np.zeros((2 * n, 80), F32)
    n_len = mel.shape[1]
    i0, i1 = min(off, n_len), min(off + 2 * n, n_len)
    w[:i1 - i0] = mel[:, i0:i1].T
    return wn.r16(w), np.zeros((2 * n, 80))


def ref_conv1(W, x16):
    pre, err = conv(x16, W["encoder.conv1.weight"], 1)
    b = W["encoder.conv1.bias"].reshape(-1)
    pre = pre + b
    err = err + 2.0 ** -23 * (np.abs(pre) + np.abs(b))
    out = wn.gelu(pre).astype(F64)
    return out, gelu_tol(pre, err, out)


def ref_conv2(W, c16, n, halo=None):
    """halo: the rows conv2 reads as its zero padding (tests only: a stale halo)"""
    pre, err = conv(c16, W["encoder.conv2.weight"], 2)
    if halo is not None:
        w2 = W["encoder.conv2.weight"]
        pre[0] += halo[0] @ w2[:, :, 0].T.astype(F64)
        pre[n - 1] += halo[1] @ w2[:, :, 2].T.astype(F64)
    b = W["encoder.conv2.bias"].reshape(-1)
    pre = pre + b
    err = err + 2.0 ** -23 * (np.abs(pre) + np.abs(b))
    g = wn.gelu(pre).astype(F64)
    out = g + W["encoder.positional_embedding"][:n]
    return out, gelu_tol(pre, err, g) + 2.0 ** -23 * np.abs(out)


def ref_qkv(W, il, x):
    """[n][3d] = Q | K | V before the head-major / transposed stores"""
    a, delta = layer_norm(x, W.blk(il, "attn_ln.weight"), W.blk(il, "attn_ln.bias"))
    Wqkv = np.concatenate([W.blk(il, "attn.query.weight"), W.blk(il, "attn.key.weight"), W.blk(il, "attn.value.weight")])
    bias = np.concatenate([W.blk(il, "attn.query.bias"), np.zeros(W.d, F32), W.blk(il, "attn.value.bias")])
    y, err = gemm(wn.r16(a), Wqkv, flip_step(a, delta))
    y = y + bias
    err = err + 2.0 ** -23 * (np.abs(y) + np.abs(bias))
    return wn.r16(y).astype(F64), err + ulp16(np.abs(y) + err)


def ref_mlp_in(W, il, x, attn16):
    """x_mid = x + attn Wo^T + bo (float64, with its bound e1), then the MLP hidden gelu(LN2(x_mid) W1^T + b1)"""
    ao, e1 = gemm(attn16, W.blk(il, "attn.out.weight"))
    bo = W.blk(il, "attn.out.bias")
    xm = np.asarray(x, F64) + ao + bo
    e1 = e1 + 2.0 ** -23 * (np.abs(xm) + np.abs(ao) + np.abs(bo) + np.abs(x))
    a, delta = layer_norm(xm, W.blk(il, "mlp_ln.weight"), W.blk(il, "mlp_ln.bias"), dx=e1)
    pre, err = gemm(wn.r16(a), W.blk(il, "mlp.0.weight"), flip_step(a, delta))
    b1 = W.blk(il, "mlp.0.bias")
    pre = pre + b1
    err = err + 2.0 ** -23 * (np.abs(pre) + np.abs(b1))
    h = wn.gelu(pre).astype(F64)
    return h, gelu_tol(pre, err, h), xm, e1


def ref_mlp_out(W, il, xm, e1, h16):
    y, err = gemm(h16, W.blk(il, "mlp.2.weight"))
    b2 = W.blk(il, "mlp.2.bias")
    out = xm + y + b2
    return out, e1 + err + 2.0 ** -23 * (np.abs(out) + np.abs(xm) + np.abs(y) + np.abs(b2))


def ref_ln_post(W, x):
    """one f16 ulp of the output plus the two LayerNorms' f32 distance, which near zero (x_hat g ~ -b) is far larger than that ulp"""
    a, delta = layer_norm(x, W["encoder.ln_post.weight"], W["encoder.ln_post.bias"])
    out = wn.r16(a).astype(F64)
    return out, delta + np.maximum(ulp16(a), ulp16(out))


def ref_cross(W, l, out16):
    """[n][d] cross K (scaled) and cross V (+ bias) of decoder layer l"""
    p = "decoder.blocks.%d.cross_attn." % l
    k, ek = gemm(out16, W[p + "key.weight"])
    k, ek = k * SCALE_K, ek * SCALE_K
    ek = ek + 2.0 ** -23 * np.abs(k)
    v, ev = gemm(out16, W[p + "value.weight"])
    bv = W[p + "value.bias"]
    v = v + bv
    ev = ev + 2.0 ** -23 * (np.abs(v) + np.abs(bv))
    return (wn.r16(k).astype(F64), ek + ulp16(np.abs(k) + ek)), (wn.r16(v).astype(F64), ev + ulp16(np.abs(v) + ev))


# ---------------------------------------------------------------------------------------------------------------------------------
# comparison with a report of where it fails
class Check:
    """Collects the stage comparisons of one run.  A failure names the slot, the row (and whether it is a chunk's edge row), the
    column band and the largest error; `worst` keeps the largest error / tolerance seen per stage over the whole module."""

    worst = {}

    def __init__(self, record=True):
        self.fails = []
        self.record = record

    def __call__(self, stage, slot, got, want, tol, band):
        got = np.asarray(got, F64)
        err = np.abs(got - want)
        bad = ~(err <= tol)                      # NaN is bad
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = np.where(tol > 0, err / np.where(tol > 0, tol, 1.0), np.where(err > 0, np.inf, 0.0))
        ratio = np.where(np.isnan(err), np.inf, ratio)
        if self.record and ratio.size:
            Check.worst[stage] = max(Check.worst.get(stage, 0.0), float(ratio.max()))
        if not bad.any():
            return
        rows, cols = np.nonzero(bad)
        i, j = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
        R = got.shape[0]
        edge = " (first row of the chunk)" if i == 0 else " (last row of the chunk)" if i == R - 1 else ""
        self.fails.append((stage, slot, "%s, slot %d: %d of %d elements over tolerance in rows %s, bands %s; worst at row %d%s, col %d (%s): "
                           "got %.6g want %.6g err %.3g tol %.3g" % (
                               stage, slot, rows.size, bad.size, _ranges(np.unique(rows)), sorted({band(c) for c in np.unique(cols)})[:8],
                               i, edge, j, band(j), got[i, j], want[i, j], err[i, j], tol[i, j])))

    def failed(self, stage, slot=None):
        return any(s == stage and (slot is None or b == slot) for s, b, _ in self.fails)

    def done(self, what):
        if self.fails:
            pytest.fail("%s\n" % what + "\n".join(f[2] for f in self.fails[:24]))


def _ranges(idx):
    out, s = [], None
    for k, v in enumerate(idx):
        if s is None:
            s = v
        if k + 1 == len(idx) or idx[k + 1] != v + 1:
            out.append(str(s) if s == v else "%d..%d" % (s, v))
            s = None
    return ", ".join(out[:10]) + (" ..." if len(out) > 10 else "")


def _bands(d):
    qkv = lambda c: "%s head %d cols %d..%d" % ("QKV"[c // d], (c % d) // 64, c - c % 32, c - c % 32 + 31)
    head = lambda c: "head %d cols %d..%d" % (c // 64, c - c % 32, c - c % 32 + 31)
    plain = lambda c: "cols %d..%d" % (c - c % 32, c - c % 32 + 31)
    return qkv, head, plain


# ---------------------------------------------------------------------------------------------------------------------------------
# snapshots: {k: [per slot {name: array}]} after an encode stopped after k layers (k = Le: all layers, then ln_post and cross-K/V)
def gpu_snapshot(c, W, batch, offsets, n, settings):
    d, H, L, Le = W.d, W.H, W.L, W.Le
    shapes = {"mel": (80, -1), "enc.input": (2 * n, 80), "enc.conv1": (2 * n, d), "enc.x": (n, d), "enc.q": (H, n, 64),
              "enc.k": (H, n, 64), "enc.vt": (H, 64, -1), "enc.attn": (n, d), "enc.h": (n, 4 * d), "encode-out": (n, d),
              "cross_k": (L, H, n, 64), "cross_v": (L, H, n, 64)}
    snap = {}
    try:
        for k in settings:
            c.set_encoder_layers(k)
            c.encode(batch, offsets)
            names = ["enc.x"]
            names += ["mel", "enc.input", "enc.conv1"] if k == 0 else ["enc.q", "enc.k", "enc.vt", "enc.attn", "enc.h"]
            names += ["encode-out", "cross_k", "cross_v"] if k == Le else []
            snap[k] = [{nm: c.get_tensor(nm, b).reshape(shapes[nm]) for nm in names} for b in range(batch)]
    finally:
        c.set_encoder_layers(-1)
    return snap


def check_snapshot(W, snap, n, offsets, layers, cross_layers, chk):
    """Every stage of every slot, each from the snapshot's own input to it."""
    d, H, Le = W.d, W.H, W.Le
    qkv_band, head_band, plain_band = _bands(d)
    n128 = (n + 127) // 128 * 128
    for b in range(len(snap[0])):
        s0 = snap[0][b]
        chk("window", b, s0["enc.input"], *ref_window(s0["mel"], offsets[b], n), lambda c: "mel band %d" % c)
        chk("conv1", b, s0["enc.conv1"], *ref_conv1(W, s0["enc.input"]), plain_band)
        chk("conv2+pos", b, s0["enc.x"], *ref_conv2(W, s0["enc.conv1"], n), plain_band)
        for il in layers:
            x, t = snap[il][b]["enc.x"], snap[il + 1][b]
            q, k, vt = t["enc.q"], t["enc.k"], t["enc.vt"]
            got = np.concatenate([q.transpose(1, 0, 2).reshape(n, d), k.transpose(1, 0, 2).reshape(n, d),
                                  vt[:, :, :n].transpose(2, 0, 1).reshape(n, d)], axis=1)
            chk("qkv", b, got, *ref_qkv(W, il, x), qkv_band)
            pad = vt[:, :, n:n128].transpose(2, 0, 1).reshape(n128 - n, d)
            chk("vt-pad", b, pad, np.zeros(pad.shape), np.zeros(pad.shape), head_band)
            want = attention_ref(q, k, vt[:, :, :n].transpose(0, 2, 1)).transpose(1, 0, 2).reshape(n, d)
            chk("attention", b, t["enc.attn"], want, ATTN_TOL + ulp16(want), head_band)
            h, tol, xm, e1 = ref_mlp_in(W, il, x, t["enc.attn"])
            chk("wo+ln2+w1", b, t["enc.h"], h, tol, plain_band)
            chk("w2+resid", b, t["enc.x"], *ref_mlp_out(W, il, xm, e1, t["enc.h"]), plain_band)
        full = snap[Le][b]
        chk("ln_post", b, full["encode-out"], *ref_ln_post(W, full["enc.x"]), plain_band)
        for l in cross_layers:
            (k, tk), (v, tv) = ref_cross(W, l, full["encode-out"])
            chk("cross-kv", b, full["cross_k"][l].transpose(1, 0, 2).reshape(n, d), k, tk, lambda c, l=l: "cross K layer %d %s" % (l, head_band(c)))
            chk("cross-kv", b, full["cross_v"][l].transpose(1, 0, 2).reshape(n, d), v, tv, lambda c, l=l: "cross V layer %d %s" % (l, head_band(c)))


def slot_inputs(batch, n):
    """(pcm, mel offset) per slot: slot 0 a 30 s clip from frame 0; slot 1 a shorter clip whose window runs past its end; the last
    slot of a batch of three or more starts past its clip's end (an all-zero window); the others at scattered offsets."""
    out = []
    for b in range(batch):
        samples = 480000 - 37000 * b
        n_len = samples // 160
        if b == 0:
            off = 0
        elif b == 1:
            off = max(0, n_len - n)
        elif b == batch - 1:
            off = n_len + 5
        else:
            off = (211 * b) % max(1, n_len - 2 * n + 1)
        out.append((synth.synth_pcm(60 + b, samples), off))
    return out


# ---------------------------------------------------------------------------------------------------------------------------------
# CPU: the comparisons have teeth
def sim_snapshot(W, mels, offsets, n):
    """What a correct encoder returns, built from the stage references themselves (all layers)."""
    d, H, Le, L = W.d, W.H, W.Le, W.L
    snap = {k: [] for k in range(Le + 1)}
    Tp = 1536
    for mel, off in zip(mels, offsets):
        x16, _ = ref_window(mel, off, n)
        c1, _ = ref_conv1(W, x16)
        x, _ = ref_conv2(W, c1, n)
        snap[0].append({"mel": mel, "enc.input": x16, "enc.conv1": c1, "enc.x": x})
        for il in range(Le):
            qkv, _ = ref_qkv(W, il, x)
            q = qkv[:, :d].reshape(n, H, 64).transpose(1, 0, 2)
            k = qkv[:, d:2 * d].reshape(n, H, 64).transpose(1, 0, 2)
            vt = np.zeros((H, 64, Tp))
            vt[:, :, :n] = qkv[:, 2 * d:].reshape(n, H, 64).transpose(1, 2, 0)
            attn = wn.r16(attention_ref(q, k, vt[:, :, :n].transpose(0, 2, 1)).transpose(1, 0, 2).reshape(n, d)).astype(F64)
            h, _, xm, e1 = ref_mlp_in(W, il, x, attn)
            x, _ = ref_mlp_out(W, il, xm, e1, h)
            snap[il + 1].append({"enc.q": q, "enc.k": k, "enc.vt": vt, "enc.attn": attn, "enc.h": h, "enc.x": x})
        out, _ = ref_ln_post(W, x)
        ck, cv = zip(*(ref_cross(W, l, out) for l in range(L)))
        snap[Le][-1].update({"encode-out": out, "cross_k": np.stack([k.reshape(n, H, 64).transpose(1, 0, 2) for k, _ in ck]),
                             "cross_v": np.stack([v.reshape(n, H, 64).transpose(1, 0, 2) for v, _ in cv])})
    return snap


def test_stage_checks_catch_mutations():
    """On micro.en-sc, a simulated correct encode passes every stage check exactly, and each of five plausible packing or epilogue
    bugs, applied to it, exceeds its stage's tolerance in the slot it hits."""
    W = Weights(synth.model_path("micro.en-sc"))
    n, d, Le = 16, W.d, W.Le
    mels = [wn.log_mel(synth.synth_pcm(70 + b, 160 * (40 - 3 * b)), W.m.filters) for b in range(3)]
    offsets = [0, 30, 50]
    snap = sim_snapshot(W, mels, offsets, n)
    layers, cross_layers = range(Le), range(W.L)

    chk = Check(record=False)
    check_snapshot(W, snap, n, offsets, layers, cross_layers, chk)
    assert not chk.fails, [f[2] for f in chk.fails]

    def mutated(fn):
        s = copy.deepcopy(snap)
        fn(s)
        chk = Check(record=False)
        check_snapshot(W, s, n, offsets, layers, cross_layers, chk)
        return chk

    def shift_row(s):            # slot 1's first row lands on slot 0's last one
        s[0][0]["enc.x"][n - 1] = s[0][1]["enc.x"][0]
    assert mutated(shift_row).failed("conv2+pos", 0)

    def stale_halo(s):           # conv2 of slot 1 reads a leftover conv1 row as its trailing zero padding
        halo = (np.zeros(d), s[0][0]["enc.conv1"][0])
        s[0][1]["enc.x"] = ref_conv2(W, s[0][1]["enc.conv1"], n, halo=halo)[0]
    assert mutated(stale_halo).failed("conv2+pos", 1)

    def drop_bias_band(s):       # Q columns 32..63 of head 0 without their bias
        q = s[1][2]["enc.q"]
        q[0, :, 32:] = wn.r16(q[0, :, 32:] - W.blk(0, "attn.query.bias")[32:64]).astype(F64)
    assert mutated(drop_bias_band).failed("qkv", 2)

    def swap_qk(s):              # Q and K of head 1 exchanged
        t = s[2][1]
        t["enc.q"][1], t["enc.k"][1] = t["enc.k"][1].copy(), t["enc.q"][1].copy()
    assert mutated(swap_qk).failed("qkv", 1)

    def cross_wrong_slot(s):     # decoder layer 2's cross K of slot 0 written into slot 1
        s[Le][1]["cross_k"][2] = s[Le][0]["cross_k"][2]
    chk = mutated(cross_wrong_slot)
    assert chk.failed("cross-kv", 1) and not chk.failed("cross-kv", 0)


# ---------------------------------------------------------------------------------------------------------------------------------
# GPU
_open = {}


def open_model(name):
    """(Weights, Engine) of one model at a time: the wide models' float32 weights take gigabytes of host memory"""
    if name not in _open:
        for v in _open.values():
            v[1].close()
            v[2].close()
        _open.clear()
        path = synth.model_path(name)
        m = capi.Model(path)
        _open[name] = (Weights(path), capi.Engine(m, 0), m)
    return _open[name][:2]


@pytest.fixture(scope="module", autouse=True)
def report_margins():
    yield
    for v in _open.values():
        v[1].close()
        v[2].close()
    _open.clear()
    if Check.worst:
        print("\nlargest error / tolerance per stage: " + ", ".join("%s %.3g" % kv for kv in Check.worst.items()))


def run_case(W, e, c, n, batch, layers, cross_layers, single=None):
    """Encode `batch` slots of slot_inputs at audio_ctx n in context c, check every stage, and with `single` (a one-slot context)
    require every stage tensor of every slot to equal, bit for bit, that slot's clip and offset encoded alone."""
    inputs = slot_inputs(batch, n)
    offsets = [o for _, o in inputs]
    for b, (pcm, _) in enumerate(inputs):
        c.pcm_to_mel(b, pcm)
    settings = sorted({0, W.Le} | set(layers) | {il + 1 for il in layers})
    c.set_audio_ctx(n)
    snap = gpu_snapshot(c, W, batch, offsets, n, settings)
    chk = Check()
    check_snapshot(W, snap, n, offsets, layers, cross_layers, chk)
    chk.done("n = %d, batch %d of max_batch %d" % (n, batch, c.max_batch))
    if single is None:
        return
    # V^T columns past n rounded up to 128 are not part of an encode at n (an earlier, longer one may have left values there)
    n128 = (n + 127) // 128 * 128
    single.set_audio_ctx(n)
    for b in range(batch):
        single.set_mel(0, snap[0][b]["mel"])
        alone = gpu_snapshot(single, W, 1, [offsets[b]], n, settings)
        for k in settings:
            for nm, a in alone[k][0].items():
                want = snap[k][b][nm]
                if nm == "enc.vt":
                    a, want = a[:, :, :n128], want[:, :, :n128]
                assert np.array_equal(a, want), "n = %d: %s after %d layers of slot %d differs from the same clip encoded alone" % (n, nm, k, b)


SMALL_N = [1500, 1499, 750, 257, 129, 128, 127, 100, 16, 1]


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["micro.en-sc", "tiny.en-sc"])
@pytest.mark.parametrize("n", SMALL_N)
def test_stages_small_models(model, n):
    """Three slots of an eight-slot context, every layer and every decoder layer's cross-K/V; below n = 1500 each slot also equals
    itself encoded alone."""
    W, e = open_model(model)
    c, single = capi.Context(e, 8), capi.Context(e, 1)
    try:
        run_case(W, e, c, n, 3, range(W.Le), range(W.L), single if n < 1500 else None)
    finally:
        c.close()
        single.close()


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["base.en-sc", "medium-sc", "large-sc"])
def test_stages_wide_models(model):
    """The first and the last layer, cross-K/V of decoder layers 0, L/2 and L - 1: one slot at n = 1500, then three at n = 129 (each
    equal to itself encoded alone) in the same four-slot context."""
    W, e = open_model(model)
    c, single = capi.Context(e, 4), capi.Context(e, 1)
    try:
        layers, cross = [0, W.Le - 1], [0, W.L // 2, W.L - 1]
        run_case(W, e, c, 1500, 1, layers, cross)
        run_case(W, e, c, 129, 3, layers, cross, single)
    finally:
        c.close()
        single.close()


@pytest.mark.gpu
def test_stages_across_settings():
    """One eight-slot context moves through audio contexts and batch sizes; after every encode each stage of each slot matches the
    independent reference, so no halo row, V^T pad column or cross-K/V row left by the previous setting survives."""
    W, e = open_model("micro.en-sc")
    c = capi.Context(e, 8)
    try:
        for n, batch in ((1500, 8), (100, 8), (1500, 3), (129, 8), (129, 3), (16, 1)):
            run_case(W, e, c, n, batch, range(W.Le), range(W.L))
    finally:
        c.close()
