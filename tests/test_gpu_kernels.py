"""Kernel-level numerics on an H100, through the C ABI test hooks: the wgmma GEMM, the wgmma flash attention, the skinny
(decoder) GEMM and LayerNorm, each against a plain numpy reference of the same arithmetic (f16 operands, f32 accumulate)."""
import numpy as np
import pytest

from whisper_b200 import capi

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M,N,K,bn", [
    (128, 128, 64, 128),      # one tile, one k-block
    (128, 256, 128, 256),
    (300, 384, 200, 128),     # ragged M and K (TMA zero fill), K not a multiple of 64
    (1500, 1024, 1024, 256),  # one chunk of the medium encoder
    (3000, 384, 384, 128),    # tiny
    (777, 640, 72, 128),
    (12000, 1280, 1280, 256),  # large-v2 width, batch of 8 chunks
])
def test_gemm_tcgen05(M, N, K, bn):
    rng = np.random.default_rng(M * 7 + N)
    A = (rng.standard_normal((M, K)) * 0.5).astype(np.float16)
    B = (rng.standard_normal((N, K)) * 0.5).astype(np.float16)
    D, _ = capi.test_gemm(A, B, bn=bn)
    ref = A.astype(np.float32) @ B.astype(np.float32).T
    # f16 x f16 products are exact in f32; only the accumulation order differs
    err = np.abs(D - ref)
    tol = 2e-6 * K * 0.25 + 1e-4
    if err.max() > tol:   # say where: a whole tile points at the pipeline, single elements at the epilogue
        rows, cols = np.nonzero(err > tol)
        pytest.fail("max err %.3e, %d bad elements, rows %d..%d cols %d..%d, row tiles %s, col tiles %s" % (
            err.max(), rows.size, rows.min(), rows.max(), cols.min(), cols.max(), sorted(set((rows // 128).tolist()))[:12], sorted(set((cols // bn).tolist()))[:12]))


def attn_ref(Q, K, V):
    Qf, Kf, Vf = Q.astype(np.float32), K.astype(np.float32), V.astype(np.float32)
    S = np.einsum("bqd,bkd->bqk", Qf, Kf) * 0.125
    P = np.exp(S - S.max(-1, keepdims=True))
    P = (P / P.sum(-1, keepdims=True)).astype(np.float16).astype(np.float32)
    return np.einsum("bqk,bkd->bqd", P, Vf)


@pytest.mark.parametrize("BH,T", [(1, 128), (2, 200), (3, 1500), (5, 77)])
def test_flash_attention_tcgen05(BH, T):
    rng = np.random.default_rng(BH * 100 + T)
    Q, K, V = [rng.standard_normal((BH, T, 64)).astype(np.float16) for _ in range(3)]
    out, _ = capi.test_attention(Q, K, V)
    ref = attn_ref(Q, K, V)
    # output is stored as f16; P is f16 in both (rounded at slightly different points)
    assert np.abs(out - ref).max() < 3e-3


def test_flash_attention_peaked_rows():
    """Large score range: one key dominates each row — exercises the running-max rescale path."""
    rng = np.random.default_rng(9)
    BH, T = 2, 640
    Q = (rng.standard_normal((BH, T, 64)) * 4).astype(np.float16)
    K = (rng.standard_normal((BH, T, 64)) * 4).astype(np.float16)
    V = rng.standard_normal((BH, T, 64)).astype(np.float16)
    out, _ = capi.test_attention(Q, K, V)
    assert np.isfinite(out).all()
    assert np.abs(out - attn_ref(Q, K, V)).max() < 1e-2


@pytest.mark.parametrize("nOut,K,cols", [(64, 128, 1), (384, 384, 8), (1024, 1024, 8), (1024, 4096, 8), (51864, 384, 3), (3072, 1024, 24), (51865, 1024, 9)])
def test_skinny_gemm(nOut, K, cols):
    rng = np.random.default_rng(nOut + cols)
    W = (rng.standard_normal((nOut, K)) / np.sqrt(K)).astype(np.float16)
    X = rng.standard_normal((cols, K)).astype(np.float16)
    out, _ = capi.test_skinny(W, X)
    ref = X.astype(np.float32) @ W.astype(np.float32).T
    assert np.abs(out - ref).max() < 2e-5


@pytest.mark.parametrize("d", [128, 384, 512, 768, 1024, 1280])
def test_layernorm_f16(d):
    rng = np.random.default_rng(d)
    x = (rng.standard_normal((37, d)) * 2 + 0.3).astype(np.float32)
    g = (1 + 0.1 * rng.standard_normal(d)).astype(np.float32)
    b = (0.1 * rng.standard_normal(d)).astype(np.float32)
    out = capi.test_layernorm(x, g, b)
    xd = x.astype(np.float64)
    ref = ((xd - xd.mean(1, keepdims=True)) / np.sqrt(xd.var(1, keepdims=True) + 1e-5) * g + b).astype(np.float32)
    # one f16 ulp at |y| < 8
    assert np.abs(out - ref.astype(np.float16).astype(np.float32)).max() <= 2 ** -7
    assert np.abs(out - ref).max() <= 2 ** -8 + 1e-6
