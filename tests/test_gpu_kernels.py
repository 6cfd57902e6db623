"""
Kernel-level parity (through the C ABI test hooks) at the real model shapes: every dense contraction
shape of SigLIP-so400m / ds-1.3b / ds-7b, attention at head_dim 72 / 128, decode GEMV rows.
Reference = plain PyTorch fp32 of the same op on the same bf16-rounded operands.
Tolerances: fp32-accumulated kernels with fp32 output must agree to accumulation-order noise
(rtol 2e-3 / atol 2e-3 * scale); bf16 outputs to one bf16 ulp of the result (rtol 1.6e-2).
"""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from detikzify_b200 import _lib as L
    return L.load_library()


def _p(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


GEMM_SHAPES = [
    # (M, N, K, bias, act, resid, glu, out_bf16)   -- ViT so400m @384: M = B*729
    (729, 1152, 640, True, 0, False, False, False),     # patch embed (K padded 588 -> 640)
    (729, 3456, 1152, True, 0, False, False, True),     # fused qkv
    (729, 1152, 1152, True, 0, True, False, False),     # out proj + residual
    (729, 4304, 1152, True, 1, False, False, True),     # fc1 + gelu(tanh)
    (729, 1152, 4304, True, 0, True, False, False),     # fc2 + residual, K = 4304 = 134.5 * 32 (ragged K tile)
    (1458, 4304, 1152, True, 2, False, False, True),    # fc1 + gelu(erf), B = 2
    (243, 2048, 3456, True, 0, False, False, False),    # projector 1.3b
    (243, 6144, 2048, False, 0, False, False, False),   # llama qkv 1.3b (fp32 out)
    (243, 11008, 2048, False, 0, False, True, True),    # gate/up interleaved + SiLU*mul
    (243, 2048, 5504, False, 0, True, False, False),    # down + residual
    (1, 1152, 1152, True, 0, False, False, False),      # M = 1 (pool head probe)
    (130, 264, 72, False, 0, False, False, False),      # ragged everything
    (300, 32256, 256, False, 0, False, False, False),   # wide N (lm_head all-logits path)
    (5832, 4304, 1152, True, 1, False, False, True),    # ViT fc1 at B = 8: 782 tiles of 128 x 256 over 132 persistent CTAs
    (5832, 1152, 4304, True, 0, True, False, False),    # ViT fc2 at B = 8 (fp32 out + residual, ragged K)
    (2047, 11008, 2048, False, 0, False, True, True),   # prefill gate/up at the 2k context (GLU, bf16 out)
    # batched decode (M = number of rollouts): the swapped-operand wgmma tile
    (32, 6144, 2048, False, 0, False, False, False),    # qkv, 32 rollouts
    (32, 2048, 5504, False, 0, True, False, False),     # down + residual, ragged K tile
    (17, 11008, 2048, False, 0, False, True, True),     # gate/up GLU, odd M
    (8, 32256, 2048, False, 0, False, False, False),    # lm_head, 8 rollouts
    (6, 264, 72, False, 0, False, False, False),        # tiny-model shapes
    (63, 1000, 264, True, 0, False, False, False),
]


@pytest.mark.parametrize("impl", [0, 1, 2], ids=["mma_sync", "tcgen05", "tcgen05_persistent"])
@pytest.mark.parametrize("M,N,K,bias,act,resid,glu,obf", GEMM_SHAPES)
def test_gemm_matches_torch(M, N, K, bias, act, resid, glu, obf, impl):
    """The dense-GEMM implementations (mma.sync bring-up kernel, one-tile 128 x 128 wgmma/TMA kernel, persistent 128 x 256
    wgmma kernel; the parameter ids keep their historical names) against torch fp32."""
    prev = _lib().dtk_dbg_gemm_impl(-1)
    _lib().dtk_dbg_gemm_impl(impl)
    try:
        _gemm_case(M, N, K, bias, act, resid, glu, obf)
    finally:
        _lib().dtk_dbg_gemm_impl(prev)


SPLIT_SHAPES = [
    # (M, N, K, bias, resid, glu, out_bf16): the batched-decode tile (weights as the wgmma M side) with cluster split-K
    (32, 4096, 4096, False, True, False, False),      # 7b o-proj + residual
    (32, 4096, 11008, False, True, False, False),     # 7b down + residual
    (32, 22016, 4096, False, False, True, True),      # 7b gate/up GLU
    (48, 6144, 2048, True, False, False, False),      # NB = 64 tile, bias
    (5, 1000, 264, False, False, False, False),       # ragged N and K, fewer k-blocks than ranks allow
]


@pytest.mark.parametrize("split", [0, 1, 2, 3, 8])
@pytest.mark.parametrize("M,N,K,bias,resid,glu,obf", SPLIT_SHAPES)
def test_batched_decode_gemm_cluster_split_k(M, N, K, bias, resid, glu, obf, split):
    """Split-K over a thread-block cluster with the DSMEM reduction on rank 0: every factor gives the torch result, and the
    result does not depend on run-to-run timing (ranks are added in order)."""
    prev = _lib().dtk_dbg_gemm_impl(-1)
    _lib().dtk_dbg_gemm_impl(1 | (split << 8))
    try:
        _gemm_case(M, N, K, bias, 0, resid, glu, obf)
    finally:
        _lib().dtk_dbg_gemm_impl(prev)


def _gemm_case(M, N, K, bias, act, resid, glu, obf):
    torch.manual_seed(M * 131 + N * 7 + K)
    dev = "cuda"
    A = (torch.randn(M, K, device=dev) * 0.5).bfloat16()
    W = (torch.randn(N, K, device=dev) * (1.0 / math.sqrt(K))).bfloat16()
    b = (torch.randn(N, device=dev) * 0.1).bfloat16() if bias else None
    No = N // 2 if glu else N
    R = torch.randn(M, No, device=dev) if resid else None
    ref = A.float() @ W.float().t()
    if bias:
        ref = ref + b.float()
    if act == 1:
        ref = torch.nn.functional.gelu(ref, approximate="tanh")
    elif act == 2:
        ref = torch.nn.functional.gelu(ref)
    if glu:
        ref = torch.nn.functional.silu(ref[:, 0::2]) * ref[:, 1::2]
    if resid:
        ref = ref + R
    out32 = None if obf else torch.full((M, No), float("nan"), device=dev)
    out16 = torch.full((M, No), float("nan"), device=dev, dtype=torch.bfloat16) if obf else None
    rc = _lib().dtk_dbg_gemm(_p(A), _p(W), _p(b), _p(R), M, N, K, act, int(glu), _p(out32), _p(out16), _stream())
    assert rc == 0
    torch.cuda.synchronize()
    if obf:
        torch.testing.assert_close(out16.float(), ref, rtol=1.6e-2, atol=1e-2)
    else:
        torch.testing.assert_close(out32, ref, rtol=2e-3, atol=2e-3)


ATTN_CASES = [
    # (B, heads, Tq, Tk, D, causal, q_pos0)
    (2, 16, 729, 729, 72, 0, 0),      # ViT so400m
    (1, 2, 16, 16, 72, 0, 0),         # tiny ViT
    (3, 3, 81, 81, 72, 0, 0),
    (1, 16, 243, 243, 128, 1, 0),     # 1.3b prefill of the image prefix
    (1, 32, 300, 300, 128, 1, 0),
    (1, 4, 57, 300, 128, 1, 243),     # suffix prefill on top of a cached prefix (MCTS prefix reuse)
    (1, 2, 1, 65, 128, 1, 64),        # single query row
    (1, 16, 2048, 2048, 128, 1, 0),   # max context
]


@pytest.mark.parametrize("B,heads,Tq,Tk,D,causal,q_pos0", ATTN_CASES)
def test_flash_attention_matches_torch(B, heads, Tq, Tk, D, causal, q_pos0):
    torch.manual_seed(Tq * 17 + Tk + D)
    dev = "cuda"
    q = torch.randn(B, Tq, heads, D, device=dev).bfloat16()
    k = torch.randn(B, Tk, heads, D, device=dev).bfloat16()
    v = torch.randn(B, Tk, heads, D, device=dev).bfloat16()
    o = torch.full((B, Tq, heads, D), float("nan"), device=dev, dtype=torch.bfloat16)
    scale = 1.0 / math.sqrt(D)
    rc = _lib().dtk_dbg_flash_attn(_p(q), _p(k), _p(v), _p(o), B, heads, Tq, Tk, D, causal, q_pos0, scale, _stream())
    assert rc == 0
    torch.cuda.synchronize()
    s = torch.einsum("bqhd,bkhd->bhqk", q.float(), k.float()) * scale
    if causal:
        qi = torch.arange(Tq, device=dev)[:, None] + q_pos0
        kj = torch.arange(Tk, device=dev)[None, :]
        s = s.masked_fill(kj > qi, float("-inf"))
    ref = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, dim=-1), v.float())
    # P is rounded to bf16 before the PV product (as FlashAttention does): 1 bf16 ulp of O plus P rounding
    torch.testing.assert_close(o.float(), ref, rtol=2e-2, atol=2e-2)


@pytest.mark.parametrize("B,heads,N", [(2, 16, 729), (1, 2, 16), (3, 3, 81), (1, 16, 900), (5, 4, 130), (64, 16, 729)])
def test_tcgen05_vit_attention_matches_torch(B, heads, N):
    """attn_tc.cu: the ViT attention on wgmma (fused qkv layout in, head_dim 72 padded to 80 by TMA zero fill, ragged last
    key block masked) against fp32 softmax attention of the same bf16 inputs; 729 = v1 tower, 900 = v2 tower."""
    torch.manual_seed(B * 31 + N)
    dev, D = "cuda", heads * 72
    qkv = torch.randn(B * N, 3 * D, device=dev).bfloat16()
    NP = (N + 127) // 128 * 128
    vt = torch.full((B * heads * 80, NP), float("nan"), device=dev, dtype=torch.bfloat16)
    o = torch.full((B * N, D), float("nan"), device=dev, dtype=torch.bfloat16)
    scale = 1.0 / math.sqrt(72)
    rc = _lib().dtk_dbg_attn_tc(_p(qkv), _p(vt), _p(o), B, heads, N, scale, _stream())
    assert rc == 0
    torch.cuda.synchronize()
    q, k, v = (t.reshape(B, N, heads, 72).float() for t in qkv.split(D, dim=1))
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * scale
    ref = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, dim=-1), v).reshape(B * N, D)
    torch.testing.assert_close(o.float(), ref, rtol=2e-2, atol=2e-2)


GEMV_CASES = [
    # (N, K, mode, norm)
    (6144, 2048, 0, True),     # 1.3b qkv-shaped rows (store mode exercises the same inner loop)
    (2048, 2048, 1, False),    # o proj + residual
    (11008, 2048, 2, True),    # 1.3b gate/up glu
    (2048, 5504, 1, False),    # down, K = 21.5 * 256 (ragged K loop)
    (32256, 2048, 0, True),    # lm_head
    (22016, 4096, 2, True),    # 7b gate/up
    (4096, 11008, 1, False),   # 7b down
    (512, 256, 0, True),       # tiny
]


@pytest.mark.parametrize("N,K,mode,norm", GEMV_CASES)
def test_decode_gemv_matches_torch(N, K, mode, norm):
    torch.manual_seed(N + K + mode)
    dev = "cuda"
    W = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
    x = torch.randn(K, device=dev)
    nw = (1 + 0.1 * torch.randn(K, device=dev)).bfloat16() if norm else None
    eps = 1e-6
    xin = x
    if norm:
        xin = x * torch.rsqrt(x.pow(2).mean() + eps) * nw.float()
    y = W.float() @ xin
    No = N // 2 if mode == 2 else N
    out = torch.randn(No, device=dev)
    base = out.clone()
    if mode == 0:
        ref = y
    elif mode == 1:
        ref = base + y
    else:
        ref = torch.nn.functional.silu(y[0::2]) * y[1::2]
    rc = _lib().dtk_dbg_gemv(_p(W), _p(x), _p(nw), eps, N, K, mode, _p(out), _stream())
    assert rc == 0
    torch.cuda.synchronize()
    torch.testing.assert_close(out, ref, rtol=2e-3, atol=2e-3)
