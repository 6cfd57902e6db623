"""
FP8 weight-only quantization on the CPU side: the per-row power-of-two e4m3 quantizer (exactness, error bound, edge cases)
and ``load(..., quantize="fp8")``, which rewrites exactly the four decoder-layer matrices of the packed arena.
"""
import re

import pytest
import torch

from detikzify_b200.quant import fp8_row_exponents, quantize_fp8_rows

E4M3 = torch.float8_e4m3fn


def _pow2(k):
    return torch.ldexp(torch.ones(k.shape, dtype=torch.float64), k.to(torch.int64))


def _matrix(seed=0, rows=64, cols=96):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(rows, cols, generator=g) * 0.02
    w *= torch.logspace(-30, 30, rows, base=2.0)[:, None]      # rows spanning many binades
    return w.to(torch.bfloat16)


def test_quantized_rows_are_e4m3_times_power_of_two():
    w = _matrix()
    wq = quantize_fp8_rows(w)
    assert wq.dtype == torch.bfloat16 and wq.shape == w.shape
    k = fp8_row_exponents(w)
    q = wq.double() / _pow2(k)[:, None]
    assert torch.equal(q.to(E4M3).double(), q)                 # every row of W~ / 2^k_r is an e4m3 value
    assert q.abs().max() <= 448
    assert torch.equal(wq.double().to(torch.bfloat16).double(), wq.double())
    assert torch.equal(quantize_fp8_rows(wq).view(torch.int16), wq.view(torch.int16))   # idempotent, bit for bit


def test_row_exponent_is_the_smallest_that_fits():
    w = _matrix(1)
    k = fp8_row_exponents(w)
    amax = w.double().abs().amax(1)
    assert (amax <= 448 * _pow2(k)).all()
    assert (amax > 448 * _pow2(k - 1)).all()


def test_error_bound():
    w = _matrix(2, rows=128, cols=256)
    wq = quantize_fp8_rows(w)
    k = fp8_row_exponents(w).double()[:, None]
    err = (wq.double() - w.double()).abs()
    normal = (w.double().abs() / torch.exp2(k)) >= 2.0 ** -6
    assert (err[normal] <= 2.0 ** -4 * w.double().abs()[normal]).all()
    assert (err[~normal] <= torch.exp2(k - 10).expand_as(err)[~normal]).all()


def test_zero_rows_and_signed_zeros():
    w = _matrix(3, rows=8, cols=32)
    w[2] = 0
    w[5] = -0.0
    wq = quantize_fp8_rows(w)
    k = fp8_row_exponents(w)
    assert k[2] == 0 and k[5] == 0
    assert (wq[2] == 0).all() and (wq[5] == 0).all()
    assert torch.equal(wq[[0, 1, 3]], quantize_fp8_rows(w[[0, 1, 3]]))   # rows are independent


def test_exponent_clamp_keeps_bf16_normals():
    w = torch.zeros(3, 16, dtype=torch.bfloat16)
    w[0, 0] = 2.0 ** -130                                  # tiny row: k would be -139, clamped to -117
    w[0, 1] = 2.0 ** -126
    w[1, :] = 2.0 ** -118
    w[2, 3] = 3 * 2.0 ** -126                              # k would be -133: clamped as well
    k = fp8_row_exponents(w)
    assert k.tolist() == [-117, -117, -117]
    wq = quantize_fp8_rows(w)
    nz = wq.float()[wq.float() != 0].abs()
    assert (nz >= 2.0 ** -126).all()                       # no bf16 subnormals
    assert wq[0, 0] == 0 and wq[0, 1] == 2.0 ** -126       # 2^-130 rounds to zero at the coarsest e4m3 step 2^-126
    assert (wq[1] == 2.0 ** -118).all()


def test_rounded_max_landing_on_224_times_scale():
    # max 229 * 2^-10 needs k = -10 (229 > 224), and 229 rounds down to 224 (e4m3 step 16 in [128, 256)): the max of W~ is
    # 224 * 2^-10 = 448 * 2^-11, so W~ itself derives k = -11 and must still be reproduced exactly
    w = torch.tensor([[229 * 2.0 ** -10, -0.37 * 2.0 ** -10, 1e-3, 3 * 2.0 ** -19]]).to(torch.bfloat16)
    assert float(w[0, 0]) == 229 * 2.0 ** -10
    assert int(fp8_row_exponents(w)[0]) == -10
    wq = quantize_fp8_rows(w)
    assert float(wq[0, 0]) == 224 * 2.0 ** -10
    assert int(fp8_row_exponents(wq)[0]) == -11
    assert torch.equal(quantize_fp8_rows(wq).view(torch.int16), wq.view(torch.int16))


@pytest.mark.parametrize("bad", [float("inf"), float("-inf"), float("nan")])
def test_non_finite_weights_are_refused(bad):
    w = _matrix(4, rows=4, cols=16)
    w[1, 7] = bad
    with pytest.raises(ValueError):
        quantize_fp8_rows(w)


class _FakeEngine:
    def __init__(self):
        self.options = {}

    def set_option(self, k, v):
        self.options[k] = v


class _FakeModel:
    """Stands in for DetikzifyForCausalLM (which needs a GPU): records the arena load() would hand to the engine."""
    def __init__(self, cfg, arena, **kw):
        self.cfg, self.arena, self.engine = cfg, arena.clone(), _FakeEngine()


def test_load_quantizes_exactly_the_layer_matrices(monkeypatch):
    import detikzify_b200.model as M
    from detikzify_b200.engine import to_c_config, weight_table
    monkeypatch.setattr(M, "DetikzifyForCausalLM", _FakeModel)
    plain, _ = M.load("tiny", seed=0)
    quant, _ = M.load("tiny", seed=0, quantize="fp8")
    assert quant.engine.options == {"decode_fp8": 1} and plain.engine.options == {}
    a, b = plain.arena, quant.arena
    changed = torch.zeros(a.numel(), dtype=torch.bool)
    names = []
    for info in weight_table(to_c_config(plain.cfg)):
        name = info.name.decode()
        if re.fullmatch(r"dec\.L\d+\.(wqkv|wo|wgu|wd)", name):
            names.append(name)
            sl = slice(info.offset // 2, info.offset // 2 + info.rows * info.cols)
            changed[sl] = True
            want = quantize_fp8_rows(a[sl].view(info.rows, info.cols)).reshape(-1)
            assert torch.equal(b[sl].view(torch.int16), want.view(torch.int16)), name
    assert len(names) == 4 * plain.cfg.num_hidden_layers
    assert torch.equal(a.view(torch.int16)[~changed], b.view(torch.int16)[~changed])   # every other byte unchanged
    assert not torch.equal(a, b)


@pytest.mark.parametrize("mode", ["int4", "fp16", "FP8", "e4m3", ""])
def test_load_refuses_other_quantize_modes(mode):
    from detikzify_b200.model import load
    with pytest.raises(ValueError):
        load("tiny", seed=0, quantize=mode)
