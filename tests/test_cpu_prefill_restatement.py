"""
The fp64 prefill restatement (tests/prefill_restatement.py) against the HF model: with no rounding point and its own fp64
cache, ``restate_layer`` chained through every layer and ``restate_head`` at the end must give the fp32 oracle's logits at
every position. This checks the restatement's wiring before it judges the kernels: the embedding splice of an image span,
the causal mask over a cached prefix (a suffix at start_pos > 0), the GQA head mapping, RoPE (plain, and llama3 past the
original context at ``tiny-v2``) and the arena layouts. The rounded ``"prefill"`` path and its error model run end to end.
"""
import pytest
import torch

from conftest import model_bundle
from decode_restatement import Weights, bf16
from prefill_restatement import flip_eps, head_noise, layer_noise, restate_head, restate_layer

MODELS = ["tiny", "tiny-tl", "tiny-v2"]


def _setup(name):
    from detikzify_b200.engine import pack_arena, to_c_config
    cfg, sd, oracle = model_bundle(name)
    w = Weights(cfg, pack_arena(cfg, sd), to_c_config(cfg), device="cpu")
    return cfg, w, oracle


def _prompt(cfg, name, seed, image=False):
    """ids [T] (tiny-v2: T = 100, past the llama3 original context of 64) and, with ``image``, an image span of
    num_patches rows in the middle: (ids, img rows float32 or None, span start)."""
    g = torch.Generator().manual_seed(seed)
    T = 100 if name == "tiny-v2" else 40
    ids = torch.randint(0, cfg.vocab_size, (T,), generator=g)
    ids[ids == cfg.image_token_id] = 3
    if not image:
        return ids, None, 0
    n, start = cfg.num_patches, T // 2 - cfg.num_patches // 2
    ids[start:start + n] = cfg.image_token_id
    img = torch.randn(n, cfg.hidden_size, generator=g) * 0.05
    return ids, img, start


def _oracle_logits(oracle, ids, img):
    with torch.no_grad():
        emb = oracle.spliced_embeds(ids[None], None if img is None else img[None])
        return oracle.llm(inputs_embeds=emb).logits[0].double()


def _embed(w, cfg, ids, img, start):
    x = w("dec.embed")[ids].clone()
    if img is not None:
        x[start:start + img.shape[0]] = img.double()
    return x


class Cache:
    """fp64 K / V [kv_heads, n, hd] per layer, appended row block by row block."""

    def __init__(self, cfg):
        z = torch.zeros(cfg.num_key_value_heads, 0, cfg.head_dim, dtype=torch.float64)
        self.k = [z] * cfg.num_hidden_layers
        self.v = [z] * cfg.num_hidden_layers

    def __call__(self, l, n):
        assert self.k[l].shape[1] >= n, (l, n)
        return self.k[l][:, :n], self.v[l][:, :n]

    def put(self, l, pos0, k, v):
        """rows [pos0, pos0 + T) of layer l from k, v [T, kv_heads, hd]."""
        self.k[l] = torch.cat([self.k[l][:, :pos0], k.transpose(0, 1)], 1)
        self.v[l] = torch.cat([self.v[l][:, :pos0], v.transpose(0, 1)], 1)


def _chain(w, x, start_pos, cache, path=None):
    """Every layer over x at positions [start_pos, start_pos + T), then the head. The "prefill" path reads the new rows
    from the cache as the kernel does (rope_kv_prefill writes them before attention reads them): a first call gives the
    rows, rounded to bf16 into the cache, the second reads them back."""
    for l in range(w.cfg.num_hidden_layers):
        if path is None:
            r = restate_layer(w, l, x, start_pos, cache, None)
            cache.put(l, start_pos, r["k"], r["v"])
        else:
            pad = torch.zeros(x.shape[0], w.cfg.num_key_value_heads, w.cfg.head_dim, dtype=torch.float64)
            cache.put(l, start_pos, pad, pad)
            r = restate_layer(w, l, x, start_pos, cache, path)
            cache.put(l, start_pos, bf16(r["k"]), bf16(r["v"]))
            r = restate_layer(w, l, x, start_pos, cache, path)
        x = r["x"]
    return x, restate_head(w, x, path)


def _rel(got, want):
    return ((got - want).abs().amax(-1) / want.pow(2).mean(-1).sqrt()).max().item()


@pytest.mark.parametrize("name", MODELS)
def test_restatement_with_image_span_matches_hf_model(name):
    cfg, w, oracle = _setup(name)
    ids, img, start = _prompt(cfg, name, 7, image=True)
    want = _oracle_logits(oracle, ids, img)
    x, head = _chain(w, _embed(w, cfg, ids, img, start), 0, Cache(cfg))
    assert _rel(head["logits"], want) < 2e-5
    assert _rel(head["last_logits"][None], want[-1:]) < 2e-5
    lse = torch.logsumexp(want, -1)
    assert (head["lse"] - lse).abs().max().item() < 2e-5 * lse.abs().max().item()


@pytest.mark.parametrize("name", MODELS)
def test_restatement_of_a_suffix_matches_hf_model(name):
    """A prefix prefilled first, then a suffix at start_pos > 0 over its cache: the suffix rows' logits are the full
    sequence's."""
    cfg, w, oracle = _setup(name)
    ids, _, _ = _prompt(cfg, name, 8)
    want = _oracle_logits(oracle, ids, None)
    cut = 23
    cache = Cache(cfg)
    _, head0 = _chain(w, _embed(w, cfg, ids[:cut], None, 0), 0, cache)
    _, head1 = _chain(w, _embed(w, cfg, ids[cut:], None, 0), cut, cache)
    assert _rel(head0["logits"], want[:cut]) < 2e-5
    assert _rel(head1["logits"], want[cut:]) < 2e-5


def test_prefill_path_runs_end_to_end():
    """The rounded path on its own bf16 cache stays near the exact restatement, and its error model gives a finite,
    positive noise scale at every check the GPU test makes."""
    name = "tiny-tl"
    cfg, w, oracle = _setup(name)
    ids, img, start = _prompt(cfg, name, 9, image=True)
    x0 = _embed(w, cfg, ids, img, start)
    _, exact = _chain(w, x0, 0, Cache(cfg))
    cache = Cache(cfg)
    x, head = _chain(w, x0, 0, cache, "prefill")
    assert _rel(head["logits"], exact["logits"]) < 3e-2
    ref = restate_layer(w, 0, x0, 0, cache, "prefill")
    sig = layer_noise(w, 0, x0, 0, cache, "prefill", ref)
    for k in ("x", "k", "v"):
        assert torch.isfinite(sig[k]).all() and (sig[k] > 0).all(), k
    assert (ref["kv_eps"][0] >= 0).all()
    assert torch.isfinite(flip_eps(w, 0, x0, 0, cache, ref)).all()
    targets = torch.randint(0, cfg.vocab_size, (ids.numel(),))
    hs = head_noise(w, x, "prefill", head, targets)
    for k in ("logits", "last_logits", "lse", "logprob"):
        assert torch.isfinite(hs[k]).all() and (hs[k] > 0).all(), k
