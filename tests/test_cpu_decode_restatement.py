"""
The fp64 decode restatement (tests/decode_restatement.py) against the HF model: with no rounding point and its own fp64 cache,
stepping it through a teacher-forced sequence must give the fp32 oracle's logits at every position. This checks the
restatement's wiring before it judges the kernels: arena layouts (fused qkv, interleaved gate/up), the GQA head mapping,
RoPE (plain, and llama3 over all three frequency bands at ``tiny-v2``) and the cache layout.
"""
import pytest
import torch

from conftest import model_bundle
from decode_restatement import Weights, restate_step, rope_table


@pytest.mark.parametrize("name", ["tiny", "tiny-tl", "tiny-v2"])
def test_restatement_matches_hf_model(name):
    from detikzify_b200.engine import pack_arena, to_c_config
    cfg, sd, oracle = model_bundle(name)
    w = Weights(cfg, pack_arena(cfg, sd), to_c_config(cfg), device="cpu")
    g = torch.Generator().manual_seed(7)
    T = 40 if name != "tiny-v2" else 100     # tiny-v2: positions past the llama3 original context (64)
    ids = torch.randint(0, cfg.vocab_size, (T,), generator=g)
    want = oracle.forward_logits(ids[None], None)[0][0].double()
    L = cfg.num_hidden_layers
    cache = [([], []) for _ in range(L)]

    def kv(b, l, n):
        ks, vs = cache[l]
        assert len(ks) == n
        z = torch.zeros(cfg.num_key_value_heads, 0, cfg.head_dim, dtype=torch.float64)
        return (torch.stack(ks, 1) if ks else z), (torch.stack(vs, 1) if vs else z)

    worst = 0.0
    for t in range(T):
        r = restate_step(w, [t], [int(ids[t])], kv, path=None)
        for l in range(L):
            cache[l][0].append(r["k"][l][0])
            cache[l][1].append(r["v"][l][0])
        err = (r["logits"][0] - want[t]).abs().max().item() / want[t].pow(2).mean().sqrt().item()
        worst = max(worst, err)
    assert worst < 2e-5, worst   # fp32 oracle: its own roundings only


def test_rope_table_follows_hf_inv_freq():
    """fp32 inv_freq (linear or llama3 scaling in fp32) and fp32 angles: at every position the model's context allows, the
    table's cos / sin equal those of HF's inv_freq within a few fp32 ulps of the angle."""
    from transformers import LlamaConfig
    from transformers.models.llama.modeling_llama import LlamaRotaryEmbedding
    from detikzify_b200.model.configuration import preset
    for name in ("nllg/detikzify-ds-1.3b", "v2-8b-2l", "tiny-v2"):
        cfg = preset(name)
        T = cfg.model_max_length
        tab = rope_table(cfg, T).double()
        rs = ({"rope_type": "llama3", "factor": cfg.rope_factor, "low_freq_factor": cfg.rope_low_freq_factor,
               "high_freq_factor": cfg.rope_high_freq_factor,
               "original_max_position_embeddings": cfg.rope_original_max_position} if cfg.rope_type == "llama3" else
              {"rope_type": "linear", "factor": cfg.rope_factor} if cfg.rope_factor != 1.0 else None)
        lc = LlamaConfig(hidden_size=cfg.hidden_size, num_attention_heads=cfg.num_attention_heads, head_dim=cfg.head_dim,
                         rope_theta=cfg.rope_theta, rope_scaling=rs, max_position_embeddings=cfg.max_position_embeddings)
        inv = LlamaRotaryEmbedding(lc).inv_freq
        ang = torch.arange(T, dtype=torch.float32)[:, None] * inv.float()[None]
        assert (tab[..., 0] - ang.double().cos()).abs().max() < 4e-6, name
        assert (tab[..., 1] - ang.double().sin()).abs().max() < 4e-6, name
