"""
Golden vectors for TikZero text conditioning, produced by the REFERENCE's own adapter code
(detikzify/model/adapter/modeling_adapter.py, read from /root/reference, never copied): the real ``CrossAttentionAdapterMixin``
mixed into the reference's v2 ``DetikzifyForConditionalGeneration`` (set up as in make_reference_golden_v2.py), with a tiny
``LlamaModel`` embedder OBJECT passed to ``init_cross_attn_adapter``. Its forward pre-hooks run the cross layers before the
vision layers, build the key-padding mask with ``_prepare_4d_attention_mask`` and feed ``dummy_input.clamp(-1, 1)`` when
there is no image. Recorded on the ``tiny-v2`` model weights (seed 0) and the ``tiny`` adapter weights (seed 1), CPU fp32:

  * embedder ``last_hidden_state`` and connector output of one caption;
  * adapted vision ``last_hidden_state`` and prefill logits for (image, caption) and (no image, caption);
  * adapted vision states of a right-padded batch of two captions of different lengths (no image);
  * greedy ids of a generation driven like ``GenerationMixin.generate`` drives the reference (its own
    ``prepare_inputs_for_generation`` + ``forward``; the image features are passed back as ``image_hidden_states`` after the
    first step, which makes the reference's hook drop the adapter inputs), logits processors of infer/generate.py:218-227.

The package ``__init__`` files are stubbed as in make_reference_golden_v2.py; ``detikzify.model.adapter`` is a stub package
that exposes the REAL mixin from the reference's modeling_adapter.py. transformers here is 5.5.0: both names the module imports
(``_prepare_4d_attention_mask``, ``is_flash_attn_greater_or_equal_2_10``) exist.

Run in the build container:  python tests/golden/make_reference_golden_adapter.py   -> tests/golden/reference_adapter_tiny.pt
"""
import importlib.util
import sys
import types
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(Path(__file__).resolve().parent))
REF = Path("/root/reference/detikzify/model")

from detikzify_b200.model import adapter as A                    # noqa: E402
from oracle.hf_oracle import synthetic_pixels                    # noqa: E402


def load_reference_v2_with_adapter():
    """As make_reference_golden_v2.load_reference_v2, but ``detikzify.model.adapter`` exposes the REAL mixin."""
    for pkg in ("detikzify", "detikzify.model", "detikzify.model.adapter"):
        m = types.ModuleType(pkg)
        m.__path__ = []
        sys.modules[pkg] = m

    def load(name, path):
        spec = importlib.util.spec_from_file_location(name, path)
        mod = importlib.util.module_from_spec(spec)
        sys.modules[spec.name] = mod
        spec.loader.exec_module(mod)
        return mod
    ad = load("detikzify.model.adapter.modeling_adapter", REF / "adapter" / "modeling_adapter.py")
    sys.modules["detikzify.model.adapter"].CrossAttentionAdapterMixin = ad.CrossAttentionAdapterMixin
    cfgm = load("detikzify.model.configuration_detikzify", REF / "configuration_detikzify.py")
    modm = load("detikzify.model.modeling_detikzify", REF / "modeling_detikzify.py")
    orig = modm.DetikzifyForConditionalGeneration.tie_weights   # transformers 5.x post_init shim, see the v2 script
    modm.DetikzifyForConditionalGeneration.tie_weights = lambda self, *a, **k: orig(self)
    return cfgm, modm


def build():
    import make_reference_golden_v2 as v2
    from transformers import LlamaConfig, LlamaModel
    v2.load_reference_v2 = load_reference_v2_with_adapter
    cfg, model = v2.build("tiny-v2", seed=0)
    acfg = A.adapter_preset("tiny")
    asd = A.random_init(cfg, acfg, seed=1)
    lcfg = LlamaConfig(
        hidden_size=acfg.hidden_size, intermediate_size=acfg.intermediate_size, num_hidden_layers=acfg.num_hidden_layers,
        num_attention_heads=acfg.num_attention_heads, num_key_value_heads=acfg.num_key_value_heads, head_dim=acfg.head_dim,
        vocab_size=acfg.vocab_size, max_position_embeddings=4096, rms_norm_eps=acfg.rms_norm_eps, rope_theta=acfg.rope_theta,
        rope_scaling={"rope_type": "llama3", "factor": acfg.rope_factor, "low_freq_factor": acfg.rope_low_freq_factor,
                      "high_freq_factor": acfg.rope_high_freq_factor,
                      "original_max_position_embeddings": acfg.rope_original_max_position},
        hidden_act="silu", attention_bias=False, mlp_bias=False, pad_token_id=acfg.pad_token_id, attn_implementation="eager")
    emb = LlamaModel(lcfg).eval()
    missing, unexpected = emb.load_state_dict({k[len("embedding_model."):]: v for k, v in asd.items()
                                               if k.startswith("embedding_model.")}, strict=False)
    assert not unexpected and all("rotary" in k or "inv_freq" in k for k in missing), (missing, unexpected)
    model.config.vision_config._attn_implementation = "eager"
    model.init_cross_attn_adapter(emb)
    model.adapter.load_state_dict({k[len("adapter."):]: v for k, v in asd.items() if k.startswith("adapter.")}, strict=True)
    return cfg, acfg, model.float().eval()


def main():
    cfg, acfg, model = build()
    assert model.has_adapter()
    P = cfg.num_patches
    g = torch.Generator().manual_seed(2468)
    cap_a = torch.randint(2, 600, (9,), generator=g)
    cap_b = torch.randint(2, 600, (4,), generator=g)
    post = torch.randint(0, 590, (3,), generator=g)
    prompt = torch.cat([torch.full((P,), cfg.patch_token_id), post]).long()
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=77)
    captured = []
    model.model.vision_model.register_forward_hook(lambda m, a, o: captured.append(o.last_hidden_state.detach().clone()))
    out = {"seed": 0, "adapter_seed": 1, "pixel_seed": 77, "caption": cap_a, "caption_b": cap_b, "prompt": prompt}
    with torch.no_grad():
        h = model.embedding_model(input_ids=cap_a[None], attention_mask=torch.ones(1, cap_a.numel(), dtype=torch.long)).last_hidden_state
        out["embed_hidden"], out["connector"] = h[0], model.adapter.connect(h)[0]
        mask = torch.ones(1, cap_a.numel(), dtype=torch.long)
        for key, p in (("image", pix), ("text", None)):
            captured.clear()
            lg = model(input_ids=prompt[None], pixel_values=p, adapter_input_ids=cap_a[None], adapter_attention_mask=mask).logits
            out[f"{key}_vision"], out[f"{key}_logits"] = captured[0][0], lg[0].float()
        # right-padded batch of two captions of different lengths, no image
        ids2 = torch.full((2, cap_a.numel()), acfg.pad_token_id)
        m2 = torch.zeros(2, cap_a.numel(), dtype=torch.long)
        for i, c in enumerate((cap_a, cap_b)):
            ids2[i, : c.numel()], m2[i, : c.numel()] = c, 1
        captured.clear()
        model(input_ids=prompt[None].repeat(2, 1), adapter_input_ids=ids2, adapter_attention_mask=m2)
        out["batch_ids"], out["batch_mask"], out["batch_vision"] = ids2, m2, captured[0]
        # greedy generation, text only and image + text
        from transformers import DynamicCache
        for key, p in (("image", pix), ("text", None)):
            cache, gen, ihs = DynamicCache(), prompt[None].clone(), None
            for step in range(16):
                seen = cache.get_seq_length()
                inputs = model.prepare_inputs_for_generation(
                    gen, past_key_values=cache, cache_position=torch.arange(seen, gen.shape[1]), attention_mask=torch.ones_like(gen),
                    pixel_values=p, image_hidden_states=ihs, use_cache=True, adapter_input_ids=cap_a[None], adapter_attention_mask=mask)
                o = model(**inputs)
                ihs = o.image_hidden_states
                lg = o.logits[0, -1].float()
                lg[cfg.image_token_id] = -float("inf")            # bad_words_ids=[[image_token_id]]
                if step == 0:
                    lg[cfg.eos_token_id] = -float("inf")          # begin_suppress_tokens=[eos]
                tok = int(lg.argmax())
                gen = torch.cat([gen, torch.tensor([[tok]])], dim=1)
                if tok == cfg.eos_token_id:
                    break
            out[f"{key}_generate_ids"] = gen[0]
    path = Path(__file__).parent / "reference_adapter_tiny.pt"
    torch.save(out, path)
    print("wrote", path, {k: (tuple(v.shape) if hasattr(v, "shape") else v) for k, v in out.items()})


if __name__ == "__main__":
    main()
