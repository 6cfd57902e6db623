"""
Golden vectors of the REFERENCE's own v1 model code for the TinyLlama-based checkpoint (detikzify-tl-1.1b: head_dim 64,
GQA 32/4). Same harness as make_reference_golden.py (its ``build()`` loads detikzify/model/v1/modeling_detikzify.py from the
reference checkout under the same stubs, and ``restore_v4_cache_truthiness()`` applies the same transformers-5 shim).

  * ``tiny-tl`` (head_dim 64, GQA 8/1, V 520): full prompt logits with the image span in mid-prompt, one
    ``prepare_inputs_for_generation`` cached decode step, the vision features and greedy ``generate()`` ids.
  * ``tl-1.1b`` at the real shape (random init from the seed): last-row logits of an image-prefix prompt and one cached
    decode step, as reference_v1_ds13b.pt has for ds-1.3b.

Run (in the build container, where /root/reference exists):  python tests/golden/make_reference_golden_tl.py
Writes tests/golden/reference_v1_tl.pt.
"""
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
from make_reference_golden import build, restore_v4_cache_truthiness   # noqa: E402
from oracle.hf_oracle import synthetic_pixels                           # noqa: E402


def cached_step(model, ids, pix, res):
    nxt = res.logits[0, -1].argmax()[None, None]
    inputs = model.prepare_inputs_for_generation(torch.cat([ids, nxt], dim=1), past_key_values=res.past_key_values,
                                                 use_cache=True, pixel_values=pix)
    res2 = model(**{k: v for k, v in inputs.items() if v is not None}, return_dict=True)
    return int(nxt), res2.logits[0, -1].clone()


@torch.no_grad()
def tiny_tl():
    cfg, model = build("tiny-tl")
    P = cfg.num_patches
    g = torch.Generator().manual_seed(4343)
    text = torch.randint(0, cfg.patch_token_id, (9,), generator=g)
    ids = torch.cat([text[:3], torch.full((P,), cfg.patch_token_id), text[3:]]).long()[None]
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=78)
    res = model(input_ids=ids, pixel_values=pix, use_cache=True, return_dict=True)
    logits = res.logits[0].clone()
    nxt, dec = cached_step(model, ids, pix, res)
    feats = model.model.get_vision_features(pix)[0].clone()
    prompt = torch.cat([torch.full((P,), cfg.patch_token_id), text[:4]]).long()[None]
    gen = model.generate(input_ids=prompt, pixel_values=pix, bad_words_ids=[[cfg.patch_token_id]],
                         begin_suppress_tokens=[cfg.eos_token_id], max_length=prompt.shape[1] + 24, do_sample=False,
                         pad_token_id=cfg.pad_token_id)
    print("tiny-tl logits", tuple(logits.shape), "max|logit|", float(logits.abs().max()))
    return {"input_ids": ids[0], "pixel_seed": 78, "seed": 0, "logits": logits, "next_id": nxt, "decode_logits": dec,
            "vision_features": feats, "generate_prompt": prompt[0], "generate_ids": gen[0].clone()}


@torch.no_grad()
def tl_real():
    cfg, model = build("nllg/detikzify-tl-1.1b")
    P = cfg.num_patches
    g = torch.Generator().manual_seed(1111)
    ids = torch.cat([torch.full((P,), cfg.patch_token_id), torch.randint(3, 32000, (5,), generator=g)]).long()[None]
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=11)
    res = model(input_ids=ids, pixel_values=pix, use_cache=True, return_dict=True)
    last = res.logits[0, -1].clone()
    nxt, dec = cached_step(model, ids, pix, res)
    print("tl-1.1b: max|logit|", float(last.abs().max()), "next", nxt)
    return {"input_ids": ids[0], "pixel_seed": 11, "seed": 0, "last_logits": last, "next_id": nxt, "decode_logits": dec}


def main():
    restore_v4_cache_truthiness()
    torch.manual_seed(0)
    out = {"tiny-tl": tiny_tl(), "tl-1.1b": tl_real()}
    path = Path(__file__).with_name("reference_v1_tl.pt")
    torch.save(out, path)
    print("wrote", path)


if __name__ == "__main__":
    main()
