"""
Golden vectors for ``forward(labels=...)``, produced by the REFERENCE's own model code (read from /root/reference, never
copied): the v1 ``DetikzifyForCausalLM.forward`` (detikzify/model/v1/modeling_detikzify.py:218-283: shift by one,
``CrossEntropyLoss`` with ``ignore_index=-100``) on the ``tiny`` fixture weights, and the v2
``DetikzifyForConditionalGeneration.forward`` (detikzify/model/modeling_detikzify.py:320-389: with an ``attention_mask`` only
shifted positions whose mask is set are counted) on the ``tiny-v2`` fixture weights, CPU fp32. The reference models are
built by the loaders of ``make_reference_golden.py`` and ``make_reference_golden_v2.py`` (same stubs and shims).

Cases (labels = ids with -100 on the image span, on padding and on a few text positions):
  * v1 and v2: one unpadded row -> loss and logits;
  * v2: a two-row batch, right padded and left padded, with ``attention_mask`` -> loss (the first real token of a
    left-padded row is labelled -100: its prediction would come from a padded position);
  * every case also stores the shifted labels the loss counted (-100 elsewhere).

Run (where /root/reference exists):  python tests/golden/make_reference_golden_loss.py   -> tests/golden/reference_loss_tiny.pt
"""
import sys
from pathlib import Path

import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))

import make_reference_golden as golden_v1      # noqa: E402
import make_reference_golden_v2 as golden_v2   # noqa: E402
from oracle.hf_oracle import synthetic_pixels  # noqa: E402


def counted(labels, mask, v1):
    """Shifted labels as the reference's loss counts them (-100 = not counted)."""
    sh = labels[:, 1:].clone()
    if not v1 and mask is not None:
        sh[mask[:, 1:] == 0] = -100
    return sh


def prompt(cfg, g, pre, post):
    P = cfg.num_patches
    lim = min(cfg.vocab_size, cfg.patch_token_id)
    return torch.cat([torch.randint(0, lim, (pre,), generator=g), torch.full((P,), cfg.patch_token_id),
                      torch.randint(0, lim, (post,), generator=g)]).long()


def labels_for(cfg, ids, mask, g):
    lab = ids.clone()
    lab[ids == cfg.patch_token_id] = -100
    lab[(torch.rand(ids.shape, generator=g) < 0.2)] = -100
    if mask is not None:
        lab[mask == 0] = -100
    return lab


def pad_batch(cfg, rows, left):
    T = max(r.numel() for r in rows)
    ids = torch.full((len(rows), T), cfg.pad_token_id, dtype=torch.long)
    mask = torch.zeros(len(rows), T, dtype=torch.long)
    for b, r in enumerate(rows):
        sl = slice(T - r.numel(), T) if left else slice(0, r.numel())
        ids[b, sl], mask[b, sl] = r, 1
    return ids, mask


@torch.no_grad()
def main():
    golden_v1.restore_v4_cache_truthiness()
    out = {}
    # v1 (tiny): one unpadded row
    cfg, model = golden_v1.build("tiny")
    g = torch.Generator().manual_seed(5151)
    ids = prompt(cfg, g, 3, 12)[None]
    lab = labels_for(cfg, ids, None, g)
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=77)
    res = model(input_ids=ids, pixel_values=pix, labels=lab, return_dict=True)
    out["v1"] = {"input_ids": ids, "labels": lab, "pixel_seed": 77, "loss": res.loss.float(), "logits": res.logits.float(),
                 "counted": counted(lab, None, True)}
    print("v1 loss", float(res.loss))

    # v2 (tiny-v2): one unpadded row, then right- and left-padded two-row batches with an attention mask
    cfg, model = golden_v2.build("tiny-v2")
    g = torch.Generator().manual_seed(6262)
    ids = prompt(cfg, g, 3, 12)[None]
    lab = labels_for(cfg, ids, None, g)
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=77)
    res = model(input_ids=ids, pixel_values=pix, labels=lab, return_dict=True)
    out["v2"] = {"input_ids": ids, "labels": lab, "pixel_seed": 77, "loss": res.loss.float(), "logits": res.logits.float(),
                 "counted": counted(lab, None, False)}
    print("v2 loss", float(res.loss))
    rows = [prompt(cfg, g, 2, 14), prompt(cfg, g, 4, 5)]
    pix2 = synthetic_pixels(2, cfg.vision_config.image_size, seed=78)
    for name, left in (("v2_right", False), ("v2_left", True)):
        ids, mask = pad_batch(cfg, rows, left)
        lab = labels_for(cfg, ids, mask, g)
        if left:
            for b in range(ids.shape[0]):
                lab[b, int(mask[b].argmax())] = -100
        res = model(input_ids=ids, attention_mask=mask, pixel_values=pix2, labels=lab, return_dict=True)
        out[name] = {"input_ids": ids, "attention_mask": mask, "labels": lab, "pixel_seed": 78, "loss": res.loss.float(),
                     "counted": counted(lab, mask, False)}
        print(name, "loss", float(res.loss))
    path = HERE / "reference_loss_tiny.pt"
    torch.save(out, path)
    print("wrote", path)


if __name__ == "__main__":
    main()
