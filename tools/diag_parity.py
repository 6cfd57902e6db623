"""Where does the logits error of a model shape come from? (dev tool) prefill last row, batch-1 decode on the
persistent kernel and on the per-op kernels, each against the fp32 oracle; plus persistent vs per-op."""
import sys
import torch
sys.path.insert(0, "."); sys.path.insert(0, "tests")
from conftest import engine_for, model_bundle
from oracle.hf_oracle import synthetic_pixels
for name in sys.argv[1:] or ["ds-7b-2l"]:
    cfg, sd, oracle = model_bundle(name)
    eng = engine_for(name, max_seqs=2, max_batch=1)
    pix = synthetic_pixels(1, cfg.vision_config.image_size)
    img = eng.image_embeds(pix.cuda())[0]
    ref_img = oracle.image_embeds(pix)[0]
    print(f"{name}: image embeds err {(img.cpu() - ref_img).abs().max():.4f} (|ref| max {ref_img.abs().max():.2f})")
    g = torch.Generator().manual_seed(7000)
    P = cfg.num_patches
    ids = torch.cat([torch.full((P,), cfg.patch_token_id), torch.randint(0, min(32000, cfg.vocab_size - 100), (50,), generator=g)]).long()
    T0, steps = ids.numel(), 6
    ref_ids = oracle.generate(ids[None], pix, max_length=T0 + steps, stop_on_eos=False)[0]
    ref_all, _ = oracle.forward_logits(ref_ids[None], pix)
    print(f"  |logits| max {ref_all.abs().max():.2f} rms {ref_all.pow(2).mean().sqrt():.3f}")
    slot = eng.seq_alloc()
    out = {}
    for impl in (1, 0):
        eng.set_option("decode_impl", impl)
        last, _ = eng.prefill(slot, ids.cuda(), 0, img, 0)
        print(f"  impl {impl}: prefill last-row err {(last.cpu() - ref_all[0, T0 - 1]).abs().max():.4f}")
        errs, rows = [], []
        for t in range(T0, T0 + steps - 1):
            lg = eng.decode([slot], [t], ref_ids[t:t + 1].cuda())[0].cpu()
            d = (lg - ref_all[0, t]).abs()
            errs.append(d.max().item()); rows.append(lg)
            if d.max() > 0.5:
                bad = (d > 0.5).nonzero().flatten()
                print(f"    step {t}: {bad.numel()} logits off by > 0.5, index range [{int(bad.min())}, {int(bad.max())}], "
                      f"first {bad[:8].tolist()}, lg {lg[bad[:4]].tolist()} ref {ref_all[0, t][bad[:4]].tolist()}")
                again = eng.decode([slot], [t], ref_ids[t:t + 1].cuda())[0].cpu()
                print(f"    same step launched again: err {(again - ref_all[0, t]).abs().max():.4f}")
        out[impl] = torch.stack(rows)
        print(f"  impl {impl}: decode errs " + " ".join(f"{e:.4f}" for e in errs))
    print(f"  persistent vs per-op max diff {(out[1] - out[0]).abs().max():.5f}")
    eng.set_option("decode_impl", 1)
    eng.seq_free(slot)
