"""Host logic of ``DetikzifyForCausalLM.forward`` / ``score`` on CPU: a fake engine defined here runs the fp32 oracle
(stock HF LLaMA) over each slot's whole token history, so logits, losses and log-probs can be compared with the reference
goldens, and the engine calls (slots, start positions, row counts, image splices) can be checked."""
from pathlib import Path

import pytest
import torch

from detikzify_b200.engine import EngineError
from detikzify_b200.model.modeling import DetikzifyForCausalLM
from oracle.hf_oracle import synthetic_pixels

GOLDEN = Path(__file__).resolve().parent / "golden" / "reference_loss_tiny.pt"


class OracleEngine:
    """Stand-in for ``Engine``: per slot the embedded input rows it holds; ``score``/``prefill`` run the oracle over them."""

    def __init__(self, cfg, oracle, max_seqs=3):
        self.cfg, self.oracle = cfg, oracle
        self.device, self.max_len = torch.device("cpu"), cfg.model_max_length
        self.Vocab, self.P, self.H = cfg.vocab_size, cfg.num_patches, cfg.hidden_size
        self.max_seqs, self.used, self.rows, self.calls = max_seqs, set(), {}, []

    def seq_alloc(self):
        for s in range(self.max_seqs):
            if s not in self.used:
                self.used.add(s)
                return s
        raise EngineError("dtk_seq_alloc: no free KV sequence slot")

    def seq_free(self, s):
        assert s in self.used
        self.used.discard(s)
        self.calls.append(("free", s))

    def seq_share(self, base, dst, n):
        assert base in self.used and dst in self.used and base != dst
        self.rows[dst] = self.rows.get(base, torch.zeros(0, self.H))[:n]
        self.calls.append(("share", base, dst, n))

    def image_embeds(self, pix):
        self.calls.append(("image_embeds", pix.shape[0]))
        return self.oracle.image_embeds(pix.float())

    def _run(self, slot, ids, start_pos, img, img_start):
        assert slot in self.used
        held = self.rows.get(slot, torch.zeros(0, self.H))
        assert held.shape[0] >= start_pos, (held.shape, start_pos)
        emb = self.oracle.llm.model.embed_tokens(ids).detach().clone()
        if img is not None:
            for t in range(ids.numel()):
                if int(ids[t]) == self.cfg.image_token_id:
                    emb[t] = img[start_pos + t - img_start]
        self.rows[slot] = torch.cat([held[:start_pos], emb])
        with torch.no_grad():
            lg = self.oracle.llm(inputs_embeds=self.rows[slot][None]).logits[0].float()
        return lg[start_pos:]

    def prefill(self, slot, ids, start_pos=0, img_embeds=None, img_start=0, want_all_logits=False):
        self.calls.append(("prefill", slot, start_pos, ids.numel(), img_embeds is not None))
        lg = self._run(slot, ids, start_pos, img_embeds, img_start)
        return lg[-1], (lg if want_all_logits else None)

    def score(self, slot, ids, start_pos=0, img_embeds=None, img_start=0, targets=None, want_all_logits=False, *, logits_out=None):
        self.calls.append(("score", slot, start_pos, ids.numel(), img_embeds is not None))
        assert targets.numel() == ids.numel()
        lg = self._run(slot, ids, start_pos, img_embeds, img_start)
        lse = torch.logsumexp(lg, -1)
        ok = (targets >= 0) & (targets < self.Vocab)
        lp = torch.where(ok, lg.gather(1, targets.clamp(0, self.Vocab - 1)[:, None])[:, 0] - lse, torch.zeros_like(lse))
        if logits_out is not None:
            logits_out.copy_(lg)
        return lp, lse, logits_out if logits_out is not None else (lg if want_all_logits else None)


def make_model(name, max_seqs=3):
    from conftest import model_bundle
    cfg, _, oracle = model_bundle(name)
    eng = OracleEngine(cfg, oracle, max_seqs=max_seqs)
    return DetikzifyForCausalLM(cfg, engine=eng), eng, oracle


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN)


@pytest.mark.parametrize("case,name", [("v1", "tiny"), ("v2", "tiny-v2"), ("v2_right", "tiny-v2"), ("v2_left", "tiny-v2")])
def test_forward_matches_reference_loss_and_logits(golden, case, name):
    g = golden[case]
    model, eng, _ = make_model(name)
    S = model.config.vision_config.image_size
    B = g["input_ids"].shape[0]
    pix = synthetic_pixels(B, S, seed=g["pixel_seed"])
    out = model(input_ids=g["input_ids"], pixel_values=pix, attention_mask=g.get("attention_mask"), labels=g["labels"])
    assert out.past_key_values is None and out.loss.dtype == torch.float32 and out.loss.dim() == 0
    assert abs(float(out.loss) - float(g["loss"])) <= 5e-5, (float(out.loss), float(g["loss"]))
    assert out["loss"] is out.loss and out[0] is out.loss and out[1] is out.logits
    if "logits" in g:
        assert (out.logits - g["logits"]).abs().max() <= 2e-5
    else:   # padded batch: valid rows match the unpadded forward, masked rows are 0
        m = g["attention_mask"].bool()
        assert out.logits[~m].abs().max() == 0
    assert eng.used == {0}   # the scratch slot was freed
    t = model(input_ids=g["input_ids"], pixel_values=pix, attention_mask=g.get("attention_mask"), labels=g["labels"],
              return_dict=False)
    assert len(t) == 2 and torch.equal(t[0], out.loss) and torch.equal(t[1], out.logits)
    assert len(model(input_ids=g["input_ids"], pixel_values=pix, attention_mask=g.get("attention_mask"), return_dict=False)) == 1


def test_forward_padded_rows_equal_unpadded_rows(golden):
    g = golden["v2_left"]
    model, _, _ = make_model("tiny-v2")
    pix = synthetic_pixels(2, model.config.vision_config.image_size, seed=g["pixel_seed"])
    out = model(input_ids=g["input_ids"], pixel_values=pix, attention_mask=g["attention_mask"])
    assert out.loss is None
    for b in range(2):
        m = g["attention_mask"][b].bool()
        one = model(input_ids=g["input_ids"][b][m][None], pixel_values=pix[b:b + 1]).logits[0]
        assert (out.logits[b][m] - one).abs().max() <= 2e-5   # the batched tower rounds differently from a single image
        assert not out.logits[b][~m].any()


def test_forward_loss_nan_when_nothing_counted():
    model, _, _ = make_model("tiny")
    ids = torch.randint(0, 400, (1, 6))
    assert torch.isnan(model(input_ids=ids, labels=torch.full((1, 6), -100)).loss)


def test_forward_rejects_bad_inputs(golden):
    model, eng, _ = make_model("tiny")
    V = model.config.vocab_size
    ids = torch.randint(0, 400, (2, 8))
    right = torch.tensor([[1] * 8, [1] * 5 + [0] * 3])
    lab = ids.clone()
    # v1 counts every non-ignored shifted label: the label at position 6 of row 1 is predicted from masked position 5
    with pytest.raises(ValueError, match="masked position"):
        model(input_ids=ids, attention_mask=right, labels=lab)
    lab[1, 5:] = -100
    model(input_ids=ids, attention_mask=right, labels=lab)
    for bad in (V, -5):
        lab2 = lab.clone()
        lab2[0, 3] = bad
        with pytest.raises(ValueError, match="labels must be"):
            model(input_ids=ids, attention_mask=right, labels=lab2)
    with pytest.raises(ValueError, match="contiguous"):
        model(input_ids=ids, attention_mask=torch.tensor([[1] * 8, [1, 1, 0, 1, 1, 1, 1, 1]]))
    with pytest.raises(ValueError, match="contiguous"):
        model(input_ids=ids, attention_mask=torch.tensor([[1] * 8, [0] * 8]))
    with pytest.raises(ValueError):
        model(input_ids=ids, inputs_embeds=torch.zeros(2, 8, model.config.hidden_size))
    with pytest.raises(ValueError):
        model(input_ids=ids, past_key_values=object())
    for k in ("output_attentions", "output_hidden_states"):
        with pytest.raises(ValueError):
            model(input_ids=ids, **{k: True})
    model(input_ids=ids, use_cache=True, output_attentions=False)
    # v2 with a left-padded row: the first real token's label would be predicted from the padding
    g = golden["v2_left"]
    m2, _, _ = make_model("tiny-v2")
    pix = synthetic_pixels(2, m2.config.vision_config.image_size, seed=g["pixel_seed"])
    lab = g["input_ids"].clone()
    lab[g["attention_mask"] == 0] = -100
    with pytest.raises(ValueError, match="masked position"):
        m2(input_ids=g["input_ids"], attention_mask=g["attention_mask"], pixel_values=pix, labels=lab)
    # splice validation and messages as in generate()
    P, patch = model.config.num_patches, model.config.image_token_id
    pix1 = synthetic_pixels(1, model.config.vision_config.image_size, seed=1)
    with pytest.raises(ValueError, match="same as the number of image patches"):
        model(input_ids=torch.tensor([[3] + [patch] * (P - 1) + [4]]), pixel_values=pix1)
    with pytest.raises(ValueError, match="consecutive"):
        model(input_ids=torch.tensor([[patch] * (P - 1) + [4, patch]]), pixel_values=pix1)
    assert eng.used == {0}


def test_forward_without_free_slot_borrows_the_lru_cache_slot():
    model, eng, _ = make_model("tiny", max_seqs=1)
    model._slot_tokens = [1, 2, 3]
    ids = torch.randint(0, 400, (1, 7))
    out = model(input_ids=ids, labels=ids)
    assert model._slot_tokens == [] and eng.used == {0}
    ref, _, _ = make_model("tiny")
    assert torch.equal(out.logits, ref(input_ids=ids).logits)


def _reference_scores(oracle, q, start, img=None):
    emb = oracle.spliced_embeds(torch.tensor([q]), None if img is None else img[None])
    with torch.no_grad():
        lp = torch.log_softmax(oracle.llm(inputs_embeds=emb).logits[0].float(), -1)
    return torch.stack([lp[start + k - 1, q[start + k]] for k in range(len(q) - start)])


def _scores(model, eng, seqs, pix=None, start=1):
    eng.calls.clear()
    out = model.score([torch.tensor(q) for q in seqs], pix, start=start)
    calls = [c for c in eng.calls if c[0] in ("prefill", "score", "share")]
    return out, calls


def test_score_prefix_sharing_and_ranges():
    model, eng, oracle = make_model("tiny")
    P, patch = model.config.num_patches, model.config.image_token_id
    S = model.config.vision_config.image_size
    pix = synthetic_pixels(1, S, seed=3)
    img = oracle.image_embeds(pix)[0]
    g = torch.Generator().manual_seed(9)

    def rnd(n):
        return torch.randint(0, 400, (n,), generator=g).tolist()
    head = rnd(20) + [patch] * P            # image span [20, 20 + P)
    seqs = [head + rnd(6), head + rnd(9), head + rnd(4)]

    # scoring starts right after the image span (the v1 prompt layout): the base holds the whole span, each sequence
    # borrows all but its last row and recomputes that row, which predicts the first scored token
    out, calls = _scores(model, eng, seqs, pix, start=len(head))
    assert calls[0] == ("prefill", calls[0][1], 0, len(head), True)
    base = calls[0][1]
    for i, q in enumerate(seqs):
        assert calls[1 + 2 * i][0] == "share" and calls[1 + 2 * i][2:] == (calls[2][1], len(head) - 1)
        assert calls[2 + 2 * i][1:] == (calls[2][1], len(head) - 1, len(q) - len(head), True)
        assert out[i].shape == (len(q) - len(head),)
        assert (out[i] - _reference_scores(oracle, q, len(head), img)).abs().max() < 1e-4
    assert base not in eng.used and eng.used == {0}

    # a cap inside the image span falls back to the span start: the image goes to each sequence's own prefill
    out, calls = _scores(model, eng, seqs, pix, start=len(head) - 2)
    assert calls[0][2:] == (0, 20, False)
    for i, q in enumerate(seqs):
        assert calls[1 + 2 * i][3] == 20 and calls[2 + 2 * i][2:] == (20, len(q) - 21, True)
        assert (out[i] - _reference_scores(oracle, q, len(head) - 2, img)).abs().max() < 1e-4

    # start inside the common prefix: the base holds min(start) positions, each sequence borrows up to start_i - 1
    out, calls = _scores(model, eng, seqs, pix, start=[18, 30, 27])
    assert calls[0][2:] == (0, 18, False)
    for i, (q, st) in enumerate(zip(seqs, [18, 30, 27])):
        s0 = min(18, st - 1)
        assert calls[1 + 2 * i][3] == s0 and calls[2 + 2 * i][2:] == (s0, len(q) - 1 - s0, True)
        assert (out[i] - _reference_scores(oracle, q, st, img)).abs().max() < 1e-4

    # a common prefix shorter than 16 positions is not shared
    short = [rnd(10) + rnd(8) for _ in range(2)]
    short[1][:10] = short[0][:10]
    out, calls = _scores(model, eng, short, start=2)
    assert [c[0] for c in calls] == ["score", "score"] and all(c[2] == 0 for c in calls)
    for i, q in enumerate(short):
        assert (out[i] - _reference_scores(oracle, q, 2)).abs().max() < 1e-4

    # one image per sequence: nothing is shared, each sequence splices its own image
    pix2 = synthetic_pixels(2, S, seed=4)
    imgs = oracle.image_embeds(pix2)
    out, calls = _scores(model, eng, seqs[:2], pix2, start=3)
    assert [c[0] for c in calls] == ["score", "score"] and all(c[2] == 0 and c[4] for c in calls)
    for i in range(2):
        assert (out[i] - _reference_scores(oracle, seqs[i], 3, imgs[i])).abs().max() < 1e-4


def test_score_rejects_bad_start():
    model, _, _ = make_model("tiny")
    for st in (0, 5):
        with pytest.raises(ValueError, match="start"):
            model.score([torch.arange(5)], start=st)
    with pytest.raises(ValueError, match="one int per sequence"):
        model.score([torch.arange(5), torch.arange(6)], start=[1])
    assert model.score([]) == []
