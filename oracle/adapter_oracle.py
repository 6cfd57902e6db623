"""
TEST INFRASTRUCTURE — NOT PRODUCT CODE. fp32 CPU oracle of the TikZero text-conditioned path.

The caption embedder is the installed transformers ``LlamaModel`` (``last_hidden_state``: final RMSNorm applied); the adapter
is restated from the reference (detikzify/model/adapter/modeling_adapter.py):

  * connector ``Linear(E -> D, bias)``                                 .. :372-376, :499-502
  * cross layer before vision layer l iff (l + 1) % n == 0, as a forward pre-hook of that layer (it sees the residual stream
    entering the layer)                                               .. :365-370, :494-509
  * x += sigmoid(g_attn) * out_proj(attn(LN1 x, cond));  x += sigmoid(g_mlp) * fc2(act(fc1(LN2 x)))        .. :326-352
  * attention: q = q_proj(x), k / v = k_proj / v_proj(cond), split into heads, per-head LayerNorm q_norm / k_norm, scale
    head_dim^-1/2, padded caption keys masked (``_prepare_4d_attention_mask``), softmax in fp32   .. :38-120, :386-391
  * without pixel_values the tower input is ``dummy_input.clamp(-1, 1)``                                   .. :486-491

Decoder, projector and splice are ``hf_oracle.Oracle``'s.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import torch
import torch.nn.functional as F
from transformers import LlamaConfig, LlamaModel

from .hf_oracle import Oracle

EMB, AD = "embedding_model.", "adapter."


def embedder(acfg, state_dict: Dict[str, torch.Tensor]) -> LlamaModel:
    lcfg = LlamaConfig(
        hidden_size=acfg.hidden_size, intermediate_size=acfg.intermediate_size, num_hidden_layers=acfg.num_hidden_layers,
        num_attention_heads=acfg.num_attention_heads, num_key_value_heads=acfg.num_key_value_heads, head_dim=acfg.head_dim,
        vocab_size=acfg.vocab_size, max_position_embeddings=131072, rms_norm_eps=acfg.rms_norm_eps, rope_theta=acfg.rope_theta,
        rope_scaling=({"rope_type": "llama3", "factor": acfg.rope_factor, "low_freq_factor": acfg.rope_low_freq_factor,
                       "high_freq_factor": acfg.rope_high_freq_factor,
                       "original_max_position_embeddings": acfg.rope_original_max_position}
                      if acfg.rope_type == "llama3" else None),
        hidden_act="silu", attention_bias=False, mlp_bias=False, pad_token_id=acfg.pad_token_id, attn_implementation="eager")
    with torch.device("meta"):
        m = LlamaModel(lcfg)
    m = m.to_empty(device="cpu")
    sd = {k[len(EMB):]: v.float() for k, v in state_dict.items() if k.startswith(EMB)}
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    assert all("rotary" in k or "inv_freq" in k for k in missing), missing
    m.rotary_emb = type(m.rotary_emb)(lcfg)
    return m.float().eval()


class AdapterOracle(Oracle):
    def __init__(self, cfg: dict, state_dict: Dict[str, torch.Tensor], acfg, adapter_state_dict: Dict[str, torch.Tensor]):
        super().__init__(cfg, state_dict)
        self.acfg = acfg
        self.emb = embedder(acfg, adapter_state_dict)
        self.ad = {k[len(AD):]: v.float() for k, v in adapter_state_dict.items() if k.startswith(AD)}
        vc = cfg["vision_config"]
        self.heads, self.eps = vc["num_attention_heads"], vc["layer_norm_eps"]
        self.act = {"gelu_pytorch_tanh": lambda x: F.gelu(x, approximate="tanh"), "gelu": F.gelu}[vc["hidden_act"]]
        self._cond = None

    @torch.no_grad()
    def caption_states(self, ids: torch.Tensor, mask: Optional[torch.Tensor] = None):
        """(embedder last_hidden_state [B,T,E], connector output [B,T,D]) of a right-padded caption batch."""
        ids = ids[None] if ids.dim() == 1 else ids
        h = self.emb(input_ids=ids, attention_mask=mask).last_hidden_state
        return h, F.linear(h, self.ad["connector.weight"], self.ad["connector.bias"])

    def _cross(self, l: int, x: torch.Tensor, cond: torch.Tensor, mask: Optional[torch.Tensor]) -> torch.Tensor:
        p = f"layers.{l}."
        w = lambda n: self.ad[p + n]
        D = x.shape[-1]
        dh = D // self.heads
        h = F.layer_norm(x, (D,), w("layer_norm1.weight"), w("layer_norm1.bias"), self.eps)
        B, Nq, Tk = x.shape[0], x.shape[1], cond.shape[1]
        q = F.linear(h, w("cross_attn.q_proj.weight"), w("cross_attn.q_proj.bias")).view(B, Nq, self.heads, dh).transpose(1, 2)
        k = F.linear(cond, w("cross_attn.k_proj.weight"), w("cross_attn.k_proj.bias")).view(B, Tk, self.heads, dh).transpose(1, 2)
        v = F.linear(cond, w("cross_attn.v_proj.weight"), w("cross_attn.v_proj.bias")).view(B, Tk, self.heads, dh).transpose(1, 2)
        q = F.layer_norm(q, (dh,), w("cross_attn.q_norm.weight"), w("cross_attn.q_norm.bias"), self.eps)
        k = F.layer_norm(k, (dh,), w("cross_attn.k_norm.weight"), w("cross_attn.k_norm.bias"), self.eps)
        s = q @ k.transpose(2, 3) * dh ** -0.5
        if mask is not None:
            s = s.masked_fill(~mask.bool()[:, None, None, :], torch.finfo(s.dtype).min)
        a = (torch.softmax(s, dim=-1, dtype=torch.float32) @ v).transpose(1, 2).reshape(B, Nq, D)
        x = x + torch.sigmoid(w("cross_attn_attn_gate")) * F.linear(a, w("cross_attn.out_proj.weight"), w("cross_attn.out_proj.bias"))
        h = F.layer_norm(x, (D,), w("layer_norm2.weight"), w("layer_norm2.bias"), self.eps)
        h = F.linear(self.act(F.linear(h, w("mlp.fc1.weight"), w("mlp.fc1.bias"))), w("mlp.fc2.weight"), w("mlp.fc2.bias"))
        return x + torch.sigmoid(w("cross_attn_mlp_gate")) * h

    def dummy_pixels(self, batch: int = 1) -> torch.Tensor:
        return self.ad["dummy_input"].clamp(-1, 1)[None].repeat(batch, 1, 1, 1)

    @torch.no_grad()
    def vision_cond(self, pixel_values: Optional[torch.Tensor], ids: torch.Tensor, mask: Optional[torch.Tensor] = None):
        """Adapted tower: (last_hidden_state, pooler_output); pixel_values None -> the clamped dummy input."""
        ids = ids[None] if ids.dim() == 1 else ids
        if pixel_values is None:
            pixel_values = self.dummy_pixels(ids.shape[0])
        _, cond = self.caption_states(ids, mask)
        vm = self.vit.vision_model
        x = vm.embeddings(pixel_values.float())
        n = self.acfg.cross_attn_every_n_layers
        for l, layer in enumerate(vm.encoder.layers):
            if (l + 1) % n == 0:
                x = self._cross(l, x, cond, mask)
            out = layer(x, None)
            x = out[0] if isinstance(out, tuple) else out
        x = vm.post_layernorm(x)
        return x, vm.head(x)

    def vision(self, pixel_values: torch.Tensor):
        if self._cond is None:
            return super().vision(pixel_values)
        return self.vision_cond(pixel_values, *self._cond)

    @torch.no_grad()
    def forward_logits_cond(self, input_ids: torch.Tensor, pixel_values: Optional[torch.Tensor], caption: torch.Tensor):
        """Prefill logits of a prompt whose image span is encoded by the adapted tower under ``caption``."""
        self._cond = (caption[None] if caption.dim() == 1 else caption, None)
        try:
            pix = pixel_values if pixel_values is not None else self.dummy_pixels()
            return self.forward_logits(input_ids, pix)[0]
        finally:
            self._cond = None

    @torch.no_grad()
    def generate_cond(self, input_ids: torch.Tensor, pixel_values: Optional[torch.Tensor], caption: torch.Tensor,
                      max_length: int) -> torch.Tensor:
        self._cond = (caption[None] if caption.dim() == 1 else caption, None)
        try:
            pix = pixel_values if pixel_values is not None else self.dummy_pixels()
            return self.generate(input_ids, pix, max_length)
        finally:
            self._cond = None
