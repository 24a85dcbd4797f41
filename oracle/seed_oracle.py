"""CPU oracle for `seeddot_nll` (SEED-Encoder, model/models.py:201-221).  TEST INFRASTRUCTURE ONLY: only tests/ and
oracle/make_golden_seed.py import it; the product (ance_b200/) never does.

It restates in plain PyTorch (fp32, or fp64 with dtype=torch.float64) what the reference's SEEDEncoderDot_NLL_LN
computes, over the reference's own parameter names.  The encoder half that `query_emb` / `body_emb` run is the fairseq
TransformerSentenceEncoder (num_segments=0, encoder_normalize_before=True, post-LN layers).  Pinned by
tests/golden/encoder_seed.npz and tests/golden/seed_grads.npz, which oracle/make_golden_seed.py generates from the
reference's own class.
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

from ance_b200.synthetic import random_seed_state_dict  # noqa: F401  (seeded checkpoints are data, shared with tools)


def _ln(x, g, b, eps):
    return F.layer_norm(x, (x.shape[-1],), g, b, eps)


class SEEDDotOracle:
    """model/models.py:201-221 (seeddot_nll): the SEED-Encoder's sentence encoder (transformer_sentence_encoder.py:
    695-925, modules.py) -> CLS -> embeddingHead -> norm, restated over the reference's parameter names:
      key padding mask = ids == pad_token_id (the attention_mask argument is ignored), masked keys get -inf
      positions        = make_positions: cumsum(ids != pad) * (ids != pad) + pad                  (modules.py:89-99)
      x                = emb_layer_norm(embed_tokens[ids] + embed_positions[positions]), padding rows zeroed
      layer            = LN(out_proj(attn(x)) + x) ; LN(fc2(gelu_erf(fc1(.))) + .), every LayerNorm at eps 1e-5
    No gradient mode is imposed: with parameters that require grad (`leaves()`) the embeddings are differentiable.
    `dtype` float64 gives the fp64 restatement.  A row made only of padding yields NaN, as the reference's does."""

    P = "seed_encoder.encoder.sentence_encoder."

    def __init__(self, sd, n_layer=12, heads=12, pad_id=1, dtype=torch.float32, device="cpu"):
        self.sd = {k: v.detach().to(device=device, dtype=dtype) for k, v in sd.items()
                   if not k.startswith("classification_heads.")}
        self.n_layer, self.heads, self.pad_id = n_layer, heads, pad_id
        self.device, self.dtype = torch.device(device), dtype

    def leaves(self) -> Dict[str, torch.Tensor]:
        """Make every parameter a leaf that requires grad; -> the dict (reference names) whose .grad autograd fills."""
        self.sd = {k: v.detach().clone().requires_grad_(True) for k, v in self.sd.items()}
        return self.sd

    def w(self, name):
        return self.sd[self.P + name]

    def query_emb(self, input_ids, attention_mask=None):
        ids = torch.as_tensor(input_ids).long().to(self.device)
        B, L = ids.shape
        pad = ids.eq(self.pad_id)
        keep = (~pad).long()
        pos = torch.cumsum(keep, dim=1) * keep + self.pad_id
        x = self.w("embed_tokens.weight")[ids] + self.w("embed_positions.weight")[pos]
        x = _ln(x, self.w("emb_layer_norm.weight"), self.w("emb_layer_norm.bias"), 1e-5)
        x = x * (~pad).unsqueeze(-1).to(x.dtype)
        kbias = torch.zeros((B, 1, 1, L), dtype=x.dtype, device=x.device).masked_fill(pad[:, None, None, :],
                                                                                       float("-inf"))
        H = x.shape[-1]
        dh = H // self.heads
        for l in range(self.n_layer):
            lp = f"layers.{l}."

            def lin(nm, t):
                return F.linear(t, self.w(lp + nm + ".weight"), self.w(lp + nm + ".bias"))

            q = (lin("self_attn.q_proj", x) * dh ** -0.5).view(B, L, self.heads, dh).transpose(1, 2)
            k = lin("self_attn.k_proj", x).view(B, L, self.heads, dh).transpose(1, 2)
            v = lin("self_attn.v_proj", x).view(B, L, self.heads, dh).transpose(1, 2)
            a = torch.softmax(q @ k.transpose(-1, -2) + kbias, dim=-1) @ v
            a = lin("self_attn.out_proj", a.transpose(1, 2).reshape(B, L, H))
            x = _ln(a + x, self.w(lp + "self_attn_layer_norm.weight"), self.w(lp + "self_attn_layer_norm.bias"), 1e-5)
            h = lin("fc2", F.gelu(lin("fc1", x)))
            x = _ln(h + x, self.w(lp + "final_layer_norm.weight"), self.w(lp + "final_layer_norm.bias"), 1e-5)
        cls = F.linear(x[:, 0], self.sd["embeddingHead.weight"], self.sd["embeddingHead.bias"])
        return _ln(cls, self.sd["norm.weight"], self.sd["norm.bias"], 1e-5)

    def body_emb(self, input_ids, attention_mask=None):
        return self.query_emb(input_ids, attention_mask)

    def nll_loss(self, q_ids, a_ids, b_ids):
        """NLL.forward's triplet loss (models.py:58-84): mean of -log_softmax([q.a, q.b])[0]."""
        q, a, b = self.query_emb(q_ids), self.body_emb(a_ids), self.body_emb(b_ids)
        lm = torch.stack([(q * a).sum(-1), (q * b).sum(-1)], dim=1)
        return (-torch.log_softmax(lm, dim=1)[:, 0]).mean()


def grad_sketch(g: torch.Tensor, name: str, k: int = 4) -> torch.Tensor:
    """A gradient's fingerprint: [norm, k projections onto unit random directions seeded by the tensor's name], fp64."""
    g = g.detach().double().reshape(-1).cpu()
    gen = torch.Generator().manual_seed(sum((i + 1) * ord(c) for i, c in enumerate(name)))
    d = torch.randn(k, g.numel(), generator=gen, dtype=torch.float64)
    d = d / d.norm(dim=1, keepdim=True)
    return torch.cat([g.norm().reshape(1), d @ g])


