"""BERT for pre-training (MLM + NSP) with the reference's *untied* decoder.

Architecture parity with ``BERT/bert/transformers/modeling.py:59-522`` (``BertConfig``, embeddings,
self-attention, ``BertLayer``, pooler, ``BertPreTrainingHeads``) and with the stage-split module lists
``BERT/bert/models/bert/depth=N`` (``StartingStage`` = embeddings + L/N layers, ``IntermediateStage``,
``EndingStage`` = layers + pooler + heads, whose decoder matrix is a *fresh* embedding-shaped
parameter, ``depth=4/__init__.py:17``) => BERT-base has 133,547,324 parameters, the paper's 133.5 M.

Fresh implementation: fused QKV projection, ``F.scaled_dot_product_attention`` (the reference does
matmul -> softmax -> matmul on the full [B,12,S,S] score tensor), ``F.layer_norm`` instead of apex, or with
``fuse_ln=True`` the encoder's dropout + residual + LayerNorm sites on the fused kernels of ``ops/fused_ln.py``, and
with ``fuse_xent=True`` the masked-LM loss on the fused softmax cross-entropy of ``ops/fused_xent.py``, and with
``sparse_mlm=True`` the masked-LM head on the labelled rows only, gathered by ``ops/mlm_gather.py``, and with
``fuse_attn=True`` self-attention on the fused kernels of ``ops/fused_attn.py``, and with ``fuse_emb=True`` the
embedding sum + LayerNorm + dropout on the fused kernels of ``ops/fused_emb.py``.
"""
from __future__ import annotations

import json
import math
from dataclasses import dataclass
from typing import List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F


@dataclass
class BertConfig:
    vocab_size: int = 30522
    hidden_size: int = 768
    num_hidden_layers: int = 12
    num_attention_heads: int = 12
    intermediate_size: int = 3072
    hidden_act: str = "gelu"
    hidden_dropout_prob: float = 0.1
    attention_probs_dropout_prob: float = 0.1
    max_position_embeddings: int = 512
    type_vocab_size: int = 2
    initializer_range: float = 0.02
    layer_norm_eps: float = 1e-12

    @classmethod
    def from_json_file(cls, path: str) -> "BertConfig":
        with open(path) as f:
            d = json.load(f)
        return cls(**{k: v for k, v in d.items() if k in cls.__dataclass_fields__})

    @classmethod
    def bert_base(cls) -> "BertConfig":
        return cls()

    @classmethod
    def bert_large(cls) -> "BertConfig":
        return cls(hidden_size=1024, num_hidden_layers=24, num_attention_heads=16, intermediate_size=4096)


def _act(name: str):
    return {"gelu": F.gelu, "relu": F.relu, "tanh": torch.tanh}[name]


class BertEmbeddings(nn.Module):
    """``fuse_emb`` (default off) runs the whole block through the fused kernels of ``ops/fused_emb.py``, which count
    ids and token types outside their tables in the non-persistent buffer ``id_overflow`` instead of faulting;
    parameters and ``state_dict`` keys are the same either way."""

    def __init__(self, c: BertConfig):
        super().__init__()
        self.word_embeddings = nn.Embedding(c.vocab_size, c.hidden_size)
        self.position_embeddings = nn.Embedding(c.max_position_embeddings, c.hidden_size)
        self.token_type_embeddings = nn.Embedding(c.type_vocab_size, c.hidden_size)
        self.LayerNorm = nn.LayerNorm(c.hidden_size, eps=c.layer_norm_eps)
        self.dropout = nn.Dropout(c.hidden_dropout_prob)
        self.fuse_emb = False
        self.register_buffer("id_overflow", torch.zeros(1, dtype=torch.int64), persistent=False)

    def forward(self, input_ids: torch.Tensor, token_type_ids: torch.Tensor) -> torch.Tensor:
        if self.fuse_emb:
            from ..ops.fused_emb import embedding_layer_norm
            return embedding_layer_norm(input_ids, token_type_ids, self, self.dropout.p if self.training else 0.0)
        pos = torch.arange(input_ids.size(1), device=input_ids.device).unsqueeze(0)
        e = self.word_embeddings(input_ids) + self.position_embeddings(pos) + self.token_type_embeddings(token_type_ids)
        return self.dropout(self.LayerNorm(e))


class BertSelfAttention(nn.Module):
    """``fuse_attn`` (default off) runs the attention of the packed projection through the fused kernels of
    ``ops/fused_attn.py``; parameters, buffers and ``state_dict`` keys are the same either way."""

    def __init__(self, c: BertConfig):
        super().__init__()
        self.h, self.dh = c.num_attention_heads, c.hidden_size // c.num_attention_heads
        self.qkv = nn.Linear(c.hidden_size, 3 * c.hidden_size)          # same parameter count as 3 separate projections
        self.p_drop = c.attention_probs_dropout_prob
        self.fuse_attn = False

    def forward(self, x: torch.Tensor, mask: Optional[torch.Tensor]) -> torch.Tensor:
        if self.fuse_attn:
            from ..ops.fused_attn import self_attention
            return self_attention(self.qkv(x), self.h, mask, self.p_drop if self.training else 0.0)
        b, s, _ = x.shape
        q, k, v = self.qkv(x).view(b, s, 3, self.h, self.dh).permute(2, 0, 3, 1, 4)
        o = F.scaled_dot_product_attention(q, k, v, attn_mask=mask, dropout_p=self.p_drop if self.training else 0.0)
        return o.transpose(1, 2).reshape(b, s, self.h * self.dh)


class BertLayer(nn.Module):
    """``fuse_ln`` (default off) runs both ``LayerNorm(x + dropout(a))`` sites through the fused kernels of
    ``ops/fused_ln.py``; parameters, buffers and ``state_dict`` keys are the same either way."""

    def __init__(self, c: BertConfig):
        super().__init__()
        self.fuse_ln = False
        self.attention = BertSelfAttention(c)
        self.attn_out = nn.Linear(c.hidden_size, c.hidden_size)
        self.attn_norm = nn.LayerNorm(c.hidden_size, eps=c.layer_norm_eps)
        self.intermediate = nn.Linear(c.hidden_size, c.intermediate_size)
        self.output = nn.Linear(c.intermediate_size, c.hidden_size)
        self.out_norm = nn.LayerNorm(c.hidden_size, eps=c.layer_norm_eps)
        self.dropout = nn.Dropout(c.hidden_dropout_prob)
        self.act = _act(c.hidden_act)

    def forward(self, x: torch.Tensor, mask: Optional[torch.Tensor]) -> torch.Tensor:
        if self.fuse_ln:
            from ..ops.fused_ln import residual_dropout_layer_norm
            p = self.dropout.p if self.training else 0.0
            x = residual_dropout_layer_norm(x, self.attn_out(self.attention(x, mask)), self.attn_norm, p)
            return residual_dropout_layer_norm(x, self.output(self.act(self.intermediate(x))), self.out_norm, p)
        a = self.dropout(self.attn_out(self.attention(x, mask)))
        x = self.attn_norm(x + a)
        f = self.dropout(self.output(self.act(self.intermediate(x))))
        return self.out_norm(x + f)


class BertPooler(nn.Module):
    def __init__(self, c: BertConfig):
        super().__init__()
        self.dense = nn.Linear(c.hidden_size, c.hidden_size)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return torch.tanh(self.dense(x[:, 0]))


class BertPreTrainingHeads(nn.Module):
    """MLM head (dense + act + LN + decoder) and NSP head.  ``decoder_weight`` is an independent
    ``[vocab, hidden]`` parameter (untied, see module docstring) plus a vocab-sized bias.

    ``forward(seq, pooled)`` returns ``(scores [B, S, V], nsp)``.  Given the masked-LM labels ``[B, S]`` (-1 = not
    masked) it also returns the targets of the scores' rows: with ``sparse_mlm`` off ``(scores [B, S, V], nsp,
    labels)``; with it on the MLM head runs on the labelled rows only, gathered by ``ops/mlm_gather.py`` into
    ``capacity_rows(B S, mlm_capacity)`` rows, and returns ``(scores [M, V], nsp, tgt [M])``.  Labelled rows past the
    capacity are left out of the loss and counted in the non-persistent buffer ``mlm_overflow``."""

    def __init__(self, c: BertConfig):
        super().__init__()
        self.transform = nn.Linear(c.hidden_size, c.hidden_size)
        self.transform_norm = nn.LayerNorm(c.hidden_size, eps=c.layer_norm_eps)
        self.act = _act(c.hidden_act)
        self.decoder_weight = nn.Parameter(torch.empty(c.vocab_size, c.hidden_size).normal_(std=c.initializer_range))
        self.decoder_bias = nn.Parameter(torch.zeros(c.vocab_size))
        self.seq_relationship = nn.Linear(c.hidden_size, 2)
        self.sparse_mlm = False
        self.mlm_capacity = 0.25
        self.register_buffer("mlm_overflow", torch.zeros(1, dtype=torch.int64), persistent=False)

    def forward(self, seq: torch.Tensor, pooled: torch.Tensor, labels: Optional[torch.Tensor] = None):
        if labels is not None and self.sparse_mlm:
            from ..ops.mlm_gather import capacity_rows, gather_labelled
            m = capacity_rows(labels.numel(), self.mlm_capacity)
            xg, tgt = gather_labelled(seq.reshape(-1, seq.size(-1)), labels.reshape(-1), m, -1, self.mlm_overflow)
            h = self.transform_norm(self.act(self.transform(xg)))
            return F.linear(h, self.decoder_weight, self.decoder_bias), self.seq_relationship(pooled), tgt
        h = self.transform_norm(self.act(self.transform(seq)))
        scores, nsp = F.linear(h, self.decoder_weight, self.decoder_bias), self.seq_relationship(pooled)
        return (scores, nsp) if labels is None else (scores, nsp, labels)


def extended_attention_mask(input_mask: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
    """``(1 - m) * -10000`` additive mask ``[B,1,1,S]`` (``BERT/bert/main_bert.py:616-639``)."""
    return ((1.0 - input_mask[:, None, None, :].to(dtype)) * -10000.0)


# ---- stage-split module lists (depth=N) --------------------------------------------------------
class StartingStage(nn.Module):
    def __init__(self, c: BertConfig, n_layers: int):
        super().__init__()
        self.embeddings = BertEmbeddings(c)
        self.layers = nn.ModuleList(BertLayer(c) for _ in range(n_layers))

    def forward(self, input_ids, token_type_ids, mask):
        x = self.embeddings(input_ids, token_type_ids)
        for l in self.layers:
            x = l(x, mask)
        return x


class IntermediateStage(nn.Module):
    def __init__(self, c: BertConfig, n_layers: int):
        super().__init__()
        self.layers = nn.ModuleList(BertLayer(c) for _ in range(n_layers))

    def forward(self, x, mask):
        for l in self.layers:
            x = l(x, mask)
        return x


class EndingStage(nn.Module):
    def __init__(self, c: BertConfig, n_layers: int):
        super().__init__()
        self.layers = nn.ModuleList(BertLayer(c) for _ in range(n_layers))
        self.pooler = BertPooler(c)
        self.heads = BertPreTrainingHeads(c)

    def forward(self, x, mask, labels=None):
        for l in self.layers:
            x = l(x, mask)
        return self.heads(x, self.pooler(x), labels)


def build_stages(c: BertConfig, depth: int = 4) -> List[nn.Module]:
    """``models.bert<L>.depth=<N>``: N sub-modules run back to back on one GPU (the reference's
    data-parallel ``StageRuntime`` instantiates every stage on every rank, ``BERT/runtime.py:128-151``)."""
    L = c.num_hidden_layers
    assert depth >= 2 and L % depth == 0, "depth must divide the layer count"
    per = L // depth
    return [StartingStage(c, per)] + [IntermediateStage(c, per) for _ in range(depth - 2)] + [EndingStage(c, per)]


class PretrainingCriterion(nn.Module):
    """CE(MLM, ignore_index=-1) + CE(NSP) (``BERT/runtime.py:585-596``).  ``fuse_xent`` (default off) runs the MLM term
    through the fused softmax cross-entropy of ``ops/fused_xent.py``; the NSP term stays stock."""

    def __init__(self, vocab_size: int):
        super().__init__()
        self.vocab_size = vocab_size
        self.fuse_xent = False

    def forward(self, prediction_scores, seq_relationship_score, masked_lm_labels, next_sentence_labels):
        scores, labels = prediction_scores.view(-1, self.vocab_size), masked_lm_labels.view(-1)
        if self.fuse_xent:
            from ..ops.fused_xent import softmax_cross_entropy
            mlm = softmax_cross_entropy(scores, labels, ignore_index=-1)
        else:
            mlm = F.cross_entropy(scores, labels, ignore_index=-1)
        nsp = F.cross_entropy(seq_relationship_score.view(-1, 2), next_sentence_labels.view(-1))
        return mlm + nsp


class BertForPreTraining(nn.Module):
    """``fuse_ln=True`` (or ``net.fuse_ln = True`` at any time) sets ``BertLayer.fuse_ln`` on every encoder layer;
    ``fuse_xent=True`` (or ``net.fuse_xent``) sets ``PretrainingCriterion.fuse_xent``; ``sparse_mlm=True`` (or
    ``net.sparse_mlm``) runs the masked-LM head on the labelled rows only when labels are given, gathered into
    ``mlm_capacity`` (or ``net.mlm_capacity``) times B·S rows, rounded up to a multiple of 8 (``BertPreTrainingHeads``);
    ``fuse_attn=True`` (or ``net.fuse_attn``) sets ``BertSelfAttention.fuse_attn`` on every encoder layer;
    ``fuse_emb=True`` (or ``net.fuse_emb``) sets ``BertEmbeddings.fuse_emb``."""

    def __init__(self, config: Optional[BertConfig] = None, depth: int = 4, recompute: bool = False,
                 fuse_ln: bool = False, fuse_xent: bool = False, sparse_mlm: bool = False, mlm_capacity: float = 0.25,
                 fuse_attn: bool = False, fuse_emb: bool = False):
        super().__init__()
        self.config = config or BertConfig()
        self.recompute = recompute           # ``--recompute_step`` (BERT/runtime.py:546-557, modeling.py:414-431)
        self.stages = nn.ModuleList(build_stages(self.config, depth))
        self.criterion = PretrainingCriterion(self.config.vocab_size)
        self.apply(self._init)
        nn.init.normal_(self.stages[-1].heads.decoder_weight, std=self.config.initializer_range)
        self.fuse_ln = fuse_ln
        self.fuse_xent = fuse_xent
        self.sparse_mlm = sparse_mlm
        self.mlm_capacity = mlm_capacity
        self.fuse_attn = fuse_attn
        self.fuse_emb = fuse_emb

    @property
    def fuse_emb(self) -> bool:
        """True when the embedding sum + LayerNorm + dropout runs through the fused kernels."""
        return self.stages[0].embeddings.fuse_emb

    @fuse_emb.setter
    def fuse_emb(self, on: bool) -> None:
        self.stages[0].embeddings.fuse_emb = bool(on)

    @property
    def fuse_attn(self) -> bool:
        """True when every encoder layer runs its self-attention through the fused kernels."""
        return all(m.fuse_attn for m in self.modules() if isinstance(m, BertSelfAttention))

    @fuse_attn.setter
    def fuse_attn(self, on: bool) -> None:
        for m in self.modules():
            if isinstance(m, BertSelfAttention):
                m.fuse_attn = bool(on)

    @property
    def sparse_mlm(self) -> bool:
        """True when the masked-LM head runs on the gathered labelled rows only."""
        return self.stages[-1].heads.sparse_mlm

    @sparse_mlm.setter
    def sparse_mlm(self, on: bool) -> None:
        self.stages[-1].heads.sparse_mlm = bool(on)

    @property
    def mlm_capacity(self) -> float:
        """The gathered rows of the sparse masked-LM head, as a fraction of the batch's B·S token rows."""
        return self.stages[-1].heads.mlm_capacity

    @mlm_capacity.setter
    def mlm_capacity(self, fraction: float) -> None:
        from ..ops.mlm_gather import capacity_rows
        capacity_rows(1, fraction)                           # validates: 0 < fraction <= 1
        self.stages[-1].heads.mlm_capacity = float(fraction)

    @property
    def fuse_xent(self) -> bool:
        """True when the masked-LM loss runs through the fused softmax cross-entropy."""
        return self.criterion.fuse_xent

    @fuse_xent.setter
    def fuse_xent(self, on: bool) -> None:
        self.criterion.fuse_xent = bool(on)

    @property
    def fuse_ln(self) -> bool:
        """True when every encoder layer runs its two residual LayerNorms through the fused kernels."""
        return all(m.fuse_ln for m in self.modules() if isinstance(m, BertLayer))

    @fuse_ln.setter
    def fuse_ln(self, on: bool) -> None:
        for m in self.modules():
            if isinstance(m, BertLayer):
                m.fuse_ln = bool(on)

    def _init(self, m: nn.Module) -> None:
        if isinstance(m, (nn.Linear, nn.Embedding)):
            nn.init.normal_(m.weight, std=self.config.initializer_range)
            if isinstance(m, nn.Linear) and m.bias is not None:
                nn.init.zeros_(m.bias)
        elif isinstance(m, nn.LayerNorm):
            nn.init.ones_(m.weight)
            nn.init.zeros_(m.bias)

    def forward(self, input_ids, token_type_ids=None, attention_mask=None, masked_lm_labels=None,
                next_sentence_label=None):
        if token_type_ids is None:
            token_type_ids = torch.zeros_like(input_ids)
        mask = None if attention_mask is None else extended_attention_mask(attention_mask)
        x = self.stages[0](input_ids, token_type_ids, mask)
        for st in self.stages[1:-1]:
            if self.recompute and self.training:
                from torch.utils.checkpoint import checkpoint
                x = checkpoint(st, x, mask, use_reentrant=False)
            else:
                x = st(x, mask)
        if self.sparse_mlm and masked_lm_labels is not None and next_sentence_label is not None:
            scores, nsp, tgt = self.stages[-1](x, mask, masked_lm_labels)
            return self.criterion(scores, nsp, tgt, next_sentence_label)
        scores, nsp = self.stages[-1](x, mask)
        if masked_lm_labels is not None and next_sentence_label is not None:
            return self.criterion(scores, nsp, masked_lm_labels, next_sentence_label)
        return scores, nsp


def bert_base(depth: int = 4) -> BertForPreTraining:
    return BertForPreTraining(BertConfig.bert_base(), depth)


def synthetic_batch(batch: int, seq: int, vocab: int = 30522, device="cpu", generator=None, mask_prob: float = 0.15):
    """Wikipedia-shaped synthetic pre-training batch: ``input_ids, segment_ids, input_mask, lm_label_ids`` of
    ``[B,S]`` int64 (-1 = not masked) and ``is_next [B]`` (``BERT/bert/main_bert.py:535-614`` feature layout)."""
    g = generator
    ids = torch.randint(1000, vocab, (batch, seq), generator=g)
    seg = (torch.arange(seq).unsqueeze(0) >= torch.randint(seq // 4, 3 * seq // 4, (batch, 1), generator=g)).long()
    lens = torch.randint(seq // 2, seq + 1, (batch, 1), generator=g)
    mask = (torch.arange(seq).unsqueeze(0) < lens).long()
    sel = (torch.rand(batch, seq, generator=g) < mask_prob) & mask.bool()
    labels = torch.where(sel, ids, torch.full_like(ids, -1))
    ids = torch.where(sel, torch.full_like(ids, 103), ids) * mask
    is_next = torch.randint(0, 2, (batch,), generator=g)
    out = (ids, seg, mask, labels, is_next)
    return tuple(t.to(device) for t in out)
