"""BERT task models on top of the stage-split encoder: ``BertModel`` and the fine-tuning heads of the reference's
``modeling.py`` (``BertForMaskedLM :828``, ``BertForNextSentencePrediction :889``, ``BertForSequenceClassification :950``,
``BertForMultipleChoice :1016``, ``BertForTokenClassification :1085``, ``BertForQuestionAnswering :1159``).

All of them share one encoder class (the same ``StartingStage`` / ``IntermediateStage`` blocks the pre-training model is
built from, so a pre-training checkpoint loads into any head with ``load_pretraining_encoder``), use the fused-QKV /
SDPA attention of ``models/bert.py`` and return the loss when labels are given, logits otherwise — the reference's
calling convention.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .bert import (BertConfig, BertLayer, BertEmbeddings, BertPooler, BertPreTrainingHeads, extended_attention_mask)


class BertModel(nn.Module):
    """Embeddings + L transformer layers + pooler; returns ``(sequence_output, pooled_output)``."""

    def __init__(self, config: Optional[BertConfig] = None):
        super().__init__()
        self.config = config or BertConfig()
        c = self.config
        self.embeddings = BertEmbeddings(c)
        self.layers = nn.ModuleList(BertLayer(c) for _ in range(c.num_hidden_layers))
        self.pooler = BertPooler(c)
        self.apply(self._init)

    def _init(self, m: nn.Module) -> None:
        if isinstance(m, (nn.Linear, nn.Embedding)):
            nn.init.normal_(m.weight, std=self.config.initializer_range)
            if isinstance(m, nn.Linear) and m.bias is not None:
                nn.init.zeros_(m.bias)
        elif isinstance(m, nn.LayerNorm):
            nn.init.ones_(m.weight)
            nn.init.zeros_(m.bias)

    def forward(self, input_ids, token_type_ids=None, attention_mask=None):
        if token_type_ids is None:
            token_type_ids = torch.zeros_like(input_ids)
        mask = None if attention_mask is None else extended_attention_mask(attention_mask)
        x = self.embeddings(input_ids, token_type_ids)
        for l in self.layers:
            x = l(x, mask)
        return x, self.pooler(x)


def load_pretraining_encoder(model: nn.Module, pretraining_state: dict) -> int:
    """Copy the encoder of a ``BertForPreTraining`` checkpoint (``stages.N.*`` names) into ``model.bert``; returns the
    number of tensors loaded (the reference re-maps its per-stage checkpoints in ``compute_glue_scores.py:698-760``)."""
    bert: BertModel = model.bert if hasattr(model, "bert") else model
    own = bert.state_dict()
    per_stage = {}
    for k in pretraining_state:
        if k.startswith("stages."):
            s = int(k.split(".")[1])
            if ".layers." in k:
                li = int(k.split(".layers.")[1].split(".")[0])
                per_stage[s] = max(per_stage.get(s, 0), li + 1)
    loaded, base = 0, {}
    acc = 0
    for s in sorted(per_stage):
        base[s] = acc
        acc += per_stage[s]
    for k, v in pretraining_state.items():
        if not k.startswith("stages."):
            continue
        parts = k.split(".")
        s, rest = int(parts[1]), ".".join(parts[2:])
        if rest.startswith("layers."):
            li = int(rest.split(".")[1])
            name = "layers.%d.%s" % (base.get(s, 0) + li, ".".join(rest.split(".")[2:]))
        elif rest.startswith(("embeddings.", "pooler.")):
            name = rest
        else:
            continue
        if name in own and own[name].shape == v.shape:
            own[name].copy_(v)
            loaded += 1
    return loaded


class _Head(nn.Module):
    def __init__(self, config: Optional[BertConfig]):
        super().__init__()
        self.config = config or BertConfig()
        self.bert = BertModel(self.config)
        self.dropout = nn.Dropout(self.config.hidden_dropout_prob)

    def _init_head(self, *mods: nn.Module) -> None:
        for m in mods:
            nn.init.normal_(m.weight, std=self.config.initializer_range)
            nn.init.zeros_(m.bias)


class BertForSequenceClassification(_Head):
    def __init__(self, config: Optional[BertConfig] = None, num_labels: int = 2):
        super().__init__(config)
        self.num_labels = num_labels
        self.classifier = nn.Linear(self.config.hidden_size, num_labels)
        self._init_head(self.classifier)

    def forward(self, input_ids, token_type_ids=None, attention_mask=None, labels=None):
        _, pooled = self.bert(input_ids, token_type_ids, attention_mask)
        logits = self.classifier(self.dropout(pooled))
        if labels is None:
            return logits
        if self.num_labels == 1:                                  # regression (STS-B)
            return F.mse_loss(logits.view(-1), labels.view(-1).float())
        return F.cross_entropy(logits.view(-1, self.num_labels), labels.view(-1))


class BertForMultipleChoice(_Head):
    def __init__(self, config: Optional[BertConfig] = None, num_choices: int = 2):
        super().__init__(config)
        self.num_choices = num_choices
        self.classifier = nn.Linear(self.config.hidden_size, 1)
        self._init_head(self.classifier)

    def forward(self, input_ids, token_type_ids=None, attention_mask=None, labels=None):
        flat = lambda t: None if t is None else t.view(-1, t.size(-1))   # noqa: E731
        _, pooled = self.bert(flat(input_ids), flat(token_type_ids), flat(attention_mask))
        logits = self.classifier(self.dropout(pooled)).view(-1, self.num_choices)
        return logits if labels is None else F.cross_entropy(logits, labels)


class BertForTokenClassification(_Head):
    def __init__(self, config: Optional[BertConfig] = None, num_labels: int = 2):
        super().__init__(config)
        self.num_labels = num_labels
        self.classifier = nn.Linear(self.config.hidden_size, num_labels)
        self._init_head(self.classifier)

    def forward(self, input_ids, token_type_ids=None, attention_mask=None, labels=None):
        seq, _ = self.bert(input_ids, token_type_ids, attention_mask)
        logits = self.classifier(self.dropout(seq))
        if labels is None:
            return logits
        if attention_mask is not None:                            # loss only on real tokens (modeling.py:1147-1153)
            active = attention_mask.view(-1) == 1
            return F.cross_entropy(logits.view(-1, self.num_labels)[active], labels.view(-1)[active])
        return F.cross_entropy(logits.view(-1, self.num_labels), labels.view(-1))


class BertForQuestionAnswering(_Head):
    def __init__(self, config: Optional[BertConfig] = None):
        super().__init__(config)
        self.qa_outputs = nn.Linear(self.config.hidden_size, 2)
        self._init_head(self.qa_outputs)

    def forward(self, input_ids, token_type_ids=None, attention_mask=None, start_positions=None, end_positions=None):
        seq, _ = self.bert(input_ids, token_type_ids, attention_mask)
        start, end = self.qa_outputs(seq).unbind(-1)
        if start_positions is None or end_positions is None:
            return start, end
        S = start.size(1)                                         # positions outside the window are ignored
        sp, ep = start_positions.clamp(0, S), end_positions.clamp(0, S)
        return 0.5 * (F.cross_entropy(start, sp, ignore_index=S) + F.cross_entropy(end, ep, ignore_index=S))


class BertForMaskedLM(_Head):
    """``fuse_xent`` (default off, a run-time switch) computes the loss with the fused softmax cross-entropy of
    ``ops/fused_xent.py``; ``sparse_mlm`` (default off, a run-time switch) runs the head on the labelled rows only,
    gathered into ``mlm_capacity`` times B·S rows, when labels are given (``BertPreTrainingHeads``)."""

    def __init__(self, config: Optional[BertConfig] = None, fuse_xent: bool = False, sparse_mlm: bool = False,
                 mlm_capacity: float = 0.25):
        super().__init__(config)
        self.heads = BertPreTrainingHeads(self.config)
        self.fuse_xent = fuse_xent
        self.sparse_mlm = sparse_mlm
        self.mlm_capacity = mlm_capacity

    @property
    def sparse_mlm(self) -> bool:
        return self.heads.sparse_mlm

    @sparse_mlm.setter
    def sparse_mlm(self, on: bool) -> None:
        self.heads.sparse_mlm = bool(on)

    @property
    def mlm_capacity(self) -> float:
        return self.heads.mlm_capacity

    @mlm_capacity.setter
    def mlm_capacity(self, fraction: float) -> None:
        from ..ops.mlm_gather import capacity_rows
        capacity_rows(1, fraction)                           # validates: 0 < fraction <= 1
        self.heads.mlm_capacity = float(fraction)

    def forward(self, input_ids, token_type_ids=None, attention_mask=None, masked_lm_labels=None):
        seq, pooled = self.bert(input_ids, token_type_ids, attention_mask)
        if masked_lm_labels is None:
            return self.heads(seq, pooled)[0]
        scores, _, labels = self.heads(seq, pooled, masked_lm_labels)
        scores, labels = scores.view(-1, self.config.vocab_size), labels.view(-1)
        if self.fuse_xent:
            from ..ops.fused_xent import softmax_cross_entropy
            return softmax_cross_entropy(scores, labels, ignore_index=-1)
        return F.cross_entropy(scores, labels, ignore_index=-1)


class BertForNextSentencePrediction(_Head):
    def __init__(self, config: Optional[BertConfig] = None):
        super().__init__(config)
        self.seq_relationship = nn.Linear(self.config.hidden_size, 2)
        self._init_head(self.seq_relationship)

    def forward(self, input_ids, token_type_ids=None, attention_mask=None, next_sentence_label=None):
        _, pooled = self.bert(input_ids, token_type_ids, attention_mask)
        logits = self.seq_relationship(pooled)
        return logits if next_sentence_label is None else F.cross_entropy(logits, next_sentence_label.view(-1))
