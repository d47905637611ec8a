"""Fused embedding sum + LayerNorm + dropout for BERT's input block (``csrc/embedding.cu``).

``embedding_layer_norm(input_ids, token_type_ids, emb, p)`` computes ``BertEmbeddings``'s

    dropout(LayerNorm(word[ids] + position[arange(S)] + token_type[tt]), p)

on CUDA with one kernel forward and three backward, instead of three gathers, two adds, ``layer_norm`` and a dropout
forward and dropout, ``layer_norm`` backward and three ``embedding_dense_backward`` calls (each a sort of the ids and a
zero-filled dense table gradient) backward.  Only ``[mean; rstd]`` per token is saved: the backward pass recomputes the
sum from the tables and the ids, and regenerates the mask.

Forward: the three rows are added in fp32 in the stock order ``(w + p) + t``, so the sum is bit for bit the stock one;
the mean and rstd are taken as in ``ops/fused_ln.py`` (the mean, then the mean squared deviation from it).

Dropout: exactly the scheme of ``ops/fused_ln.py``: one int64 seed per call drawn on the device from torch's CUDA
generator, Philox4x32-10 with counter ``i // 4`` and word ``i % 4`` over the element index ``i`` of ``y``, kept iff
below ``keep_threshold(p)``, and no generator call at ``p = 0``.  So the op is safe under CUDA graphs and
``torch.utils.checkpoint``.

Gradients: the LayerNorm parameters' from per-CTA partials added in a fixed order; the three tables' dense, every
element written once (no memset, no sort, no float atomics).  A word-table row is the sum of the gradient of the
embedding sum over the tokens with that id, added in token order, or exactly 0; a position row ``s < S`` the sum over
the batch in ``b`` order, the rows from ``S`` on 0; a token-type row the sum over the tokens of that type in token
order.  Both backward calls of one input give bitwise equal gradients.  The word table's gradient stays dense because
Ok-Topk reads ``p.grad`` in place.

Out-of-range ids: an id outside ``[0, vocab)`` or a type outside ``[0, type_vocab)`` is never used as an address.  Its
table row contributes 0 to the sum and gets no gradient, and the forward pass adds one per such index to ``emb.id_overflow``
(a non-persistent int64 buffer of ``BertEmbeddings``, read by whoever wants to check it).  Stock ``nn.Embedding`` fires a
device assert on them instead.

Types: the tables and the LayerNorm are fp32.  Under bf16 or fp16 autocast stock ``embedding`` and ``layer_norm`` stay
fp32, and so does this op: it runs the same fp32 kernels and returns fp32 ``y``.

Falls back to exactly the stock expression wherever the fast path does not apply: CPU tensors, ids that are not a 2-D
``[B, S]`` integer matrix with token types of the same shape, more than 4096 tokens, H outside 128, 256, ..., 1024,
tables or LayerNorm parameters that are not fp32 (or a LayerNorm without them), an embedding with ``sparse=True``,
``padding_idx``, ``max_norm`` or ``scale_grad_by_freq`` set, S larger than the position table, ``p`` outside
[0, 1), or no native extension.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import ext
from .ext import dense16
from .fused_ln import keep_threshold


def _plain(e: torch.nn.Embedding, H: int, dev) -> bool:
    w = e.weight
    return (not e.sparse and e.padding_idx is None and e.max_norm is None and not e.scale_grad_by_freq
            and w.dtype == torch.float32 and w.device == dev and w.dim() == 2 and w.size(1) == H and w.size(0) > 0)


def _fast_path_ok(ids: torch.Tensor, tt: torch.Tensor, emb, p: float) -> bool:
    if not (ids.is_cuda and ids.dim() == 2 and ids.numel() > 0 and ext.available()):
        return False
    B, S = ids.shape
    dev = ids.device
    word, pos, typ, ln = emb.word_embeddings, emb.position_embeddings, emb.token_type_embeddings, emb.LayerNorm
    H = word.embedding_dim
    w, b = ln.weight, ln.bias
    ints = (torch.int64, torch.int32)
    return (0.0 <= p < 1.0 and ids.dtype in ints and tt.dtype in ints and tt.shape == ids.shape and tt.device == dev
            and B * S <= 4096 and H % 128 == 0 and 128 <= H <= 1024 and S <= pos.num_embeddings
            and all(_plain(e, H, dev) for e in (word, pos, typ)) and tuple(ln.normalized_shape) == (H,)
            and w is not None and b is not None and w.dtype == torch.float32 and b.dtype == torch.float32
            and w.device == dev and b.device == dev)


def _stock(ids, tt, emb, p):
    pos = torch.arange(ids.size(1), device=ids.device).unsqueeze(0)
    e = emb.word_embeddings(ids) + emb.position_embeddings(pos) + emb.token_type_embeddings(tt)
    return F.dropout(emb.LayerNorm(e), p, p > 0)


class _EmbeddingLN(torch.autograd.Function):
    @staticmethod
    def forward(ctx, ids, tt, word, pos, typ, gamma, beta, p, eps, ovf):
        C = ext.require()
        B, S = ids.shape
        R, H = B * S, word.size(1)
        seed = torch.empty(1, dtype=torch.int64, device=ids.device).random_() if p > 0 else None
        y = torch.empty((B, S, H), dtype=torch.float32, device=ids.device)
        stats = torch.empty(2 * R, dtype=torch.float32, device=ids.device)         # [mean; rstd] per token
        thr, scale = keep_threshold(p), 1.0 / (1.0 - p)
        C.emb_forward(ids.data_ptr(), tt.data_ptr(), word.data_ptr(), pos.data_ptr(), typ.data_ptr(), gamma.data_ptr(),
                      beta.data_ptr(), y.data_ptr(), stats.data_ptr(), 0 if ovf is None else ovf.data_ptr(),
                      0 if seed is None else seed.data_ptr(), R, S, H, word.size(0), pos.size(0), typ.size(0), thr,
                      scale, eps, torch.cuda.current_stream().cuda_stream)
        ctx.save_for_backward(ids, tt, word, pos, typ, gamma, stats, seed)
        ctx.thr, ctx.scale = thr, scale
        return y

    @staticmethod
    def backward(ctx, dy):
        C = ext.require()
        ids, tt, word, pos, typ, gamma, stats, seed = ctx.saved_tensors
        B, S = ids.shape
        R, H = B * S, word.size(1)
        dev = ids.device
        dy = dense16(dy.float())                        # y is fp32, so is its gradient
        de = torch.empty((R, H), dtype=torch.float32, device=dev)
        partial = torch.empty(C.ln_bwd_grid(R) * 2 * H, dtype=torch.float32, device=dev)
        dgb = torch.empty(2 * H, dtype=torch.float32, device=dev)              # [dgamma | dbeta]
        dword, dpos, dtyp = torch.empty_like(word), torch.empty_like(pos), torch.empty_like(typ)
        C.emb_backward(ids.data_ptr(), tt.data_ptr(), word.data_ptr(), pos.data_ptr(), typ.data_ptr(), gamma.data_ptr(),
                       stats.data_ptr(), dy.data_ptr(), 0 if seed is None else seed.data_ptr(), de.data_ptr(),
                       partial.data_ptr(), dgb.data_ptr(), dgb.data_ptr() + 4 * H, dword.data_ptr(),
                       dpos.data_ptr(), dtyp.data_ptr(), R, S, H, word.size(0), pos.size(0), typ.size(0), ctx.thr,
                       ctx.scale, torch.cuda.current_stream().cuda_stream)
        return None, None, dword, dpos, dtyp, dgb[:H], dgb[H:], None, None, None


def embedding_layer_norm(input_ids: torch.Tensor, token_type_ids: torch.Tensor, emb, p: float) -> torch.Tensor:
    """``BertEmbeddings`` ``emb``'s ``dropout(LayerNorm(word + position + token_type), p)`` (``p = 0``: no dropout, as
    in eval mode); see the module docstring."""
    p = float(p)
    if _fast_path_ok(input_ids, token_type_ids, emb, p):
        ovf = getattr(emb, "id_overflow", None)
        if ovf is not None and (ovf.device != input_ids.device or ovf.dtype != torch.int64 or ovf.numel() != 1):
            ovf = None
        with torch.autocast("cuda", enabled=False):
            return _EmbeddingLN.apply(input_ids.long().contiguous(), token_type_ids.long().contiguous(),
                                      dense16(emb.word_embeddings.weight), dense16(emb.position_embeddings.weight),
                                      dense16(emb.token_type_embeddings.weight), dense16(emb.LayerNorm.weight),
                                      dense16(emb.LayerNorm.bias), p, float(emb.LayerNorm.eps), ovf)
    return _stock(input_ids, token_type_ids, emb, p)
