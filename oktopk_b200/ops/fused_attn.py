"""Fused self-attention for BERT's encoder layers (``csrc/attention.cu``).

``self_attention(qkv, heads, mask, p)`` takes the packed projection ``qkv`` [B, S, 3·H·D] of ``BertSelfAttention`` and
returns ``[B, S, H·D]``: per sequence b, head h and query i, with D = 64,

    s_ij = (q_i · k_j) / sqrt(D) + m_bj,    P_ij = softmax_j(s_ij),    O_i = sum_j keep(b,h,i,j) / (1-p) · P_ij · v_j

which is what ``F.scaled_dot_product_attention(q, k, v, attn_mask=mask, dropout_p=p)`` computes with the additive
``[B, 1, 1, S]`` key-padding mask (dropout on the normalised probabilities).  On CUDA it is one kernel forward and two
backward, reading Q, K and V straight out of ``qkv`` and writing the output and d(qkv) in their final layouts, with no
S x S tensor stored: the backward pass recomputes P from each row's saved max and log-sum, kept apart so that the sum
survives beside a max of any magnitude.  d(qkv) is the only gradient.

Dropout (``ops/fused_ln.py``'s convention): each call draws one int64 seed on the device from torch's default CUDA
generator, and element (b, h, i, j), flat index ``((b·H + h)·S + i)·S + j`` over [B, H, S, S], is kept iff word
``idx % 4`` of Philox4x32-10 at counter ``idx // 4`` is below ``floor((1-p) 2^32)``.  So ``torch.manual_seed`` makes runs
reproducible, ``torch.utils.checkpoint`` recomputes the same mask, and a CUDA graph draws a fresh mask at each replay.
The masks are not torch's own dropout masks.  ``p = 0`` runs no generator.  The backward pass regenerates the mask.

Types: ``qkv`` is fp32, bf16 or fp16; the output and d(qkv) have its type, and every sum (scores, softmax, products) is
fp32.  bf16 / fp16 run on the tensor cores (``mma.sync``, P and dS rounded to the 16-bit type before their products);
fp32 runs 3xTF32 tensor-core products, which keep about fp32 accuracy.  Under CUDA autocast the ``qkv`` Linear hands
over a 16-bit tensor and the mask stays fp32: the kernels read the fp32 mask as it is, where stock autocast SDPA first
rounds the mask to the 16-bit type (BERT's -10000 becomes -9984 in bf16; either way a padded key's weight is 0 in fp32).
The backward pass is deterministic: no atomics, a fixed order of every sum.

A finite mask entry always gives a finite score, even where the kernels' conversion to base 2 (``mask · log2 e``) would
overflow fp32: it saturates at the largest finite float.  So a sequence masked at every key with a finite value, BERT's
``(1 - m) · -10000`` or ``torch.finfo(torch.float32).min`` alike, gets a softmax over its scores as float64 computes
it; with ``finfo.min``, whose scores all round to the same value, that is the uniform average of V.  A sequence whose
mask is -inf at every key has no finite score in any row: its output and its rows of d(qkv) are NaN, as
``torch.softmax`` over an all -inf row is.

Falls back to exactly today's expression (view, permute, ``F.scaled_dot_product_attention``, transpose, reshape)
wherever the fast path does not apply: CPU tensors or no native extension, ``qkv`` not a 3-d fp32 / bf16 / fp16 tensor,
a last dimension other than ``3·heads·64``, S outside 1..512, B or heads above 65535 (the kernels' grid), a mask other
than ``None`` or exactly ``[B, 1, 1, S]`` on ``qkv``'s device in fp32 or ``qkv``'s type, a mask that requires a
gradient, or ``p`` outside [0, 1).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import ext
from .ext import DTYPE_CODE, dense16
from .fused_ln import keep_threshold

HEAD_DIM = 64


def _fast_path_ok(qkv: torch.Tensor, heads: int, mask, p: float) -> bool:
    if not (qkv.is_cuda and qkv.dim() == 3 and qkv.dtype in DTYPE_CODE and ext.available()):
        return False
    B, S, W = qkv.shape
    if not (0.0 <= p < 1.0 and heads >= 1 and W == 3 * heads * HEAD_DIM and ext.require().attn_supported(B, S, heads)):
        return False
    if mask is None:
        return True
    return (isinstance(mask, torch.Tensor) and tuple(mask.shape) == (B, 1, 1, S) and mask.device == qkv.device
            and mask.dtype in (torch.float32, qkv.dtype) and not mask.requires_grad)


class _FusedAttention(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv, mask, heads, p):
        C = ext.require()
        B, S, _ = qkv.shape
        seed = torch.empty(1, dtype=torch.int64, device=qkv.device).random_() if p > 0 else None
        out = torch.empty((B, S, heads * HEAD_DIM), dtype=qkv.dtype, device=qkv.device)
        lse = torch.empty((B, heads, S, 2), dtype=torch.float32, device=qkv.device)    # each row's max, log2 of its sum
        thr, scale = keep_threshold(p), 1.0 / (1.0 - p)
        C.attn_forward(qkv.data_ptr(), 0 if mask is None else mask.data_ptr(), 0 if seed is None else seed.data_ptr(),
                       out.data_ptr(), lse.data_ptr(), B, S, heads, thr, scale, DTYPE_CODE[qkv.dtype],
                       torch.cuda.current_stream().cuda_stream)
        ctx.save_for_backward(qkv, out, lse, mask, seed)
        ctx.heads, ctx.thr, ctx.scale = heads, thr, scale
        return out

    @staticmethod
    def backward(ctx, dout):
        C = ext.require()
        qkv, out, lse, mask, seed = ctx.saved_tensors
        B, S, _ = qkv.shape
        dout = dense16(dout.to(qkv.dtype))
        dqkv = torch.empty_like(qkv)
        delta = torch.empty((B, ctx.heads, S), dtype=torch.float32, device=qkv.device)
        C.attn_backward(qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), 0 if mask is None else mask.data_ptr(),
                        0 if seed is None else seed.data_ptr(), lse.data_ptr(), delta.data_ptr(), dqkv.data_ptr(), B, S,
                        ctx.heads, ctx.thr, ctx.scale, DTYPE_CODE[qkv.dtype], torch.cuda.current_stream().cuda_stream)
        return dqkv, None, None, None


def self_attention(qkv: torch.Tensor, heads: int, mask, p: float) -> torch.Tensor:
    """Multi-head self-attention of the packed projection ``qkv`` [B, S, 3·heads·D] with the additive mask ``mask``
    (``None`` or [B, 1, 1, S]) and attention dropout ``p`` (0 in eval mode); returns [B, S, heads·D].  See the module
    docstring."""
    p = float(p)
    if _fast_path_ok(qkv, heads, mask, p):
        B, S, _ = qkv.shape
        m = None if mask is None else dense16(mask.reshape(B, S).float())
        return _FusedAttention.apply(dense16(qkv), m, int(heads), p)
    b, s, w = qkv.shape
    dh = w // (3 * heads)
    q, k, v = qkv.view(b, s, 3, heads, dh).permute(2, 0, 3, 1, 4)
    o = F.scaled_dot_product_attention(q, k, v, attn_mask=mask, dropout_p=p)
    return o.transpose(1, 2).reshape(b, s, heads * dh)
