"""Persistent LSTM recurrence for DeepSpeech's uni-directional layers (``csrc/lstm.cu``).

``lstm_layer(x, lengths, rnn)`` returns what ``BatchRNN`` returns after its batch norm: ``rnn`` run over the time-major
``x`` (T x N x I) with per-utterance ``lengths`` through ``pack_padded_sequence`` / ``pad_packed_sequence``, i.e. the
hidden states h_t for t < len_b and exactly 0 after.  torch's ``nn.LSTM`` conventions: gate order i, f, g, o,
``c_t = f c_{t-1} + i g``, ``h_t = o tanh(c_t)``, zero initial state.

The native path runs one cooperative kernel per pass instead of cuDNN's small GEMM + element-wise kernel per timestep:

* forward: the input projection ``x W_ih^T + b_ih + b_hh`` of all timesteps is one GEMM; then ``lstm_forward`` walks the
  timesteps, each CTA holding the 4u rows of ``W_hh`` of its u hidden units in shared memory, with one grid barrier per
  step.  It writes y and keeps the activated gates and c_t for the backward pass;
* backward: ``lstm_backward`` walks t from T-1 down to 0, each CTA holding the 4H x u columns of ``W_hh`` of the same
  units, and writes the gates' pre-activation gradients; ``dx``, ``dW_ih``, ``dW_hh`` and the bias gradients are GEMMs
  and sums over them in torch.

Everything is summed in fp32 in a fixed order (no atomics), so results are bitwise reproducible.  The native path
needs: CUDA fp32 tensors with autocast off, the native extension, ``rnn`` a single-layer, uni-directional ``nn.LSTM``
with bias, ``proj_size == 0`` and ``batch_first=False``, lengths in [1, T], and an (H, N) that ``lstm_geometry``
accepts on the current device.  Everything else -- the CPU, fp64, bidirectional layers, and in fp32 the PTB model's
H = 1500, whose 288 KB of recurrent weights per CTA do not fit on chip -- runs the stock pack -> ``rnn`` -> pad sequence
and returns exactly what ``BatchRNN`` returns without the switch.

Under bf16 / fp16 CUDA autocast the layer is stock too, unless ``lstm_layer(..., autocast=True)`` asks for the 16-bit
kernels: ``x``, ``W_ih``, ``W_hh`` and ``b_ih + b_hh`` are cast to the autocast type (the parameters stay fp32), the
input projection runs in it, and W_hh (in shared memory, half the bytes: H = 1500 fits), the input projection, y, dy
and the gates' gradients are 16-bit; the saved gates and c, the cell state and every sum stay fp32.  A stored y_t or
dgates_t is rounded to nearest even (an fp16 overflow gives inf, for loss scaling to see) and it is the rounded value
that the next step reads.  y comes back in the autocast type, as ``nn.LSTM``'s does, the parameter gradients in fp32.
This differs from cuDNN's 16-bit RNN, which also keeps c in 16 bits.
"""
from __future__ import annotations

from typing import NamedTuple, Optional, Tuple

import torch
import torch.nn as nn

from . import ext

LSTM_THREADS = 512          # csrc/lstm.cu kLstmThreads
MAX_BATCH = 64              # the largest N the native path takes


class LstmGeometry(NamedTuple):
    units: int              # hidden units per CTA (u)
    grid: int               # CTAs: ceil(H / u), one per SM
    fwd_rows: int           # rows of h_{t-1} staged in shared memory at a time by the forward kernel
    bwd_rows: int           # rows of dgates_{t+1} staged at a time by the backward kernel
    fwd_smem: int           # dynamic shared memory per CTA, bytes
    bwd_smem: int


def lstm_geometry(H: int, N: int, sms: int, smem_per_block: int, elem: int = 4) -> Optional[LstmGeometry]:
    """How the kernels split a layer of H hidden units at batch N over ``sms`` SMs with ``smem_per_block`` bytes of
    (opt-in) shared memory per CTA, or None when they cannot.  ``elem``: bytes per element of W_hh and of the operand
    staged every step, 4 (fp32) or 2 (bf16 / fp16).  Each CTA owns u = ceil(H / sms) units, so the grid is one CTA per
    SM at most, and keeps their 4u x H slice of W_hh (4 elem u H bytes) in shared memory next to u x N fp32 cell states
    (forward) or carried dc (backward), the step's 4u x N fp32 gate sums (u x N dh sums), and as many rows of the
    operand it reads every step (h_{t-1}: H elements a row; dgates_{t+1}: 4H elements a row) as fit, at least one.  H must be a
    multiple of 4 (the kernels move four elements at a time) and 1 <= N <= MAX_BATCH.  On an H100 (132 SMs, 227 KB):
    H = 800 gives u = 7 on 115 CTAs with 89.6 KB of fp32 weights (44.8 KB of 16-bit ones); H = 1500 gives u = 12 on 125
    CTAs and needs 288 KB in fp32, which is rejected, and 144 KB in 16 bits."""
    if H <= 0 or H % 4 or not 1 <= N <= MAX_BATCH or sms <= 0 or elem not in (2, 4):
        return None
    u = -(-H // sms)
    grid = -(-H // u)
    w = 4 * elem * u * H
    fwd_fixed = w + 4 * (4 * u * N + u * N)
    bwd_fixed = w + 4 * (u * N + u * N)
    fr = min(N, (smem_per_block - fwd_fixed) // (elem * H))
    br = min(N, (smem_per_block - bwd_fixed) // (4 * elem * H))
    if fr < 1 or br < 1:
        return None
    return LstmGeometry(u, grid, fr, br, fwd_fixed + elem * H * fr, bwd_fixed + 4 * elem * H * br)


def _device_geometry(H: int, N: int, dev: torch.device, elem: int = 4) -> Optional[LstmGeometry]:
    p = torch.cuda.get_device_properties(dev)
    return lstm_geometry(H, N, p.multi_processor_count, p.shared_memory_per_block_optin, elem)


_DTYPE_CODE = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}      # csrc/oktopk.cuh BnDtype


def stock_layer(x: torch.Tensor, lengths: torch.Tensor, rnn: nn.Module) -> torch.Tensor:
    """``BatchRNN``'s recurrence on the stock modules: pack (unsorted lengths), run ``rnn``, pad back to T, and add the
    two directions of a bidirectional layer."""
    total = x.size(0)
    x = nn.utils.rnn.pack_padded_sequence(x, lengths.cpu(), enforce_sorted=False)
    x, _ = rnn(x)
    x, _ = nn.utils.rnn.pad_packed_sequence(x, total_length=total)
    if rnn.bidirectional:
        x = x.view(x.size(0), x.size(1), 2, -1).sum(2)
    return x


def _native_ok(x: torch.Tensor, lengths: torch.Tensor, rnn: nn.Module,
               autocast: bool) -> Optional[Tuple[LstmGeometry, torch.dtype]]:
    """The geometry and the kernels' storage type when the native path applies, else None."""
    if not (isinstance(rnn, nn.LSTM) and rnn.num_layers == 1 and not rnn.bidirectional and rnn.bias
            and rnn.proj_size == 0 and not rnn.batch_first):
        return None
    if not (x.is_cuda and x.dim() == 3 and x.size(2) == rnn.input_size):
        return None
    dt = torch.float32
    if torch.is_autocast_enabled(x.device.type):
        dt = torch.get_autocast_dtype(x.device.type)
        if not autocast or dt not in (torch.bfloat16, torch.float16):
            return None
    if x.dtype not in (torch.float32, dt) or not ext.available():
        return None
    ps = (rnn.weight_ih_l0, rnn.weight_hh_l0, rnn.bias_ih_l0, rnn.bias_hh_l0)
    if any(p.dtype != torch.float32 or p.device != x.device for p in ps):
        return None
    T, N = x.size(0), x.size(1)
    if lengths.dim() != 1 or lengths.numel() != N or T == 0:
        return None
    host = lengths.cpu()
    if int(host.min()) < 1 or int(host.max()) > T:          # stock raises on these; let it
        return None
    geom = _device_geometry(rnn.hidden_size, N, x.device, dt.itemsize)
    return None if geom is None else (geom, dt)


class _LstmLayer(torch.autograd.Function):
    """``dt``: the kernels' storage type.  fp32: every tensor is fp32.  bf16 / fp16: x and the parameters are cast to it
    here, once per forward, and both passes run with autocast off, so that neither depends on the ambient state."""

    @staticmethod
    def forward(ctx, x, lens, w_ih, w_hh, b_ih, b_hh, geom, dt):
        C = ext.require()
        T, N, I = x.shape
        H = w_hh.size(1)
        with torch.autocast(x.device.type, enabled=False):
            xs, w_ih, w_hh, b = x.to(dt), w_ih.to(dt), w_hh.to(dt), (b_ih + b_hh).to(dt)
            gx = torch.addmm(b, xs.reshape(T * N, I), w_ih.t())                # (T N) x 4H
        y = torch.empty(T, N, H, device=x.device, dtype=dt)
        gates = torch.empty(T, N, 4 * H, device=x.device, dtype=torch.float32)
        cs = torch.empty(T, N, H, device=x.device, dtype=torch.float32)
        bar = torch.zeros(1, dtype=torch.int64, device=x.device)
        C.lstm_forward(gx.data_ptr(), w_hh.data_ptr(), lens.data_ptr(), y.data_ptr(), gates.data_ptr(), cs.data_ptr(),
                       bar.data_ptr(), T, N, H, geom.units, geom.fwd_rows, torch.cuda.current_stream().cuda_stream,
                       _DTYPE_CODE[dt])
        ctx.save_for_backward(xs, lens, w_ih, w_hh, y, gates, cs)
        ctx.geom = geom
        ctx.x_dtype = x.dtype
        return y

    @staticmethod
    def backward(ctx, dy):
        C = ext.require()
        x, lens, w_ih, w_hh, y, gates, cs = ctx.saved_tensors
        T, N, I = x.shape
        H = w_hh.size(1)
        dt = y.dtype
        dy = dy.to(dt).contiguous()
        dg = torch.empty(T, N, 4 * H, device=x.device, dtype=dt)
        bar = torch.zeros(1, dtype=torch.int64, device=x.device)
        C.lstm_backward(dy.data_ptr(), gates.data_ptr(), cs.data_ptr(), w_hh.data_ptr(), lens.data_ptr(), dg.data_ptr(),
                        bar.data_ptr(), T, N, H, ctx.geom.units, ctx.geom.bwd_rows,
                        torch.cuda.current_stream().cuda_stream, _DTYPE_CODE[dt])
        g2 = dg.view(T * N, 4 * H)
        need = ctx.needs_input_grad
        with torch.autocast(x.device.type, enabled=False):      # GEMMs in dt; the parameters' gradients come back fp32
            dx = (g2 @ w_ih).view(T, N, I).to(ctx.x_dtype) if need[0] else None
            dw_ih = (g2.t() @ x.reshape(T * N, I)).float() if need[2] else None
            # h_{t-1} = y_{t-1}
            dw_hh = (dg[1:].reshape(-1, 4 * H).t() @ y[:-1].reshape(-1, H)).float() if need[3] else None
            db = g2.sum(0, dtype=torch.float32) if need[4] or need[5] else None
        db_ih = db if need[4] else None
        db_hh = (db.clone() if need[4] else db) if need[5] else None             # two tensors, never one aliased
        return dx, None, dw_ih, dw_hh, db_ih, db_hh, None, None


def lstm_layer(x: torch.Tensor, lengths: torch.Tensor, rnn: nn.Module, dev_lengths: Optional[torch.Tensor] = None,
               autocast: bool = False) -> torch.Tensor:
    """``rnn`` over ``x`` (T x N x I) with per-utterance ``lengths`` (host int tensor), as ``BatchRNN`` runs it; see the
    module docstring.  ``dev_lengths``: the same lengths as int32 on ``x``'s device, to share one copy between
    layers.  ``autocast``: under bf16 / fp16 CUDA autocast, take the 16-bit kernels instead of the stock layer."""
    ok = _native_ok(x, lengths, rnn, autocast)
    if ok is None:
        return stock_layer(x, lengths, rnn)
    geom, dt = ok
    if dev_lengths is None or dev_lengths.device != x.device or dev_lengths.dtype != torch.int32:
        dev_lengths = lengths.to(device=x.device, dtype=torch.int32)
    w_hh = rnn.weight_hh_l0.contiguous()
    if dt == torch.float32 and w_hh.data_ptr() % 16:         # read as 16-byte vectors; a 16-bit copy is a fresh tensor
        w_hh = w_hh.clone()
    return _LstmLayer.apply(x.contiguous(), dev_lengths.contiguous(), rnn.weight_ih_l0, w_hh, rnn.bias_ih_l0,
                            rnn.bias_hh_l0, geom, dt)
