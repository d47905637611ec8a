"""Persistent LSTM recurrence for DeepSpeech's LSTM layers (``csrc/lstm.cu``).

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
accepts on the current device.  Everything else -- the CPU, fp64, bidirectional layers (unless asked for, below), and
in fp32 the PTB model's H = 1500, whose 288 KB of recurrent weights per CTA do not fit on chip -- runs the stock pack ->
``rnn`` -> pad sequence and returns exactly what ``BatchRNN`` returns without the switch.

``lstm_layer(..., bidirectional=True)`` takes a single-layer bidirectional ``nn.LSTM`` too, on the same conditions.  Both
directions run in one launch per pass, each on half of the SMs (``lstm_geometry`` at ``sms // 2``, so H = 800 on an H100
is u = 13 on 62 + 62 CTAs): the reverse direction is the forward recurrence run over each utterance's own
``len - 1, ..., 0``, so it starts from a zero state at the last frame, as the packed stock layer does.  Each direction
has its own input projection GEMM; the output is the sum of the two directions' y, which is what ``BatchRNN`` returns,
and ``dx`` is two accumulating GEMMs.  A layer whose two directions do not fit together runs stock.

Under bf16 / fp16 CUDA autocast the layer is stock too, unless ``lstm_layer(..., autocast=True)`` asks for the 16-bit
kernels: ``x``, ``W_ih``, ``W_hh`` and ``b_ih + b_hh`` are cast to the autocast type (the parameters stay fp32), the
input projection runs in it, and W_hh (in shared memory, half the bytes: H = 1500 fits), the input projection, y, dy
and the gates' gradients are 16-bit; the saved gates and c, the cell state and every sum stay fp32.  A stored y_t or
dgates_t is rounded to nearest even (an fp16 overflow gives inf, for loss scaling to see) and it is the rounded value
that the next step reads.  y comes back in the autocast type, as ``nn.LSTM``'s does, the parameter gradients in fp32.
This differs from cuDNN's 16-bit RNN, which also keeps c in 16 bits.

``lstm_layer_device(x, lengths, rnn, ...)`` takes the lengths as an int32 device tensor and never reads them on the host,
so that a whole training step can be captured in a CUDA graph; it runs the native path or raises, never the stock layer.

``lstm_stack(x, hx, rnn, dropout_p, training)`` runs a multi-layer ``nn.LSTM`` from a carried state (the PTB language
model) under bf16 / fp16 autocast on a second pair of kernels, whose step product runs on the tensor cores, and with
``fp32=True`` in fp32 on the fp32 forms of the same kernels; see its docstring.
"""
from __future__ import annotations

from typing import NamedTuple, Optional, Tuple

import torch
import torch.nn as nn

from . import ext
from .ext import DTYPE_CODE

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


def _device_geometry(H: int, N: int, dev: torch.device, elem: int = 4, dirs: int = 1) -> Optional[LstmGeometry]:
    """The geometry of one direction of a ``dirs``-direction layer: the directions split the SMs between them."""
    p = torch.cuda.get_device_properties(dev)
    return lstm_geometry(H, N, p.multi_processor_count // dirs, p.shared_memory_per_block_optin, elem)


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


def _native_ok(x: torch.Tensor, lengths: torch.Tensor, rnn: nn.Module, autocast: bool,
               bidirectional: bool) -> Optional[Tuple[LstmGeometry, torch.dtype]]:
    """The geometry (of one direction) and the kernels' storage type when the native path applies, else None."""
    ok = _native_layer_ok(x, rnn, autocast, bidirectional)
    if ok is None or lengths.dim() != 1 or lengths.numel() != x.size(1):
        return None
    host = lengths.cpu()
    if int(host.min()) < 1 or int(host.max()) > x.size(0):        # stock raises on these; let it
        return None
    return ok


def _native_layer_ok(x: torch.Tensor, rnn: nn.Module, autocast: bool,
                     bidirectional: bool) -> Optional[Tuple[LstmGeometry, torch.dtype]]:
    """``_native_ok`` without the lengths: nothing here reads device memory."""
    if not (isinstance(rnn, nn.LSTM) and rnn.num_layers == 1 and (bidirectional or not rnn.bidirectional) and rnn.bias
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
    if any(p.dtype != torch.float32 or p.device != x.device for p in _params(rnn)):
        return None
    T, N = x.size(0), x.size(1)
    if T == 0:
        return None
    geom = _device_geometry(rnn.hidden_size, N, x.device, dt.itemsize, 2 if rnn.bidirectional else 1)
    return None if geom is None else (geom, dt)


def _params(rnn: nn.LSTM) -> Tuple[torch.Tensor, ...]:
    """W_ih, W_hh, b_ih, b_hh of each direction, forward direction first."""
    return tuple(getattr(rnn, n + sfx) for sfx in (("_l0", "_l0_reverse") if rnn.bidirectional else ("_l0",))
                 for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"))


class _LstmLayer(torch.autograd.Function):
    """``dt``: the kernels' storage type.  fp32: every tensor is fp32.  bf16 / fp16: x and the parameters are cast to it
    here, once per forward, and both passes run with autocast off, so that neither depends on the ambient state.
    ``ps``: W_ih, W_hh, b_ih, b_hh of one direction, or of the forward then the reverse direction."""

    @staticmethod
    def forward(ctx, x, lens, geom, dt, *ps):
        C = ext.require()
        T, N, I = x.shape
        dirs = len(ps) // 4
        H = ps[1].size(1)
        with torch.autocast(x.device.type, enabled=False):
            xs = x.to(dt)
            w_ih = [ps[4 * d].to(dt) for d in range(dirs)]
            w_hh = [ps[4 * d + 1].to(dt) for d in range(dirs)]
            gx = torch.empty(dirs, T * N, 4 * H, device=x.device, dtype=dt)
            for d in range(dirs):
                b = (ps[4 * d + 2] + ps[4 * d + 3]).to(dt)
                torch.addmm(b, xs.reshape(T * N, I), w_ih[d].t(), out=gx[d])        # (T N) x 4H
        y = torch.empty(dirs * T, N, H, device=x.device, dtype=dt)       # [dirs, T, N, H]; one direction: the output
        gates = torch.empty(dirs, T, N, 4 * H, device=x.device, dtype=torch.float32)
        cs = torch.empty(dirs, T, N, H, device=x.device, dtype=torch.float32)
        bar = torch.zeros(dirs, dtype=torch.int64, device=x.device)
        C.lstm_forward(gx.data_ptr(), w_hh[0].data_ptr(), lens.data_ptr(), y.data_ptr(), gates.data_ptr(),
                       cs.data_ptr(), bar.data_ptr(), T, N, H, geom.units, geom.fwd_rows,
                       torch.cuda.current_stream().cuda_stream, DTYPE_CODE[dt], w_hh[1].data_ptr() if dirs == 2 else 0)
        ctx.save_for_backward(xs, lens, y, gates, cs, *w_ih, *w_hh)
        ctx.geom = geom
        ctx.x_dtype = x.dtype
        return y if dirs == 1 else y[:T] + y[T:]                 # stock_layer's sum of the two directions

    @staticmethod
    def backward(ctx, dy):
        C = ext.require()
        x, lens, y, gates, cs, *ws = ctx.saved_tensors
        dirs = len(ws) // 2
        w_ih, w_hh = ws[:dirs], ws[dirs:]
        T, N, I = x.shape
        y = y.view(dirs, T, N, -1)
        H = w_hh[0].size(1)
        dt = y.dtype
        dy = dy.to(dt).contiguous()
        dg = torch.empty(dirs, T, N, 4 * H, device=x.device, dtype=dt)
        bar = torch.zeros(dirs, dtype=torch.int64, device=x.device)
        C.lstm_backward(dy.data_ptr(), gates.data_ptr(), cs.data_ptr(), w_hh[0].data_ptr(), lens.data_ptr(),
                        dg.data_ptr(), bar.data_ptr(), T, N, H, ctx.geom.units, ctx.geom.bwd_rows,
                        torch.cuda.current_stream().cuda_stream, DTYPE_CODE[dt],
                        w_hh[1].data_ptr() if dirs == 2 else 0)
        need = ctx.needs_input_grad
        grads = []
        dx = None
        with torch.autocast(x.device.type, enabled=False):      # GEMMs in dt; the parameters' gradients come back fp32
            for d in range(dirs):
                g2 = dg[d].view(T * N, 4 * H)
                n_ih, n_hh, n_bih, n_bhh = need[4 + 4 * d:8 + 4 * d]
                if need[0]:
                    dx = g2 @ w_ih[d] if d == 0 else dx.addmm_(g2, w_ih[d])
                dw_ih = (g2.t() @ x.reshape(T * N, I)).float() if n_ih else None
                # h_{t-1} = y_{t-1} forward; in reverse the previous step's h is y_{t+1}, which is 0 at t + 1 >= len
                if d == 0:
                    dw_hh = (dg[0, 1:].reshape(-1, 4 * H).t() @ y[0, :-1].reshape(-1, H)).float() if n_hh else None
                else:
                    dw_hh = (dg[1, :-1].reshape(-1, 4 * H).t() @ y[1, 1:].reshape(-1, H)).float() if n_hh else None
                db = g2.sum(0, dtype=torch.float32) if n_bih or n_bhh else None
                db_ih = db if n_bih else None
                db_hh = (db.clone() if n_bih else db) if n_bhh else None         # two tensors, never one aliased
                grads += [dw_ih, dw_hh, db_ih, db_hh]
        if dx is not None:
            dx = dx.view(T, N, I).to(ctx.x_dtype)
        return (dx, None, None, None, *grads)


def lstm_layer(x: torch.Tensor, lengths: torch.Tensor, rnn: nn.Module, dev_lengths: Optional[torch.Tensor] = None,
               autocast: bool = False, bidirectional: bool = False) -> torch.Tensor:
    """``rnn`` over ``x`` (T x N x I) with per-utterance ``lengths`` (host int tensor), as ``BatchRNN`` runs it; see the
    module docstring.  ``dev_lengths``: the same lengths as int32 on ``x``'s device, to share one copy between
    layers.  ``autocast``: under bf16 / fp16 CUDA autocast, take the 16-bit kernels instead of the stock layer.
    ``bidirectional``: a bidirectional ``rnn`` takes the kernels too, both directions in one launch, instead of the stock
    layer."""
    ok = _native_ok(x, lengths, rnn, autocast, bidirectional)
    if ok is None:
        return stock_layer(x, lengths, rnn)
    geom, dt = ok
    if dev_lengths is None or dev_lengths.device != x.device or dev_lengths.dtype != torch.int32:
        dev_lengths = lengths.to(device=x.device, dtype=torch.int32)
    return _native_layer(x, dev_lengths, geom, dt, rnn)


def _native_layer(x: torch.Tensor, dev_lengths: torch.Tensor, geom: LstmGeometry, dt: torch.dtype,
                  rnn: nn.Module) -> torch.Tensor:
    ps = list(_params(rnn))
    for i in range(1, len(ps), 4):
        w_hh = ps[i].contiguous()
        if dt == torch.float32 and w_hh.data_ptr() % 16:     # read as 16-byte vectors; a 16-bit copy is a fresh tensor
            w_hh = w_hh.clone()
        ps[i] = w_hh
    return _LstmLayer.apply(x.contiguous(), dev_lengths.contiguous(), geom, dt, *ps)


def lstm_layer_device(x: torch.Tensor, lengths: torch.Tensor, rnn: nn.Module, autocast: bool = False,
                      bidirectional: bool = False) -> torch.Tensor:
    """``lstm_layer`` with the lengths on the device only: ``lengths`` is an int32 tensor of N lengths on ``x``'s device,
    each in [1, T], and nothing is read back to the host, so the layer can be captured in a CUDA graph.  It always runs
    the native path and raises ``RuntimeError`` where ``lstm_layer`` would take the stock one (which packs with host
    lengths).  The kernels stop at the longest length (``csrc/lstm.cu``), so frames padded past it cost the recurrence
    nothing; y there is exactly 0, as at every t >= len_b.  A length outside [1, T] is not checked: the longest one is
    capped at T, and the rows' results are undefined."""
    if not (isinstance(lengths, torch.Tensor) and lengths.dtype == torch.int32 and lengths.dim() == 1
            and lengths.device == x.device and lengths.numel() == (x.size(1) if x.dim() == 3 else -1)):
        raise RuntimeError("lstm_layer_device needs int32 lengths, one per batch row, on the input's device")
    ok = _native_layer_ok(x, rnn, autocast, bidirectional)
    if ok is None:
        raise RuntimeError("the fused LSTM kernels do not apply to this layer and input (a single-layer nn.LSTM with "
                           "bias on CUDA, fp32 or, with autocast=True, under bf16 / fp16 autocast; bidirectional only "
                           "with bidirectional=True; H %% 4 == 0 and N <= %d), and the stock layer needs host lengths"
                           % MAX_BATCH)
    geom, dt = ok
    return _native_layer(x, lengths, geom, dt, rnn)


# ---- stacked layers from a carried state (the PTB language model) -----------------------------------------------------

LSTM_WARPS = LSTM_THREADS // 32


class LstmSeqGeometry(NamedTuple):
    units: int              # hidden units per CTA (u)
    grid: int               # CTAs: ceil(H / u), one per SM
    fwd_rows: int           # rows of h_{t-1} staged in shared memory at a time by the forward kernel
    bwd_rows: int           # rows of dgates_{t+1} staged at a time by the backward kernel
    fwd_smem: int           # dynamic shared memory per CTA, bytes
    bwd_smem: int


def _seq_ld(K: int) -> int:
    """csrc/lstm.cu lstm_seq_ld: the shared-memory row stride of a K-element operand row."""
    return -(-K // 16) * 16 + 8


def _seq_ksplit(rows: int, R: int, K: int) -> int:
    """csrc/lstm.cu lstm_seq_ksplit."""
    tiles = -(-rows // 16) * -(-R // 8)
    return max(1, min(LSTM_WARPS // tiles, -(-K // 16)))


def _seq_fwd_smem(H: int, N: int, u: int, rows: int) -> int:
    R = 4 * u
    return 2 * (R + rows) * _seq_ld(H) + 4 * (_seq_ksplit(rows, R, H) * rows * R + R * N + u * N)


def _seq_bwd_smem(H: int, N: int, u: int, rows: int) -> int:
    return 2 * (u + rows) * _seq_ld(4 * H) + 4 * (_seq_ksplit(rows, u, 4 * H) * rows * u + 2 * u * N)


def lstm_seq_geometry(H: int, N: int, sms: int, smem_per_block: int) -> Optional[LstmSeqGeometry]:
    """How the 16-bit stacked-layer kernels (``lstm_seq_forward`` / ``lstm_seq_backward``) split a layer of H units at
    batch N over ``sms`` SMs with ``smem_per_block`` bytes of opt-in shared memory per CTA, or None when they cannot.
    As ``lstm_geometry``, each CTA owns u = ceil(H / sms) units and keeps its slice of W_hh (4u rows forward, u columns
    backward) in shared memory, here with each row padded to ``_seq_ld`` elements for the tensor-core fragments, next to
    as many staged rows of the step's operand as fit (at least one), the K-split partial sums of the step product, and
    the fp32 gate sums and cell state (forward) or dh sums and carried dc (backward).  H % 4 == 0, 1 <= N <= MAX_BATCH.
    On an H100 (132 SMs, 232 448 B): H = 1500, N = 20 is u = 12 on 125 CTAs with all 20 rows of h_{t-1} staged forward
    (214 272 B) and 6 rows of dgates_{t+1} at a time backward (220 512 B)."""
    if H <= 0 or H % 4 or not 1 <= N <= MAX_BATCH or sms <= 0:
        return None
    u = -(-H // sms)
    rows = []
    for smem in (_seq_fwd_smem, _seq_bwd_smem):
        r = next((r for r in range(N, 0, -1) if smem(H, N, u, r) <= smem_per_block), 0)
        if r == 0:
            return None
        rows.append(r)
    return LstmSeqGeometry(u, -(-H // u), rows[0], rows[1], _seq_fwd_smem(H, N, u, rows[0]),
                           _seq_bwd_smem(H, N, u, rows[1]))


# fp32: the CTA's W_hh slice (288 KB at H = 1500) does not fit in shared memory.  The first r_on of its weight rows stay
# on chip and the others are read from L2 at every step; the step operand is staged F32_CHUNK columns at a time.
F32_CHUNK = 256             # columns of h_{t-1} / dgates_{t+1} per staged chunk (a multiple of 8)
F32_MAX_ROWS = 8 * LSTM_WARPS       # weight rows per CTA the fp32 step takes: 8 per warp


class LstmSeqF32Geometry(NamedTuple):
    units: int              # hidden units per CTA (u)
    grid: int               # CTAs: ceil(H / u), one per SM
    fwd_r_on: int           # of the CTA's 4u gate rows of W_hh, how many are held in shared memory
    fwd_kc: int             # columns of h_{t-1} staged at a time
    bwd_r_on: int           # of its u columns of W_hh (rows of W_hh^T), how many are held in shared memory
    bwd_kc: int             # columns of dgates_{t+1} staged at a time
    fwd_smem: int           # dynamic shared memory per CTA, bytes
    bwd_smem: int
    fwd_l2_bytes: int       # weight bytes all CTAs together read from L2 at each step
    bwd_l2_bytes: int


def _f32_ld(K: int) -> int:
    """csrc/lstm.cu lstm_f32_ld: the shared-memory row stride of a K-float weight row, = 4 (mod 8)."""
    return -(-K // 8) * 8 + 4


def _f32_ksplit(R: int) -> int:
    """csrc/lstm.cu lstm_f32_ksplit."""
    return max(1, LSTM_WARPS // -(-R // 8))


def _f32_fixed_smem(N: int, R: int, kc: int, cell: int) -> int:
    """Everything but the on-chip weight rows: two staged chunks, the K-split partial sums and ``cell`` fp32 values
    (gate sums and c forward, dh sums and carried dc backward)."""
    return 4 * (2 * N * (kc + 4) + _f32_ksplit(R) * N * R + cell)


def lstm_seq_f32_geometry(H: int, N: int, sms: int, smem_per_block: int) -> Optional[LstmSeqF32Geometry]:
    """How the fp32 stacked-layer kernels split a layer of H units at batch N over ``sms`` SMs with ``smem_per_block``
    bytes of opt-in shared memory per CTA, or None when they cannot.  Each CTA owns u = ceil(H / sms) units, as in
    ``lstm_seq_geometry``.  Forward its weight rows are its 4u gate rows of W_hh (K = H columns), backward its u columns
    (K = 4H); it stages the step operand's N rows ``min(F32_CHUNK, K rounded up to 8)`` columns at a time in two
    buffers, and keeps as many weight rows in shared memory as fit next to them, ``_f32_ld(K)`` floats apart; the
    remaining rows are read from L2 at every step.  H % 4 == 0, 1 <= N <= MAX_BATCH, 4u <= F32_MAX_ROWS.  On an H100
    (132 SMs, 232 448 B): H = 1500, N = 20 is u = 12 on 125 CTAs, 29 of 48 rows on chip forward (229 008 B) and 7 of
    12 backward (219 312 B), in 256-column chunks; the other rows are 14.25 MB forward and 15 MB backward per step."""
    if H <= 0 or H % 4 or not 1 <= N <= MAX_BATCH or sms <= 0:
        return None
    u = -(-H // sms)
    grid = -(-H // u)
    if 4 * u > F32_MAX_ROWS:
        return None
    split = []
    for R, K, cell in ((4 * u, H, 5 * u * N), (u, 4 * H, 2 * u * N)):
        kc = min(F32_CHUNK, -(-K // 8) * 8)
        fixed = _f32_fixed_smem(N, R, kc, cell)
        r_on = min(R, (smem_per_block - fixed) // (4 * _f32_ld(K)))
        if r_on < 0:
            return None
        split.append((r_on, kc, fixed + 4 * r_on * _f32_ld(K)))
    (fr, fkc, fsm), (br, bkc, bsm) = split
    fwd_l2 = bwd_l2 = 0
    for b in range(grid):                   # the last CTA may own fewer units; its rows past them are not read
        nu = min(u, H - b * u)
        fwd_l2 += sum(1 for lr in range(fr, 4 * u) if lr % u < nu) * H * 4
        bwd_l2 += max(0, nu - br) * 4 * H * 4
    return LstmSeqF32Geometry(u, grid, fr, fkc, br, bkc, fsm, bsm, fwd_l2, bwd_l2)


def _stack_params(rnn: nn.LSTM, layer: int) -> Tuple[torch.Tensor, ...]:
    return tuple(getattr(rnn, "%s_l%d" % (n, layer)) for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"))


def _stack_ok(x: torch.Tensor, hx, rnn: nn.Module, fp32: bool = False):
    """The geometry (``LstmSeqGeometry``, or ``LstmSeqF32Geometry`` in fp32) and the kernels' storage type when
    ``lstm_stack`` runs the native path, else None."""
    if not (isinstance(rnn, nn.LSTM) and rnn.num_layers >= 1 and not rnn.bidirectional and rnn.bias
            and rnn.proj_size == 0 and not rnn.batch_first):
        return None
    if not (x.is_cuda and x.dim() == 3 and x.size(2) == rnn.input_size and x.size(0) > 0):
        return None
    if torch.is_autocast_enabled("cuda"):
        dt = torch.get_autocast_dtype("cuda")
        if dt not in (torch.bfloat16, torch.float16):
            return None
    elif fp32:
        dt = torch.float32
    else:
        return None
    if x.dtype not in (torch.float32, dt) or not ext.available():
        return None
    if any(p.dtype != torch.float32 or p.device != x.device for p in rnn.parameters()):
        return None
    L, N, H = rnn.num_layers, x.size(1), rnn.hidden_size
    if hx is not None:
        if not (isinstance(hx, (tuple, list)) and len(hx) == 2):
            return None
        for h in hx:
            if not (isinstance(h, torch.Tensor) and tuple(h.shape) == (L, N, H) and h.device == x.device
                    and h.dtype in (torch.float32, dt)):
                return None
    p = torch.cuda.get_device_properties(x.device)
    geometry = lstm_seq_f32_geometry if dt == torch.float32 else lstm_seq_geometry
    geom = geometry(H, N, p.multi_processor_count, p.shared_memory_per_block_optin)
    return None if geom is None else (geom, dt)


class _LstmSeqLayer(torch.autograd.Function):
    """One layer from (h0, c0) on the stacked-layer kernels: returns y [T, N, H] and h_n (both of type ``dt``) and c_n
    (fp32).  x, h0 and the parameters are cast to ``dt`` here, once per forward, and both passes run with autocast off.
    ``h0`` of the input's type or ``dt``, ``c0`` fp32 or ``dt``; their gradients come back in their types.  With
    ``dt`` fp32 nothing is cast, ``geom`` is an ``LstmSeqF32Geometry``, and the backward kernel reads W_hh^T, a copy
    made per backward pass."""

    @staticmethod
    def forward(ctx, x, h0, c0, geom, dt, w_ih, w_hh, b_ih, b_hh):
        C = ext.require()
        ctx.set_materialize_grads(False)
        T, N, I = x.shape
        H = w_hh.size(1)
        with torch.autocast(x.device.type, enabled=False):
            xs = x.to(dt).contiguous()
            w_ih_s, w_hh_s = w_ih.to(dt), ext.dense16(w_hh.to(dt))
            h0s, c0f = ext.dense16(h0.to(dt)), c0.float().contiguous()
            gx = torch.addmm((b_ih + b_hh).to(dt), xs.view(T * N, I), w_ih_s.t())      # (T N) x 4H
        y = torch.empty(T, N, H, device=x.device, dtype=dt)
        gates = torch.empty(T, N, 4 * H, device=x.device, dtype=torch.float32)
        cs = torch.empty(T, N, H, device=x.device, dtype=torch.float32)
        bar = torch.zeros(1, dtype=torch.int64, device=x.device)
        split = (N, geom.fwd_r_on, geom.fwd_kc) if dt == torch.float32 else (geom.fwd_rows, 0, 0)
        C.lstm_seq_forward(gx.data_ptr(), w_hh_s.data_ptr(), h0s.data_ptr(), c0f.data_ptr(), y.data_ptr(),
                           gates.data_ptr(), cs.data_ptr(), bar.data_ptr(), T, N, H, geom.units, split[0],
                           torch.cuda.current_stream().cuda_stream, DTYPE_CODE[dt], split[1], split[2])
        ctx.save_for_backward(xs, h0s, c0f, y, gates, cs, w_ih_s, w_hh_s)
        ctx.geom = geom
        ctx.dtypes = (x.dtype, h0.dtype, c0.dtype)
        return y, y[T - 1].clone(), cs[T - 1].clone()

    @staticmethod
    def backward(ctx, dy, dhn, dcn):
        C = ext.require()
        x, h0, c0, y, gates, cs, w_ih, w_hh = ctx.saved_tensors
        T, N, I = x.shape
        H = w_hh.size(1)
        dt = y.dtype
        dy = torch.zeros_like(y) if dy is None else dy.to(dt).contiguous()
        dhn = None if dhn is None else dhn.to(dt).contiguous()
        dcn = None if dcn is None else dcn.float().contiguous()
        dg = torch.empty(T, N, 4 * H, device=x.device, dtype=dt)
        dc0 = torch.empty(N, H, device=x.device, dtype=torch.float32)
        bar = torch.zeros(1, dtype=torch.int64, device=x.device)
        geom = ctx.geom
        if dt == torch.float32:                                 # fp32 streams rows of W_hh^T from L2
            whh, split = w_hh.t().contiguous(), (N, geom.bwd_r_on, geom.bwd_kc)
        else:
            whh, split = w_hh, (geom.bwd_rows, 0, 0)
        C.lstm_seq_backward(dy.data_ptr(), gates.data_ptr(), cs.data_ptr(), whh.data_ptr(), c0.data_ptr(),
                            0 if dhn is None else dhn.data_ptr(), 0 if dcn is None else dcn.data_ptr(), dg.data_ptr(),
                            dc0.data_ptr(), bar.data_ptr(), T, N, H, geom.units, split[0],
                            torch.cuda.current_stream().cuda_stream, DTYPE_CODE[dt], split[1], split[2])
        del whh
        need = ctx.needs_input_grad
        x_dt, h0_dt, c0_dt = ctx.dtypes
        g2 = dg.view(T * N, 4 * H)
        with torch.autocast(x.device.type, enabled=False):      # GEMMs in dt; the parameters' gradients come back fp32
            dx = (g2 @ w_ih).view(T, N, I).to(x_dt) if need[0] else None
            dh0 = (dg[0] @ w_hh).to(h0_dt) if need[1] else None
            dw_ih = (g2.t() @ x.view(T * N, I)).float() if need[5] else None
            if need[6]:                                         # h_{t-1}: h0, then y[:-1]
                hp = torch.cat([h0.unsqueeze(0), y[:-1]]).view(T * N, H)
                dw_hh = (g2.t() @ hp).float()
            else:
                dw_hh = None
            db = g2.sum(0, dtype=torch.float32) if need[7] or need[8] else None
        db_ih = db if need[7] else None
        db_hh = (db.clone() if need[7] else db) if need[8] else None             # two tensors, never one aliased
        return dx, dh0, dc0.to(c0_dt) if need[2] else None, None, None, dw_ih, dw_hh, db_ih, db_hh


def lstm_stack(x: torch.Tensor, hx, rnn: nn.Module, dropout_p: float, training: bool, fp32: bool = False):
    """``rnn(x, hx)`` for a uni-directional, multi-layer ``nn.LSTM`` over the time-major ``x`` (T x N x I): returns
    ``(y, (h_n, c_n))`` with h_n and c_n [L, N, H], as ``nn.LSTM`` does.  ``hx`` = (h0, c0), each [L, N, H], or None
    (zeros).

    Under bf16 / fp16 CUDA autocast its layers run one after another on the stacked-layer kernels (``lstm_seq_forward``
    / ``lstm_seq_backward``): each layer from its own (h0, c0), every row of length T, the step product on the tensor
    cores, W_hh held in shared memory in the autocast type (at H = 1500 that needs 16 bits: the fp32 slice, 288 KB per
    CTA, does not fit).  Between layers, in training, ``F.dropout(p=dropout_p)``, where ``nn.LSTM`` places its dropout
    (cuDNN draws its own masks, so the stock and fused layers see different ones).  y and h_n come back in the autocast
    type and c_n in fp32: the kernels keep the cell state in fp32, where cuDNN's 16-bit RNN keeps it in 16 bits.  The
    parameter gradients are fp32; h0 and c0 may be fp32 or of the autocast type, and their gradients have their types.
    Numerics otherwise as the module docstring's 16-bit layer: W_hh, gx, y, dy and dgates 16-bit, rounded to nearest
    even (an fp16 overflow is inf), everything else fp32, bitwise reproducible.

    With ``fp32=True`` and autocast off, an fp32 ``x`` runs on the fp32 forms of the same kernels (``hx`` fp32 too):
    y, h_n and c_n come back fp32.  The CTA keeps as many of its W_hh rows in shared memory as fit and reads the rest
    from L2 at every step (``lstm_seq_f32_geometry``), and the step product runs in 3xTF32 on the tensor cores, about
    fp32 accuracy, whatever ``torch.backends.cuda.matmul.allow_tf32`` says.  The input projection, dx, dh0, dW_ih and
    dW_hh are torch GEMMs and follow that switch, as ``lstm_layer``'s do.  Under autocast ``fp32`` changes nothing.

    Needs the native extension, fp32 parameters on x's device, bias, ``proj_size == 0``, ``batch_first=False``, x of
    fp32 or the autocast type, T >= 1, hx of the right shape, and an (H, N) that ``lstm_seq_geometry`` (in fp32
    ``lstm_seq_f32_geometry``) accepts on the device.  Anything else -- autocast off without ``fp32``, the CPU, fp64, a
    bidirectional ``rnn``, a layer too large -- returns exactly ``rnn(x, hx)``."""
    ok = _stack_ok(x, hx, rnn, fp32)
    if ok is None:
        return rnn(x, hx)
    geom, dt = ok
    L, N, H = rnn.num_layers, x.size(1), rnn.hidden_size
    if hx is None:
        z = torch.zeros(L, N, H, device=x.device, dtype=dt)
        hx = (z, z.float())
    h0, c0 = hx
    hs, cs = [], []
    for layer in range(L):
        if layer > 0 and training and dropout_p > 0:
            x = nn.functional.dropout(x, dropout_p, True)
        x, h, c = _LstmSeqLayer.apply(x.contiguous(), h0[layer], c0[layer], geom, dt, *_stack_params(rnn, layer))
        hs.append(h)
        cs.append(c)
    return x, (torch.stack(hs), torch.stack(cs))
