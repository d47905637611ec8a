"""DeepSpeech-style acoustic model "lstman4" (the reference's LSTM workload).

Architecture parity with ``VGG/models/lstm_models.py:148-239`` and the factory defaults of
``VGG/models/lstman4.py:8-33`` (hidden 800, 5 uni-directional LSTM layers, look-ahead context 20,
29 labels): two masked Conv2d+BN+Hardtanh blocks over the (freq, time) spectrogram, a stack of
BatchNorm+LSTM layers on packed sequences, a look-ahead convolution, BatchNorm + bias-free Linear.
27,569,568 parameters in 40 tensors.  Input ``(B, 1, 161, T)`` + lengths; output ``(B, T', classes)``
logits (softmax only in eval mode) + output lengths; trained with CTC.

``fuse_lstm=True`` (or ``net.fuse_lstm = True`` at any time) runs the uni-directional LSTM layers on the persistent
recurrence kernels of ``ops/fused_lstm.py`` instead of packing the sequences for cuDNN; parameters, buffers and
``state_dict`` keys are the same either way.  Under bf16 / fp16 autocast those layers are stock again unless
``fuse_lstm_autocast=True`` (``net.fuse_lstm_autocast``) is set as well, which runs the 16-bit forms of the kernels.
The bidirectional network (``bidirectional=True``) keeps stock layers under ``fuse_lstm`` unless
``fuse_lstm_bidirectional=True`` (``net.fuse_lstm_bidirectional``) is set as well, which runs both directions of each
layer in one launch of the kernels.  ``fuse_ctc=True`` (``net.fuse_ctc``, a plain attribute) asks the trainer to compute
the CTC loss with the fused softmax + CTC kernels (``ops/fused_ctc``); it does not change the network.
``fuse_bn=True`` (or ``net.fuse_bn = True`` at any time) runs the seven batch-norm sites on the kernels of
``ops/fused_frame_bn.py``: each conv block's mask -> BatchNorm2d -> mask -> Hardtanh -> mask in one kernel per pass, and
the BatchNorm1d in front of LSTM layers 1-4 and of ``fc`` likewise, with the lengths copied to the device once per
forward pass and shared with the LSTM layers.  Their statistics stop at the longest utterance, so a batch padded past it
(``Trainer(an4_pad_multiple=m)``) gives the unpadded batch's loss and gradients to rounding.  Off the kernels' domain (CPU, eval mode, ...)
those sites are the stock modules.
``fuse_lookahead=True`` (or ``net.fuse_lookahead = True`` at any time) runs the look-ahead convolution and its Hardtanh
on the kernels of ``ops/fused_lookahead.py``, one kernel per pass, the frames past each length read as 0 and written +0,
with the same device copy of the lengths; the bidirectional network has no look-ahead and refuses it (``ValueError``).
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops.fused_frame_bn import conv_block_bn, seq_bn
from ..ops.fused_lookahead import lookahead_hardtanh
from ..ops.fused_lstm import lstm_layer, lstm_layer_device, lstm_stack, stock_layer

AN4_LABELS = "_'ABCDEFGHIJKLMNOPQRSTUVWXYZ "     # 29 symbols, index 0 = CTC blank


class _TimeMaskedConv(nn.Module):
    """Conv stack that re-zeroes the padded time steps after every layer (``MaskConv``, :43-70)."""

    def __init__(self, seq: nn.Sequential):
        super().__init__()
        self.seq_module = seq

    def forward(self, x: torch.Tensor, lengths: torch.Tensor,
                bn_lengths: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``bn_lengths`` (the lengths on ``x``'s device): each Conv2d is followed by ``conv_block_bn`` on the
        BatchNorm2d in place of the mask / batch-norm / Hardtanh modules."""
        if bn_lengths is not None:
            mods = list(self.seq_module)
            for conv, bn in zip(mods[0::3], mods[1::3]):
                x = conv_block_bn(conv(x), bn, bn_lengths)
            return x
        t = torch.arange(x.size(3), device=x.device).view(1, 1, 1, -1)
        for m in self.seq_module:
            x = m(x)
            if t.size(3) != x.size(3):
                t = torch.arange(x.size(3), device=x.device).view(1, 1, 1, -1)
            x = x.masked_fill(t >= lengths.to(x.device).view(-1, 1, 1, 1), 0)
        return x


class _SeqBN(nn.Module):
    """BatchNorm1d applied on (T*N, H) (``SequenceWise``, :21-40)."""

    def __init__(self, module: nn.Module):
        super().__init__()
        self.module = module

    def forward(self, x: torch.Tensor, bn_lengths: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``bn_lengths`` (the lengths on ``x``'s device): the batch-norm (the module, or the first of a Sequential)
        runs as ``seq_bn``."""
        t, n = x.size(0), x.size(1)
        if bn_lengths is None:
            return self.module(x.reshape(t * n, -1)).view(t, n, -1)
        if isinstance(self.module, nn.Sequential):
            x = seq_bn(x, self.module[0], bn_lengths)
            return self.module[1:](x.reshape(t * n, -1)).view(t, n, -1)
        return seq_bn(x, self.module, bn_lengths)


class BatchRNN(nn.Module):
    """``fuse`` (default off) runs the recurrence through ``ops/fused_lstm.lstm_layer``, which falls back to the stock
    pack -> rnn -> pad sequence wherever its kernels do not apply; with ``fuse_autocast`` (default off) it takes the
    16-bit kernels under bf16 / fp16 autocast, where ``fuse`` alone is stock; with ``fuse_bidirectional`` (default off)
    a bidirectional layer takes them too, where ``fuse`` alone is stock."""

    def __init__(self, input_size: int, hidden_size: int, rnn_type=nn.LSTM, bidirectional: bool = False,
                 batch_norm: bool = True, fuse: bool = False, fuse_autocast: bool = False,
                 fuse_bidirectional: bool = False):
        super().__init__()
        self.bidirectional = bidirectional
        self.fuse = fuse
        self.fuse_autocast = fuse_autocast
        self.fuse_bidirectional = fuse_bidirectional
        self.batch_norm = _SeqBN(nn.BatchNorm1d(input_size)) if batch_norm else None
        self.rnn = rnn_type(input_size=input_size, hidden_size=hidden_size, bidirectional=bidirectional, bias=True)

    def forward(self, x: torch.Tensor, lengths: Optional[torch.Tensor],
                dev_lengths: Optional[torch.Tensor] = None, bn_lengths: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``lengths``: host int tensor; ``dev_lengths``: optionally the same as int32 on the device (fused path);
        ``bn_lengths``: the same on ``x``'s device, to run the batch-norm as ``seq_bn``.
        ``lengths=None``: the lengths are ``dev_lengths`` only and are never read on the host (``lstm_layer_device``);
        the layer must then take the fused kernels, else ``RuntimeError``."""
        if lengths is None and not self.fuse:
            raise RuntimeError("device-only lengths need the fused LSTM layer (fuse_lstm)")
        if self.batch_norm is not None:
            x = self.batch_norm(x, bn_lengths)
        if lengths is None:
            return lstm_layer_device(x, dev_lengths, self.rnn, autocast=self.fuse_autocast,
                                     bidirectional=self.fuse_bidirectional)
        if self.fuse:
            return lstm_layer(x, lengths, self.rnn, dev_lengths, autocast=self.fuse_autocast,
                              bidirectional=self.fuse_bidirectional)
        return stock_layer(x, lengths, self.rnn)


class Lookahead(nn.Module):
    """Look-ahead convolution (Wang et al. 2016): per-feature weighted sum over the next ``context``
    frames -- a depthwise 1-D convolution (the reference materialises a TxNxHx(context+1) tensor, :119-132)."""

    def __init__(self, n_features: int, context: int):
        super().__init__()
        assert context > 0
        self.n_features, self.context = n_features, context
        self.weight = nn.Parameter(torch.empty(n_features, context + 1))
        stdv = 1.0 / math.sqrt(context + 1)
        nn.init.uniform_(self.weight, -stdv, stdv)

    def forward(self, x: torch.Tensor) -> torch.Tensor:          # T x N x H
        y = F.pad(x.permute(1, 2, 0), (0, self.context))          # N x H x (T + context)
        y = F.conv1d(y, self.weight.unsqueeze(1), groups=self.n_features)
        return y.permute(2, 0, 1).contiguous()


class DeepSpeech(nn.Module):
    def __init__(self, rnn_hidden_size: int = 800, nb_layers: int = 5, labels: str = AN4_LABELS,
                 rnn_type=nn.LSTM, bidirectional: bool = False, context: int = 20, sample_rate: int = 16000,
                 window_size: float = 0.02, fuse_lstm: bool = False, fuse_lstm_autocast: bool = False,
                 fuse_lstm_bidirectional: bool = False, fuse_ctc: bool = False, fuse_bn: bool = False,
                 fuse_lookahead: bool = False):
        super().__init__()
        self._labels = labels
        self._bidirectional = bidirectional
        num_classes = len(labels)
        self.conv = _TimeMaskedConv(nn.Sequential(
            nn.Conv2d(1, 32, kernel_size=(41, 11), stride=(2, 2), padding=(20, 5)),
            nn.BatchNorm2d(32), nn.Hardtanh(0, 20, inplace=True),
            nn.Conv2d(32, 32, kernel_size=(21, 11), stride=(2, 1), padding=(10, 5)),
            nn.BatchNorm2d(32), nn.Hardtanh(0, 20, inplace=True)))
        f = int(math.floor(sample_rate * window_size / 2) + 1)          # 161 frequency bins
        f = int(math.floor(f + 2 * 20 - 41) / 2 + 1)
        f = int(math.floor(f + 2 * 10 - 21) / 2 + 1)
        rnn_in = f * 32
        rnns = [BatchRNN(rnn_in, rnn_hidden_size, rnn_type, bidirectional, batch_norm=False)]
        for _ in range(nb_layers - 1):
            rnns.append(BatchRNN(rnn_hidden_size, rnn_hidden_size, rnn_type, bidirectional))
        self.rnns = nn.ModuleList(rnns)
        self.lookahead = None if bidirectional else nn.Sequential(
            Lookahead(rnn_hidden_size, context=context), nn.Hardtanh(0, 20, inplace=True))
        self.fc = _SeqBN(nn.Sequential(nn.BatchNorm1d(rnn_hidden_size),
                                       nn.Linear(rnn_hidden_size, num_classes, bias=False)))
        self.fuse_lstm = fuse_lstm
        self.fuse_lstm_autocast = fuse_lstm_autocast
        self.fuse_lstm_bidirectional = fuse_lstm_bidirectional
        self.fuse_ctc = bool(fuse_ctc)
        self.fuse_bn = fuse_bn
        self.fuse_lookahead = fuse_lookahead

    @property
    def fuse_lookahead(self) -> bool:
        """Whether the look-ahead convolution and its Hardtanh take the fused kernels of ``ops/fused_lookahead.py``.
        Setting it on the bidirectional network, which has no look-ahead, raises ``ValueError``."""
        return self._fuse_lookahead

    @fuse_lookahead.setter
    def fuse_lookahead(self, on: bool) -> None:
        if on and self.lookahead is None:
            raise ValueError("fuse_lookahead needs the look-ahead convolution: the bidirectional network has none")
        self._fuse_lookahead = bool(on)

    @property
    def fuse_bn(self) -> bool:
        """Whether the batch-norm sites take the fused kernels of ``ops/fused_frame_bn.py``, with statistics over the
        frames of the longest utterance."""
        return self._fuse_bn

    @fuse_bn.setter
    def fuse_bn(self, on: bool) -> None:
        self._fuse_bn = bool(on)

    @property
    def fuse_lstm(self) -> bool:
        """Whether every ``BatchRNN`` layer takes the fused recurrence kernels (``ops/fused_lstm.py``)."""
        return all(m.fuse for m in self.rnns)

    @fuse_lstm.setter
    def fuse_lstm(self, on: bool) -> None:
        for m in self.rnns:
            m.fuse = bool(on)

    @property
    def fuse_lstm_autocast(self) -> bool:
        """Whether every fused ``BatchRNN`` layer keeps its kernels (their 16-bit forms) under bf16 / fp16 autocast."""
        return all(m.fuse_autocast for m in self.rnns)

    @fuse_lstm_autocast.setter
    def fuse_lstm_autocast(self, on: bool) -> None:
        for m in self.rnns:
            m.fuse_autocast = bool(on)

    @property
    def fuse_lstm_bidirectional(self) -> bool:
        """Whether every fused bidirectional ``BatchRNN`` layer runs both directions on the kernels (one launch)."""
        return all(m.fuse_bidirectional for m in self.rnns)

    @fuse_lstm_bidirectional.setter
    def fuse_lstm_bidirectional(self, on: bool) -> None:
        for m in self.rnns:
            m.fuse_bidirectional = bool(on)

    def get_seq_lens(self, input_length: torch.Tensor) -> torch.Tensor:
        seq = input_length
        for m in self.conv.modules():
            if isinstance(m, nn.Conv2d):
                seq = (seq + 2 * m.padding[1] - m.dilation[1] * (m.kernel_size[1] - 1) - 1) // m.stride[1] + 1
        return seq.int()

    def device_lengths_error(self, cuda: bool = True, autocast: bool = False) -> Optional[str]:
        """Why ``forward(..., device_lengths=True)`` cannot run on a CUDA (``cuda``) input with bf16 / fp16 autocast on
        (``autocast``) or off, or None: every LSTM layer must take the fused kernels, since the stock layers pack their
        sequences with host lengths."""
        if not cuda:
            return "device lengths need a CUDA input"
        if not self.fuse_lstm:
            return "device lengths need fuse_lstm: the stock LSTM layers pack with host lengths"
        if autocast and not self.fuse_lstm_autocast:
            return "device lengths under autocast need fuse_lstm_autocast: the LSTM layers would be stock"
        if self._bidirectional and not self.fuse_lstm_bidirectional:
            return "device lengths with bidirectional layers need fuse_lstm_bidirectional: the layers would be stock"
        return None

    def forward(self, x: torch.Tensor, lengths: torch.Tensor,
                device_lengths: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
        """``lengths``: the input frames of each utterance.  ``device_lengths=True``: ``lengths`` is an int32 tensor on
        ``x``'s device, each in [1, T], and is never read on the host: the conv masks, every LSTM layer
        (``lstm_layer_device``) and the returned output lengths stay on the device, so the step can be captured in a CUDA
        graph.  It raises ``RuntimeError`` where a layer would be stock (``device_lengths_error``).  Default: the
        lengths are copied to the host once, as they always were."""
        if device_lengths:
            why = self.device_lengths_error(x.is_cuda, torch.is_autocast_enabled("cuda"))
            if why is not None:
                raise RuntimeError(why)
            if lengths.dtype != torch.int32 or lengths.device != x.device:
                raise RuntimeError("device lengths must be an int32 tensor on the input's device")
            return self._forward(x, self.get_seq_lens(lengths), None)
        out_lens = self.get_seq_lens(lengths.cpu().int())
        return self._forward(x, out_lens, out_lens)

    def _forward(self, x: torch.Tensor, out_lens: torch.Tensor,
                 host_lens: Optional[torch.Tensor]) -> Tuple[torch.Tensor, torch.Tensor]:
        """``out_lens`` on the host (``host_lens`` the same tensor) or on the device only (``host_lens`` None)."""
        # the fused batch-norm, LSTM layers and look-ahead read the lengths on the device: one copy for all of them
        bn_lens = out_lens.to(x.device) if self.fuse_bn else None
        x = self.conv(x, out_lens, bn_lens)
        b, c, d, t = x.size()
        x = x.view(b, c * d, t).permute(2, 0, 1).contiguous()        # T x N x H
        dev_lens = None
        if x.is_cuda and any(m.fuse for m in self.rnns):
            dev_lens = bn_lens if bn_lens is not None else out_lens.to(x.device)
        for rnn in self.rnns:
            x = rnn(x, host_lens, dev_lens, bn_lens)
        if self.lookahead is not None:
            if self.fuse_lookahead:
                la_lens = dev_lens if dev_lens is not None else bn_lens if bn_lens is not None else out_lens.to(x.device)
                x = lookahead_hardtanh(x, self.lookahead[0].weight, la_lens)
            else:
                x = self.lookahead(x)
        x = self.fc(x, bn_lens).transpose(0, 1)                       # N x T x classes
        if not self.training:
            x = F.softmax(x, dim=-1)
        return x, out_lens


def lstman4(hidden_size: int = 800, hidden_layers: int = 5, bidirectional: bool = False,
            fuse_lstm: bool = False, fuse_lstm_autocast: bool = False,
            fuse_lstm_bidirectional: bool = False, fuse_ctc: bool = False, fuse_bn: bool = False,
            fuse_lookahead: bool = False) -> DeepSpeech:
    """``VGG/models/lstman4.py:8`` defaults."""
    return DeepSpeech(rnn_hidden_size=hidden_size, nb_layers=hidden_layers, bidirectional=bidirectional,
                      fuse_lstm=fuse_lstm, fuse_lstm_autocast=fuse_lstm_autocast,
                      fuse_lstm_bidirectional=fuse_lstm_bidirectional, fuse_ctc=fuse_ctc, fuse_bn=fuse_bn,
                      fuse_lookahead=fuse_lookahead)


class PTBLSTM(nn.Module):
    """2-layer 1500-hidden word-level LSTM language model (``VGG/models/lstm.py:5-40``), vocab 10k.

    ``fuse_lstm=True`` (or ``net.fuse_lstm = True`` at any time) runs the stacked ``nn.LSTM`` through
    ``ops/fused_lstm.lstm_stack``: under bf16 / fp16 CUDA autocast, on the 16-bit stacked-layer kernels with the carried
    state in and out; anywhere else exactly the stock layer, unless ``fuse_lstm_fp32=True`` (``net.fuse_lstm_fp32``) is
    set as well, which runs fp32 on CUDA on the fp32 forms of the kernels (W_hh partly streamed from L2, the step in
    3xTF32).  The returned c_n is fp32 either way.  ``fuse_lstm_fp32`` alone is the stock layer.  ``fuse_xent=True`` (``net.fuse_xent``) asks the trainer to compute the loss with the fused softmax
    cross-entropy (``ops/fused_xent``).  Parameters, buffers and ``state_dict`` keys are the same either way."""

    def __init__(self, vocab_size: int = 10000, embedding_dim: int = 1500, num_steps: int = 35, batch_size: int = 20,
                 num_layers: int = 2, dp_keep_prob: float = 0.35, fuse_lstm: bool = False, fuse_xent: bool = False,
                 fuse_lstm_fp32: bool = False):
        super().__init__()
        self.fuse_lstm = bool(fuse_lstm)
        self.fuse_lstm_fp32 = bool(fuse_lstm_fp32)
        self.fuse_xent = bool(fuse_xent)
        self.embedding_dim, self.num_layers = embedding_dim, num_layers
        self.dropout = nn.Dropout(1 - dp_keep_prob)
        self.word_embeddings = nn.Embedding(vocab_size, embedding_dim)
        self.lstm = nn.LSTM(embedding_dim, embedding_dim, num_layers=num_layers, dropout=1 - dp_keep_prob)
        self.sm_fc = nn.Linear(embedding_dim, vocab_size)
        for w in (self.word_embeddings.weight, self.sm_fc.weight):
            nn.init.uniform_(w, -0.1, 0.1)
        nn.init.zeros_(self.sm_fc.bias)

    def init_hidden(self, batch_size: int, device=None):
        z = torch.zeros(self.num_layers, batch_size, self.embedding_dim, device=device)
        return (z, z.clone())

    def forward(self, inputs: torch.Tensor, hidden):
        emb = self.dropout(self.word_embeddings(inputs))
        if self.fuse_lstm:
            out, hidden = lstm_stack(emb, hidden, self.lstm, self.lstm.dropout, self.training, self.fuse_lstm_fp32)
        else:
            out, hidden = self.lstm(emb, hidden)
        out = self.dropout(out)
        logits = self.sm_fc(out.view(-1, self.embedding_dim))
        return logits.view(inputs.size(0), inputs.size(1), -1), hidden
