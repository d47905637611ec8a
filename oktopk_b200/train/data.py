"""Data pipelines: synthetic generators of every dataset shape the reference trains on, with the
same sharding semantics (``DistributedSampler`` when world > 1, ``VGG/dl_trainer.py:312-467``), plus
optional real-data loaders when the files are already on disk (there is no network here).

Shapes: CIFAR-10 ``[B,3,32,32]``/10 classes, ImageNet ``[B,3,224,224]``/1000, MNIST ``[B,1,28,28]``,
AN4 spectrograms ``[B,1,161,T]`` + transcripts for CTC (the reference's ``audio_data`` loader is
missing from its repo, SURVEY D1), PTB ``[35,B]`` token windows, Wikipedia-shaped BERT pre-training
features ``input_ids/segment_ids/input_mask/lm_label_ids [B,128]`` + ``is_next [B]``
(``BERT/bert/main_bert.py:535-639``).

Batches are produced in pinned host memory; ``Prefetcher`` moves them to the device on a side stream
(H2D overlapped with compute) -- the reference does a synchronous ``.cuda()`` per step.
"""
from __future__ import annotations

import math
from typing import Dict, Iterator, List, NamedTuple, Optional, Tuple

import torch
from torch.utils.data import DataLoader, Dataset, DistributedSampler

DATASET_CLASSES = {"cifar10": 10, "imagenet": 1000, "mnist": 10, "an4": 29, "ptb": 10000, "wikipedia": 30522}


def teacher_labels(images: torch.Tensor, classes: int, seed: int = 4242) -> torch.Tensor:
    """Learnable synthetic labels: argmax of a fixed random linear map of the image.  (Purely random labels make
    training collapse to the uniform prediction within ~50 steps, after which gradients -- and the sparse selection
    the benchmark is about -- degenerate.)"""
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(images[0].numel(), classes, generator=g)
    return (images.flatten(1) @ w).argmax(1)


class SyntheticImages(Dataset):
    def __init__(self, n: int, shape: Tuple[int, int, int], classes: int, seed: int = 0):
        g = torch.Generator().manual_seed(seed)
        self.n, self.shape, self.classes = n, shape, classes
        # a small pool of distinct images re-indexed cyclically keeps host memory bounded
        self.pool = torch.randn((min(n, 2048),) + shape, generator=g)
        self.pool_labels = teacher_labels(self.pool, classes)

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        j = i % self.pool.size(0)
        return self.pool[j], self.pool_labels[j]

    def __getitems__(self, idxs):
        """Batched fetch (DataLoader calls this with the whole index list): two gathers instead of 2 x batch tensor
        views + a stack -- the host side of a 1.2 ms GPU step must stay in the tens of microseconds."""
        j = torch.as_tensor(idxs, dtype=torch.long) % self.pool.size(0)
        return self.pool.index_select(0, j), self.pool_labels.index_select(0, j)

    @staticmethod
    def collate_batched(batch):
        return batch                       # already a (images, labels) pair of stacked tensors


def an4_templates(labels: int = 29, seed: int = 4243) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return torch.randn(labels, 161, generator=g)


def an4_utterance(target: torch.Tensor, frames_per_char: int, templates: torch.Tensor, gen: torch.Generator,
                  noise: float = 0.5) -> torch.Tensor:
    """A learnable synthetic utterance: every character is ``frames_per_char`` frames of its spectral template + noise."""
    base = templates[target.long()].repeat_interleave(frames_per_char, dim=0).t()          # [161, T]
    return base + noise * torch.randn(base.shape, generator=gen)


class SyntheticAN4(Dataset):
    """Variable-length spectrogram + transcript pairs (AN4: ~1-5 s utterances, 161 frequency bins, 100-400 frames)."""

    def __init__(self, n: int = 948, min_frames: int = 100, max_frames: int = 400, seed: int = 0, labels: int = 29):
        g = torch.Generator().manual_seed(seed)
        self.n = n
        self.fpc = 12
        self.tlen = torch.randint(max(min_frames // self.fpc, 2), max_frames // self.fpc + 1, (n,), generator=g)
        self.frames = self.tlen * self.fpc
        self.seed, self.labels = seed, labels
        self.templates = an4_templates(labels)

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        g = torch.Generator().manual_seed(self.seed * 1_000_003 + i)
        target = torch.randint(1, self.labels, (int(self.tlen[i]),), generator=g)
        return an4_utterance(target, self.fpc, self.templates, g), target


def an4_collate(batch):
    """Sort by length (longest first), pad spectrograms, concatenate targets (deepspeech convention)."""
    batch = sorted(batch, key=lambda s: s[0].size(1), reverse=True)
    T = batch[0][0].size(1)
    B = len(batch)
    inputs = torch.zeros(B, 1, 161, T)
    in_pct = torch.empty(B)
    tsizes = torch.empty(B, dtype=torch.int32)
    targets = []
    for i, (sp, tg) in enumerate(batch):
        inputs[i, 0, :, :sp.size(1)] = sp
        in_pct[i] = sp.size(1) / float(T)
        tsizes[i] = tg.numel()
        targets.append(tg)
    return inputs, torch.cat(targets).int(), in_pct, tsizes


AN4_MAX_TARGETS = 2047          # ops/fused_ctc's fast-path limit on a batch's targets (csrc/ctc.cu kCtcMaxTargets)


class PaddedAN4Batch(NamedTuple):
    """An AN4 training batch staged for a fixed-shape step (``pad_an4_batch``): every tensor's shape depends on the batch
    size and the padded frame count ``T_b`` only, and no field needs a host read of device memory."""
    inputs: torch.Tensor        # [B, 1, 161, T_b]: the batch, then zero frames
    lengths: torch.Tensor       # int32 [B] on the device: (in_pct * T).int() clamped to [1, T], T the unpadded length
    targets: torch.Tensor       # int32 [capacity]: the concatenated targets, then zeros ([ntargets] if over capacity)
    tsizes: torch.Tensor        # int32 [B]: target sizes
    ntargets: int               # the batch's number of targets (a host value: targets.numel() before padding)
    over_capacity: bool         # ntargets > capacity: the targets are not padded, and the shape is the batch's own


def an4_padded_frames(T: int, multiple: int) -> int:
    """``T`` rounded up to a multiple of ``multiple`` (>= 1)."""
    return -(-T // multiple) * multiple


def an4_target_capacity(B: int, out_frames: int) -> int:
    """The targets a padded batch holds: one per output frame of every utterance, at most ``AN4_MAX_TARGETS``."""
    return min(B * out_frames, AN4_MAX_TARGETS)


def pad_an4_batch(batch, multiple: int, out_frames) -> PaddedAN4Batch:
    """Stage the trainer's AN4 batch ``(inputs [B, 1, 161, T], targets, in_pct, tsizes)`` (device tensors) into a
    ``PaddedAN4Batch`` with ``T_b = an4_padded_frames(T, multiple)`` frames.  ``out_frames(T_b)``: the model's output
    frames for ``T_b`` input frames, which sets the target capacity.  A few tensor ops on the current stream; every size
    comes from the shapes, so nothing is read back to the host."""
    inputs, targets, in_pct, tsizes = batch
    B, T = inputs.size(0), inputs.size(3)
    Tb = an4_padded_frames(T, multiple)
    padded = torch.nn.functional.pad(inputs, (0, Tb - T)) if Tb > T else inputs
    lengths = (in_pct * T).int().clamp_(1, T)           # the eager formula, kept inside the tensor
    n = targets.numel()
    cap = an4_target_capacity(B, out_frames(Tb))
    tg = targets.to(torch.int32)
    if n <= cap:
        tg = torch.cat([tg, tg.new_zeros(cap - n)])
    return PaddedAN4Batch(padded, lengths, tg, tsizes.to(torch.int32), n, n > cap)


class SyntheticPTB(Dataset):
    def __init__(self, n_tokens: int = 929_589, vocab: int = 10000, batch_size: int = 20, num_steps: int = 35, seed: int = 0):
        g = torch.Generator().manual_seed(seed)
        self.data = torch.randint(0, vocab, (n_tokens,), generator=g)
        self.num_steps = num_steps
        self.n = (n_tokens - 1) // num_steps

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        s = i * self.num_steps
        return self.data[s:s + self.num_steps], self.data[s + 1:s + 1 + self.num_steps]


class SyntheticWikipedia(Dataset):
    def __init__(self, n: int = 100_000, seq: int = 128, vocab: int = 30522, seed: int = 0):
        self.n, self.seq, self.vocab, self.seed = n, seq, vocab, seed

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        from ..models.bert import synthetic_batch
        g = torch.Generator().manual_seed(self.seed * 7_000_003 + i)
        ids, seg, mask, labels, nxt = synthetic_batch(1, self.seq, self.vocab, generator=g)
        return ids[0], seg[0], mask[0], labels[0], nxt[0]


class PTBText(Dataset):
    """Penn Treebank from ``ptb.{train,valid,test}.txt`` (``VGG/ptb_reader.py``: whitespace tokens, ``<eos>`` per line,
    vocabulary sorted by frequency) as ``num_steps`` windows of (input, shifted target)."""

    def __init__(self, data_dir: str, split: str = "train", num_steps: int = 35, vocab: Optional[Dict[str, int]] = None):
        import collections
        import os

        def read(path):
            with open(path, "r", encoding="utf-8") as f:
                return f.read().replace("\n", " <eos> ").split()
        if vocab is None:
            words = read(os.path.join(data_dir, "ptb.train.txt"))
            cnt = collections.Counter(words)
            vocab = {w: i for i, (w, _) in enumerate(sorted(cnt.items(), key=lambda kv: (-kv[1], kv[0])))}
        self.vocab = vocab
        unk = vocab.get("<unk>", 0)
        toks = read(os.path.join(data_dir, "ptb.%s.txt" % split))
        self.data = torch.tensor([vocab.get(w, unk) for w in toks], dtype=torch.long)
        self.num_steps = num_steps
        self.n = max((self.data.numel() - 1) // num_steps, 0)

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        s = i * self.num_steps
        return self.data[s:s + self.num_steps], self.data[s + 1:s + 1 + self.num_steps]


class AN4Manifest(Dataset):
    """AN4-style speech corpus from a manifest (``wav_path,transcript_path`` per line -- the deepspeech.pytorch layout
    the reference's missing ``audio_data/data_loader.py`` consumed, SURVEY D1): 16 kHz wav -> log-magnitude STFT
    spectrogram (20 ms window, 10 ms stride => 161 bins), per-utterance normalisation, transcript -> label ids."""

    def __init__(self, manifest: str, labels: str, sample_rate: int = 16000, window_size: float = 0.02,
                 window_stride: float = 0.01, normalize: bool = True):
        import os
        self.items = []
        base = os.path.dirname(os.path.abspath(manifest))
        with open(manifest) as f:
            for line in f:
                line = line.strip()
                if line:
                    a, b = line.split(",")[:2]
                    self.items.append((a if os.path.isabs(a) else os.path.join(base, a),
                                       b if os.path.isabs(b) else os.path.join(base, b)))
        self.labels_map = {c: i for i, c in enumerate(labels)}
        self.sr, self.n_fft, self.hop = sample_rate, int(sample_rate * window_size), int(sample_rate * window_stride)
        self.normalize = normalize

    def __len__(self):
        return len(self.items)

    def spectrogram(self, wav_path: str) -> torch.Tensor:
        from scipy.io import wavfile
        sr, y = wavfile.read(wav_path)
        y = torch.as_tensor(y.astype("float32"))
        if y.dim() > 1:
            y = y.mean(1)
        if y.abs().max() > 1.5:
            y = y / 32768.0
        win = torch.hamming_window(self.n_fft, periodic=False)
        spec = torch.stft(y, self.n_fft, self.hop, self.n_fft, window=win, return_complex=True).abs()
        spec = torch.log1p(spec)
        if self.normalize:
            spec = (spec - spec.mean()) / (spec.std() + 1e-8)
        return spec                                            # [n_fft // 2 + 1 = 161, frames]

    def __getitem__(self, i):
        wav, txt = self.items[i]
        with open(txt, "r", encoding="utf-8") as f:
            t = f.read().strip().upper()
        target = torch.tensor([self.labels_map[c] for c in t if c in self.labels_map], dtype=torch.long)
        return self.spectrogram(wav), target


class ImageNetHDF5(Dataset):
    """ImageNet packed in one HDF5 file (``VGG/datasets.py:8-36``): datasets ``<split>_img`` uint8 ``[N,H,W,3]`` and
    ``<split>_labels``.  Needs ``h5py`` (not in this image: raises ImportError, callers fall back to synthetic)."""

    def __init__(self, path: str, train: bool = True):
        import h5py                                             # noqa: WPS433
        self.f = h5py.File(path, "r")
        k = "train" if train else "val"
        self.img, self.lab = self.f[k + "_img"], self.f[k + "_labels"]
        self.mean = torch.tensor([0.485, 0.456, 0.406]).view(3, 1, 1)
        self.std = torch.tensor([0.229, 0.224, 0.225]).view(3, 1, 1)

    def __len__(self):
        return int(self.lab.shape[0])

    def __getitem__(self, i):
        x = torch.from_numpy(self.img[i]).permute(2, 0, 1).float() / 255.0
        return (x - self.mean) / self.std, int(self.lab[i])


def build_dataset(name: str, data_dir: Optional[str] = None, train: bool = True, seed: int = 0, **kw) -> Dataset:
    """Real data if it is already on disk under ``data_dir`` (never downloads), else synthetic."""
    name = name.lower()
    if data_dir and name in ("cifar10", "mnist"):
        try:
            import torchvision
            import torchvision.transforms as T
            if name == "cifar10":
                tf = T.Compose(([T.RandomCrop(32, padding=4), T.RandomHorizontalFlip()] if train else []) +
                               [T.ToTensor(), T.Normalize((0.4914, 0.4822, 0.4465), (0.2023, 0.1994, 0.2010))])
                return torchvision.datasets.CIFAR10(data_dir, train=train, download=False, transform=tf)
            tf = T.Compose([T.ToTensor(), T.Normalize((0.1307,), (0.3081,))])
            return torchvision.datasets.MNIST(data_dir, train=train, download=False, transform=tf)
        except Exception:  # noqa: BLE001 - fall back to synthetic
            pass
    if data_dir and name in ("ptb", "an4", "imagenet"):
        import os
        try:
            if name == "ptb" and os.path.isfile(os.path.join(data_dir, "ptb.train.txt")):
                return PTBText(data_dir, "train" if train else "valid", kw.get("num_steps", 35))
            if name == "an4":
                man = os.path.join(data_dir, "an4_train_manifest.csv" if train else "an4_val_manifest.csv")
                if os.path.isfile(man):
                    from ..models.deepspeech import AN4_LABELS
                    return AN4Manifest(man, AN4_LABELS)
            if name == "imagenet":
                for cand in ("imagenet-shuffled.hdf5", "imagenet.hdf5"):
                    if os.path.isfile(os.path.join(data_dir, cand)):
                        return ImageNetHDF5(os.path.join(data_dir, cand), train)
        except Exception:  # noqa: BLE001 - fall back to synthetic
            pass
    if name == "cifar10":
        return SyntheticImages(50_000 if train else 10_000, (3, 32, 32), 10, seed)
    if name == "imagenet":
        return SyntheticImages(kw.get("n", 12_800), (3, 224, 224), 1000, seed)
    if name == "mnist":
        return SyntheticImages(60_000 if train else 10_000, (1, 28, 28), 10, seed)
    if name == "an4":
        return SyntheticAN4(948 if train else 130, seed=seed)
    if name == "ptb":
        return SyntheticPTB(seed=seed, **{k: v for k, v in kw.items() if k in ("batch_size", "num_steps")})
    if name in ("wikipedia", "bert"):
        if data_dir:
            # a real corpus on disk: <data_dir>/{train,valid}.txt (or corpus.txt) + optional vocab.txt
            import os
            from ..utils.tokenization import BertTokenizer
            from .bert_data import BERTDataset
            for cand in (("train.txt" if train else "valid.txt"), "corpus.txt"):
                path = os.path.join(data_dir, cand)
                if os.path.isfile(path):
                    vf = os.path.join(data_dir, "vocab.txt")
                    tok = BertTokenizer(vf) if os.path.isfile(vf) else BertTokenizer.synthetic()
                    return BERTDataset(path, tok, seq_len=kw.get("seq", 128), seed=seed)
        return SyntheticWikipedia(seq=kw.get("seq", 128), seed=seed)
    raise ValueError("unknown dataset %r" % name)


def build_loader(dataset: Dataset, name: str, batch_size: int, rank: int, world: int, train: bool = True,
                 num_workers: int = 0, seed: int = 0):
    sampler = DistributedSampler(dataset, num_replicas=world, rank=rank, shuffle=train, seed=seed) if world > 1 else None
    collate = an4_collate if name == "an4" else getattr(dataset, "collate_batched", None)
    loader = DataLoader(dataset, batch_size=batch_size, shuffle=(train and sampler is None), sampler=sampler,
                        num_workers=num_workers, pin_memory=False, drop_last=train, collate_fn=collate)
    return loader, sampler


class Prefetcher:
    """Endless iterator over a DataLoader that stages batches on the device from pinned memory on a side stream.

    Optionally (``OKTOPK_PREFETCH_THREAD=1`` / ``threaded=True``) a background thread runs the host side of the pipeline (DataLoader iteration + collate, copy into a reusable
    pinned buffer, H2D enqueue on the side stream) up to ``depth`` batches ahead, so the training thread's per-step cost is
    a queue pop and an event wait: with 1.2 ms GPU steps the few hundred microseconds of Python per batch must not sit on
    the critical path (the reference does a synchronous ``.cuda()`` per step).  By default everything stays on the
    calling thread: ``next(defer=True)`` + ``advance()`` overlap the staging of the next batch with the running step."""

    def __init__(self, loader: DataLoader, device: torch.device, sampler=None, depth: int = 3, threaded: Optional[bool] = None):
        import os
        self.loader, self.device, self.sampler = loader, device, sampler
        self.epoch = 0
        self.it: Optional[Iterator] = None
        self.stream = torch.cuda.Stream() if device.type == "cuda" else None
        self.next_batch = None
        self.h2d_bytes = 0
        self._pinned = {}
        self._ring = 0
        self._nring = max(depth + 1, 8)
        self._ring_events = {}
        if threaded is None:
            # opt-in: at millisecond steps the extra Python thread buys nothing over the single-threaded host path and adds
            # GIL / CPU-quota interference
            threaded = device.type == "cuda" and os.environ.get("OKTOPK_PREFETCH_THREAD", "0") == "1"
        self.threaded = bool(threaded) and self.stream is not None
        self._q = None
        self._stop = False
        self._thread = None
        self._err = None
        if self.threaded:
            import queue
            import threading
            self._q = queue.Queue(maxsize=max(depth, 1))
            self._thread = threading.Thread(target=self._worker, name="okt-prefetch", daemon=True)
            self._thread.start()
        else:
            self._preload()

    def _raw_next(self):
        if self.it is None:
            if self.sampler is not None:
                self.sampler.set_epoch(self.epoch)
            self.it = iter(self.loader)
        try:
            return next(self.it)
        except StopIteration:
            self.epoch += 1
            self.it = None
            return self._raw_next()

    SIDE_STREAM_MIN_BYTES = 4 << 20

    def _stage(self):
        """Host batch -> reusable pinned buffers -> device.  Returns (device batch, H2D-done event or None, bytes).

        Small batches (< 4 MB: a CIFAR batch is 0.2 MB, 8 us of copy time) are copied on the CONSUMER's stream, in order
        with the step that uses them: no second stream, no cross-stream events, no ``record_stream`` bookkeeping in the
        caching allocator -- nothing to overlap anyway.  Large batches (ImageNet: ~150 MB) go through the side stream so
        that the copy overlaps the previous step."""
        batch = self._raw_next()
        if self.stream is None:
            return batch, None, 0
        nbytes = sum(t.numel() * t.element_size() for t in batch if torch.is_tensor(t))
        side = nbytes >= self.SIDE_STREAM_MIN_BYTES or self.threaded     # (a staging THREAD has no consumer stream of its own)
        # a small ring of reusable pinned buffers (no per-step cudaHostAlloc, no pin thread)
        self._ring = (self._ring + 1) % self._nring
        ev = self._ring_events.get(self._ring)
        if ev is not None:
            ev.synchronize()          # the host may run steps ahead of the device: never overwrite a slot still being copied
        stream = self.stream if side else torch.cuda.current_stream()
        with torch.cuda.stream(stream):
            out = []
            for j, t in enumerate(batch):
                if torch.is_tensor(t):
                    key = (self._ring, j)
                    buf = self._pinned.get(key)
                    if buf is None or buf.numel() < t.numel() or buf.dtype != t.dtype:
                        # cudaHostAlloc synchronises the device (and takes milliseconds): allocate the staging buffers
                        # of ALL ring slots at once, with head-room for variable-length batches, the first time a size is
                        # seen -- never one slot at a time in the middle of a run
                        cap = max(t.numel(), 1)
                        if buf is not None:
                            cap = int(cap * 1.5)
                        for r in range(self._nring):
                            self._pinned[(r, j)] = torch.empty(cap, dtype=t.dtype).pin_memory()
                        buf = self._pinned[key]
                    host = buf[:t.numel()].view(t.shape)
                    host.copy_(t)
                    out.append(host.to(self.device, non_blocking=True))
                else:
                    out.append(t)
            done = torch.cuda.Event(blocking=True)       # a host wait on it sleeps instead of spinning a core
            done.record(stream)
            self._ring_events[self._ring] = done
        return tuple(out), (done if side else None), nbytes

    def _worker(self):
        import queue
        try:
            torch.cuda.set_device(self.device)
            torch.set_num_threads(1)         # OpenMP's thread count is per calling thread: without this the staging thread
            while not self._stop:            # splits its 200 KB copies over a full OpenMP team (measured: 0.3 -> 3 ms per batch)
                item = self._stage()
                while not self._stop:
                    try:
                        self._q.put(item, timeout=0.2)
                        break
                    except queue.Full:
                        continue
        except BaseException as e:  # noqa: BLE001 - surfaced on the training thread by next()
            self._err = e
            try:
                self._q.put_nowait((None, None, 0))
            except Exception:  # noqa: BLE001
                pass

    def _preload(self):
        batch, done, nbytes = self._stage()
        self.next_batch = (batch, done, nbytes)

    def next(self, defer: bool = False):
        """The next staged batch (device tensors).  Non-threaded mode: with ``defer=True`` the host work for the FOLLOWING
        batch is postponed until ``advance()``, which the trainer calls right after it has enqueued the step."""
        if self.threaded:
            batch, done, nbytes = self._q.get()
            if batch is None and self._err is not None:
                raise RuntimeError("prefetch thread failed: %r" % (self._err,))
        else:
            if self.next_batch is None:
                self._preload()
            batch, done, nbytes = self.next_batch
            self.next_batch = None
        self.h2d_bytes += nbytes
        if self.stream is not None and done is not None:          # side-stream copy: order it before the consumer
            cur = torch.cuda.current_stream()
            cur.wait_event(done)
            for t in batch:
                if torch.is_tensor(t):
                    t.record_stream(cur)
        if not self.threaded and not defer:
            self._preload()
        return batch

    def advance(self) -> None:
        if not self.threaded and self.next_batch is None:
            self._preload()

    def close(self) -> None:
        self._stop = True
        if self._thread is not None:
            try:
                while True:
                    self._q.get_nowait()
            except Exception:  # noqa: BLE001
                pass
            self._thread.join(timeout=2.0)
            self._thread = None
