"""Early pack: which ranges of a bucket a threshold-reuse Ok-Topk call packs during backward, and which it packs itself.

The bucket's big gradients exist long before its last one (VGG-16: layers 9 - 13, 80 % of the bucket, while backward
still runs layers 8 -> 1).  The pack pass of a threshold-reuse call (acc = g + residual, |acc| > carried threshold ->
send slot) needs nothing but the element itself, so it can run over those ranges as soon as their gradients are ready:
``oktopk_run(..., pack_ranges=ranges, segment=1)``.  The call that follows packs what no segment covered
(``pack_ranges=rest``) and publishes.  ``PackPlanner`` decides both, on the host and without a device, so that every
element of the bucket is packed exactly once per call.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

Range = Tuple[int, int]


class PackPlanner:
    """Parameter i of the bucket owns the span [offsets[i], offsets[i + 1]) (the last one up to the bucket's end), clipped
    to the bucket's whole float4 vectors [0, 4 (n // 4)): padding after a parameter belongs to it, the scalar tail of a
    bucket whose length is not a multiple of 4 is always left to the call.

    ``ready(i)`` marks parameter i's gradient as produced.  Once the ready spans that no segment packed yet hold at least
    ``min_elems`` elements, it returns them as one segment -- the maximal runs of adjacent such spans, in bucket order --
    and marks them packed; otherwise None.  One segment late in backward rather than one per layer: the big gradients of
    a CNN come first, and the backward kernels that follow them run small grids next to which a segment finds free SMs.
    ``rest()`` lists the ranges no segment covered.  Segments hold at most ``max_ranges - 1`` ranges in all, so that
    ``rest()`` never has more than ``max_ranges``."""

    def __init__(self, offsets: Sequence[int], n: int, min_elems: int, max_ranges: int):
        order = sorted(range(len(offsets)), key=lambda i: offsets[i])
        if any(int(offsets[i]) % 4 for i in order):
            raise ValueError("parameter offsets must be multiples of 4 elements")
        self.n, self.min_elems, self.max_ranges = int(n), max(int(min_elems), 1), int(max_ranges)
        top = 4 * (self.n // 4)
        self._pos = {i: k for k, i in enumerate(order)}          # parameter -> span number (bucket order)
        starts = [min(int(offsets[i]), top) for i in order]
        ends = starts[1:] + [top]
        if starts:
            starts[0] = 0                                        # elements before the first parameter go with it
        self._span = list(zip(starts, ends))
        self.reset()

    def reset(self) -> None:
        """Start of a call: nothing ready, nothing packed."""
        self._state = [0] * len(self._span)                      # 0 not ready, 1 ready, 2 packed by a segment
        self._pending = 0                                        # elements of the ready, unpacked spans
        self._segments: List[List[Range]] = []
        self._packed_runs = 0

    @property
    def segments(self) -> List[List[Range]]:
        return [list(s) for s in self._segments]

    def _runs(self, want: int) -> List[Range]:
        out: List[Range] = []
        for (a, b), s in zip(self._span, self._state):
            if s != want or a == b:
                continue
            if out and out[-1][1] == a:
                out[-1] = (out[-1][0], b)
            else:
                out.append((a, b))
        return out

    def ready(self, i: int) -> Optional[List[Range]]:
        k = self._pos[i]
        if self._state[k]:
            return None
        self._state[k] = 1
        self._pending += self._span[k][1] - self._span[k][0]
        if self._pending < self.min_elems:
            return None
        runs = self._runs(1)
        if self._packed_runs + len(runs) > self.max_ranges - 1:
            return None
        for q, s in enumerate(self._state):
            if s == 1:
                self._state[q] = 2
        self._pending = 0
        self._packed_runs += len(runs)
        self._segments.append(runs)
        return runs

    def rest(self) -> List[Range]:
        """The ranges of the bucket's whole vectors that no segment of this call covered, in bucket order."""
        out: List[Range] = []
        for (a, b), s in zip(self._span, self._state):
            if s == 2 or a == b:
                continue
            if out and out[-1][1] == a:
                out[-1] = (out[-1][0], b)
            else:
                out.append((a, b))
        return out
