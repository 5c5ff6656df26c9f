"""Offline placement of a lowered program's activation buffers in one arena, by live interval.

Pure host arithmetic (no torch, no library) so it can be tested on its own.  A buffer is a size in bytes and an
inclusive interval [first, last] of op positions on the program's timeline (the cond ops followed by the step ops).
Persistent buffers (the cond outputs the step ops read) are laid out one after another at
the front; every temporary is placed behind them, greedily by size into the lowest offset that no temporary with an
overlapping interval occupies.  Every offset and size is a multiple of ALIGN: the TMA maps of the tensor-core kernels
need 16-byte-aligned addresses and strides.  Buffers of different kinds (element type and size) never share a start
offset, so every address an op names is the start of exactly one typed buffer.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

ALIGN = 256


def align(n: int) -> int:
    return (n + ALIGN - 1) // ALIGN * ALIGN


def overlaps(a: Tuple[int, int], b: Tuple[int, int]) -> bool:
    return a[0] <= b[1] and b[0] <= a[1]


def _first_fit(busy: List[Tuple[int, int]], n: int, at: int) -> int:
    """lowest offset >= at where n bytes miss every [lo, hi) of ``busy`` (sorted by lo)"""
    for lo, hi in busy:
        if hi <= at:
            continue
        if at + n <= lo:
            break
        at = max(at, hi)
    return at


def place(sizes: Sequence[int], intervals: Sequence[Optional[Tuple[int, int]]],
          kinds: Optional[Sequence[object]] = None) -> Tuple[List[int], int, int]:
    """(offset of every buffer, persistent bytes, temporary bytes).  ``intervals[i]`` None marks buffer i
    persistent; temporaries' offsets start at the persistent bytes.  With ``kinds``, two temporaries of different
    kinds never start at the same offset."""
    offs = [0] * len(sizes)
    pers = 0
    for i, iv in enumerate(intervals):
        if iv is None:
            offs[i] = pers
            pers += align(sizes[i])
    temps = [i for i, iv in enumerate(intervals) if iv is not None]
    temps.sort(key=lambda i: (-align(sizes[i]), intervals[i][0], i))
    placed: List[Tuple[int, int, Tuple[int, int]]] = []          # (offset, aligned size, interval)
    starts = {}                                                   # offset -> kind of the temporaries starting there
    top = 0
    for i in temps:
        n, iv = align(sizes[i]), intervals[i]
        kind = None if kinds is None else kinds[i]
        busy = sorted((o, o + s) for o, s, jv in placed if overlaps(iv, jv))
        at = _first_fit(busy, n, 0)
        while starts.get(at, kind) != kind:
            at = _first_fit(busy, n, at + ALIGN)
        starts[at] = kind
        placed.append((at, n, iv))
        offs[i] = pers + at
        top = max(top, at + n)
    return offs, pers, top


def lower_bound(sizes: Sequence[int], intervals: Sequence[Optional[Tuple[int, int]]]) -> int:
    """largest sum of aligned temporary sizes live at one op: no placement of the temporaries needs less"""
    events = []
    for n, iv in zip(sizes, intervals):
        if iv is not None:
            events.append((iv[0], 0, align(n)))
            events.append((iv[1], 1, -align(n)))      # a buffer still counts at its last op
    live = best = 0
    for _, _, d in sorted(events):
        live += d
        best = max(best, live)
    return best


def check(sizes: Sequence[int], intervals: Sequence[Optional[Tuple[int, int]]], offs: Sequence[int],
          kinds: Optional[Sequence[object]] = None) -> None:
    """AssertionError unless every offset is aligned, no two buffers whose intervals overlap share a byte (persistent
    buffers overlap every interval) and, with ``kinds``, no two buffers of different kinds start at one offset"""
    if kinds is not None:
        seen = {}
        for i, o in enumerate(offs):
            if sizes[i]:
                assert seen.setdefault(o, kinds[i]) == kinds[i], f"buffers of kinds {seen[o]} and {kinds[i]} start at {o}"
    full = (-1, 1 << 62)
    spans = sorted((offs[i], offs[i] + sizes[i], intervals[i] or full, i) for i in range(len(sizes)) if sizes[i])
    for o, _, _, i in spans:
        assert o % ALIGN == 0, f"buffer {i} at offset {o} is not {ALIGN}-byte aligned"
    for a in range(len(spans)):
        lo, hi, iv, i = spans[a]
        for b in range(a + 1, len(spans)):
            lo2, hi2, iv2, j = spans[b]
            if lo2 >= hi:
                break
            assert not overlaps(iv, iv2), \
                f"buffers {i} [{lo}, {hi}) and {j} [{lo2}, {hi2}) share bytes while both are live ({iv}, {iv2})"
