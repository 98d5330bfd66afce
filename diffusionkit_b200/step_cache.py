"""Skip decision of the opt-in first-block step cache (MMDiT.set_step_cache, DESIGN.md §10).  Pure host logic, so it
can be driven without a GPU.

Per forward on B' sequences, the first block's residual r0 = a - e (image stream after block 0 minus the image stream
before it) is compared with r0prev, the r0 of the last fully computed forward:
    rel_b = Σ|r0_b - r0prev_b| / Σ|r0prev_b|        (a zero denominator: do not skip)
The forward is skipped, batch-wide, iff the cache is on, this is not the first forward since the last reset,
max_b rel_b < threshold and fewer than max_consecutive_skips forwards in a row have been skipped (None: no cap).
r0prev moves only on full forwards, so drift cannot chain through skipped ones.
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence, Tuple


def max_relative_change(sums: Sequence[Tuple[float, float]]) -> float:
    """max over sequences of Σ|r0 - r0prev| / Σ|r0prev|, from the per-sequence (numerator, denominator) pairs; inf when
    a denominator is zero, NaN when a numerator is not finite (neither ever skips)."""
    worst = 0.0
    for num, den in sums:
        num, den = float(num), float(den)
        if not math.isfinite(num) or not math.isfinite(den):
            return math.nan
        rel = math.inf if den == 0.0 else num / den
        worst = max(worst, rel)
    return worst


class StepCachePolicy:
    """threshold: skip while max rel < threshold (0 never skips, inf always skips after the first forward);
    max_consecutive_skips: at most this many skipped forwards in a row (None: no cap)."""

    def __init__(self, threshold: float, max_consecutive_skips: Optional[int] = None):
        threshold = float(threshold)
        if math.isnan(threshold) or threshold < 0:
            raise ValueError(f"step cache threshold must be >= 0 (or None to turn the cache off), got {threshold}")
        if max_consecutive_skips is not None:
            if int(max_consecutive_skips) != max_consecutive_skips or max_consecutive_skips < 0:
                raise ValueError(f"max_consecutive_skips must be a non-negative integer or None, got "
                                 f"{max_consecutive_skips!r}")
            max_consecutive_skips = int(max_consecutive_skips)
        self.threshold = threshold
        self.max_consecutive_skips = max_consecutive_skips
        self.log: List[Tuple[Optional[float], bool]] = []
        self.reset()

    def reset(self):
        """The next forward runs in full (and has no rel); the log starts again."""
        self._have_prev = False
        self._consecutive = 0
        self.log = []

    @property
    def needs_full(self) -> bool:
        """True when the next forward runs in full whatever its residual (first forward since a reset)."""
        return not self._have_prev

    def decide(self, rel: Optional[float]) -> bool:
        """Record one forward whose max relative change is `rel` (None on the first forward since a reset) and return
        whether it is skipped."""
        if not self._have_prev:
            rel = None
        cap_ok = self.max_consecutive_skips is None or self._consecutive < self.max_consecutive_skips
        skip = rel is not None and rel < self.threshold and cap_ok
        if skip:
            self._consecutive += 1
        else:
            self._consecutive = 0
            self._have_prev = True
        self.log.append((rel, skip))
        return skip

    def step(self, sums: Sequence[Tuple[float, float]]) -> bool:
        """decide() from the per-sequence (Σ|r0 - r0prev|, Σ|r0prev|) pairs of this forward"""
        return self.decide(max_relative_change(sums) if self._have_prev else None)
