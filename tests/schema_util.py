"""Random registrations for the differential tests, and the kernel the engine picks for one on each tick path.

``random_schema`` reaches element sizes with sub-word tails (1, 2, 3, 5, 7 B) next to whole-word ones, up to seven
optional columns (every bit of the mask byte), checksum ranges that are none, the whole element, or unaligned and
partial, and rows of an exact width in words (24 / 25 and 49 / 50 are where the NVRTC kernel and the one-launch
program stop taking the registration).

TEST INFRASTRUCTURE: nothing in the product package imports this file.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np
import pytest

from bevy_ggrs_b200 import capi

OPT = capi.BGR_STRATEGY_OPTIONAL
SIZES = [1, 2, 3, 5, 7, 8, 12, 40]   # 1024 B is passed explicitly: one such element is a 256-word row

# tick paths: (environment, engine flags)
WIDE_PATHS = {"generic": ({}, 0), "stepwise_tma": ({}, capi.BGR_CFG_FORCE_STEPWISE),
              "stepwise_flat": ({"BGR_TUNE_TMA": "0"}, capi.BGR_CFG_FORCE_STEPWISE),
              "stepwise_tma_stages2": ({"BGR_TUNE_TMA_STAGES": "2"}, capi.BGR_CFG_FORCE_STEPWISE)}


def path_env(monkeypatch, path, generic_kernel):
    """Sets the environment of a WIDE_PATHS entry and returns its flags; the stepwise paths run once (they do not
    depend on the generic kernel)."""
    if path != "generic" and generic_kernel != "interpreter":
        pytest.skip("the stepwise path does not depend on the generic kernel: run once")
    env, flags = WIDE_PATHS[path]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    return flags


def expected_kind(path, words, n_sys, nvrtc_ranges, generic_kernel):
    """The kernel bgr_build / submit pick for this registration (engine.cu bgr_build, jit_specialise, run_stepwise)."""
    tma_stages = words <= 49   # at least two one-tile stages in 200 KB of shared memory (BGR_TUNE_TMA_STAGES=2 keeps two)
    if path == "generic" and words <= 49 and n_sys <= 8:
        if generic_kernel != "interpreter" and words <= 24 and nvrtc_ranges:
            return "generic_nvrtc"
        return "generic_interpreter"
    if path == "stepwise_flat":
        return "stepwise_flat"
    return "stepwise_tma" if tma_stages else "stepwise_flat"


@dataclass
class Schema:
    sizes: List[int]
    optional: List[bool]
    cks: List[Tuple[int, int, int]]                  # (column, byte offset, byte length)
    systems: List[Tuple[int, List[int], List[int]]]  # (BGR_SYS_*, columns, params)

    @property
    def words(self) -> int:
        return sum((s + 3) // 4 for s in self.sizes)

    @property
    def nvrtc_ranges(self) -> bool:   # the ranges the NVRTC kernel accepts: whole words, 4..64 bytes
        return all(off % 4 == 0 and ln % 4 == 0 and 4 <= ln <= 64 for _, off, ln in self.cks)

    def register(self, w) -> List[int]:
        """Registers the schema on an Engine or an oracle world (before build)."""
        cols = [w.rollback_component(f"C{i}", s, (capi.BGR_STRATEGY_COPY | OPT) if o else capi.BGR_STRATEGY_CLONE)
                for i, (s, o) in enumerate(zip(self.sizes, self.optional))]
        for i, off, ln in self.cks:
            w.checksum_component(cols[i], off, ln)
        for kind, c, p in self.systems:
            w.add_system(kind, [cols[i] for i in c], p)
        return cols

    def values(self, rng, n) -> List[np.ndarray]:
        """Random element bytes for n rows; u32 fields small enough that SATSUB despawns some rows (not most) within
        ~30 ticks."""
        data = [rng.integers(0, 256, (n, s), dtype=np.uint8) for s in self.sizes]
        for i, s in enumerate(self.sizes):
            if s % 4 == 0:
                data[i].view(np.uint32)[:] = rng.integers(20, 300, (n, s // 4), dtype=np.uint32)
        return data


def random_schema(rng, words: Optional[int] = None, sizes: Optional[Sequence[int]] = None, n_opt: Optional[int] = None,
                  ranges: Sequence[str] = ("none", "whole", "partial"), store_call_count: bool = False) -> Schema:
    """A registration of the given element sizes, or of random SIZES that add up to exactly `words` word planes.
    `n_opt` optional columns (random when None; at least one column stays required: a row exists iff it holds one).
    Up to six checksummed columns, each range drawn from `ranges`.  Systems: U32_ADD and U32_SATSUB_DESPAWN on columns
    with u32 fields, and with `store_call_count` one U32_STORE_CALL_COUNT, whose value differs on every re-simulation."""
    if sizes is None:
        sizes, rem = [], words
        if store_call_count:
            sizes, rem = [8], words - 2
        while rem > 0:
            s = int(rng.choice([s for s in SIZES if (s + 3) // 4 <= rem]))
            sizes.append(s)
            rem -= (s + 3) // 4
    sizes = [int(s) for s in sizes]
    n = len(sizes)
    n_opt = min(n - 1, 7, int(rng.integers(0, 8)) if n_opt is None else n_opt)
    optional = [False] + [i < n_opt for i in range(n - 1)]
    perm = rng.permutation(n)
    optional = [optional[int(k)] for k in perm]
    cks = []
    for i in sorted(int(k) for k in rng.permutation(n)[:6]):
        kind, s = str(rng.choice(list(ranges))), sizes[i]
        if kind == "whole":
            cks.append((i, 0, s))
        elif kind == "partial" and s >= 2:
            off = int(rng.integers(1, s))   # an unaligned start ...
            cks.append((i, off, int(rng.integers(1, s - off + 1))))   # ... and any end inside the element
    u32 = [i for i, s in enumerate(sizes) if s % 4 == 0]
    systems = []
    for i in u32[:2]:
        kind = int(rng.choice([capi.BGR_SYS_U32_ADD, capi.BGR_SYS_U32_SATSUB_DESPAWN]))
        systems.append((kind, [i], [4 * int(rng.integers(0, sizes[i] // 4)), int(rng.integers(1, 4))]))
    if store_call_count:
        i = int(rng.choice(u32))
        systems.append((capi.BGR_SYS_U32_STORE_CALL_COUNT, [i], [4 * int(rng.integers(0, sizes[i] // 4))]))
    return Schema(sizes, optional, cks, systems)
