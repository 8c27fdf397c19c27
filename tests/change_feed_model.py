"""numpy reference model of the change feed (include/bevy_ggrs_b200.h "change feed"), and a host replica its records
are applied to.

A live world is a ``WorldState``: the row count and, per row below it, whether the row is alive, per column whether it
is present and the element bytes.  The model keeps, per row, the (state, field bytes) it last reported and reports the
rows whose current ones differ, lowest rows first, at most ``cap`` of them.

TEST INFRASTRUCTURE: nothing in the product package imports this file.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Sequence, Tuple

import numpy as np

from bevy_ggrs_b200.engine import FeedInfo, feed_record_dtype


@dataclass
class WorldState:
    rows: int
    alive: np.ndarray                  # [rows] bool
    present: Dict[int, np.ndarray]     # column -> [rows] bool (False where not alive)
    elems: Dict[int, np.ndarray]       # column -> [rows, elem_bytes] u8


def world_of(w, cols: Sequence[int]) -> WorldState:
    """The live world of an Engine or an oracle world, for the columns a feed tracks."""
    rows = w.row_count()
    alive = w.read_alive(0, rows).astype(bool) if rows else np.zeros(0, bool)
    present = {c: (w.has_component(c, 0, rows).astype(bool) if rows else np.zeros(0, bool)) for c in set(cols)}
    elems = {c: (w.read_component(c, 0, rows) if rows else np.zeros((0, 1), np.uint8)) for c in set(cols)}
    return WorldState(rows, alive, present, elems)


class FeedModel:
    def __init__(self, fields: Sequence[Tuple[int, int, int]], max_rows: int):
        self.fields = [tuple(f) for f in fields]
        self.dtype = feed_record_dtype(self.fields)
        self.state = np.zeros(max_rows, np.uint32)
        self.bytes = [np.zeros((max_rows, ln), np.uint8) for _, _, ln in self.fields]

    def reset(self) -> None:
        self.state[:] = 0
        for b in self.bytes:
            b[:] = 0

    def current(self, world: WorldState) -> Tuple[np.ndarray, List[np.ndarray]]:
        """(state, field bytes) of every row of the model's range in ``world``."""
        n = len(self.state)
        state = np.zeros(n, np.uint32)
        state[: world.rows] = world.alive.astype(np.uint32)
        out = []
        for k, (c, off, ln) in enumerate(self.fields):
            pres = np.zeros(n, bool)
            pres[: world.rows] = world.present[c] & world.alive
            state |= pres.astype(np.uint32) << np.uint32(1 + k)
            b = np.zeros((n, ln), np.uint8)
            b[: world.rows] = world.elems[c][:, off:off + ln]
            b[~pres] = 0
            out.append(b)
        return state, out

    def differing(self, world: WorldState) -> np.ndarray:
        state, fb = self.current(world)
        d = state != self.state
        for k in range(len(self.fields)):
            d |= (fb[k] != self.bytes[k]).any(axis=1)
        return np.nonzero(d)[0]

    def report(self, world: WorldState, cap: int) -> Tuple[np.ndarray, FeedInfo]:
        state, fb = self.current(world)
        rows = self.differing(world)
        take = rows[:cap]
        recs = np.zeros(len(take), self.dtype)
        recs["row"] = take
        recs["state"] = state[take]
        for k in range(len(self.fields)):
            recs[f"f{k}"] = fb[k][take]
            self.bytes[k][take] = fb[k][take]
        self.state[take] = state[take]
        return recs, FeedInfo(len(take), len(rows) - len(take), world.rows, self.dtype.itemsize)


class Replica:
    """What a host mirror knows after applying records: per row existence, per field presence and bytes."""

    def __init__(self, n_fields: int, field_lens: Sequence[int], max_rows: int):
        self.state = np.zeros(max_rows, np.uint32)
        self.bytes = [np.zeros((max_rows, ln), np.uint8) for ln in field_lens]

    def apply(self, recs: np.ndarray) -> None:
        r = recs["row"].astype(np.int64)
        self.state[r] = recs["state"]
        for k in range(len(self.bytes)):
            self.bytes[k][r] = recs[f"f{k}"]

    def matches(self, model: FeedModel, world: WorldState) -> bool:
        state, fb = model.current(world)
        return bool(np.array_equal(self.state, state) and all(np.array_equal(a, b) for a, b in zip(self.bytes, fb)))


def host_edits(worlds, rng, optional_col: int, value_col: int, value_bytes: int) -> None:
    """The same random host-side edits between ticks on every world (an Engine and its oracle): spawn, despawn,
    remove / insert of the optional column, write_component of one row."""
    w0 = worlds[0]
    rows = w0.row_count()
    alive = np.nonzero(w0.read_alive(0, rows))[0] if rows else np.zeros(0, int)
    picks = [int(r) for r in rng.choice(alive, min(3, len(alive)), replace=False)] if len(alive) else []
    val = rng.integers(0, 256, value_bytes, dtype=np.uint8)
    ins = rng.integers(0, 256, worlds[0].elem_bytes[optional_col], dtype=np.uint8)
    for w in worlds:
        if len(picks) >= 3:
            r = picks[0]
            if w.has_component(optional_col, r, 1)[0]:
                w.remove_component(optional_col, r)
            else:
                w.insert_component(optional_col, r, ins)
            w.write_component(value_col, picks[1], val[None, :])
            w.despawn(picks[2])
        w.spawn(3)
