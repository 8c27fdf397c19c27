"""Desync capture and diff restated on the oracle (the CPU restatement of the World), independently of the engine.

``CaptureOracleWorld`` is ``OracleWorld`` plus what ``BGR_CFG_DESYNC_CAPTURE`` adds to the engine: it keeps the first
snapshot of every frame with the engine's release rules (ring.hpp) and compares it with the frame's current snapshot
in numpy, from the oracle's per-frame maps.  Request vectors are replayed one request at a time (handle_requests is a
plain loop over the vector, schedule_systems.rs:222-269), so every Save can be read back before a later request of the
same vector replaces it.

What the oracle does not expose is restated here: ``Time<GgrsTime>::elapsed`` at a Save of frame f is f * 1e9 / fps
(time.rs:63-76), and ``ParticleRng`` is not compared (the worlds checked with this have no spawn_particles system).
The per-row mask byte of the engine is rebuilt from per-column presence: bit 0 = the row exists (it holds any column),
bit 1+k = optional column k absent.  Every world checked with this has at least one non-optional column.

TEST INFRASTRUCTURE: nothing in the product package imports this file.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.desync import NO_INDEX, RECORD_DTYPE, DesyncColumn, DesyncReport
from bevy_ggrs_b200.session import SAVE
from oracle_backend import OracleWorld


def _is_older(stored: int, incoming: int) -> bool:  # GgrsSnapshots::push's wrap-aware test (mod.rs:156-161)
    diff = abs(stored - incoming)
    wrapped = diff > 0x7FFFFFFF
    return not ((stored >= incoming and not wrapped) or (incoming >= stored and wrapped))


class CaptureOracleWorld(OracleWorld):
    def __init__(self, max_entities: int = 0, max_depth: int = 9, fps: int = 60, **kw):
        super().__init__(max_entities, max_depth, fps, **kw)
        self.fps = fps
        self.names: List[str] = []
        self.absent_bit: List[int] = []
        self.ck_range: List[tuple] = []
        self._first: Dict[int, dict] = {}   # frame -> its retained first snapshot
        self._latest: Dict[int, dict] = {}  # frame -> its most recent snapshot

    # ---- registration: remember what the engine's registration knows ----
    def rollback_component(self, name, elem_bytes, strategy=0):
        col = super().rollback_component(name, elem_bytes, strategy)
        n_opt = sum(1 for b in self.absent_bit if b)
        self.absent_bit.append((2 << n_opt) if strategy & capi.BGR_STRATEGY_OPTIONAL else 0)
        self.names.append(name)
        self.ck_range.append((0, 0))
        return col

    def checksum_component(self, col, byte_offset, byte_len, flags=0):
        super().checksum_component(col, byte_offset, byte_len, flags)
        self.ck_range[col] = (byte_offset, byte_offset + byte_len) if byte_len else (0, 0)

    # ---- capture ----
    def _snapshot(self, frame: int) -> dict:
        rows = self.row_count()
        cols = []
        for c, eb in enumerate(self.elem_bytes):
            data, alive = self.peek(frame, c, 0, rows)
            cw = (eb + 3) // 4
            padded = np.zeros((rows, cw * 4), np.uint8)
            padded[:, :eb] = data
            cols.append((padded.view("<u4").reshape(rows, cw), alive.astype(bool), data))
        return {"rows": rows, "elapsed": frame * 1_000_000_000 // self.fps, "cols": cols}

    def handle_requests(self, session_info, requests):
        out = []
        for r in requests:
            if r.kind != SAVE:
                out += super().handle_requests(session_info, [r])
                continue
            frame = self.rollback_frame_count()  # the frame SaveWorld pushes
            before = set(self.snapshot_frames())
            out += super().handle_requests(session_info, [r])
            after = set(self.snapshot_frames())
            confirmed = self.confirmed_frame_count()
            for f in list(self._first):  # released: below the confirmed frame ...
                if f < confirmed:
                    del self._first[f]
            for f in before - after:     # ... or evicted from the old end of the ring
                if _is_older(f, frame):
                    self._first.pop(f, None)
            snap = self._snapshot(frame)
            self._first.setdefault(frame, snap)
            self._latest[frame] = snap
        return out

    def reset_session(self):
        super().reset_session()
        self._first.clear()

    # ---- the engine's desync surface ----
    def desync_frames(self) -> List[int]:
        return [f for f in self.snapshot_frames() if f in self._first and self._first[f] is not self._latest.get(f)]

    def peek_first(self, frame, col, first_row, count):
        snap = self._first.get(frame)
        if snap is None:
            return None
        _, alive, data = snap["cols"][col]
        out = np.zeros((count, self.elem_bytes[col]), np.uint8)
        a = np.zeros(count, np.uint8)
        n = max(0, min(count, snap["rows"] - first_row))
        out[:n] = data[first_row:first_row + n]
        a[:n] = alive[first_row:first_row + n]
        return out, a

    def _masks(self, snap: dict, n: int) -> np.ndarray:
        exists = np.zeros(n, bool)
        for _, alive, _ in snap["cols"]:
            exists[: len(alive)] |= alive
        m = np.zeros(n, np.uint32)
        m[exists] = 1
        for (_, alive, _), bit in zip(snap["cols"], self.absent_bit):
            if bit:
                present = np.zeros(n, bool)
                present[: len(alive)] = alive
                m[exists & ~present] |= bit
        return m

    def desync_diff(self, frame: int, max_records: int = 64) -> Optional[DesyncReport]:
        if frame not in self._first or frame not in self.snapshot_frames():
            return None
        a, b = self._first[frame], self._latest[frame]
        n = max(a["rows"], b["rows"])
        ma, mb = self._masks(a, n), self._masks(b, n)
        both = (ma != 0) & (mb != 0)
        existence = (ma != 0) != (mb != 0)
        recs = [np.stack([np.nonzero(existence)[0], np.full(existence.sum(), NO_INDEX), np.full(existence.sum(), NO_INDEX),
                          ma[existence], mb[existence]], axis=1).astype(np.uint64)]
        any_row = existence.copy()
        words_total = 0
        columns = {}
        for c, eb in enumerate(self.elem_bytes):
            bit = self.absent_bit[c]
            pa, pb = both & ((ma & bit) == 0), both & ((mb & bit) == 0)
            presence = pa != pb
            recs.append(np.stack([np.nonzero(presence)[0], np.full(presence.sum(), c), np.full(presence.sum(), NO_INDEX),
                                  ma[presence], mb[presence]], axis=1).astype(np.uint64))
            cw = (eb + 3) // 4
            wa, wb = np.zeros((n, cw), np.uint32), np.zeros((n, cw), np.uint32)
            wa[: a["rows"]] = a["cols"][c][0]
            wb[: b["rows"]] = b["cols"][c][0]
            differ = (wa != wb) & (pa & pb)[:, None]
            r, w = np.nonzero(differ)
            recs.append(np.stack([r, np.full(len(r), c), w, wa[r, w], wb[r, w]], axis=1).astype(np.uint64))
            lo, hi = self.ck_range[c]
            in_ck = np.array([4 * k < hi and 4 * k + 4 > lo for k in range(cw)], bool)
            columns[c] = DesyncColumn(c, self.names[c], int(differ.any(axis=1).sum()),
                                      int((differ & in_ck[None, :]).any(axis=1).sum()), int(presence.sum()))
            any_row |= presence | differ.any(axis=1)
            words_total += len(r)
        allr = np.concatenate(recs) if recs else np.zeros((0, 5), np.uint64)
        order = np.lexsort((allr[:, 2], allr[:, 1], allr[:, 0]))
        allr = allr[order][:max_records]
        out = np.zeros(len(allr), RECORD_DTYPE)
        for k, name in enumerate(RECORD_DTYPE.names):
            out[name] = allr[:, k]
        host = 2 if a["elapsed"] != b["elapsed"] else 0
        return DesyncReport(frame, a["rows"], b["rows"], int(any_row.sum()), int(existence.sum()), words_total, host,
                            a["elapsed"], b["elapsed"], columns, out)
