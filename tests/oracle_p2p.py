"""P2P desync reports restated on the oracle (the CPU restatement of the World), independently of the engine.

``RetainOracleWorld`` is ``CaptureOracleWorld`` plus what ``bgr_retain_confirmed`` adds: it records the latest
snapshot of every frame from the oracle's per-frame maps, and keeps the last ``count`` frames f >= 0, f % interval == 0
that leave the oracle's own ring from the old end.  ``frame_digest`` restates the digest words from those snapshots with
the oracle's seahash, and ``two_world_diff`` restates the keyed-map diff of two worlds' images of a frame on a list of
512-row blocks.  Nothing here reads the engine.

TEST INFRASTRUCTURE: nothing in the product package imports this file.
"""
from __future__ import annotations

import struct
from typing import Dict, List, Optional

import numpy as np

from bevy_ggrs_b200.desync import NO_INDEX, RECORD_DTYPE, DesyncColumn, DesyncReport
from bevy_ggrs_b200.session import SAVE
from oracle_backend import OracleWorld
from oracle_desync import CaptureOracleWorld, _is_older

BLOCK = 512  # BGR_DIGEST_BLOCK_ROWS, the wire format's block size


class RetainOracleWorld(CaptureOracleWorld):
    def __init__(self, *a, order_base: int = 0, **kw):
        super().__init__(*a, order_base=order_base, **kw)
        self.order_base = order_base
        self.interval, self.count = 1, 0
        self._retained: List[int] = []  # oldest first

    def retain_confirmed(self, interval: int, count: int) -> None:
        self.interval, self.count = interval, count

    def handle_requests(self, session_info, requests):
        out = []
        for r in requests:
            if r.kind != SAVE:
                out += OracleWorld.handle_requests(self, session_info, [r])
                continue
            frame = self.rollback_frame_count()
            if frame in self._retained:          # a new save of a retained frame replaces it
                self._retained.remove(frame)
            before = set(self.snapshot_frames())
            out += OracleWorld.handle_requests(self, session_info, [r])
            for f in sorted(before - set(self.snapshot_frames())):
                if _is_older(f, frame) and self.count and f >= 0 and f % self.interval == 0:
                    self._retained.append(f)     # left from the old end: confirmed or evicted for depth
                    del self._retained[:-self.count]
            self._latest[frame] = self._snapshot(frame)
        return out

    def reset_session(self):
        super().reset_session()
        self._retained = []

    def retained_frames(self) -> List[int]:
        return self._retained[::-1]

    def image(self, frame: int) -> Optional[dict]:
        """The snapshot the engine would hold for ``frame``: queued first, then retained."""
        if frame in self.snapshot_frames() or frame in self._retained:
            return self._latest[frame]
        return None

    def _seahash(self, b: bytes) -> int:
        return self._lib.orc_seahash(b, len(b))

    def frame_digest(self, frame: int):
        """(rows, active, words[n_blocks, n_columns + 1]) of ``frame``, or None."""
        snap = self.image(frame)
        if snap is None:
            return None
        rows = snap["rows"]
        n_cols = len(self.elem_bytes)
        masks = self._masks(snap, rows)
        words = np.zeros(((rows + BLOCK - 1) // BLOCK, n_cols + 1), np.uint64)
        for r in np.nonzero(masks)[0]:
            order = self.order_base + int(r)
            for c in range(n_cols):
                if not masks[r] & self.absent_bit[c]:
                    h = self._seahash(snap["cols"][c][2][r].tobytes())
                    words[r // BLOCK, c] ^= np.uint64(self._seahash(struct.pack("<QQ", order, h)))
            words[r // BLOCK, n_cols] ^= np.uint64(self._seahash(struct.pack("<QQ", order, int(masks[r]))))
        return rows, int(np.count_nonzero(masks)), words


def two_world_diff(a: RetainOracleWorld, b: RetainOracleWorld, frame: int, blocks, max_records: int) -> DesyncReport:
    """The keyed-map diff (component_snapshot.rs:99-115) of a's image of ``frame`` (first) against b's (latest), on the
    rows of ``blocks`` (b's exported blocks) and of a's blocks at or past b's block count (rows only a has), in
    ascending (row, column, word) order."""
    sa, sb = a.image(frame), b.image(frame)
    n = max(sa["rows"], sb["rows"], max(blocks, default=-1) * BLOCK + BLOCK)
    sel = np.zeros(n, bool)
    for blk in blocks:
        sel[blk * BLOCK:(blk + 1) * BLOCK] = True
    sel[-(-sb["rows"] // BLOCK) * BLOCK: -(-sa["rows"] // BLOCK) * BLOCK] = True
    ma, mb = a._masks(sa, n), b._masks(sb, n)
    both = (ma != 0) & (mb != 0) & sel
    existence = ((ma != 0) != (mb != 0)) & sel
    recs = [np.stack([np.nonzero(existence)[0], np.full(existence.sum(), NO_INDEX), np.full(existence.sum(), NO_INDEX),
                      ma[existence], mb[existence]], axis=1).astype(np.uint64)]
    any_row = existence.copy()
    words_total = 0
    columns: Dict[int, DesyncColumn] = {}
    for c, eb in enumerate(a.elem_bytes):
        bit = a.absent_bit[c]
        pa, pb = both & ((ma & bit) == 0), both & ((mb & bit) == 0)
        presence = pa != pb
        recs.append(np.stack([np.nonzero(presence)[0], np.full(presence.sum(), c), np.full(presence.sum(), NO_INDEX),
                              ma[presence], mb[presence]], axis=1).astype(np.uint64))
        cw = (eb + 3) // 4
        wa, wb = np.zeros((n, cw), np.uint32), np.zeros((n, cw), np.uint32)
        wa[: sa["rows"]] = sa["cols"][c][0]
        wb[: sb["rows"]] = sb["cols"][c][0]
        differ = (wa != wb) & (pa & pb)[:, None]
        r, w = np.nonzero(differ)
        recs.append(np.stack([r, np.full(len(r), c), w, wa[r, w], wb[r, w]], axis=1).astype(np.uint64))
        lo, hi = a.ck_range[c]
        in_ck = np.array([4 * k < hi and 4 * k + 4 > lo for k in range(cw)], bool)
        columns[c] = DesyncColumn(c, a.names[c], int(differ.any(axis=1).sum()),
                                  int((differ & in_ck[None, :]).any(axis=1).sum()), int(presence.sum()))
        any_row |= presence | differ.any(axis=1)
        words_total += len(r)
    allr = np.concatenate(recs)
    allr = allr[np.lexsort((allr[:, 2], allr[:, 1], allr[:, 0]))][:max_records]
    out = np.zeros(len(allr), RECORD_DTYPE)
    for k, name in enumerate(RECORD_DTYPE.names):
        out[name] = allr[:, k]
    host = 2 if sa["elapsed"] != sb["elapsed"] else 0
    return DesyncReport(frame, sa["rows"], sb["rows"], int(any_row.sum()), int(existence.sum()), words_total, host,
                        sa["elapsed"], sb["elapsed"], columns, out)
