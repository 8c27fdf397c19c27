"""What ``bgr_desync_diff`` reports, as a Python value (``Engine.desync_diff``, ``App.desync_report``).

The report compares a frame's first-recorded snapshot (what the SyncTest compared against) with its re-saved one, with
the keyed-map semantics of ``component_snapshot.rs:99-115`` (see ``include/bevy_ggrs_b200.h``, "desync capture").
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict

import numpy as np

NO_INDEX = 0xFFFFFFFF  # BGR_DESYNC_NO_INDEX: the word of existence / presence records, the column of existence records
HOST_RNG, HOST_TIME = 1, 2  # host_state_differs bits: ParticleRng, Time<GgrsTime>

RECORD_DTYPE = np.dtype([("row", "<u4"), ("column", "<u4"), ("word", "<u4"), ("first", "<u4"), ("latest", "<u4")])


@dataclass
class DesyncColumn:
    index: int
    name: str
    rows: int              # rows with a word difference
    rows_in_checksum: int  # ... of which a differing word overlaps the checksummed byte range
    presence: int          # rows where the component is present in one image only


@dataclass
class DesyncReport:
    frame: int
    rows_first: int
    rows_latest: int
    rows_differing: int
    existence_differing: int
    words_differing: int
    host_state_differs: int
    elapsed_ns_first: int
    elapsed_ns_latest: int
    columns: Dict[int, DesyncColumn] = field(default_factory=dict)
    records: np.ndarray = field(default_factory=lambda: np.zeros(0, RECORD_DTYPE))

    @property
    def by_name(self) -> Dict[str, DesyncColumn]:
        return {c.name: c for c in self.columns.values()}

    @property
    def empty(self) -> bool:
        """No difference in any state the engine holds: the mismatch came from host-held state (resources such as
        FrameCount, host-side component tables)."""
        return self.rows_differing == 0 and self.host_state_differs == 0

    def summary_tuple(self) -> tuple:
        return (self.frame, self.rows_first, self.rows_latest, self.rows_differing, self.existence_differing,
                self.words_differing, self.host_state_differs, self.elapsed_ns_first, self.elapsed_ns_latest)

    def __str__(self) -> str:
        if self.empty:
            return (f"frame {self.frame}: no difference in engine-held state; the mismatch comes from host-held state "
                    f"(resources, host-side component tables)")
        lines = [f"frame {self.frame}: {self.rows_differing} rows differ ({self.existence_differing} exist in one "
                 f"snapshot only), {self.words_differing} words"]
        if self.host_state_differs & HOST_RNG:
            lines.append("  ParticleRng differs")
        if self.host_state_differs & HOST_TIME:
            lines.append(f"  Time<GgrsTime> differs: {self.elapsed_ns_first} ns vs {self.elapsed_ns_latest} ns")
        for c in self.columns.values():
            if c.rows or c.presence:
                lines.append(f"  {c.name}: {c.rows} rows ({c.rows_in_checksum} inside the checksum), "
                             f"{c.presence} presence")
        for r in self.records[:8]:
            where = "exists" if r["column"] == NO_INDEX else (
                f"{self.columns[int(r['column'])].name} present" if r["word"] == NO_INDEX else
                f"{self.columns[int(r['column'])].name} word {int(r['word'])}")
            lines.append(f"  row {int(r['row'])} {where}: {int(r['first']):#x} -> {int(r['latest']):#x}")
        return "\n".join(lines)
