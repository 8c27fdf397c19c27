"""Thin object wrapper over the C ABI (``include/bevy_ggrs_b200.h``): numpy in, numpy out.

Every method is one C-ABI call.  Nothing here computes: columns, snapshots, checksums and the
re-simulation all happen in the CUDA library.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np

from . import capi
from .capi import BgrError
from .desync import RECORD_DTYPE, DesyncColumn, DesyncReport


_KERNEL_KINDS = {capi.BGR_KERNEL_NONE: "none", capi.BGR_KERNEL_STEPWISE_TMA: "stepwise_tma",
                 capi.BGR_KERNEL_STEPWISE_FLAT: "stepwise_flat", capi.BGR_KERNEL_BUNDLE: "bundle",
                 capi.BGR_KERNEL_GENERIC_INTERPRETER: "generic_interpreter", capi.BGR_KERNEL_GENERIC_NVRTC: "generic_nvrtc"}


class LastKernel(NamedTuple):
    """bgr_last_kernel decoded.  vec / mode / tier / passive_tma describe the bundle kernel (0 / False otherwise);
    item_rows is set for the bundle and the NVRTC kernel.  tier: 0 unconstrained, 1 768 and 2 1024 threads per SM.
    deferred_live: the vector did not write the live image (BGR_TUNE_DEFER_LIVE); from_deferred: it started from the
    base slot of the previous vector's deferred live image.  passive_tma: the bundle ran in its passive-TMA
    configuration; passive_planes: the bundle launch read or wrote passive planes at all (clear on ticks whose slots
    already hold them); held_saves: at least one of its Saves stored nothing, its slot already holding that content."""
    kind: str
    vec: int
    mode: int
    tier: int
    passive_tma: bool
    item_rows: int
    raw: int
    deferred_live: bool = False
    from_deferred: bool = False
    passive_planes: bool = False
    stable_planes: bool = False
    held_saves: bool = False

    @property
    def batched(self) -> bool:
        """The vector ran inside a world batch's launch (BGR_KERNEL_BATCHED, EngineBatch)."""
        return bool(self.raw & capi.BGR_KERNEL_BATCHED)

    @property
    def replay(self) -> bool:
        """The last replay ran on the generated kernel's replay entry point (BGR_KERNEL_REPLAY), not in chunks."""
        return bool(self.raw & capi.BGR_KERNEL_REPLAY)

    @property
    def warp_fold(self) -> bool:
        """The bundle launch reduced each Save's checksum partials over the warp (BGR_KERNEL_WARP_FOLD): its lane slots
        would have cost it a resident block per SM."""
        return bool(self.raw & capi.BGR_KERNEL_WARP_FOLD)

    @staticmethod
    def decode(v: int) -> "LastKernel":
        return LastKernel(_KERNEL_KINDS.get(v & 0xF, f"unknown({v & 0xF})"), (v >> 4) & 0xF, (v >> 8) & 0x3,
                          (v >> 10) & 0x3, bool((v >> 12) & 1), (v >> 16) & 0x3FF, v,
                          bool(v & capi.BGR_KERNEL_DEFERRED_LIVE), bool(v & capi.BGR_KERNEL_FROM_DEFERRED),
                          bool(v & capi.BGR_KERNEL_PASSIVE_PLANES), bool(v & capi.BGR_KERNEL_STABLE_PLANES),
                          bool(v & capi.BGR_KERNEL_HELD_SAVES))


class FeedInfo(NamedTuple):
    """bgr_feed_info: records written, differing rows left for the next report (cap), rows compared, bytes per record."""
    n_records: int
    pending: int
    rows: int
    record_bytes: int


EDIT_DTYPE = np.dtype([(name, "<u4") for name, _ in capi.bgr_edit._fields_])   # one bgr_edit record


def feed_record_dtype(fields: Sequence[Tuple[int, int, int]]) -> np.dtype:
    """A change-feed record: u32 row, u32 state (bit 0 exists, bit 1+k field k present), then field k's bytes as
    ``f<k>``."""
    return np.dtype([("row", "<u4"), ("state", "<u4")] + [(f"f{k}", np.uint8, (ln,)) for k, (_, _, ln) in enumerate(fields)])


class Engine:
    def __init__(self, max_entities: int, max_depth: int = 9, fps: int = 60, device: int = 0, flags: int = 0,
                 order_base: int = 0, stream: Optional[int] = None):
        self._lib = capi.load_library()
        cfg = capi.bgr_config(capi.BGR_ABI_VERSION, device, max_entities, max_depth, fps, flags, order_base,
                              C.c_void_p(stream) if stream else None)
        handle = C.c_void_p()
        self._h = None
        self._check(self._lib.bgr_engine_create(C.byref(cfg), C.byref(handle)))
        self._h = handle
        self.elem_bytes: List[int] = []
        self.names: List[str] = []
        self.max_entities = max_entities
        self._pinned: List[C.c_void_p] = []
        self._feed_dtypes: Dict[int, np.dtype] = {}
        self._feed_tickets: Dict[int, Tuple[int, np.ndarray]] = {}

    # ---- plumbing ----
    def _check(self, status: int) -> None:
        if status != capi.BGR_OK:
            raise BgrError(status, self._lib.bgr_last_error().decode("utf-8", "replace"))

    def close(self) -> None:
        if self._h is not None:
            self._lib.bgr_engine_destroy(self._h)  # waits for every download in flight
            self._h = None
            for p in self._pinned:
                self._lib.bgr_host_free(p)
            self._pinned = []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- registration (RollbackApp) ----
    def rollback_component(self, name: str, elem_bytes: int, strategy: int = capi.BGR_STRATEGY_COPY) -> int:
        col = C.c_uint32()
        self._check(self._lib.bgr_rollback_component(self._h, name.encode(), elem_bytes, strategy, C.byref(col)))
        self.elem_bytes.append(elem_bytes)
        self.names.append(name)
        return col.value

    def checksum_component(self, col: int, byte_offset: int, byte_len: int, flags: int = 0) -> None:
        self._check(self._lib.bgr_checksum_component(self._h, col, capi.BGR_HASH_BYTES, byte_offset, byte_len, flags))

    def add_system(self, system: int, cols: Sequence[int], params: Sequence[int] = ()) -> None:
        ca = (C.c_uint32 * max(1, len(cols)))(*cols)
        pa = (C.c_uint32 * max(1, len(params)))(*params)
        self._check(self._lib.bgr_add_system(self._h, system, ca, len(cols), pa, len(params)))

    def build(self) -> None:
        self._check(self._lib.bgr_build(self._h))

    def run_startup_system(self, system: int) -> None:
        self._check(self._lib.bgr_run_startup_system(self._h, system))

    # ---- capacity (flags=BGR_CFG_GROWABLE: row-creating calls grow it) ----
    def reserve(self, rows: int) -> None:
        """Capacity >= rows afterwards (BGR_CFG_GROWABLE engines; others only accept rows <= their capacity)."""
        self._check(self._lib.bgr_reserve(self._h, rows))

    def capacity(self) -> Tuple[int, int]:
        """(rows held without growing, most rows the engine can ever hold)."""
        cap, ceiling = C.c_uint32(), C.c_uint32()
        self._check(self._lib.bgr_capacity(self._h, C.byref(cap), C.byref(ceiling)))
        return cap.value, ceiling.value

    # ---- entities ----
    def spawn(self, count: int) -> int:
        first = C.c_uint32()
        self._check(self._lib.bgr_spawn(self._h, count, C.byref(first)))
        return first.value

    def despawn(self, row: int) -> None:
        self._check(self._lib.bgr_despawn(self._h, row))

    def row_count(self) -> int:
        v = C.c_uint32()
        self._check(self._lib.bgr_row_count(self._h, C.byref(v)))
        return v.value

    def active_count(self) -> int:
        v = C.c_uint64()
        self._check(self._lib.bgr_active_count(self._h, C.byref(v)))
        return v.value

    def write_component(self, col: int, first_row: int, values: np.ndarray) -> None:
        eb = self.elem_bytes[col]
        a = np.ascontiguousarray(values).view(np.uint8).reshape(-1, eb)
        self._check(self._lib.bgr_write_component(self._h, col, first_row, a.shape[0], a.ctypes.data, eb))

    def read_component(self, col: int, first_row: int, count: int) -> np.ndarray:
        eb = self.elem_bytes[col]
        out = np.zeros((count, eb), dtype=np.uint8)
        self._check(self._lib.bgr_read_component(self._h, col, first_row, count, out.ctypes.data, eb))
        return out

    def read_alive(self, first_row: int, count: int) -> np.ndarray:
        out = np.zeros(count, dtype=np.uint8)
        self._check(self._lib.bgr_read_alive(self._h, first_row, count, out.ctypes.data))
        return out

    # ---- per-entity presence of BGR_STRATEGY_OPTIONAL columns ----
    def remove_component(self, col: int, row: int) -> None:
        self._check(self._lib.bgr_remove_component(self._h, col, row))

    def insert_component(self, col: int, row: int, value) -> None:
        a = np.ascontiguousarray(value).view(np.uint8).reshape(-1)
        assert a.size == self.elem_bytes[col]
        self._check(self._lib.bgr_insert_component(self._h, col, row, a.ctypes.data))

    def has_component(self, col: int, first_row: int, count: int) -> np.ndarray:
        out = np.zeros(count, dtype=np.uint8)
        self._check(self._lib.bgr_has_component(self._h, col, first_row, count, out.ctypes.data))
        return out

    # ---- host edits (bgr_apply_edits) ----
    def apply_edits(self, edits: np.ndarray, values: bytes = b"") -> None:
        """One queued batch of live-world edits: ``edits`` is an ``EDIT_DTYPE`` array (kind, column, row, count,
        byte_offset, byte_len, value_offset, reserved), ``values`` the bytes its WRITE / INSERT records point into.
        Returns without waiting for the GPU; both buffers are free on return."""
        e = np.ascontiguousarray(edits, dtype=EDIT_DTYPE)
        v = np.frombuffer(bytes(values), dtype=np.uint8)
        self._check(self._lib.bgr_apply_edits(self._h, e.ctypes.data, len(e), v.ctypes.data if v.size else None, v.size))

    # ---- asynchronous mirror download (bgr_download_begin / bgr_download_wait) ----
    def host_alloc(self, count: int, byte_len: int) -> np.ndarray:
        """Page-locked (count, byte_len) u8 array for download_begin; freed with the engine."""
        p = C.c_void_p()
        self._check(self._lib.bgr_host_alloc(count * byte_len, C.byref(p)))
        self._pinned.append(p)
        buf = (C.c_uint8 * max(1, count * byte_len)).from_address(p.value)
        return np.frombuffer(buf, dtype=np.uint8, count=count * byte_len).reshape(count, byte_len)

    def download_begin(self, col: int, byte_offset: int, byte_len: int, first_row: int, count: int, dst: np.ndarray) -> int:
        assert dst.dtype == np.uint8 and dst.flags.c_contiguous and dst.size >= count * byte_len
        t = C.c_uint32()
        self._check(self._lib.bgr_download_begin(self._h, col, byte_offset, byte_len, first_row, count, dst.ctypes.data,
                                                 C.byref(t)))
        return t.value

    def download_wait(self, ticket: int) -> None:
        self._check(self._lib.bgr_download_wait(self._h, ticket))

    # ---- change feed (bgr_feed_*): the live rows whose existence, presence or tracked bytes changed ----
    def feed_create(self, fields: Sequence[Tuple[int, int, int]]) -> int:
        """A feed over ``fields`` = [(column, byte_offset, byte_len), ...]; its first report lists every existing row."""
        fields = [tuple(int(x) for x in f) for f in fields]
        arr = (capi.bgr_feed_field * max(1, len(fields)))(*[capi.bgr_feed_field(*f) for f in fields])
        feed = C.c_uint32()
        self._check(self._lib.bgr_feed_create(self._h, arr, len(fields), C.byref(feed)))
        self._feed_dtypes[feed.value] = feed_record_dtype(fields)
        return feed.value

    def feed_reset(self, feed: int) -> None:
        self._check(self._lib.bgr_feed_reset(self._h, feed))

    def feed_record_dtype(self, feed: int) -> np.dtype:
        return self._feed_dtypes[feed]

    def feed_alloc(self, feed: int, cap: int) -> np.ndarray:
        """Page-locked buffer for ``cap`` records of ``feed``; freed with the engine."""
        return self.host_alloc(max(1, cap), self._feed_dtypes[feed].itemsize)

    def feed_begin(self, feed: int, buf: np.ndarray, cap: int) -> int:
        """Starts a report of at most ``cap`` records into ``buf`` (from feed_alloc); returns its ticket."""
        assert buf.dtype == np.uint8 and buf.flags.c_contiguous and buf.size >= cap * self._feed_dtypes[feed].itemsize
        t = C.c_uint32()
        self._check(self._lib.bgr_feed_begin(self._h, feed, buf.ctypes.data, cap, C.byref(t)))
        self._feed_tickets[t.value] = (feed, buf)
        return t.value

    def feed_wait(self, ticket: int) -> Tuple[np.ndarray, FeedInfo]:
        """(records, info) of a report: a structured array (row, state, f0, f1, ...) copied out of the buffer."""
        info = capi.bgr_feed_info()
        self._check(self._lib.bgr_feed_wait(self._h, ticket, C.byref(info)))
        feed, buf = self._feed_tickets.pop(ticket)
        dt = self._feed_dtypes[feed]
        assert info.record_bytes == dt.itemsize
        recs = np.empty(info.n_records, dt)
        C.memmove(recs.ctypes.data, buf.ctypes.data, info.n_records * dt.itemsize)  # only the records, not the buffer
        return recs, FeedInfo(info.n_records, info.pending, info.rows, info.record_bytes)

    # ---- frame resources ----
    def rollback_frame_count(self) -> int:
        v = C.c_int32()
        self._check(self._lib.bgr_rollback_frame_count(self._h, C.byref(v)))
        return v.value

    def set_rollback_frame_count(self, frame: int) -> None:
        self._check(self._lib.bgr_set_rollback_frame_count(self._h, frame))

    def confirmed_frame_count(self) -> int:
        v = C.c_int32()
        self._check(self._lib.bgr_confirmed_frame_count(self._h, C.byref(v)))
        return v.value

    def max_prediction_window(self) -> int:
        v = C.c_uint32()
        self._check(self._lib.bgr_max_prediction_window(self._h, C.byref(v)))
        return v.value

    # ---- ring ----
    def set_depth(self, depth: int) -> None:
        self._check(self._lib.bgr_set_depth(self._h, depth))

    def confirm(self, frame: int) -> None:
        self._check(self._lib.bgr_confirm(self._h, frame))

    def snapshot_frames(self) -> List[int]:
        buf = (C.c_int32 * 128)()
        n = C.c_uint32()
        self._check(self._lib.bgr_snapshot_frames(self._h, buf, 128, C.byref(n)))
        return [buf[i] for i in range(n.value)]

    def peek(self, frame: int, col: int, first_row: int, count: int) -> Optional[Tuple[np.ndarray, np.ndarray]]:
        eb = self.elem_bytes[col]
        out = np.zeros((count, eb), dtype=np.uint8)
        alive = np.zeros(count, dtype=np.uint8)
        found = C.c_int32()
        self._check(self._lib.bgr_peek(self._h, frame, col, first_row, count, out.ctypes.data, eb,
                                       alive.ctypes.data, C.byref(found)))
        return (out, alive) if found.value else None

    # ---- desync capture (flags=BGR_CFG_DESYNC_CAPTURE) ----
    def desync_frames(self) -> List[int]:
        """Frames whose first-recorded snapshot is retained and that were saved again since, newest first."""
        buf = (C.c_int32 * 128)()
        n = C.c_uint32()
        self._check(self._lib.bgr_desync_frames(self._h, buf, 128, C.byref(n)))
        return [buf[i] for i in range(min(n.value, 128))]

    def desync_diff(self, frame: int, max_records: int = 64) -> Optional[DesyncReport]:
        """First-recorded vs current snapshot of ``frame`` (bgr_desync_diff); None if either is not held."""
        s = capi.bgr_desync_summary()
        cols = (capi.bgr_desync_column * max(1, len(self.elem_bytes)))()
        recs = np.zeros(max_records, RECORD_DTYPE)
        n, found = C.c_uint32(), C.c_int32()
        self._check(self._lib.bgr_desync_diff(self._h, frame, C.byref(s), cols, len(self.elem_bytes),
                                              recs.ctypes.data_as(C.POINTER(capi.bgr_desync_record)), max_records,
                                              C.byref(n), C.byref(found)))
        if not found.value:
            return None
        return DesyncReport(s.frame, s.rows_first, s.rows_latest, s.rows_differing, s.existence_differing,
                            s.words_differing, s.host_state_differs, s.elapsed_ns_first, s.elapsed_ns_latest,
                            {i: DesyncColumn(i, self.names[i], cols[i].rows, cols[i].rows_in_checksum, cols[i].presence)
                             for i in range(len(self.elem_bytes))},
                            recs[: n.value].copy())

    def peek_first(self, frame: int, col: int, first_row: int, count: int) -> Optional[Tuple[np.ndarray, np.ndarray]]:
        """``peek`` of the first-recorded snapshot of ``frame``."""
        eb = self.elem_bytes[col]
        out = np.zeros((count, eb), dtype=np.uint8)
        alive = np.zeros(count, dtype=np.uint8)
        found = C.c_int32()
        self._check(self._lib.bgr_peek_first(self._h, frame, col, first_row, count, out.ctypes.data, eb,
                                             alive.ctypes.data, C.byref(found)))
        return (out, alive) if found.value else None

    # ---- P2P desync reports ----
    def retain_confirmed(self, interval: int, count: int) -> None:
        """Before build: keep the last ``count`` confirmed frames that are multiples of ``interval``."""
        self._check(self._lib.bgr_retain_confirmed(self._h, interval, count))

    def retained_frames(self) -> List[int]:
        """Retained frames, the most recently retained first."""
        buf = (C.c_int32 * 64)()
        n = C.c_uint32()
        self._check(self._lib.bgr_retained_frames(self._h, buf, 64, C.byref(n)))
        return [buf[i] for i in range(min(n.value, 64))]

    def frame_digest(self, frame: int) -> Optional[Tuple["capi.bgr_frame_digest_header", np.ndarray]]:
        """(header, words[n_blocks, n_columns + 1]) of a queued or retained frame; None if neither holds it."""
        h = capi.bgr_frame_digest_header()
        found = C.c_int32()
        per = len(self.elem_bytes) + 1
        words = np.zeros(-(-self.capacity()[0] // capi.BGR_DIGEST_BLOCK_ROWS) * per, np.uint64)  # any frame fits: one call
        self._check(self._lib.bgr_frame_digest(self._h, frame, C.byref(h), words.ctypes.data, words.size, C.byref(found)))
        if not found.value:
            return None
        return h, words[: h.n_blocks * per].reshape(h.n_blocks, per).copy()

    def export_blocks(self, frame: int, blocks: Sequence[int]) -> Optional[bytes]:
        """The export blob of ``blocks`` of a queued or retained frame; None if neither holds it."""
        ba = np.ascontiguousarray(blocks, dtype=np.uint32)
        size, found = C.c_size_t(), C.c_int32()
        self._check(self._lib.bgr_frame_export(self._h, frame, ba.ctypes.data, len(ba), None, 0, C.byref(size), C.byref(found)))
        if not found.value:
            return None
        out = np.zeros(size.value, np.uint8)
        self._check(self._lib.bgr_frame_export(self._h, frame, ba.ctypes.data, len(ba), out.ctypes.data, out.size,
                                               C.byref(size), C.byref(found)))
        return out.tobytes()

    def diff_remote(self, frame: int, blob: bytes, max_records: int = 64) -> Optional[DesyncReport]:
        """The local image of ``frame`` ("first") against a peer's exported blocks ("latest"), plus the local blocks
        past the peer's block count, whose rows only this side has."""
        s = capi.bgr_desync_summary()
        cols = (capi.bgr_desync_column * max(1, len(self.elem_bytes)))()
        recs = np.zeros(max_records, RECORD_DTYPE)
        n, found = C.c_uint32(), C.c_int32()
        self._check(self._lib.bgr_desync_diff_remote(self._h, frame, blob, len(blob), C.byref(s), cols, len(self.elem_bytes),
                                                     recs.ctypes.data_as(C.POINTER(capi.bgr_desync_record)), max_records,
                                                     C.byref(n), C.byref(found)))
        if not found.value:
            return None
        return DesyncReport(s.frame, s.rows_first, s.rows_latest, s.rows_differing, s.existence_differing,
                            s.words_differing, s.host_state_differs, s.elapsed_ns_first, s.elapsed_ns_latest,
                            {i: DesyncColumn(i, self.names[i], cols[i].rows, cols[i].rows_in_checksum, cols[i].presence)
                             for i in range(len(self.elem_bytes))},
                            recs[: n.value].copy())

    # ---- world checkpoints ----
    def checkpoint(self, frame: int) -> Optional[bytes]:
        """The checkpoint blob of a queued or retained frame (include/bevy_ggrs_b200.h "world checkpoints"); None if
        neither holds it."""
        size, found = C.c_size_t(), C.c_int32()
        self._check(self._lib.bgr_checkpoint_save(self._h, frame, None, 0, C.byref(size), C.byref(found)))
        if not found.value:
            return None
        out = np.empty(size.value, np.uint8)   # an upper bound: the call reports the exact size
        self._check(self._lib.bgr_checkpoint_save(self._h, frame, out.ctypes.data, out.size, C.byref(size), C.byref(found)))
        return out[: size.value].tobytes()

    def restore(self, blob: bytes) -> None:
        """Replace the world with a checkpoint's; the ring then holds the checkpoint's frame alone."""
        self._check(self._lib.bgr_checkpoint_restore(self._h, blob, len(blob)))

    def checkpoint_delta(self, frame: int, base_frame: int) -> Optional[bytes]:
        """The checkpoint delta of ``frame`` against ``base_frame`` (include/bevy_ggrs_b200.h "checkpoint deltas"): the
        blocks of the two frames' canonical images XORed and coded as a checkpoint's.  Both frames queued or retained;
        None if either is not.  ``restore_delta(checkpoint(base_frame), delta)`` restores ``frame``."""
        size, found = C.c_size_t(), C.c_int32()
        self._check(self._lib.bgr_checkpoint_save_delta(self._h, frame, base_frame, None, 0, C.byref(size), C.byref(found)))
        if not found.value:
            return None
        out = np.empty(size.value, np.uint8)   # an upper bound: the call reports the exact size
        self._check(self._lib.bgr_checkpoint_save_delta(self._h, frame, base_frame, out.ctypes.data, out.size, C.byref(size),
                                                        C.byref(found)))
        return out[: size.value].tobytes()

    def restore_delta(self, base: bytes, delta: bytes) -> None:
        """Replace the world with a delta's target frame, given the full checkpoint the delta was written against; the
        engine ends exactly as ``restore`` of the target's full checkpoint leaves it."""
        self._check(self._lib.bgr_checkpoint_restore_delta(self._h, base, len(base), delta, len(delta)))

    # ---- schedules ----
    def save_world(self) -> Tuple[int, int]:
        cs = capi.bgr_checksum()
        self._check(self._lib.bgr_save_world(self._h, C.byref(cs)))
        return cs.frame, (cs.hi << 64) | cs.lo

    def load_world(self) -> None:
        self._check(self._lib.bgr_load_world(self._h))

    def advance_world(self, inputs: Sequence[int] = (), status: Sequence[int] = ()) -> None:
        n = len(inputs)
        ia = (C.c_uint8 * capi.BGR_MAX_PLAYERS)(*[v & 0xFF for v in inputs])
        sa = (C.c_uint8 * capi.BGR_MAX_PLAYERS)(*list(status)[:n])
        self._check(self._lib.bgr_advance_world(self._h, ia, sa, n))

    # ---- the hot loop ----
    def handle_requests(self, session_info: Sequence[int], requests) -> List[Tuple[int, int]]:
        reqs = list(requests)
        arr = capi.make_requests(reqs)
        info = capi.make_session_info(session_info)
        out = (capi.bgr_checksum * capi.BGR_MAX_REQUESTS)()
        n = C.c_uint32()
        self._check(self._lib.bgr_handle_requests(self._h, C.byref(info), arr, len(reqs), out,
                                                  capi.BGR_MAX_REQUESTS, C.byref(n)))
        return [(out[i].frame, (out[i].hi << 64) | out[i].lo) for i in range(n.value)]

    def replay(self, inputs: np.ndarray, checksum_interval: int = 0) -> List[Tuple[int, int]]:
        """Run a recorded input log, ``inputs[n_frames, n_players]`` (uint8), from the current frame f0 in one call:
        what ``[Save(f) if checksum_interval and f % checksum_interval == 0] + [Advance(inputs[j])]`` for every frame
        f = f0 + j would do, without pushing snapshots.  Returns [(frame, checksum), ...] of the checksum frames in
        order.  A non-finite value at a checksum frame raises BgrError(BGR_ERR_NON_FINITE) after the whole log ran."""
        log = _replay_log(inputs)
        r = capi.bgr_replay(log.shape[0], log.shape[1], checksum_interval, 0, log.ctypes.data if log.size else None)
        cap = _replay_points(self.rollback_frame_count(), log.shape[0], checksum_interval)
        out = (capi.bgr_checksum * max(1, cap))()
        n = C.c_uint32()
        self._check(self._lib.bgr_replay(self._h, C.byref(r), out, cap, C.byref(n)))
        return _checksum_list(out, 0, n.value)

    def replay_keyframes(self, inputs: np.ndarray, checksum_interval: int,
                         keyframe_interval: int) -> Tuple[List[Tuple[int, int]], List[Tuple[int, bytes]]]:
        """``replay`` that also returns a world checkpoint (``checkpoint``'s blob) of every frame f = f0 + j, j < n, with
        f % keyframe_interval == 0, taken before frame f is advanced: (checksums, [(frame, blob), ...]).  Both intervals
        are required: every blob is a whole world, so the keyframe interval is the caller's memory budget.  Buffers are
        sized by the call's query (dst NULL), which runs nothing.  A non-finite value at a checksum frame raises
        BgrError(BGR_ERR_NON_FINITE) after the whole log ran, with the keyframes written."""
        log = _replay_log(inputs)
        r = capi.bgr_replay(log.shape[0], log.shape[1], checksum_interval, 0, log.ctypes.data if log.size else None)
        kf = capi.bgr_keyframes(keyframe_interval, 0, 0, None, 0, None)
        n_kf, size = C.c_uint32(), C.c_size_t()
        n = C.c_uint32()
        self._check(self._lib.bgr_replay_keyframes(self._h, C.byref(r), C.byref(kf), None, 0, C.byref(n), C.byref(n_kf),
                                                   C.byref(size)))
        buf, index = _keyframe_buffers(kf, n_kf.value, size.value)
        cap = _replay_points(self.rollback_frame_count(), log.shape[0], checksum_interval)
        out = (capi.bgr_checksum * max(1, cap))()
        self._check(self._lib.bgr_replay_keyframes(self._h, C.byref(r), C.byref(kf), out, cap, C.byref(n), C.byref(n_kf),
                                                   C.byref(size)))
        return _checksum_list(out, 0, n.value), _keyframe_list(buf, index, n_kf.value)

    def replay_trace(self, inputs: np.ndarray, checksum_interval: int, trace_interval: int,
                     fields: Sequence[Tuple[int, int, int]], first_row: int,
                     n_rows: int) -> Tuple[List[Tuple[int, int]], List[Tuple[int, int]], np.ndarray]:
        """``replay`` that also samples rows [first_row, first_row + n_rows) at every frame f = f0 + j, j < n, with
        f % trace_interval == 0, before frame f is advanced: (checksums, [(frame, rows), ...], records).  ``records`` is a
        uint8 array [n_samples, n_rows, record_bytes] of change-feed records over ``fields`` = [(column, byte_offset,
        byte_len), ...] (``feed_record_dtype(fields)`` views one); rows that do not exist are state 0 with zero bytes.
        Buffers are sized by the call's query (dst NULL), which runs nothing.  A non-finite value at a checksum frame
        raises BgrError(BGR_ERR_NON_FINITE) after the whole log ran, with every sample written."""
        log = _replay_log(inputs)
        r = capi.bgr_replay(log.shape[0], log.shape[1], checksum_interval, 0, log.ctypes.data if log.size else None)
        fa = _feed_fields(fields)
        t = capi.bgr_trace(trace_interval, first_row, n_rows, len(fields), fa, None, 0, None, 0, 0)
        n_s, size, n = C.c_uint32(), C.c_size_t(), C.c_uint32()
        self._check(self._lib.bgr_replay_trace(self._h, C.byref(r), C.byref(t), None, 0, C.byref(n), C.byref(n_s), C.byref(size)))
        records, samples = _trace_buffers(t, n_s.value, size.value, n_rows, _record_bytes(fields))
        cap = _replay_points(self.rollback_frame_count(), log.shape[0], checksum_interval)
        out = (capi.bgr_checksum * max(1, cap))()
        self._check(self._lib.bgr_replay_trace(self._h, C.byref(r), C.byref(t), out, cap, C.byref(n), C.byref(n_s),
                                               C.byref(size)))
        return _checksum_list(out, 0, n.value), _sample_list(samples, n_s.value), records

    def submit_requests(self, session_info: Sequence[int], requests) -> None:
        reqs = list(requests)
        arr = capi.make_requests(reqs)
        info = capi.make_session_info(session_info)
        self._check(self._lib.bgr_submit_requests(self._h, C.byref(info), arr, len(reqs)))

    def submit_prepared(self, info: "capi.bgr_session_info", arr, n: int) -> None:
        """submit with pre-built ctypes buffers (bench inner loop: no Python marshalling in the timed region)."""
        self._check(self._lib.bgr_submit_requests(self._h, C.byref(info), arr, n))

    def collect(self) -> List[Tuple[int, int]]:
        out = (capi.bgr_checksum * capi.BGR_MAX_REQUESTS)()
        n = C.c_uint32()
        self._check(self._lib.bgr_collect(self._h, out, capi.BGR_MAX_REQUESTS, C.byref(n)))
        return [(out[i].frame, (out[i].hi << 64) | out[i].lo) for i in range(n.value)]

    def last_partials(self) -> List["capi.bgr_partial"]:
        out = (capi.bgr_partial * capi.BGR_MAX_REQUESTS)()
        n = C.c_uint32()
        self._check(self._lib.bgr_last_partials(self._h, out, capi.BGR_MAX_REQUESTS, C.byref(n)))
        return [out[i] for i in range(n.value)]

    # ---- introspection ----
    def launch_count(self) -> int:
        v = C.c_uint64()
        self._check(self._lib.bgr_launch_count(self._h, C.byref(v)))
        return v.value

    def slot_bytes(self) -> int:
        v = C.c_uint64()
        self._check(self._lib.bgr_slot_bytes(self._h, C.byref(v)))
        return v.value

    def last_path_fused(self) -> bool:
        v = C.c_uint32()
        self._check(self._lib.bgr_last_path(self._h, C.byref(v)))
        return bool(v.value)

    def generic_specialised(self) -> bool:
        """True if bgr_build compiled this registration's own kernel (NVRTC, csrc/generic_program_jit.cuh)."""
        v = C.c_uint32()
        self._check(self._lib.bgr_generic_specialised(self._h, C.byref(v)))
        return bool(v.value)

    def last_kernel(self) -> "LastKernel":
        """What the last request vector executed (bgr_last_kernel), decoded."""
        v = C.c_uint32()
        self._check(self._lib.bgr_last_kernel(self._h, C.byref(v)))
        return LastKernel.decode(v.value)

    def held_saves(self) -> dict:
        """bgr_held_saves: Saves of the last request vector and of all so far that stored nothing, and (env
        BGR_TUNE_HELD_SAVES=2) the words in which a held Save's target differed from the registers (waits for the GPU)."""
        out = (C.c_uint64 * 3)()
        self._check(self._lib.bgr_held_saves(self._h, out, 3))
        return {"last": out[0], "total": out[1], "mismatched_words": out[2]}

    def synchronize(self) -> None:
        self._check(self._lib.bgr_synchronize(self._h))

    def stream(self) -> int:
        """cudaStream_t (as an int) the engine launches on — for timing events recorded by the caller."""
        p = C.c_void_p()
        self._check(self._lib.bgr_stream(self._h, C.byref(p)))
        return p.value or 0

    def reset_session(self) -> None:
        """schedule_systems.rs:70-79: no session -> RollbackFrameCount(0), ConfirmedFrameCount(-1), MaxPredictionWindow(8)."""
        self._check(self._lib.bgr_reset_session(self._h))

    # ---- device-side launch trace ----
    def trace_enable(self, capacity: int) -> None:
        self._check(self._lib.bgr_trace_enable(self._h, capacity))

    def trace_read(self, capacity: int) -> np.ndarray:
        """(n, 4) uint64 per traced fused launch, GPU globaltimer ns: first block start, last block end, results
        published, reserved."""
        out = np.zeros((capacity, 4), dtype=np.uint64)
        n = C.c_uint32()
        self._check(self._lib.bgr_trace_read(self._h, out.ctypes.data, capacity, C.byref(n)))
        return out[: n.value]

    def host_profile(self) -> dict:
        out = (C.c_uint64 * 8)()
        self._check(self._lib.bgr_host_profile(self._h, out, 8))
        return {"calls": out[0], "compile_ns": out[1], "launch_ns": out[2], "wait_ns": out[3], "fold_ns": out[4]}

    # ---- shard group (multi-GPU): cross-shard checksum fold inside the engine ----
    def shard_group_join(self, name: str, rank: int, world_size: int, timeout_ms: int = 0) -> None:
        self._check(self._lib.bgr_shard_group_join(self._h, name.encode(), rank, world_size, timeout_ms))

    def shard_group_leave(self) -> None:
        self._check(self._lib.bgr_shard_group_leave(self._h))


class EngineBatch:
    """A world batch (bgr_batch_*): engines with one registration on one shared stream whose request vectors run in one
    kernel launch.  Holds its engines, so none is destroyed while the batch exists."""

    def __init__(self, engines: Sequence[Engine]):
        self._lib = capi.load_library()
        self._h = None
        self.engines = list(engines)
        self._pinned: List[C.c_void_p] = []
        self._feed_tickets: Dict[int, tuple] = {}
        arr = (C.c_void_p * max(1, len(self.engines)))(*[e._h for e in self.engines])
        h = C.c_void_p()
        self._check(self._lib.bgr_batch_create(arr, len(self.engines), C.byref(h)))
        self._h = h

    def _check(self, status: int) -> None:
        if status != capi.BGR_OK:
            raise BgrError(status, self._lib.bgr_last_error().decode("utf-8", "replace"))

    def close(self) -> None:
        if self._h is not None:
            self._lib.bgr_batch_destroy(self._h)   # waits for a report in flight
            self._h = None
            for p in self._pinned:
                self._lib.bgr_host_free(p)
            self._pinned = []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def specialised(self) -> bool:
        """True if calls run as one launch; False: each world's own handle_requests runs in turn (same results)."""
        v = C.c_uint32()
        self._check(self._lib.bgr_batch_specialised(self._h, C.byref(v)))
        return bool(v.value)

    def handle_requests(self, calls) -> List[Tuple[int, List[Tuple[int, int]]]]:
        """``calls`` = [(world, session_info, requests), ...]: the listed worlds' vectors in one synchronous call.
        Returns [(status, [(frame, checksum), ...]), ...] in the same order; a world's status is what its own
        handle_requests would have returned (BGR_ERR_NON_FINITE ...).  A call refused before anything executed (bad
        index, unsaved frame, pending submits ...) raises BgrError and changes no world."""
        calls = [(w, si, list(r)) for w, si, r in calls]
        n = len(calls)
        worlds = (C.c_uint32 * max(1, n))(*[w for w, _, _ in calls])
        sessions = (capi.bgr_session_info * max(1, n))(*[capi.make_session_info(si) for _, si, _ in calls])
        reqs = capi.make_requests([q for _, _, r in calls for q in r])
        n_req = (C.c_uint32 * max(1, n))(*[len(r) for _, _, r in calls])
        cap = sum(1 for _, _, r in calls for q in r if q.kind == capi.BGR_REQ_SAVE)
        out = (capi.bgr_checksum * max(1, cap))()
        n_cs = (C.c_uint32 * max(1, n))()
        status = (C.c_int32 * max(1, n))()
        rc = self._lib.bgr_batch_handle_requests(self._h, worlds, n, sessions, reqs, n_req, out, cap, n_cs, status)
        if rc not in (capi.BGR_OK, capi.BGR_ERR_NON_FINITE):
            self._check(rc)
        res, k = [], 0
        for i in range(n):
            res.append((status[i], [(out[k + j].frame, (out[k + j].hi << 64) | out[k + j].lo) for j in range(n_cs[i])]))
            k += n_cs[i]
        return res


    def replay(self, calls) -> List[Tuple[int, List[Tuple[int, int]]]]:
        """``calls`` = [(world, inputs[n_frames, n_players] uint8, checksum_interval), ...]: Engine.replay of every
        listed world in one synchronous call (one launch when the batch is specialised).  Returns [(status, [(frame,
        checksum), ...]), ...] in the same order.  A call refused before anything executed raises BgrError and changes
        no world."""
        calls = [(w, _replay_log(x), k) for w, x, k in calls]
        n = len(calls)
        worlds = (C.c_uint32 * max(1, n))(*[w for w, _, _ in calls])
        reps = (capi.bgr_replay * max(1, n))(*[capi.bgr_replay(x.shape[0], x.shape[1], k, 0, x.ctypes.data if x.size else None)
                                               for _, x, k in calls])
        cap = 0
        for w, x, k in calls:
            if 0 <= w < len(self.engines):
                cap += _replay_points(self.engines[w].rollback_frame_count(), x.shape[0], k)
        out = (capi.bgr_checksum * max(1, cap))()
        n_cs = (C.c_uint32 * max(1, n))()
        status = (C.c_int32 * max(1, n))()
        rc = self._lib.bgr_batch_replay(self._h, worlds, n, reps, out, cap, n_cs, status)
        if rc not in (capi.BGR_OK, capi.BGR_ERR_NON_FINITE):
            self._check(rc)
        res, k = [], 0
        for i in range(n):
            res.append((status[i], _checksum_list(out, k, k + n_cs[i])))
            k += n_cs[i]
        return res


    def replay_keyframes(self, calls) -> List[Tuple[int, List[Tuple[int, int]], List[Tuple[int, bytes]]]]:
        """``calls`` = [(world, inputs, checksum_interval, keyframe_interval), ...]: Engine.replay_keyframes of every
        listed world in one synchronous call (one launch per keyframe budget when the batch is specialised).  Returns
        [(status, checksums, [(frame, blob), ...]), ...] in the same order.  Each world's buffers are sized by its own
        engine's query; a call refused before anything executed raises BgrError and changes no world."""
        calls = [(w, _replay_log(x), k, kk) for w, x, k, kk in calls]
        n = len(calls)
        worlds = (C.c_uint32 * max(1, n))(*[w for w, _, _, _ in calls])
        reps = (capi.bgr_replay * max(1, n))(*[capi.bgr_replay(x.shape[0], x.shape[1], k, 0, x.ctypes.data if x.size else None)
                                               for _, x, k, _ in calls])
        kfs = (capi.bgr_keyframes * max(1, n))()
        bufs = []
        cap = 0
        for i, (w, x, k, kk) in enumerate(calls):
            kfs[i].interval = kk
            buf, index = None, None
            if 0 <= w < len(self.engines) and kk > 0:
                q = capi.bgr_keyframes(kk, 0, 0, None, 0, None)
                n_kf, size, n_cs = C.c_uint32(), C.c_size_t(), C.c_uint32()
                if self._lib.bgr_replay_keyframes(self.engines[w]._h, C.byref(reps[i]), C.byref(q), None, 0, C.byref(n_cs),
                                                  C.byref(n_kf), C.byref(size)) == capi.BGR_OK:
                    buf, index = _keyframe_buffers(kfs[i], n_kf.value, size.value)
                cap += _replay_points(self.engines[w].rollback_frame_count(), x.shape[0], k)
            bufs.append((buf, index))
        out = (capi.bgr_checksum * max(1, cap))()
        n_cs = (C.c_uint32 * max(1, n))()
        n_kf = (C.c_uint32 * max(1, n))()
        status = (C.c_int32 * max(1, n))()
        rc = self._lib.bgr_batch_replay_keyframes(self._h, worlds, n, reps, kfs, out, cap, n_cs, n_kf, status)
        if rc not in (capi.BGR_OK, capi.BGR_ERR_NON_FINITE):
            self._check(rc)
        res, k = [], 0
        for i in range(n):
            res.append((status[i], _checksum_list(out, k, k + n_cs[i]), _keyframe_list(bufs[i][0], bufs[i][1], n_kf[i])))
            k += n_cs[i]
        return res

    def replay_trace(self, calls, fields: Sequence[Tuple[int, int, int]]):
        """``calls`` = [(world, inputs, checksum_interval, trace_interval, first_row, n_rows), ...]: Engine.replay_trace of
        every listed world over one field list in one synchronous call (one launch per trace budget when the batch is
        specialised).  Returns [(status, checksums, [(frame, rows), ...], records), ...] in the same order.  Each world's
        buffers are sized by its own engine's query; a call refused before anything executed raises BgrError and changes
        no world."""
        calls = [(w, _replay_log(x), k, tt, a, nr) for w, x, k, tt, a, nr in calls]
        n = len(calls)
        fa = _feed_fields(fields)
        worlds = (C.c_uint32 * max(1, n))(*[c[0] for c in calls])
        reps = (capi.bgr_replay * max(1, n))(*[capi.bgr_replay(x.shape[0], x.shape[1], k, 0, x.ctypes.data if x.size else None)
                                               for _, x, k, _, _, _ in calls])
        trs = (capi.bgr_trace * max(1, n))()
        bufs = []
        cap = 0
        for i, (w, x, k, tt, a, nr) in enumerate(calls):
            trs[i] = capi.bgr_trace(tt, a, nr, len(fields), fa, None, 0, None, 0, 0)
            records, samples = np.zeros((0, nr, _record_bytes(fields)), np.uint8), None
            if 0 <= w < len(self.engines):
                q = capi.bgr_trace(tt, a, nr, len(fields), fa, None, 0, None, 0, 0)
                n_s, size, n_cs = C.c_uint32(), C.c_size_t(), C.c_uint32()
                if self._lib.bgr_replay_trace(self.engines[w]._h, C.byref(reps[i]), C.byref(q), None, 0, C.byref(n_cs),
                                              C.byref(n_s), C.byref(size)) == capi.BGR_OK:
                    records, samples = _trace_buffers(trs[i], n_s.value, size.value, nr, _record_bytes(fields))
                cap += _replay_points(self.engines[w].rollback_frame_count(), x.shape[0], k)
            bufs.append((records, samples))
        out = (capi.bgr_checksum * max(1, cap))()
        n_cs = (C.c_uint32 * max(1, n))()
        n_s = (C.c_uint32 * max(1, n))()
        status = (C.c_int32 * max(1, n))()
        rc = self._lib.bgr_batch_replay_trace(self._h, worlds, n, reps, trs, out, cap, n_cs, n_s, status)
        if rc not in (capi.BGR_OK, capi.BGR_ERR_NON_FINITE):
            self._check(rc)
        res, k = [], 0
        for i in range(n):
            res.append((status[i], _checksum_list(out, k, k + n_cs[i]), _sample_list(bufs[i][1], n_s[i]), bufs[i][0]))
            k += n_cs[i]
        return res

    def checkpoint(self, calls) -> List[Optional[bytes]]:
        """``calls`` = [(world, frame), ...]: Engine.checkpoint of every listed world in one call (one encoding pass and
        one copy back).  Returns the blobs in the same order, None where the world holds that frame neither queued
        nor retained.  The buffer is sized by the call's query (dst NULL), which runs nothing; a refused call raises
        BgrError naming the world."""
        calls = list(calls)
        n = len(calls)
        worlds = (C.c_uint32 * max(1, n))(*[w for w, _ in calls])
        frames = (C.c_int32 * max(1, n))(*[f for _, f in calls])
        index = (capi.bgr_keyframe * max(1, n))()
        size = C.c_size_t()
        status = (C.c_int32 * max(1, n))()
        self._check(self._lib.bgr_batch_checkpoint_save(self._h, worlds, n, frames, None, 0, index, C.byref(size), status))
        buf = np.empty(max(1, size.value), np.uint8)   # upper bounds: the call reports the exact layout
        self._check(self._lib.bgr_batch_checkpoint_save(self._h, worlds, n, frames, buf.ctypes.data, size.value, index,
                                                        C.byref(size), status))
        return [buf[index[i].offset: index[i].offset + index[i].bytes].tobytes() if index[i].bytes else None
                for i in range(n)]

    def restore(self, calls) -> None:
        """``calls`` = [(world, blob), ...]: Engine.restore of every listed world in one call (one decoding pass).  All
        or nothing: a refused call raises BgrError (its status, and text starting with "world <index>: ") and changes
        no world."""
        calls = list(calls)
        n = len(calls)
        worlds = (C.c_uint32 * max(1, n))(*[w for w, _ in calls])
        keep = [C.c_char_p(b if isinstance(b, bytes) else bytes(b)) for _, b in calls]   # no copy of a bytes blob
        blobs = (C.c_void_p * max(1, n))(*[C.cast(k, C.c_void_p).value for k in keep])
        sizes = (C.c_size_t * max(1, n))(*[len(b) for _, b in calls])
        status = (C.c_int32 * max(1, n))()
        self._check(self._lib.bgr_batch_checkpoint_restore(self._h, worlds, n, blobs, sizes, status))

    def apply_edits(self, calls) -> None:
        """``calls`` = [(world, edits, values), ...]: Engine.apply_edits of every listed world in one queued call (at
        most one spawn launch and one patch launch over all of them).  ``edits`` is an ``EDIT_DTYPE`` array, ``values``
        the bytes its WRITE / INSERT records point into; both are free on return.  All or nothing: a refused call raises
        BgrError (its status, and text starting with "world <index>: ") and changes no world."""
        calls = [(int(w), np.ascontiguousarray(x, dtype=EDIT_DTYPE), np.frombuffer(bytes(v), dtype=np.uint8))
                 for w, x, v in calls]
        n = len(calls)
        entries = (capi.bgr_batch_edits * max(1, n))(*[
            capi.bgr_batch_edits(w, len(x), x.ctypes.data if len(x) else None, v.ctypes.data if v.size else None, v.size)
            for w, x, v in calls])
        status = (C.c_int32 * max(1, n))()
        self._check(self._lib.bgr_batch_apply_edits(self._h, entries, n, status))

    # ---- batched change feed (bgr_batch_feed_*): many members' feeds in one pass ----
    def _feed_bytes(self, calls) -> Optional[int]:
        """sum(cap) records of the first call's feed (a call has one record size), or None when the first call names no
        feed this wrapper knows (the library refuses the call)."""
        if not calls:
            return 0
        w, f, _ = calls[0]
        dt = self.engines[w]._feed_dtypes.get(f) if 0 <= w < len(self.engines) else None
        return None if dt is None else sum(cap for _, _, cap in calls) * dt.itemsize

    def feed_alloc(self, calls) -> np.ndarray:
        """Page-locked buffer for a batched report of ``calls`` = [(world, feed, cap), ...]: sum(cap) records of the
        first call's feed; freed with the batch."""
        size = self._feed_bytes(list(calls)) or 0
        p = C.c_void_p()
        self._check(self._lib.bgr_host_alloc(max(1, size), C.byref(p)))
        self._pinned.append(p)
        return np.frombuffer((C.c_uint8 * max(1, size)).from_address(p.value), dtype=np.uint8)

    def feed_begin(self, calls, buf: Optional[np.ndarray]) -> int:
        """Starts one report of every ``calls`` entry (world, feed, cap) into ``buf`` (from feed_alloc); returns its
        ticket.  A refused call raises BgrError (text starting with "world <index>: " for a refused entry) and changes
        no feed."""
        calls = [tuple(int(x) for x in c) for c in calls]
        n = len(calls)
        need = self._feed_bytes(calls)
        if need:   # the library cannot check the buffer's size: the records of every entry must fit
            assert buf is not None and buf.dtype == np.uint8 and buf.flags.c_contiguous and buf.size >= need, \
                f"feed_begin needs a buffer of {need} bytes (feed_alloc of these calls)"
        reps = (capi.bgr_batch_feed * max(1, n))(*[capi.bgr_batch_feed(*c) for c in calls])
        t = C.c_uint32()
        status = (C.c_int32 * max(1, n))()
        dst = buf.ctypes.data if buf is not None else None
        self._check(self._lib.bgr_batch_feed_begin(self._h, reps, n, dst, C.byref(t), status))
        self._feed_tickets[t.value] = (calls, buf)
        return t.value

    def feed_wait(self, ticket: int) -> List[Tuple[np.ndarray, FeedInfo]]:
        """[(records, info), ...] of a batched report, in the order of its calls: structured arrays (row, state, f0,
        ...) copied out of the buffer, entry i's from behind the earlier entries' records."""
        calls, buf = self._feed_tickets.get(ticket, ([], None))
        infos = (capi.bgr_feed_info * max(1, len(calls)))()
        self._check(self._lib.bgr_batch_feed_wait(self._h, ticket, infos))
        del self._feed_tickets[ticket]
        out, at = [], 0
        for i, (w, f, _) in enumerate(calls):
            dt = self.engines[w].feed_record_dtype(f)
            info = infos[i]
            assert info.record_bytes == dt.itemsize
            recs = np.empty(info.n_records, dt)
            if info.n_records:   # buf may be None when every cap is 0
                C.memmove(recs.ctypes.data, buf.ctypes.data + at, info.n_records * dt.itemsize)
            at += info.n_records * dt.itemsize
            out.append((recs, FeedInfo(info.n_records, info.pending, info.rows, info.record_bytes)))
        return out


def _keyframe_buffers(kf: "capi.bgr_keyframes", n_kf: int, size: int):
    """A dst of `size` bytes and an index of `n_kf` entries, installed in `kf`; the arrays must outlive the call."""
    buf = np.empty(max(1, size), np.uint8)
    index = (capi.bgr_keyframe * max(1, n_kf))()
    kf.dst, kf.dst_cap, kf.index, kf.index_cap = buf.ctypes.data, size, index, n_kf
    return buf, index


def _keyframe_list(buf, index, n: int) -> List[Tuple[int, bytes]]:
    return [(index[i].frame, buf[index[i].offset: index[i].offset + index[i].bytes].tobytes()) for i in range(n)]


def _feed_fields(fields) -> "C.Array[capi.bgr_feed_field]":
    fields = [tuple(int(x) for x in f) for f in fields]
    return (capi.bgr_feed_field * max(1, len(fields)))(*[capi.bgr_feed_field(*f) for f in fields])


def _trace_buffers(t: "capi.bgr_trace", n_samples: int, size: int, n_rows: int, rb: int):
    """Records [n_samples, n_rows, rb] (uint8) and a sample index of n_samples entries, installed in `t`; the arrays must
    outlive the call."""
    buf = np.zeros(max(1, size), np.uint8)   # never a null dst, which would be a query: a log may take no sample
    records = buf[:size].reshape(n_samples, n_rows, rb)
    samples = (capi.bgr_trace_sample * max(1, n_samples))()
    t.dst, t.dst_cap, t.samples, t.samples_cap = buf.ctypes.data, size, samples, n_samples
    return records, samples


def _record_bytes(fields) -> int:
    return 8 + sum(int(ln) for _, _, ln in fields)


def _sample_list(samples, n: int) -> List[Tuple[int, int]]:
    """[(frame, rows)] of the first n bgr_trace_sample entries, through numpy: a trace at T = 1 returns thousands."""
    if not n:
        return []
    arr = np.ctypeslib.as_array(samples)[:n]
    return list(zip(arr["frame"].tolist(), arr["rows"].tolist()))


def _replay_log(inputs) -> np.ndarray:
    log = np.ascontiguousarray(inputs, dtype=np.uint8)
    if log.ndim != 2:
        raise ValueError("a replay log is a [n_frames, n_players] array")
    return log


def _checksum_list(out, a: int, b: int) -> List[Tuple[int, int]]:
    """[(frame, checksum)] of bgr_checksum array elements [a, b), through numpy: a replay returns thousands."""
    if b <= a:
        return []
    arr = np.ctypeslib.as_array(out)[a:b]
    return [(f, (h << 64) | lo) for f, lo, h in zip(arr["frame"].tolist(), arr["lo"].tolist(), arr["hi"].tolist())]


def _replay_points(f0: int, n: int, k: int) -> int:
    """Checksum frames f0 + j, j < n, with (f0 + j) % k == 0 (the size of a replay's result)."""
    if k <= 0 or n <= 0 or f0 < 0:
        return 0
    return (f0 + n + k - 1) // k - (f0 + k - 1) // k


def fold_partials(partial: "capi.bgr_partial") -> int:
    lib = capi.load_library()
    cs = capi.bgr_checksum()
    st = lib.bgr_fold_partials(C.byref(partial), C.byref(cs))
    if st != capi.BGR_OK:
        raise BgrError(st, lib.bgr_last_error().decode())
    return (cs.hi << 64) | cs.lo


def digest_mismatch(local, remote) -> Tuple[List[int], int]:
    """(blocks that differ, host_state_differs bits) of two ``Engine.frame_digest`` results (bgr_digest_mismatch)."""
    lib = capi.load_library()
    (lh, lw), (rh, rw) = local, remote
    lw, rw = np.ascontiguousarray(lw, np.uint64), np.ascontiguousarray(rw, np.uint64)
    cap = max(lh.n_blocks, rh.n_blocks, 1)
    out = np.zeros(cap, np.uint32)
    n, host = C.c_uint32(), C.c_uint32()
    st = lib.bgr_digest_mismatch(C.byref(lh), lw.ctypes.data, C.byref(rh), rw.ctypes.data, out.ctypes.data, cap,
                                 C.byref(n), C.byref(host))
    if st != capi.BGR_OK:
        raise BgrError(st, lib.bgr_last_error().decode("utf-8", "replace"))
    return [int(b) for b in out[: n.value]], host.value


def ggrs_time_delta_bits(fps: int, frame: int) -> int:
    return capi.load_library().bgr_ggrs_time_delta_bits(fps, frame)
