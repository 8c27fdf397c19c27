"""ctypes binding of oracle/liboracle.so (the CPU restatement) with the same method surface as
``bevy_ggrs_b200.engine.Engine`` so tests can drive both with identical code.

TEST INFRASTRUCTURE: nothing in the product package imports this file.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from typing import List, Optional, Sequence, Tuple

import numpy as np

from bevy_ggrs_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
ORC_SYS_RESOURCE_U32_ADD = 100

_LIB = None


def build_oracle() -> str:
    subprocess.run(["make", "-C", ORACLE_DIR, "liboracle.so"], check=True, capture_output=True)
    return os.path.join(ORACLE_DIR, "liboracle.so")


def load_oracle() -> C.CDLL:
    global _LIB
    if _LIB is not None:
        return _LIB
    path = os.path.join(ORACLE_DIR, "liboracle.so")
    if not os.path.exists(path):
        build_oracle()
    lib = C.CDLL(path)
    vp, u32, i32, u64 = C.c_void_p, C.c_uint32, C.c_int32, C.c_uint64
    u32p, u64p = C.POINTER(u32), C.POINTER(u64)
    sig = {
        "orc_last_error": (C.c_char_p, []),
        "orc_seahash": (u64, [vp, u64]),
        "orc_checksum_part_from_u32": (u64, [u32]),
        "orc_seahash_u32_fields": (u64, [u32p, u32]),
        "orc_seahash_u64_fields": (u64, [u64p, u32]),
        "orc_ggrs_time_delta_bits": (u32, [u32, i32]),
        "orc_ring_new": (vp, [u32, C.c_int]),
        "orc_ring_free": (None, [vp]),
        "orc_ring_set_depth": (None, [vp, u32]),
        "orc_ring_depth": (u32, [vp]),
        "orc_ring_push": (None, [vp, i32, u32]),
        "orc_ring_confirm": (None, [vp, i32]),
        "orc_ring_rollback": (C.c_int, [vp, i32]),
        "orc_ring_get": (C.c_int, [vp, u32p]),
        "orc_ring_peek": (C.c_int, [vp, i32, u32p]),
        "orc_ring_len": (u32, [vp]),
        "orc_ordered_new": (vp, []),
        "orc_ordered_clone": (vp, [vp]),
        "orc_ordered_free": (None, [vp]),
        "orc_ordered_push": (None, [vp, u64]),
        "orc_ordered_order": (C.c_int, [vp, u64, u64p]),
        "orc_ordered_len": (u64, [vp]),
        "orc_ordered_iter_sorted": (u32, [vp, u64p, u32]),
        "orc_world_new": (vp, [u32, u64, u32]),
        "orc_world_free": (None, [vp]),
        "orc_rollback_component": (C.c_int, [vp, C.c_char_p, u32, u32p]),
        "orc_checksum_component": (C.c_int, [vp, u32, u32, u32, u32, u32]),
        "orc_rollback_resource": (C.c_int, [vp, C.c_char_p, vp, u32, C.c_int, u32p]),
        "orc_add_system": (C.c_int, [vp, u32, u32p, u32, u32p, u32]),
        "orc_spawn": (C.c_int, [vp, u32, u32p]),
        "orc_run_startup_system": (C.c_int, [vp, u32]),
        "orc_xoshiro_stream": (None, [u64, u32, u64p, C.POINTER(C.c_float), C.c_float, C.c_float]),
        "orc_xoshiro_from_state": (None, [u64p, u32, u64p]),
        "orc_xoshiro_seed_state": (None, [u64, u64p]),
        "orc_row_count": (u32, [vp]),
        "orc_active_count": (u64, [vp]),
        "orc_write_component": (C.c_int, [vp, u32, u32, u32, vp, u32]),
        "orc_read_component": (C.c_int, [vp, u32, u32, u32, vp, u32, vp]),
        "orc_read_alive": (C.c_int, [vp, u32, u32, vp]),
        "orc_remove_component": (C.c_int, [vp, u32, u64]),
        "orc_insert_component": (C.c_int, [vp, u32, u64, vp]),
        "orc_despawn": (C.c_int, [vp, u64]),
        "orc_peek": (C.c_int, [vp, i32, u32, u32, u32, vp, u32, vp]),
        "orc_snapshot_frames": (C.c_int, [vp, C.POINTER(i32), u32]),
        "orc_read_resource": (C.c_int, [vp, u32, vp]),
        "orc_rollback_frame_count": (i32, [vp]),
        "orc_set_rollback_frame_count": (None, [vp, i32]),
        "orc_confirmed_frame_count": (i32, [vp]),
        "orc_set_max_prediction": (None, [vp, u32]),
        "orc_reset_session": (None, [vp]),
        "orc_last_dt_bits": (u32, [vp]),
        "orc_save_world": (C.c_int, [vp, C.POINTER(capi.bgr_checksum)]),
        "orc_checksum_world": (C.c_int, [vp, C.POINTER(capi.bgr_checksum)]),
        "orc_restore": (C.c_int, [vp, i32, u32, vp, u32p, C.POINTER(vp), u64, u64p]),
        "orc_load_world": (C.c_int, [vp]),
        "orc_advance_world": (C.c_int, [vp, vp, u32]),
        "orc_last_partial": (C.c_int, [vp, C.POINTER(capi.bgr_partial)]),
        "orc_soa_new": (vp, [u32, u32, u32, u32]),
        "orc_soa_free": (None, [vp]),
        "orc_soa_set_columns": (None, [vp, vp, vp, vp]),
        "orc_soa_get_columns": (None, [vp, vp, vp, vp, vp]),
        "orc_soa_handle_requests": (C.c_int, [vp, C.POINTER(capi.bgr_session_info), C.POINTER(capi.bgr_request), u32,
                                              C.POINTER(capi.bgr_checksum), u32, u32p, u64p]),
        "orc_handle_requests": (C.c_int, [vp, C.POINTER(capi.bgr_session_info), C.POINTER(capi.bgr_request), u32,
                                          C.POINTER(capi.bgr_checksum), u32, u32p, u64p]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    _LIB = lib
    return lib


class OracleError(RuntimeError):
    def __init__(self, status, text):
        super().__init__(text)
        self.status = status


class OracleWorld:
    """Same surface as bevy_ggrs_b200.engine.Engine, backed by the CPU restatement."""

    def __init__(self, max_entities: int = 0, max_depth: int = 9, fps: int = 60, order_base: int = 0,
                 save_threads: int = 1, **_):
        self._lib = load_oracle()
        self._h = C.c_void_p(self._lib.orc_world_new(fps, order_base, save_threads))
        self.elem_bytes: List[int] = []
        self.last_elapsed_ns = 0

    def _check(self, st):
        if st != 0:
            raise OracleError(st, self._lib.orc_last_error().decode())

    def close(self):
        if self._h:
            self._lib.orc_world_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def rollback_component(self, name, elem_bytes, strategy=0):
        col = C.c_uint32()
        self._check(self._lib.orc_rollback_component(self._h, name.encode(), elem_bytes, C.byref(col)))
        self.elem_bytes.append(elem_bytes)
        return col.value

    def checksum_component(self, col, byte_offset, byte_len, flags=0):
        self._check(self._lib.orc_checksum_component(self._h, col, capi.BGR_HASH_BYTES, byte_offset, byte_len, flags))

    def rollback_resource(self, name, init: bytes, checksum: bool):
        res = C.c_uint32()
        buf = C.create_string_buffer(init, len(init))
        self._check(self._lib.orc_rollback_resource(self._h, name.encode(), buf, len(init), int(checksum), C.byref(res)))
        return res.value

    def read_resource(self, res, nbytes):
        buf = C.create_string_buffer(nbytes)
        ok = self._lib.orc_read_resource(self._h, res, buf)
        return buf.raw if ok else None

    def add_system(self, system, cols, params=()):
        ca = (C.c_uint32 * max(1, len(cols)))(*cols)
        pa = (C.c_uint32 * max(1, len(params)))(*params)
        self._check(self._lib.orc_add_system(self._h, system, ca, len(cols), pa, len(params)))

    def build(self):
        pass

    def run_startup_system(self, system):
        self._check(self._lib.orc_run_startup_system(self._h, system))

    def spawn(self, count):
        first = C.c_uint32()
        self._check(self._lib.orc_spawn(self._h, count, C.byref(first)))
        return first.value

    def despawn(self, row):
        self._check(self._lib.orc_despawn(self._h, row))

    def row_count(self):
        return self._lib.orc_row_count(self._h)

    def active_count(self):
        return self._lib.orc_active_count(self._h)

    def write_component(self, col, first_row, values):
        eb = self.elem_bytes[col]
        a = np.ascontiguousarray(values).view(np.uint8).reshape(-1, eb)
        self._check(self._lib.orc_write_component(self._h, col, first_row, a.shape[0], a.ctypes.data, eb))

    def remove_component(self, col, row):
        self._check(self._lib.orc_remove_component(self._h, col, row))

    def insert_component(self, col, row, value):
        a = np.ascontiguousarray(value).view(np.uint8).reshape(-1)
        assert a.size == self.elem_bytes[col]
        self._check(self._lib.orc_insert_component(self._h, col, row, a.ctypes.data))

    def has_component(self, col, first_row, count):
        return self.read_component_alive(col, first_row, count)[1]

    def read_component_alive(self, col, first_row, count):
        eb = self.elem_bytes[col]
        out = np.zeros((count, eb), dtype=np.uint8)
        alive = np.zeros(count, dtype=np.uint8)
        self._check(self._lib.orc_read_component(self._h, col, first_row, count, out.ctypes.data, eb, alive.ctypes.data))
        return out, alive

    def read_component(self, col, first_row, count):
        return self.read_component_alive(col, first_row, count)[0]

    def read_alive(self, first_row, count):
        alive = np.zeros(count, dtype=np.uint8)
        self._check(self._lib.orc_read_alive(self._h, first_row, count, alive.ctypes.data))
        return alive

    def rollback_frame_count(self):
        return self._lib.orc_rollback_frame_count(self._h)

    def set_rollback_frame_count(self, f):
        self._lib.orc_set_rollback_frame_count(self._h, f)

    def confirmed_frame_count(self):
        return self._lib.orc_confirmed_frame_count(self._h)

    def set_depth(self, depth):
        self._lib.orc_set_max_prediction(self._h, depth)

    def reset_session(self):
        self._lib.orc_reset_session(self._h)

    def snapshot_frames(self):
        buf = (C.c_int32 * 128)()
        n = self._lib.orc_snapshot_frames(self._h, buf, 128)
        return [buf[i] for i in range(n)]

    def peek(self, frame, col, first_row, count):
        eb = self.elem_bytes[col]
        out = np.zeros((count, eb), dtype=np.uint8)
        alive = np.zeros(count, dtype=np.uint8)
        found = self._lib.orc_peek(self._h, frame, col, first_row, count, out.ctypes.data, eb, alive.ctypes.data)
        return (out, alive) if found else None

    def save_world(self):
        cs = capi.bgr_checksum()
        self._check(self._lib.orc_save_world(self._h, C.byref(cs)))
        return cs.frame, (cs.hi << 64) | cs.lo

    def checksum_world(self):
        """The Checksum half of SaveWorld: (frame, checksum) of the current world, no snapshot pushed."""
        cs = capi.bgr_checksum()
        self._check(self._lib.orc_checksum_world(self._h, C.byref(cs)))
        return cs.frame, (cs.hi << 64) | cs.lo

    def restore_world(self, frame, mask, absent_bits, columns, elapsed_ns, rng):
        """Replaces the world with a checkpoint's content (World::restore): ``mask`` one byte per row, ``absent_bits``
        each column's mask bit (0: required), ``columns[c]`` [rows, elem_bytes] u8."""
        rows = len(mask)
        mask = np.ascontiguousarray(mask, np.uint8)
        absent = np.ascontiguousarray(absent_bits, np.uint32)
        cols = [np.ascontiguousarray(c, np.uint8).reshape(rows, eb) for c, eb in zip(columns, self.elem_bytes)]
        ptrs = (C.c_void_p * max(1, len(cols)))(*[c.ctypes.data for c in cols])
        words = np.ascontiguousarray(rng, np.uint64)
        self._check(self._lib.orc_restore(self._h, frame, rows, mask.ctypes.data,
                                          absent.ctypes.data_as(C.POINTER(C.c_uint32)), ptrs, elapsed_ns,
                                          words.ctypes.data_as(C.POINTER(C.c_uint64))))

    def load_world(self):
        self._check(self._lib.orc_load_world(self._h))

    def advance_world(self, inputs=(), status=()):
        ia = (C.c_uint8 * capi.BGR_MAX_PLAYERS)(*[v & 0xFF for v in inputs])
        self._check(self._lib.orc_advance_world(self._h, ia, len(inputs)))

    def last_dt_bits(self):
        return self._lib.orc_last_dt_bits(self._h)

    def last_partial(self):
        p = capi.bgr_partial()
        self._check(self._lib.orc_last_partial(self._h, C.byref(p)))
        return p

    def handle_requests(self, session_info, requests):
        reqs = list(requests)
        arr = capi.make_requests(reqs)
        info = capi.make_session_info(session_info)
        out = (capi.bgr_checksum * capi.BGR_MAX_REQUESTS)()
        n = C.c_uint32()
        ns = C.c_uint64()
        st = self._lib.orc_handle_requests(self._h, C.byref(info), arr, len(reqs), out, capi.BGR_MAX_REQUESTS,
                                           C.byref(n), C.byref(ns))
        self.last_elapsed_ns = ns.value
        self._check(st)
        return [(out[i].frame, (out[i].hi << 64) | out[i].lo) for i in range(n.value)]


class SoaWorld:
    """The optimised CPU SoA bar (oracle/soa_baseline.hpp): particles schema, all host cores."""

    def __init__(self, tf, vel, ttl, depth, fps=60, threads=0):
        self._lib = load_oracle()
        self.n = tf.shape[0]
        self.threads = threads or (os.cpu_count() or 1)
        self._h = C.c_void_p(self._lib.orc_soa_new(self.n, depth, fps, self.threads))
        tf = np.ascontiguousarray(tf, dtype=np.float32); vel = np.ascontiguousarray(vel, dtype=np.float32)
        ttl = np.ascontiguousarray(ttl, dtype=np.uint64)
        self._lib.orc_soa_set_columns(self._h, tf.ctypes.data, vel.ctypes.data, ttl.ctypes.data)
        self.last_elapsed_ns = 0

    def handle_requests(self, session_info, requests):
        reqs = list(requests)
        arr = capi.make_requests(reqs)
        info = capi.make_session_info(session_info)
        out = (capi.bgr_checksum * capi.BGR_MAX_REQUESTS)()
        n, ns = C.c_uint32(), C.c_uint64()
        st = self._lib.orc_soa_handle_requests(self._h, C.byref(info), arr, len(reqs), out, capi.BGR_MAX_REQUESTS,
                                               C.byref(n), C.byref(ns))
        self.last_elapsed_ns = ns.value
        if st != 0:
            raise OracleError(st, self._lib.orc_last_error().decode())
        return [(out[i].frame, (out[i].hi << 64) | out[i].lo) for i in range(n.value)]

    def columns(self):
        tf = np.zeros((self.n, 10), np.float32); vel = np.zeros((self.n, 3), np.float32)
        ttl = np.zeros(self.n, np.uint64); alive = np.zeros(self.n, np.uint8)
        self._lib.orc_soa_get_columns(self._h, tf.ctypes.data, vel.ctypes.data, ttl.ctypes.data, alive.ctypes.data)
        return tf, vel, ttl, alive

    def close(self):
        if self._h:
            self._lib.orc_soa_free(self._h)
            self._h = None
