"""Host-side mirror of the bevy_ggrs plugin surface for the hot path.

Same names and argument meaning as the reference (src/lib.rs, src/snapshot/rollback_app.rs,
src/schedule_systems.rs) so that a bevy_ggrs user — and the parity tests — read the same:

    app = App(engine)
    app.add_plugins(GgrsPlugin())
    app.insert_resource(RollbackFrameRate(60))
    app.add_systems(ReadInputs, read_local_inputs)
    t = app.rollback_component_with_clone("Transform", 40)
    app.checksum_component(t, byte_offset=0, byte_len=12, assert_finite=True)
    app.add_systems(GgrsSchedule, System(BGR_SYS_PARTICLES_UPDATE, [t, v]))
    app.insert_resource(Session.SyncTest(session))
    app.add_observer(SyncTestMismatch, on_mismatch)
    app.update()

Differences forced by the C ABI (documented in INTEGRATION.md):
  * components are registered by (name, size_of::<T>()) and the per-element hasher is a byte
    range instead of a Rust closure;
  * GgrsSchedule systems are compiled-in GPU systems named by id;
  * the "World" is the engine: columns live in HBM, the ring of snapshots too.

``backend`` is any object with the ``bevy_ggrs_b200.engine.Engine`` method surface.  This
module is pure host logic: it never touches the GPU or the oracle itself.
"""
from __future__ import annotations

import struct
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence, Tuple

from . import capi
from .host_components import HostComponents
from .session import (ADVANCE, LOAD, SAVE, GgrsError, MismatchedChecksum, P2PTraceSession, Request,
                      SyncTestSession)

DEFAULT_FPS = 60  # lib.rs:58


# ---- schedule labels (lib.rs:73-74, :148-149) ----
class GgrsSchedule:
    pass


class ReadInputs:
    pass


class Startup:
    pass


# ---- resources ----
@dataclass
class RollbackFrameRate:  # time.rs:19-26
    fps: int = DEFAULT_FPS


@dataclass
class LocalInputs:  # lib.rs:140-141
    inputs: Dict[int, int]


@dataclass
class LocalPlayers:  # lib.rs:144-145
    handles: List[int] = field(default_factory=list)


@dataclass
class SyncTestMismatch:  # lib.rs:131-137
    current_frame: int
    mismatched_frames: List[int]


class Session:  # lib.rs:79-86
    SYNCTEST, P2P, SPECTATOR = "SyncTest", "P2P", "Spectator"

    def __init__(self, kind: str, inner):
        self.kind = kind
        self.inner = inner

    @classmethod
    def SyncTest(cls, s: SyncTestSession) -> "Session":
        return cls(cls.SYNCTEST, s)

    @classmethod
    def P2PTrace(cls, s: P2PTraceSession) -> "Session":
        return cls(cls.P2P, s)


@dataclass
class System:
    """A compiled-in GgrsSchedule system: id + the columns it binds + scalar parameters."""
    system: int
    columns: Sequence[int]
    params: Sequence[int] = ()


@dataclass
class ResourceSystem:
    """A GgrsSchedule system that only touches host-side resources (e.g. box_game's increase_frame_system,
    box_game.rs:146-148): ``fn(resources: dict[str, bytearray])``.  Resources are a few bytes and not
    data-parallel, so they stay on the host (SURVEY.md §2 row 10); the shim rolls them back per frame and XORs
    their checksum parts into the engine's checksum."""
    fn: Callable


class GgrsPlugin:  # lib.rs:198-258
    def build(self, app: "App") -> None:
        app._ggrs = True


class App:
    """Mirror of ``bevy::App`` restricted to what the rollback hot path touches."""

    MANUAL_DURATION_NS = 16_666_667  # Duration::from_secs_f64(1.0 / 60.0), tests/common/mod.rs:47-49

    def __init__(self, backend):
        self.world = backend
        self._ggrs = False
        self._built = False
        self._session: Optional[Session] = None
        self._frame_rate = RollbackFrameRate()
        self._read_inputs: List[Callable[["App"], None]] = []
        self._startup: List[Callable[["App"], None]] = []
        self._observers: List[Callable[[SyncTestMismatch], None]] = []
        self._local_inputs: Optional[LocalInputs] = None
        self.local_players = LocalPlayers()
        # FixedTimestepData (lib.rs:98-114)
        self._accumulator_ns = 0
        self._run_slow = False
        self._first_update = True
        self.last_checksums: List[tuple] = []
        self.ticks = 0
        # host-side resources (rollback_resource_with_copy / checksum_resource_with_hash)
        self.resources: Dict[str, bytearray] = {}
        self._res_registered: List[str] = []
        self._res_checksummed: List[str] = []
        self._res_systems: List[Callable] = []
        self._res_store: Dict[int, Dict[str, bytes]] = {}
        self._res_frame = 0
        # host-side side table for rollback components that are not plain bytes (Sprite: particles.rs:191)
        self.host_components = HostComponents(backend)

    # ---- App ----
    def add_plugins(self, plugin) -> "App":
        plugin.build(self)
        return self

    def remove_resource(self, kind) -> "App":
        """`world.remove_resource::<Session<T>>()`: the next update takes the session-less branch."""
        if kind is Session:
            self._session = None
        else:
            raise TypeError(f"unsupported resource {kind!r}")
        return self

    def insert_resource(self, res) -> "App":
        if isinstance(res, Session):
            self._session = res
        elif isinstance(res, RollbackFrameRate):
            self._frame_rate = res
        elif isinstance(res, LocalInputs):
            self._local_inputs = res
        else:
            raise TypeError(f"unsupported resource {type(res).__name__}")
        return self

    def add_systems(self, schedule, system) -> "App":
        if schedule is GgrsSchedule:
            if isinstance(system, ResourceSystem):
                self._res_systems.append(system.fn)
                return self
            assert isinstance(system, System), "GgrsSchedule systems are compiled-in GPU systems or ResourceSystems"
            self.world.add_system(system.system, list(system.columns), list(system.params))
        elif schedule is ReadInputs:
            self._read_inputs.append(system)
        elif schedule is Startup:
            self._startup.append(system)
        else:
            raise TypeError("unknown schedule label")
        return self

    def add_observer(self, event_type, fn) -> "App":
        assert event_type is SyncTestMismatch
        self._observers.append(fn)
        return self

    # ---- RollbackApp (rollback_app.rs:31-248) ----
    def rollback_component_with_copy(self, type_name: str, size_of: int) -> int:
        return self.world.rollback_component(type_name, size_of, capi.BGR_STRATEGY_COPY)

    def rollback_component_with_clone(self, type_name: str, size_of: Optional[int] = None, clone=None):
        """``size_of`` bytes of plain data -> an HBM column (returns its index).  ``size_of=None``: the type is Clone but
        not plain bytes (``Sprite`` holds an ``Arc`` handle, particles.rs:191) -> it stays on the host in the side table
        (host_components.py) and is rolled back there by the same request vectors; returns the ``HostColumn``."""
        if size_of is None:
            return self.host_components.register(type_name, **({"clone": clone} if clone else {}))
        return self.world.rollback_component(type_name, size_of, capi.BGR_STRATEGY_CLONE)

    def rollback_optional_component_with_copy(self, type_name: str, size_of: int) -> int:
        """A component single entities may lose / regain inside the rollback window: the ``Option<&mut S::Target>``
        match of ``ComponentSnapshotPlugin::load`` (component_snapshot.rs:99-115).  ``world.remove_component`` /
        ``world.insert_component`` are the ``commands.entity(e).remove::<T>()`` / ``.insert(t)`` of code outside
        ``GgrsSchedule``."""
        return self.world.rollback_component(type_name, size_of, capi.BGR_STRATEGY_COPY | capi.BGR_STRATEGY_OPTIONAL)

    def checksum_component(self, column: int, byte_offset: int, byte_len: int, assert_finite: bool = False) -> "App":
        self.world.checksum_component(column, byte_offset, byte_len,
                                      capi.BGR_HASH_FLAG_ASSERT_FINITE_F32 if assert_finite else 0)
        return self

    def checksum_component_with_hash(self, column: int) -> "App":
        return self.checksum_component(column, 0, self.world.elem_bytes[column])

    def rollback_resource_with_copy(self, type_name: str, initial: Optional[bytes] = None) -> "App":  # rollback_app.rs:171-176
        """``initial=None`` registers a resource that is absent for now: the snapshot stores ``None`` for it
        (GgrsResourceSnapshots = GgrsSnapshots<R, Option<As>>, mod.rs:87) and a Load re-inserts / removes it."""
        self._res_registered.append(type_name)
        if initial is not None:
            self.resources[type_name] = bytearray(initial)
        return self

    rollback_resource_with_clone = rollback_resource_with_copy

    def checksum_resource_with_hash(self, type_name: str) -> "App":  # rollback_app.rs:213-218
        self._res_checksummed.append(type_name)
        return self

    # ---- desync capture ----
    def desync_report(self, frame: int, max_records: int = 64):
        """Where the re-simulation of ``frame`` diverged from its first simulation: a ``DesyncReport`` of the frame's
        first-recorded snapshot against its re-saved one, or None if the backend no longer holds both.  Meant for a
        ``SyncTestMismatch`` observer (call it with one of ``ev.mismatched_frames``); the backend must have been created
        with ``BGR_CFG_DESYNC_CAPTURE``.  Host-side resources and host component tables are not compared: an empty
        report for a mismatched frame points at them."""
        return self.world.desync_diff(frame, max_records)

    # ---- P2P desync reports ----
    # GgrsEvent::DesyncDetected { frame, .. } arrives after `frame` was confirmed: retain_confirmed (before the first
    # update) keeps the confirmed multiples of the session's desync interval, frame_digest / digest_mismatch find the
    # blocks two peers disagree on, and export_blocks / diff_remote show the rows.  Moving digests and blobs between
    # the peers is the game's job (GGRS carries no application messages).
    def retain_confirmed(self, interval: int, count: int) -> "App":
        self.world.retain_confirmed(interval, count)
        return self

    def retained_frames(self):
        return self.world.retained_frames()

    def frame_digest(self, frame: int):
        """(bgr_frame_digest_header, words[n_blocks, n_columns + 1]) of a queued or retained frame, or None."""
        self._finish()
        return self.world.frame_digest(frame)

    @staticmethod
    def digest_mismatch(local, remote):
        """(blocks whose digests differ, host_state_differs bits); bgr_digest_mismatch interprets the format."""
        from .engine import digest_mismatch
        return digest_mismatch(local, remote)

    def export_blocks(self, frame: int, blocks):
        self._finish()
        return self.world.export_blocks(frame, blocks)

    def diff_remote(self, frame: int, blob: bytes, max_records: int = 64):
        """A ``DesyncReport`` of the local image of ``frame`` ("first") against a peer's exported blocks ("latest"),
        plus the local blocks past the peer's block count, whose rows only this side has."""
        self._finish()
        return self.world.diff_remote(frame, blob, max_records)

    # ---- world checkpoints ----
    # The engine blob (include/bevy_ggrs_b200.h "world checkpoints") followed by the App's rollback resources of the
    # frame: u32 count, then per registered resource in registration order u32 present, u32 len, the bytes, zero
    # padding to a multiple of 4 (INTEGRATION.md "World checkpoints"; bevy_ggrs.hpp writes the same section).
    def _checkpoint_args(self) -> None:
        self._finish()
        if self.host_components.columns:
            raise capi.BgrError(capi.BGR_ERR_UNSUPPORTED, "an App with host-side component tables cannot be checkpointed: "
                                                          "their values are not plain bytes")

    def checkpoint(self, frame: int) -> Optional[bytes]:
        """The checkpoint of a queued or retained frame with the App's resources of that frame; None if the engine
        holds neither.  Refused when the App no longer holds the frame's resource snapshot."""
        self._checkpoint_args()
        self._check_resource_snapshot(frame)
        blob = self.world.checkpoint(frame)
        if blob is None:
            return None
        return blob + self._resource_section(self._res_store.get(frame, {}))

    def checkpoint_delta(self, frame: int, base_frame: int) -> Optional[bytes]:
        """The engine's checkpoint delta of ``frame`` against ``base_frame`` followed by the App's resources of
        ``frame``, in the section ``checkpoint`` writes; None if the engine holds either frame neither queued nor
        retained.  Refused where ``checkpoint(frame)`` is refused."""
        self._checkpoint_args()
        self._check_resource_snapshot(frame)
        delta = self.world.checkpoint_delta(frame, base_frame)
        if delta is None:
            return None
        return delta + self._resource_section(self._res_store.get(frame, {}))

    def _check_resource_snapshot(self, frame: int) -> None:
        if self._res_registered and frame not in self._res_store:
            raise capi.BgrError(capi.BGR_ERR_NO_SNAPSHOT, f"the App holds no resource snapshot of frame {frame}")

    def _resource_section(self, snap: Dict[str, Optional[bytes]]) -> bytes:
        out = [struct.pack("<I", len(self._res_registered))]
        for name in self._res_registered:
            v = snap.get(name)
            out.append(struct.pack("<II", 0 if v is None else 1, 0 if v is None else len(v)))
            if v is not None:
                out.append(bytes(v) + bytes(-len(v) % 4))
        return b"".join(out)

    def _parse_resources(self, blob: bytes, at: int, what: str) -> Dict[str, Optional[bytes]]:
        """The resource section of ``blob`` from byte ``at`` to its end (``what``: "checkpoint" or "checkpoint
        delta"), checked against the App's registration."""
        res: Dict[str, Optional[bytes]] = {}

        def take(n: int) -> bytes:
            nonlocal at
            if at + n > len(blob):
                raise capi.BgrError(capi.BGR_ERR_INVALID_ARGUMENT, f"{what} truncated: its resource section is incomplete")
            at += n
            return blob[at - n:at]
        (count,) = struct.unpack("<I", take(4))
        if count != len(self._res_registered):
            raise capi.BgrError(capi.BGR_ERR_INVALID_ARGUMENT, f"the {what} holds {count} resources, the App registers "
                                                               f"{len(self._res_registered)}")
        for name in self._res_registered:
            present, n = struct.unpack("<II", take(8))
            if present > 1 or (not present and n):
                raise capi.BgrError(capi.BGR_ERR_INVALID_ARGUMENT, f"resource {name}: bad presence or length")
            res[name] = take(n) if present else None
            if any(take(-n % 4)):
                raise capi.BgrError(capi.BGR_ERR_INVALID_ARGUMENT, f"resource {name}: non-zero padding")
        if at != len(blob):
            raise capi.BgrError(capi.BGR_ERR_INVALID_ARGUMENT, f"{what} overlong: bytes follow its resource section")
        return res

    def restore_checkpoint(self, blob: bytes) -> None:
        """Replaces the world and the App's resources with a checkpoint's.  The resource section is checked before the
        engine restores, so a refused blob changes nothing."""
        self._checkpoint_args()
        if len(blob) < capi.C.sizeof(capi.bgr_checkpoint_header):
            raise capi.BgrError(capi.BGR_ERR_INVALID_ARGUMENT, "checkpoint truncated: shorter than its header")
        h = capi.bgr_checkpoint_header.from_buffer_copy(blob)
        at = capi.C.sizeof(h) + 8 * (h.n_blocks + 1) + h.payload_bytes
        res = self._parse_resources(blob, at, "checkpoint")
        self.world.restore(blob[:at])
        self._set_restored_resources(h.frame, res)

    def restore_checkpoint_delta(self, base: bytes, delta: bytes) -> None:
        """Replaces the world and the App's resources with the target frame of ``delta`` (from ``checkpoint_delta``),
        given the App checkpoint ``base`` it was written against.  Both resource sections are checked before the engine
        restores, so a refused pair changes nothing."""
        self._checkpoint_args()
        if len(base) < capi.C.sizeof(capi.bgr_checkpoint_header):
            raise capi.BgrError(capi.BGR_ERR_INVALID_ARGUMENT, "checkpoint truncated: shorter than its header")
        if len(delta) < capi.C.sizeof(capi.bgr_checkpoint_delta_header):
            raise capi.BgrError(capi.BGR_ERR_INVALID_ARGUMENT, "checkpoint delta truncated: shorter than its header")
        bh = capi.bgr_checkpoint_header.from_buffer_copy(base)
        dh = capi.bgr_checkpoint_delta_header.from_buffer_copy(delta)
        b_at = capi.C.sizeof(bh) + 8 * (bh.n_blocks + 1) + bh.payload_bytes
        d_at = capi.C.sizeof(dh) + 8 * (dh.n_blocks + 1) + dh.payload_bytes
        self._parse_resources(base, b_at, "checkpoint")
        res = self._parse_resources(delta, d_at, "checkpoint delta")
        self.world.restore_delta(base[:b_at], delta[:d_at])
        self._set_restored_resources(dh.frame, res)

    def _set_restored_resources(self, frame: int, res: Dict[str, Optional[bytes]]) -> None:
        self.resources = {n: bytearray(v) for n, v in res.items() if v is not None}
        self._res_store = {frame: res} if self._res_registered else {}
        self._res_frame = frame

    # ---- replays (INTEGRATION.md "Replays") ----
    # App.replay(inputs, k) leaves the App as handle_requests of the stream [Save(f) if f % k == 0, Advance(inputs[j])],
    # f = f0 + j, would leave it, except that no snapshot is pushed: the engine re-simulates the world, and the App steps
    # its resources through the same frames on the host and XORs their checksum parts in.  The engine's ring is not
    # touched, so neither is the App's resource store.  Resource systems run at frames the world is not at: they must not
    # read the world.
    def replay(self, inputs, checksum_interval: int = 0) -> List[tuple]:
        """``Engine.replay`` of the App: [(frame, checksum), ...] of the checksum frames, with the resources' parts.  A
        non-finite value at a checksum frame raises BgrError(BGR_ERR_NON_FINITE) after the whole log ran and the
        resources were committed."""
        steps = self._replay_steps(len(inputs), checksum_interval, 0)
        checksums = self._replay_run(steps, lambda: self.world.replay(inputs, checksum_interval))
        return steps.fold(checksums)

    def replay_keyframes(self, inputs, checksum_interval: int, keyframe_interval: int) -> Tuple[List[tuple], List[tuple]]:
        """``Engine.replay_keyframes`` of the App: (checksums, [(frame, blob), ...]), each blob the App checkpoint
        ``checkpoint(frame)`` writes on an App that ticked to the frame and saved it."""
        steps = self._replay_steps(len(inputs), checksum_interval, keyframe_interval)
        checksums, kfs = self._replay_run(steps, lambda: self.world.replay_keyframes(inputs, checksum_interval,
                                                                                        keyframe_interval))
        return steps.fold(checksums), [(f, blob + self._resource_section(steps.snapshots.get(f, {}))) for f, blob in kfs]

    def replay_trace(self, inputs, checksum_interval: int, trace_interval: int, fields, first_row: int, n_rows: int):
        """``Engine.replay_trace`` of the App: (checksums, samples, records).  The records hold engine fields only; the
        checksums include the resources' parts."""
        steps = self._replay_steps(len(inputs), checksum_interval, 0)
        checksums, samples, records = self._replay_run(steps, lambda: self.world.replay_trace(
            inputs, checksum_interval, trace_interval, fields, first_row, n_rows))
        return steps.fold(checksums), samples, records

    def _replay_steps(self, n_frames: int, checksum_interval: int, keyframe_interval: int) -> "_ResourceSteps":
        """The App's half of a replay of ``n_frames``, before the engine runs it.  Checks that the App can replay, then
        steps the resources through the frames on a copy, as the tick's host half does for Saves and Advances: at a
        checksum frame the resource part, at a keyframe frame the resource snapshot, then the resource systems."""
        self._finish()
        if self.host_components.columns:
            raise capi.BgrError(capi.BGR_ERR_UNSUPPORTED, "an App with host-side component tables cannot replay: their rows "
                                                          "follow spawns and despawns a replay does not report frame by frame")
        steps = _ResourceSteps(n_frames, {}, [], {})
        if not self._res_registered:
            return steps
        f0 = self.world.rollback_frame_count()
        if self._res_frame != f0:
            raise capi.BgrError(capi.BGR_ERR_STATE, f"the App's resources are at frame {self._res_frame}, its world at "
                                                    f"frame {f0}")
        res = steps.resources = {n: bytearray(v) for n, v in self.resources.items()}
        for f in range(f0, f0 + n_frames):
            if checksum_interval and f % checksum_interval == 0:
                steps.parts.append(self._resource_part(res))
            if keyframe_interval and f % keyframe_interval == 0:
                steps.snapshots[f] = self._resource_snapshot(res)
            self._run_resource_systems(res, f + 1)
        return steps

    def _replay_run(self, steps: "_ResourceSteps", run: Callable):
        """``run()`` (the engine's replay) and then the commit of ``steps``.  BGR_ERR_NON_FINITE means the log ran: the
        resources are committed before it is raised.  Any other refusal commits nothing."""
        try:
            out = run()
        except capi.BgrError as e:
            if e.status == capi.BGR_ERR_NON_FINITE:
                self._replay_commit(steps)
            raise
        self._replay_commit(steps)
        return out

    def _replay_commit(self, steps: "_ResourceSteps") -> None:
        if self._res_registered:
            self.resources = steps.resources
            self._res_frame += steps.n_frames

    # ---- frame resources ----
    def rollback_frame_count(self) -> int:
        return self.world.rollback_frame_count()

    def confirmed_frame_count(self) -> int:
        return self.world.confirmed_frame_count()

    # ---- one Bevy frame ----
    def _finish(self) -> None:
        if not self._built:
            self.world.build()
            self._built = True
            for s in self._startup:
                s(self)

    def finish(self) -> "App":
        """``App::finish``: builds the engine and runs Startup once (the first update does it otherwise).  An
        ``EngineBatch`` takes built engines."""
        self._finish()
        return self

    def update(self) -> None:
        self._finish()
        # bevy Time<Real>: the first update has zero delta, later ones the manual duration
        delta = 0 if self._first_update else self.MANUAL_DURATION_NS
        self._first_update = False
        self.run_ggrs_schedules(delta)

    def step(self) -> None:
        """Exactly one GGRS tick regardless of the accumulator (benches)."""
        self._finish()
        self._tick()

    # ---- run_ggrs_schedules (schedule_systems.rs:19-83) ----
    def run_ggrs_schedules(self, delta_ns: int) -> None:
        fps = self._frame_rate.fps
        fps_delta = (1_000_000_000 * 11 // (fps * 10)) if self._run_slow else (1_000_000_000 // fps)
        self._accumulator_ns += delta_ns
        while self._accumulator_ns >= fps_delta:
            self._accumulator_ns -= fps_delta
            if self._session is None:
                # "No session has been started yet, reset time data and snapshots" (schedule_systems.rs:70-79)
                self._accumulator_ns = 0
                self._run_slow = False
                self.local_players = LocalPlayers([])
                self.world.reset_session()  # RollbackFrameCount(0), ConfirmedFrameCount(-1), MaxPredictionWindow(8)
                return
            self._tick()

    def _tick(self) -> None:
        requests = self._advance_session()
        if requests is None:
            return
        self.handle_requests(requests)
        self.ticks += 1

    def _advance_session(self) -> Optional[List[Request]]:
        """ReadInputs and the session's advance_frame of one tick: its request vector, or None when the session
        skipped the tick (a SyncTest mismatch has fired the observers)."""
        sess = self._session
        inner = sess.inner
        self.local_players = LocalPlayers(list(range(inner.num_players())))
        # world.run_schedule(ReadInputs) (:89 / :144)
        self._local_inputs = None
        for s in self._read_inputs:
            s(self)
        if self._local_inputs is None:
            raise RuntimeError("No local player inputs found. Did you insert systems into the ReadInputs schedule?")
        for handle, value in self._local_inputs.inputs.items():
            inner.add_local_input(handle, value)
        try:
            return inner.advance_frame()
        except MismatchedChecksum as e:  # :104-115
            ev = SyncTestMismatch(e.current_frame, e.mismatched_frames)
            for obs in self._observers:
                obs(ev)
            return None
        except GgrsError:
            return None

    # ---- handle_requests (schedule_systems.rs:170-289) ----
    def handle_requests(self, requests: Sequence[Request]) -> None:
        inner = self._session.inner
        self._host_requests(requests, self.world.handle_requests(inner.info(), requests))

    def _host_requests(self, requests: Sequence[Request], checksums) -> None:
        """The host half of handle_requests, given the engine's checksums of the vector: resources XORed into the
        checksums, host-side component tables, and the session's cells."""
        inner = self._session.inner
        if self._res_registered:
            checksums = self._handle_resource_requests(requests, checksums)
        if self.host_components.columns:
            self.host_components.handle_requests(requests)
        # cell.save(frame, None, checksum) (:236)
        for frame, cs in checksums:
            inner.save_cell(frame, cs)
        self.last_checksums = checksums

    # host-side half of handle_requests for resources (resource_snapshot.rs:65-93, resource_checksum.rs:63-82):
    # the same request vector, replayed on a few bytes of host state; parts are XORed into the engine's
    # checksum exactly like ChecksumPlugin::update folds every ChecksumPart (checksum.rs:88-99).
    def _handle_resource_requests(self, requests, checksums):
        out, k = [], 0
        for r in requests:
            if r.kind == SAVE:
                self._res_store[self._res_frame] = self._resource_snapshot(self.resources)
                frame, cs = checksums[k]
                out.append((frame, cs ^ self._resource_part(self.resources)))
                k += 1
            elif r.kind == LOAD:  # resource_snapshot.rs:77-93: update / insert / remove
                self._res_frame = r.frame
                for n, v in self._res_store[r.frame].items():
                    if v is None:
                        self.resources.pop(n, None)
                    else:
                        self.resources[n] = bytearray(v)
            else:
                self._res_frame += 1
                self._run_resource_systems(self.resources, self._res_frame)
        alive = set(self.world.snapshot_frames())
        self._res_store = {f: v for f, v in self._res_store.items() if f in alive}
        return out

    def _resource_snapshot(self, resources) -> Dict[str, Optional[bytes]]:  # resource_snapshot.rs:65-73: Some(clone) or None
        return {n: (bytes(resources[n]) if n in resources else None) for n in self._res_registered}

    def _resource_part(self, resources) -> int:  # resource_checksum.rs:63-82 (the resource must exist)
        import ctypes as C
        lib = capi.load_library()
        part = 0
        for name in self._res_checksummed:
            b = bytes(resources[name])
            part ^= lib.bgr_seahash(C.create_string_buffer(b, len(b)), len(b))
        return part

    def _run_resource_systems(self, resources, frame: int) -> None:
        for fn in self._res_systems:
            if fn.__code__.co_argcount >= 2:
                fn(resources, frame)   # (resources, RollbackFrameCount)
            else:
                fn(resources)


@dataclass
class _ResourceSteps:
    """An App's resources stepped through the frames of a replay, on a copy: the resources after the last frame, the
    resource parts of the checksum frames in order, and the resource snapshots of the keyframe frames."""
    n_frames: int
    resources: Dict[str, bytearray]
    parts: List[int]
    snapshots: Dict[int, Dict[str, Optional[bytes]]]

    def fold(self, checksums: List[tuple]) -> List[tuple]:
        """The engine's checksums of the replay with the resource parts XORed in (checksum.rs:88-99)."""
        if not self.parts:
            return checksums
        return [(f, cs ^ p) for (f, cs), p in zip(checksums, self.parts)]


def step_batch(apps: Sequence[App], batch) -> None:
    """Exactly one GGRS tick of every App, like ``App.step()`` on each in turn, with ONE engine call for all of them:
    ``batch`` is an ``EngineBatch`` over the Apps' engines (built: ``App.finish``).  Every App runs ReadInputs and its
    session's advance_frame (an App whose SyncTest mismatches fires its own observers and skips the tick), the batch runs
    the vectors, and each App runs the host half of handle_requests with its checksums.  A world whose call failed after
    executing (BGR_ERR_NON_FINITE) raises once every other App has finished its tick."""
    index = {id(e): i for i, e in enumerate(batch.engines)}
    ticking = []
    for app in apps:
        app._finish()
        requests = app._advance_session()
        if requests is not None:
            ticking.append((app, requests))
    results = batch.handle_requests([(index[id(app.world)], app._session.inner.info(), requests) for app, requests in ticking])
    failed = None
    for (app, requests), (status, checksums) in zip(ticking, results):
        if status != capi.BGR_OK:
            failed = failed or capi.BgrError(status, "Hashing is not stable for NaN f32 values." if status == capi.BGR_ERR_NON_FINITE
                                             else f"bgr_batch_handle_requests status {status}")
            continue
        app._host_requests(requests, checksums)
        app.ticks += 1
    if failed is not None:
        raise failed


# ---- world batches of replays: EngineBatch.replay* over many Apps, each App's resources stepped as App.replay* does ----
def replay_batch(calls, batch) -> List[List[tuple]]:
    """``App.replay`` of every listed App with ONE engine call: ``calls`` = [(app, inputs, checksum_interval), ...] over
    Apps whose built engines are in ``batch`` (an ``EngineBatch``).  Returns each App's checksums in the same order."""
    return [steps.fold(cs) for _, steps, (_, cs) in _replay_batch(calls, batch, batch.replay, 0)]


def replay_keyframes_batch(calls, batch) -> List[Tuple[List[tuple], List[tuple]]]:
    """``App.replay_keyframes`` of every listed App with ONE engine call: ``calls`` = [(app, inputs, checksum_interval,
    keyframe_interval), ...].  Returns each App's (checksums, [(frame, App checkpoint), ...]) in the same order."""
    return [(steps.fold(cs), [(f, blob + app._resource_section(steps.snapshots.get(f, {}))) for f, blob in kfs])
            for app, steps, (_, cs, kfs) in _replay_batch(calls, batch, batch.replay_keyframes, 3)]


def replay_trace_batch(calls, batch, fields):
    """``App.replay_trace`` of every listed App over one field list with ONE engine call: ``calls`` = [(app, inputs,
    checksum_interval, trace_interval, first_row, n_rows), ...].  Returns each App's (checksums, samples, records) in the
    same order."""
    return [(steps.fold(cs), samples, records)
            for _, steps, (_, cs, samples, records) in _replay_batch(calls, batch, lambda c: batch.replay_trace(c, fields), 0)]


def _replay_batch(calls, batch, run: Callable, keyframe_at: int):
    """Steps the resources of every App in ``calls`` (entries (app, inputs, checksum_interval, ...); the keyframe interval
    at index ``keyframe_at``, 0: none) on copies, runs ``run`` (the EngineBatch call, on the same entries with each App
    replaced by its world's index) and commits every App whose world ran.  A refused call commits nothing.  A world that
    reported BGR_ERR_NON_FINITE raises once every App has committed.  Returns [(app, steps, the world's result), ...]."""
    calls = [tuple(c) for c in calls]
    index = {id(e): i for i, e in enumerate(batch.engines)}
    worlds = []
    for c in calls:
        if id(c[0].world) not in index:
            raise capi.BgrError(capi.BGR_ERR_INVALID_ARGUMENT, "an App's engine is not a member of the batch")
        worlds.append(index[id(c[0].world)])
    steps = [c[0]._replay_steps(len(c[1]), c[2], c[keyframe_at] if keyframe_at else 0) for c in calls]
    results = run([(w,) + c[1:] for w, c in zip(worlds, calls)])
    failed = None
    for w, c, st, res in zip(worlds, calls, steps, results):
        if res[0] in (capi.BGR_OK, capi.BGR_ERR_NON_FINITE):
            c[0]._replay_commit(st)
        if res[0] != capi.BGR_OK:
            failed = failed or capi.BgrError(res[0], f"world {w}: " + ("Hashing is not stable for NaN f32 values."
                                                                       if res[0] == capi.BGR_ERR_NON_FINITE else f"status {res[0]}"))
    if failed is not None:
        raise failed
    return [(c[0], st, res) for c, st, res in zip(calls, steps, results)]
