"""Stand-ins for the ggrs sessions that feed ``handle_requests``.

ggrs (the netcode crate: input queues, prediction, UDP) is third-party and OUT OF SCOPE
(SURVEY.md §2 row 17).  The hot path only consumes the *request vector* a session returns
from ``advance_frame()`` (reference src/schedule_systems.rs:98,156), so this module restates
exactly that: the order of Save / Load / Advance requests and, for SyncTest, the checksum
comparison that raises ``MismatchedChecksum`` (-> ``SyncTestMismatch``, lib.rs:131-137,
schedule_systems.rs:104-115).

Restated from ggrs 0.11 ``SyncTestSession::advance_frame`` / ``adjust_gamestate`` and
``P2PSession::adjust_gamestate`` (non-sparse saving); see SURVEY.md §3.6:

    SyncTest tick, frame f > d:  [Load(f-d), Adv, Save(f-d+1), Adv, ..., Save(f-1), Adv, Save(f), Adv]
    P2P tick, no misprediction:  [Save(f), Adv]
    P2P tick, rollback of L:     [Load(f-L), Adv, Save(f-L+1), Adv, ..., Save(f), Adv]

This is pure host logic (no GPU, no oracle); it drives the engine, the oracle and the
reference arm with the same request stream.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

SAVE, LOAD, ADVANCE = 0, 1, 2
SESSION_NONE, SESSION_SYNCTEST, SESSION_P2P, SESSION_SPECTATOR = 0, 1, 2, 3
INPUT_CONFIRMED, INPUT_PREDICTED, INPUT_DISCONNECTED = 0, 1, 2
NULL_FRAME = -1


@dataclass
class Request:
    """``GgrsRequest<T>`` with ``T::Input = u8``."""

    kind: int
    frame: int = 0
    inputs: Sequence[int] = ()
    status: Sequence[int] = ()

    def __repr__(self) -> str:  # compact, for assertion messages
        name = {SAVE: "Save", LOAD: "Load", ADVANCE: "Adv"}[self.kind]
        return f"{name}({self.frame})" if self.kind != ADVANCE else f"Adv{list(self.inputs)}"


class GgrsError(Exception):
    pass


class MismatchedChecksum(GgrsError):
    """``GgrsError::MismatchedChecksum { current_frame, mismatched_frames }``."""

    def __init__(self, current_frame: int, mismatched_frames: List[int]):
        super().__init__(f"Detected checksum mismatch during rollback on frame {current_frame}, "
                         f"mismatched frames: {mismatched_frames}")
        self.current_frame = current_frame
        self.mismatched_frames = mismatched_frames


class InvalidRequest(GgrsError):
    pass


class _InputQueues:
    """Per-player confirmed inputs keyed by frame, with ggrs' frame-delay behaviour:
    an input added at frame f lands at f+delay, frames before the first delayed input hold
    the blank input (``Input::default()``)."""

    def __init__(self, num_players: int, delay: int):
        self.delay = delay
        self.frames: List[Dict[int, int]] = [dict() for _ in range(num_players)]

    def add(self, handle: int, frame: int, value: int) -> None:
        self.frames[handle][frame + self.delay] = value & 0xFF

    def get(self, frame: int) -> List[int]:
        return [q.get(frame, 0) for q in self.frames]


class SyncTestSession:
    """``ggrs::SyncTestSession``: every tick rolls back ``check_distance`` frames, resimulates
    and compares the re-saved checksums with the first ones recorded for those frames."""

    def __init__(self, num_players: int = 1, check_distance: int = 2, max_prediction: int = 8,
                 input_delay: int = 0):
        if num_players < 1 or num_players > 8:
            raise InvalidRequest("num_players")
        if check_distance >= max_prediction:
            # SessionBuilder::start_synctest_session
            raise InvalidRequest("Check distance too big.")
        self._num_players = num_players
        self._check_distance = check_distance
        self._max_prediction = max_prediction
        self.current_frame = 0
        self._inputs = _InputQueues(num_players, input_delay)
        self._local: Dict[int, int] = {}
        self._checksum_history: Dict[int, Optional[int]] = {}
        # sync_layer.saved_states: max_prediction+1 cells addressed by frame % len
        self._cells: List[Optional[tuple]] = [None] * (max_prediction + 1)

    # -- what bevy_ggrs reads (schedule_systems.rs:86,199,207) --
    def num_players(self) -> int:
        return self._num_players

    def max_prediction(self) -> int:
        return self._max_prediction

    def check_distance(self) -> int:
        return self._check_distance

    def info(self) -> tuple:
        """(kind, max_prediction, check_distance, confirmed_frame) for ``bgr_session_info``."""
        return (SESSION_SYNCTEST, self._max_prediction, self._check_distance, 0)

    def add_local_input(self, handle: int, value: int) -> None:
        if not 0 <= handle < self._num_players:
            raise InvalidRequest("The player handle you provided is not valid.")
        self._local[handle] = value

    # -- GameStateCell::save(frame, None, checksum) (schedule_systems.rs:236) --
    def save_cell(self, frame: int, checksum: Optional[int]) -> None:
        self._cells[frame % len(self._cells)] = (frame, checksum)

    def _saved_state_by_frame(self, frame: int):
        cell = self._cells[frame % len(self._cells)]
        return cell if cell is not None and cell[0] == frame else None

    def _checksums_consistent(self, frame_to_check: int) -> bool:
        oldest_allowed = self.current_frame - self._check_distance
        self._checksum_history = {k: v for k, v in self._checksum_history.items() if k >= oldest_allowed}
        cell = self._saved_state_by_frame(frame_to_check)
        if cell is None:
            return True
        frame, cs = cell
        if frame in self._checksum_history:
            return self._checksum_history[frame] == cs
        self._checksum_history[frame] = cs
        return True

    def _advance_request(self) -> Request:
        ins = self._inputs.get(self.current_frame)
        return Request(ADVANCE, 0, ins, [INPUT_CONFIRMED] * self._num_players)

    def advance_frame(self) -> List[Request]:
        requests: List[Request] = []
        d = self._check_distance
        cur = self.current_frame
        if d > 0 and cur > d:
            mismatched = [f for f in range(cur - d, cur + 1) if not self._checksums_consistent(f)]
            if mismatched:
                raise MismatchedChecksum(cur, mismatched)
            # adjust_gamestate(frame_to)
            frame_to = cur - d
            requests.append(Request(LOAD, frame_to))
            self.current_frame = frame_to
            for i in range(d):
                if i > 0:
                    requests.append(Request(SAVE, self.current_frame))
                requests.append(self._advance_request())
                self.current_frame += 1
            assert self.current_frame == cur
        if len(self._local) != self._num_players:
            raise InvalidRequest("Missing local input while calling advance_frame().")
        for handle, value in self._local.items():
            self._inputs.add(handle, self.current_frame, value)
        self._local = {}
        if d > 0:
            requests.append(Request(SAVE, self.current_frame))
        requests.append(self._advance_request())
        self.current_frame += 1
        return requests


def _splitmix64(state: int):
    mask = (1 << 64) - 1
    state = (state + 0x9E3779B97F4A7C15) & mask
    z = state
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & mask
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & mask
    return state, z ^ (z >> 31)


class Xoshiro256pp:
    """xoshiro256++ seeded through splitmix64 — the generator BASELINE.md names for all
    synthetic inputs and traces."""

    MASK = (1 << 64) - 1

    def __init__(self, seed: int):
        s = seed & self.MASK
        self.s = []
        for _ in range(4):
            s, out = _splitmix64(s)
            self.s.append(out)

    @staticmethod
    def _rotl(x: int, k: int) -> int:
        return ((x << k) | (x >> (64 - k))) & Xoshiro256pp.MASK

    def next_u64(self) -> int:
        s = self.s
        result = (self._rotl((s[0] + s[3]) & self.MASK, 23) + s[0]) & self.MASK
        t = (s[1] << 17) & self.MASK
        s[2] ^= s[0]
        s[3] ^= s[1]
        s[1] ^= s[2]
        s[0] ^= s[3]
        s[2] ^= t
        s[3] = self._rotl(s[3], 45)
        return result

    def next_f64(self) -> float:
        return (self.next_u64() >> 11) * (1.0 / (1 << 53))


class P2PTraceSession:
    """Synthetic 2-peer P2P request trace (BASELINE.md config C4): no sockets, the rollback
    depth of every tick is drawn from a seeded generator — P(no rollback) = ``p_clean``,
    otherwise uniform in 1..=max_prediction (clamped to the frames that exist)."""

    def __init__(self, num_players: int = 2, max_prediction: int = 8, input_delay: int = 2,
                 seed: int = 0xB200, p_clean: float = 0.5, desync_interval: Optional[int] = None):
        self._num_players = num_players
        # DesyncDetection::On { interval }: the checksums of confirmed frames 0, interval, 2*interval, ... go to the peer
        self._desync_interval = desync_interval
        self._checksums: Dict[int, Optional[int]] = {}
        self._reported: set = set()
        self._max_prediction = max_prediction
        self.current_frame = 0
        self._rng = Xoshiro256pp(seed)
        self._p_clean = p_clean
        self._inputs = _InputQueues(num_players, input_delay)
        self._local: Dict[int, int] = {}
        self.last_rollback_depth = 0

    def num_players(self) -> int:
        return self._num_players

    def max_prediction(self) -> int:
        return self._max_prediction

    def confirmed_frame(self) -> int:
        return self.current_frame - self._max_prediction

    def info(self) -> tuple:
        return (SESSION_P2P, self._max_prediction, 0, self.confirmed_frame())

    def add_local_input(self, handle: int, value: int) -> None:
        self._local[handle] = value

    def save_cell(self, frame: int, checksum: Optional[int]) -> None:
        if self._desync_interval and frame >= 0 and frame % self._desync_interval == 0:
            self._checksums[frame] = checksum  # a re-save after a rollback replaces the prediction's checksum

    def checksum_reports(self) -> List[tuple]:
        """The (frame, checksum) pairs GGRS would send to the peer now (desync_interval set): each multiple of the
        interval once it is confirmed, with its latest checksum."""
        out = [(f, c) for f, c in sorted(self._checksums.items())
               if f not in self._reported and f <= self.confirmed_frame()]
        self._reported.update(f for f, _ in out)
        return out

    def _advance_request(self, predicted: bool) -> Request:
        ins = self._inputs.get(self.current_frame)
        st = [INPUT_CONFIRMED] + [INPUT_PREDICTED if predicted else INPUT_CONFIRMED] * (self._num_players - 1)
        return Request(ADVANCE, 0, ins, st)

    def advance_frame(self) -> List[Request]:
        cur = self.current_frame
        depth = 0
        if self._rng.next_f64() >= self._p_clean:
            depth = 1 + int(self._rng.next_u64() % self._max_prediction)
        depth = min(depth, cur)
        self.last_rollback_depth = depth
        requests: List[Request] = []
        if depth > 0:
            self.current_frame = cur - depth
            requests.append(Request(LOAD, self.current_frame))
            for i in range(depth):
                if i > 0:
                    requests.append(Request(SAVE, self.current_frame))
                requests.append(self._advance_request(False))
                self.current_frame += 1
        for handle, value in self._local.items():
            self._inputs.add(handle, self.current_frame, value)
        self._local = {}
        requests.append(Request(SAVE, self.current_frame))
        requests.append(self._advance_request(True))
        self.current_frame += 1
        return requests


def count_advances(requests: Sequence[Request]) -> int:
    return sum(1 for r in requests if r.kind == ADVANCE)
