"""Uniform experience replay on the HBM ring.  Drop-in for
``rl_coach/memories/non_episodic/experience_replay.py:41-276`` (same constructor, methods, errors), with the fast
path ``sample_batch`` returning a :class:`~coach_b200.core_types.DeviceBatch`.

Sampling draws from numpy's *legacy global* RandomState exactly as the reference does
(``np.random.randint(num_transitions, size)``, experience_replay.py:81) so that a seeded run consumes the same random
stream and picks the same transitions; the drawn list positions are mapped to ring slots on the host (4 KB) and the
row gather runs on the GPU.
"""
import pickle
import random
from typing import List, Tuple, Union

import numpy as np
import torch

from coach_b200 import _lib
from coach_b200.core_types import DeviceBatch, Transition
from coach_b200.memories.device_ring import DeviceTransitionRing
from coach_b200.memories.memory import Memory, MemoryGranularity, MemoryParameters


class ExperienceReplayParameters(MemoryParameters):
    def __init__(self):
        super().__init__()
        self.max_size = (MemoryGranularity.Transitions, 1000000)
        self.allow_duplicates_in_batch_sampling = True
        # coach_b200 only: store every frame of stacked image observations once (device_ring, SURVEY.md 8(f1)); the
        # frame store holds (1 + frame_slack) x max_size frames
        self.frame_dedup = False
        self.frame_slack = 0.25
        self.frame_streams = 1          # environments whose transitions are store()d in turn (sizes the frame cache)

    @property
    def path(self):
        return 'coach_b200.memories.experience_replay:ExperienceReplay'


class ExperienceReplay(Memory):
    """A regular replay buffer which stores transitions without any additional structure (HBM resident)."""

    def __init__(self, max_size: Tuple[MemoryGranularity, int], allow_duplicates_in_batch_sampling: bool = True,
                 device=None, frame_dedup: bool = False, frame_slack: float = 0.25, frame_streams: int = 1):
        super().__init__(max_size)
        self.frame_dedup, self.frame_slack, self.frame_streams = bool(frame_dedup), float(frame_slack), int(frame_streams)
        if max_size[0] != MemoryGranularity.Transitions:
            raise ValueError("Experience replay size can only be configured in terms of transitions")
        self.allow_duplicates_in_batch_sampling = allow_duplicates_in_batch_sampling
        self.frozen = False
        self.lib = _lib.load()                    # no CUDA library, no replay: fail here, loudly
        self.device = torch.device(device if device is not None else "cuda")
        self.ring = DeviceTransitionRing(self._ring_capacity(), self.device)

    def _ring_capacity(self):
        size = self.max_size[1]
        if size == 0:
            raise ValueError("an unbounded replay (max_size 0) cannot be HBM resident; give a capacity")
        return size

    # ---- bookkeeping ---------------------------------------------------------------------------------------------
    def length(self) -> int:
        return self.num_transitions()

    def num_transitions(self) -> int:
        return min(self.ring.count + self.ring._pending, self.ring.capacity)

    def assert_not_frozen(self):
        assert self.frozen is False, "Memory is frozen, and cannot be changed."

    def freeze(self):
        self.frozen = True

    # ---- store ---------------------------------------------------------------------------------------------------
    def store(self, transition: Transition, lock: bool = True) -> None:
        """experience_replay.py:131-150.  The oldest transition is overwritten once the ring is full, which is what
        ``_enforce_max_length`` (:117-129, ``del transitions[0]``) amounts to."""
        self.assert_not_frozen()
        Memory.store(self, transition)
        if self.ring.stage_transition(transition):
            self._flush()
        # num_transitions() counts pending rows; cap like the reference's list would be capped
        if self.ring.count + self.ring._pending > self.ring.capacity:
            self._flush()

    def declare_schema(self, columns: dict, image_columns=()) -> None:
        """Column layout of the ring ({name: (shape, dtype)} or the agent's batch buffers), fixed before the first store
        so that ``store(Transition)`` casts to it (device_ring.DeviceTransitionRing.declare_schema).  ``image_columns``:
        the stacked-frame columns, kept frame-deduplicated when the memory was created with ``frame_dedup``."""
        if self.frame_dedup and image_columns:
            self.ring.declare_schema(columns, frame_stack=tuple(image_columns), frame_slack=self.frame_slack,
                                     frame_streams=self.frame_streams)
        else:
            self.ring.declare_schema(columns)

    def store_columns(self, columns: dict) -> None:
        """Batched ingest: {column name: array/tensor [n, ...]} with the ring's column names (see device_ring)."""
        self.assert_not_frozen()
        self._flush()
        self.ring.append_columns(columns)

    def _flush(self):
        return self.ring.flush()

    # ---- sample --------------------------------------------------------------------------------------------------
    def _draw_positions(self, size: int) -> np.ndarray:
        n = self.num_transitions()
        if self.allow_duplicates_in_batch_sampling:
            return np.random.randint(n, size=size)                      # :81
        if n >= size:
            return np.random.choice(n, size=size, replace=False)        # :85
        raise ValueError("The replay buffer cannot be sampled since there are not enough transitions yet. "
                         "There are currently {} transitions".format(n))

    def _positions_to_slots(self, pos: np.ndarray) -> np.ndarray:
        # list position p (0 = oldest) lives in slot (cursor - count + p) mod capacity
        r = self.ring
        return (r.cursor - r.count + pos) % r.capacity

    def sample_batch(self, size: int, out: dict = None, s2d: dict = None) -> DeviceBatch:
        """Fast path: one H2D copy of the drawn slots + one gather launch; returns device-resident columns.
        ``s2d``: image columns as space-to-depth operand planes (see PrioritizedExperienceReplay.sample_batch)."""
        pos = self._draw_positions(size)
        self._flush()
        return self._gather_slots(self._positions_to_slots(pos), size, out, s2d)

    def _gather_slots(self, slots: np.ndarray, size: int, out: dict = None, s2d: dict = None) -> DeviceBatch:
        """the rows of the given ring slots as a DeviceBatch: into ``out`` (persistent buffers) or fresh tensors, the
        image columns optionally as space-to-depth operand planes (``s2d``)"""
        slots = torch.from_numpy(np.asarray(slots).astype(np.int64))
        idx = slots.pin_memory().to(self.device, non_blocking=True) if self.device.type == "cuda" else slots
        if s2d is not None:
            from coach_b200.memories.prioritized_experience_replay import _LazyColumns
            ia, ni, sa, ns = self.ring.s2d_tables(s2d, out, size)
            H, W, C, S = s2d["geometry"]
            _lib.check(self.lib.cb200_gather_s2d(idx.data_ptr(), size, ia, ni, H, W, C, S, sa, ns,
                                                 self.ring.frames_ptr(), self.ring.frame_capacity, _lib.current_stream()))
            cols = {k: v for k, v in out.items() if k not in s2d["columns"]}
            cols["idx"] = idx
            return DeviceBatch(cols, size, lazy=_LazyColumns(self.ring, idx, tuple(s2d["columns"])))
        cols = self.ring.gather(idx, out)
        cols = dict(cols)
        cols["idx"] = idx
        return DeviceBatch(cols, size)

    def sample(self, size: int) -> List[Transition]:
        """API-compatible slow path (experience_replay.py:71-93): materialises Transitions on the host."""
        return self.sample_batch(size).to_transitions()

    def get_shuffled_training_data_generator(self, size: int):
        """experience_replay.py:95-115 -- epochs over the whole buffer in shuffled order (Python ``random.shuffle``,
        same stream as the reference); yields DeviceBatch objects; the tail that does not fill a batch is dropped."""
        self._flush()
        order = list(range(self.num_transitions()))
        random.shuffle(order)
        for i in range(int(len(order) / size)):
            pos = np.array(order[i * size:(i + 1) * size], dtype=np.int64)
            idx = torch.from_numpy(self._positions_to_slots(pos)).to(self.device)
            cols = dict(self.ring.gather(idx))
            cols["idx"] = idx
            yield DeviceBatch(cols, size)

    # ---- single-transition access (host materialisation; compatibility only) -------------------------------------
    def get_transition(self, transition_index: int, lock: bool = True) -> Union[None, Transition]:
        if self.length() == 0 or transition_index >= self.length():
            return None
        self._flush()
        idx = torch.tensor(self._positions_to_slots(np.array([transition_index])), dtype=torch.int64,
                           device=self.device)
        return DeviceBatch(dict(self.ring.gather(idx)), 1).to_transitions()[0]

    def get(self, transition_index: int, lock: bool = True) -> Union[None, Transition]:
        return self.get_transition(transition_index, lock)

    def remove_transition(self, transition_index: int, lock: bool = True) -> None:
        """Only removal of the oldest transition is expressible on a ring (that is the only use in the reference,
        experience_replay.py:127)."""
        self.assert_not_frozen()
        self._flush()
        if transition_index != 0:
            raise NotImplementedError("the HBM ring can only drop its oldest transition")
        if self.ring.count > 0:
            self.ring.count -= 1

    def clean(self, lock: bool = True) -> None:
        self.assert_not_frozen()
        self.ring.clear()

    def mean_reward(self):
        self._flush()
        r = self.ring
        if r.count == 0:
            return np.float64("nan")
        col = r.columns["reward"].view(torch.float64).reshape(-1)
        slots = torch.from_numpy(self._positions_to_slots(np.arange(r.count))).to(self.device)
        return col[slots].mean().item()

    def save(self, file_path: str) -> None:
        self._flush()
        n = self.num_transitions()
        idx = torch.from_numpy(self._positions_to_slots(np.arange(n))).to(self.device)
        with open(file_path, 'wb') as f:
            pickle.dump(DeviceBatch(dict(self.ring.gather(idx)), n).to_transitions(), f)

    def load_pickled(self, file_path: str) -> None:
        self.assert_not_frozen()
        with open(file_path, 'rb') as f:
            for t in pickle.load(f):
                self.store(t)
