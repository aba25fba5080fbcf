"""Episode-structured replay on the HBM ring.  Drop-in for the parts of
``rl_coach/memories/episodic/episodic_experience_replay.py:60-300`` that the replay -> learn path uses
(store / store_episode / sample / ``transitions`` / clean / counters), the default memory of ClippedPPO, DDPG, TD3
(SURVEY.md M7).  Out of scope, as in SURVEY.md: CSV / off-policy-evaluation loaders, goal relabelling.

Transitions are appended to the device ring as they arrive; episode boundaries live on the host (a list of episode
lengths).  When an episode closes, its n-step discounted returns are computed on the GPU
(``Episode.update_transitions_rewards_and_bootstrap_data``, core_types.py:803-820 -> cb200_nstep_returns) into the
``n_step_discounted_rewards`` column.  ``transitions_batch()`` hands the whole content (complete episodes first, in
arrival order) to the agent as a DeviceBatch -- the device-side counterpart of ``self.memory.transitions``
(clipped_ppo_agent.py:319).
"""
from typing import List, Tuple

import numpy as np
import torch

from coach_b200 import _lib, rl_math
from coach_b200.core_types import DeviceBatch, Transition
from coach_b200.memories.experience_replay import ExperienceReplay
from coach_b200.memories.memory import MemoryGranularity, MemoryParameters


class EpisodicExperienceReplayParameters(MemoryParameters):
    def __init__(self):
        super().__init__()
        self.max_size = (MemoryGranularity.Transitions, 1000000)
        self.n_step = -1
        self.train_to_eval_ratio = 1
        # coach_b200 only: the ring's size in transitions when max_size counts episodes
        self.transition_capacity = None

    @property
    def path(self):
        return 'coach_b200.memories.episodic_experience_replay:EpisodicExperienceReplay'


class EpisodicExperienceReplay(ExperienceReplay):
    """``max_size`` in transitions sizes the ring; in episodes (``MemoryGranularity.Episodes``) it caps the number of
    listed episodes and ``transition_capacity`` sizes the ring, which must then hold every listed episode: a store that
    would overwrite a slot of one raises ``ValueError``."""

    def __init__(self, max_size: Tuple[MemoryGranularity, int] = (MemoryGranularity.Transitions, 1000000),
                 n_step=-1, train_to_eval_ratio: int = 1, discount: float = 0.99, device=None,
                 transition_capacity: int = None):
        if max_size[0] == MemoryGranularity.Episodes:
            if transition_capacity is None:
                raise ValueError("an episode-sized replay needs transition_capacity: the ring is sized in transitions")
            if max_size[1] < 1:
                raise ValueError("an episode-sized replay holds at least one episode")
            ExperienceReplay.__init__(self, (MemoryGranularity.Transitions, int(transition_capacity)), True,
                                      device=device)
            self.max_size = max_size
        elif max_size[0] == MemoryGranularity.Transitions:
            ExperienceReplay.__init__(self, max_size, True, device=device)
        else:
            raise ValueError("max_size is counted in transitions or episodes")
        self.n_step = n_step
        self.discount = discount
        self.episode_lengths = []          # complete episodes, oldest first
        self._open_len = 0                 # transitions of the episode currently being filled
        self._returns = None               # fp64 [capacity] n-step discounted returns (valid for complete episodes)
        self._bootstrap = None             # uint8 [capacity] info['should_bootstrap_next_state'] (n_step > 1 only)

    # ---- counters (episodic_experience_replay.py:75-100) -----------------------------------------------------------
    def length(self, lock: bool = False) -> int:
        """number of episodes, counting the open one like the reference's buffer list -- except that an episode-sized
        replay counts it only when it is non-empty, as the reference's length() does (:77-85)"""
        if self.max_size[0] == MemoryGranularity.Episodes:
            return len(self.episode_lengths) + (1 if self._open_len > 0 else 0)
        return len(self.episode_lengths) + 1

    def num_complete_episodes(self):
        return len(self.episode_lengths)

    def num_transitions_in_complete_episodes(self):
        return int(sum(self.episode_lengths))

    # ---- store -------------------------------------------------------------------------------------------------------
    def num_transitions(self) -> int:
        return self.num_transitions_in_complete_episodes() + self._open_len

    def _evict(self):
        """_enforce_max_length (:215-228, Transitions granularity): whole oldest episodes go while the buffer holds
        more transitions than max_size -- checked at every store, like the reference, so the ring (capacity =
        max_size slots) never overwrites a slot of an episode that is still listed.  Episodes granularity: whole oldest
        episodes go while length() exceeds max_size; listed episodes that outgrow the ring raise."""
        if self.max_size[0] == MemoryGranularity.Episodes:
            while self.episode_lengths and self.length() > self.max_size[1]:
                self.episode_lengths.pop(0)
            if sum(self.episode_lengths) + self._open_len > self.ring.capacity:
                raise ValueError("the listed episodes need more than the ring's %d transitions (transition_capacity)"
                                 % self.ring.capacity)
            return
        while self.episode_lengths and sum(self.episode_lengths) + self._open_len > self.ring.capacity:
            self.episode_lengths.pop(0)
        if self._open_len > self.ring.capacity:
            raise ValueError("an episode longer than the replay (%d transitions) cannot be held" % self.ring.capacity)

    def store(self, transition: Transition, lock: bool = True) -> None:
        ExperienceReplay.store(self, transition)
        self._open_len += 1
        self._evict()
        if transition.game_over:
            self._close_episode()

    def store_episode(self, episode, lock: bool = True) -> None:
        """episodic_experience_replay.py:294-318: a whole episode (any object with ``.transitions``) is appended and
        closed -- whether or not its last transition carries game_over.  The reference lets this happen while another
        episode is being filled (that one then stays in the buffer, never closed); the ring cannot interleave two
        episodes, so that case raises."""
        self.assert_not_frozen()
        if self._open_len != 0:
            raise NotImplementedError("store_episode while an episode is being filled transition by transition")
        for t in episode.transitions:
            ExperienceReplay.store(self, t)
            self._open_len += 1
            self._evict()
        self._close_episode()

    def store_columns(self, columns: dict, episode_lengths: List[int] = None) -> None:
        """Batched ingest of whole episodes laid out back to back; ``episode_lengths`` defaults to the split implied
        by the game_over column (read back once: 1 byte per transition)."""
        self._flush()
        first, n = self.ring.append_columns(columns)
        if episode_lengths is None:
            done = torch.as_tensor(columns["game_over"]).cpu().numpy().astype(bool)
            ends = np.nonzero(done)[0]
            episode_lengths, prev = [], -1
            for e in ends:
                episode_lengths.append(int(e - prev))
                prev = e
            tail = n - 1 - prev
        else:
            tail = n - int(sum(episode_lengths))
        for L in episode_lengths:
            self._open_len += L
            self._close_episode()
        self._open_len += tail

    def _close_episode(self):
        """Episode.update_transitions_rewards_and_bootstrap_data (core_types.py:803-820) for the episode that just
        ended: n-step discounted returns on the GPU."""
        self._flush()
        L = self._open_len
        self._open_len = 0
        if L == 0:
            return
        if not isinstance(self.n_step, int) or (self.n_step < 1 and self.n_step != -1):
            raise ValueError("n-step should be an integer with value >= 1, or set to -1 for always setting to episode"
                             " length.")
        self.episode_lengths.append(L)
        r = self.ring
        if self._returns is None:
            self._returns = torch.zeros(r.capacity, dtype=torch.float64, device=self.device)
        start = (r.cursor - L) % r.capacity
        if start + L <= r.capacity:                   # not wrapped: compute in place
            rew = r.columns["reward"].view(torch.float64).reshape(-1)[start:start + L]
            self._returns[start:start + L] = rl_math.nstep_returns(rew.contiguous(), [L], self.discount, self.n_step)
        else:
            idx = (torch.arange(L, device=self.device) + start) % r.capacity
            rew = r.columns["reward"].view(torch.float64).reshape(-1)[idx]
            self._returns[idx] = rl_math.nstep_returns(rew.contiguous(), [L], self.discount, self.n_step)
        if self.n_step > 1:
            self._relink(start, L)
        self._evict()

    def _relink(self, start, L):
        """core_types.py:807-818 (n_step > 1): next_state of transition i becomes the state of transition i + n -- or,
        past the end of the episode, the episode's last next_state -- and info['should_bootstrap_next_state'] says
        which.  Row moves inside the HBM columns; the source rows are read before anything is written."""
        r = self.ring
        n = self.n_step if self.n_step < L else L
        slots = (torch.arange(L, device=self.device) + start) % r.capacity
        j = torch.arange(L, device=self.device) + n
        inside = j < L
        if self._bootstrap is None:
            self._bootstrap = torch.zeros(r.capacity, dtype=torch.uint8, device=self.device)
        self._bootstrap[slots] = inside.to(torch.uint8)
        src = slots[torch.clamp(j, max=L - 1)]
        for name in r.specs:
            if not name.startswith("next_state:"):
                continue
            ns_col, s_col = r.columns[name], r.columns["state:" + name[len("next_state:"):]]
            last = ns_col[slots[L - 1]].clone()
            new = torch.where(inside[:, None], s_col[src], last[None, :])
            ns_col[slots] = new

    def verify_last_episode_is_closed(self) -> None:
        pass

    # ---- read --------------------------------------------------------------------------------------------------------
    def _slots_of_complete_episodes(self, pos=None):
        """ring slots of list positions ``pos`` (default: all) of the complete episodes, oldest first"""
        r = self.ring
        n = self.num_transitions_in_complete_episodes()
        start = (r.cursor - self._open_len - n) % r.capacity
        pos = np.arange(n, dtype=np.int64) if pos is None else np.asarray(pos, dtype=np.int64)
        return (pos + start) % r.capacity

    def transitions_batch(self) -> DeviceBatch:
        """All transitions of the complete episodes, in order (``memory.transitions`` of the reference restricted to
        what ClippedPPO trains on: the agent only trains once the episode is complete, agent.py:681-699)."""
        self._flush()
        if self.num_transitions_in_complete_episodes() < 1:
            raise ValueError("The episodic replay buffer holds no complete episode yet. "
                             "There is currently 1 episodes with {} transitions".format(self._open_len))
        slots = self._slots_of_complete_episodes()
        idx = torch.from_numpy(slots).to(self.device)
        cols = dict(self.ring.gather(idx))
        cols["n_step_discounted_rewards"] = self._returns[idx] if self._returns is not None else None
        if self._bootstrap is not None and self.n_step > 1:
            cols["should_bootstrap_next_state"] = self._bootstrap[idx]
        cols["idx"] = idx
        return DeviceBatch(cols, len(slots))

    @property
    def transitions(self):
        return self.transitions_batch().to_transitions()

    def get_episode(self, episode_index: int, lock: bool = True):
        """episodic_experience_replay.py:320-336: the episode at the given index (complete episodes, oldest first) as an
        object with ``.transitions`` (host materialisation), or None"""
        from types import SimpleNamespace
        if episode_index < 0:
            episode_index += len(self.episode_lengths)
        if not 0 <= episode_index < len(self.episode_lengths):
            return None
        self._flush()
        lo = int(sum(self.episode_lengths[:episode_index]))
        pos = np.arange(lo, lo + self.episode_lengths[episode_index], dtype=np.int64)
        idx = torch.from_numpy(self._slots_of_complete_episodes(pos)).to(self.device)
        cols = dict(self.ring.gather(idx))
        if self._returns is not None:
            cols["n_step_discounted_rewards"] = self._returns[idx]
        ts = DeviceBatch(cols, len(pos)).to_transitions()
        if self._returns is not None:
            for t, r in zip(ts, cols["n_step_discounted_rewards"].cpu().numpy()):
                t.n_step_discounted_rewards = float(r)
        return SimpleNamespace(transitions=ts, length=lambda: len(ts))

    def get(self, episode_index: int, lock: bool = True):
        return self.get_episode(episode_index, lock)

    def sample_batch(self, size: int, out: dict = None, s2d: dict = None) -> DeviceBatch:
        """episodic_experience_replay.py:102-130: uniform over the transitions of complete episodes.  The batch carries
        their Monte Carlo returns as ``n_step_discounted_rewards`` (fp64), written into ``out[...]`` when ``out`` has
        that buffer.  ``s2d``: image columns as space-to-depth operand planes (ExperienceReplay.sample_batch)."""
        n = self.num_transitions_in_complete_episodes()
        if n < 1:
            raise ValueError("The episodic replay buffer cannot be sampled since there are no complete episodes yet. "
                             "There is currently 1 episodes with {} transitions".format(self._open_len))
        self._flush()
        pos = np.random.randint(n, size=size)                                   # :121
        # only the drawn positions are mapped to slots: no O(buffer) host work per step
        batch = self._gather_slots(self._slots_of_complete_episodes(pos), size, out, s2d)
        idx = batch.columns["idx"]
        ret = out.get("n_step_discounted_rewards") if out is not None else None
        if ret is not None:
            torch.index_select(self._returns, 0, idx, out=ret)
        else:
            ret = self._returns[idx]
        batch.columns["n_step_discounted_rewards"] = ret
        return batch

    def clean(self, lock: bool = True) -> None:
        self.assert_not_frozen()
        self.ring.clear()
        self.episode_lengths = []
        self._open_len = 0
