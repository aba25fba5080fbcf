"""Data carriers of the hot path, mirroring ``rl_coach/core_types.py``:

  Transition   <- core_types.py:195-310   (same constructor, same "not filled" exceptions, same __copy__)
  Batch        <- core_types.py:405-649   (host AoS->SoA view over a list of Transitions; kept for API parity)
  DeviceBatch  -- the device-resident counterpart of Batch: the same accessors (states / next_states / actions / rewards /
                  game_overs / info / size / slice) but every column is a CUDA tensor that the replay's gather kernel
                  has already staged in HBM.  ``Agent.train`` in the reference forces List[Transition] through
                  ``pre_network_filter`` and ``Batch()`` (agents/agent.py:726-741); device agents call
                  ``memory.sample_batch()`` instead and never materialise Transitions.
"""
import copy
from random import shuffle
from typing import Any, Dict, List

import numpy as np


class Transition(object):
    def __init__(self, state: Dict[str, np.ndarray] = None, action=None, reward=None,
                 next_state: Dict[str, np.ndarray] = None, game_over: bool = None, info: Dict = None):
        self._state = self.state = state
        self._action = self.action = action
        self._reward = self.reward = reward
        self._n_step_discounted_rewards = self.n_step_discounted_rewards = None
        if not next_state:
            next_state = state
        self._next_state = self._next_state = next_state
        self._game_over = self.game_over = game_over
        self.info = {} if info is None else info

    def __repr__(self):
        return str(self.__dict__)

    def _get(self, name, what):
        v = getattr(self, name)
        if v is None:
            raise Exception("The {} was not filled by any of the modules between the environment and the agent"
                            .format(what))
        return v

    state = property(lambda s: s._get("_state", "state"), lambda s, v: setattr(s, "_state", v))
    action = property(lambda s: s._get("_action", "action"), lambda s, v: setattr(s, "_action", v))
    reward = property(lambda s: s._get("_reward", "reward"), lambda s, v: setattr(s, "_reward", v))
    game_over = property(lambda s: s._get("_game_over", "done flag"), lambda s, v: setattr(s, "_game_over", v))
    next_state = property(lambda s: s._get("_next_state", "next state"), lambda s, v: setattr(s, "_next_state", v))

    @property
    def n_step_discounted_rewards(self):
        if self._n_step_discounted_rewards is None:
            raise Exception("The n_step_discounted_rewards were not filled by any of the modules between the "
                            "environment and the agent.  Make sure that you are using an episodic experience replay.")
        return self._n_step_discounted_rewards

    @n_step_discounted_rewards.setter
    def n_step_discounted_rewards(self, val):
        self._n_step_discounted_rewards = val

    def add_info(self, new_info: Dict[str, Any]) -> None:
        if not new_info.keys().isdisjoint(self.info.keys()):
            raise ValueError("The new info dictionary can not be appended to the existing info dictionary since there "
                             "are overlapping keys between the two. old keys: {}, new keys: {}"
                             .format(self.info.keys(), new_info.keys()))
        self.info.update(new_info)

    def update_info(self, new_info: Dict[str, Any]) -> None:
        self.info.update(new_info)

    def __copy__(self):
        new_transition = type(self)()
        new_transition.__dict__.update(self.__dict__)
        new_transition._state = copy.copy(new_transition._state)
        new_transition._next_state = copy.copy(new_transition._next_state)
        new_transition.info = copy.copy(new_transition.info)
        return new_transition


class Batch(object):
    """Host-side batch over a list of Transitions (lazy column extraction), API of core_types.py:405-649."""

    def __init__(self, transitions: List[Transition]):
        self.transitions = transitions
        self._reset_cache()

    def _reset_cache(self):
        self._states, self._next_states, self._info = {}, {}, {}
        self._actions = self._rewards = self._n_step_discounted_rewards = self._game_overs = self._goals = None

    def slice(self, start, end) -> None:
        self.transitions = self.transitions[start:end]
        for d in (self._states, self._next_states, self._info):
            for k, v in d.items():
                d[k] = v[start:end]
        for name in ("_actions", "_rewards", "_n_step_discounted_rewards", "_game_overs", "_goals"):
            v = getattr(self, name)
            if v is not None:
                setattr(self, name, v[start:end])

    def shuffle(self) -> None:
        order = list(range(self.size))
        shuffle(order)
        self.transitions = [self.transitions[i] for i in order]
        self._reset_cache()

    @staticmethod
    def _maybe_expand(x, expand_dims):
        return np.expand_dims(x, -1) if expand_dims else x

    def _state_like(self, cache, attr, fetches, expand_dims):
        out = {}
        for key in set(fetches).intersection(getattr(self.transitions[0], attr).keys()):
            if key not in cache:
                cache[key] = np.array([np.array(getattr(t, attr)[key]) for t in self.transitions])
            out[key] = self._maybe_expand(cache[key], expand_dims)
        return out

    def states(self, fetches: List[str], expand_dims=False) -> Dict[str, np.ndarray]:
        return self._state_like(self._states, "state", fetches, expand_dims)

    def next_states(self, fetches: List[str], expand_dims=False) -> Dict[str, np.ndarray]:
        return self._state_like(self._next_states, "next_state", fetches, expand_dims)

    def _column(self, cache_name, attr, expand_dims):
        if getattr(self, cache_name) is None:
            setattr(self, cache_name, np.array([getattr(t, attr) for t in self.transitions]))
        return self._maybe_expand(getattr(self, cache_name), expand_dims)

    def actions(self, expand_dims=False):
        return self._column("_actions", "action", expand_dims)

    def rewards(self, expand_dims=False):
        return self._column("_rewards", "reward", expand_dims)

    def n_step_discounted_rewards(self, expand_dims=False):
        return self._column("_n_step_discounted_rewards", "n_step_discounted_rewards", expand_dims)

    def game_overs(self, expand_dims=False):
        return self._column("_game_overs", "game_over", expand_dims)

    def goals(self, expand_dims=False):
        return self._column("_goals", "goal", expand_dims)

    def info_as_list(self, key) -> list:
        if key not in self._info:
            self._info[key] = [t.info[key] for t in self.transitions]
        return self._info[key]

    def info(self, key, expand_dims=False):
        lst = self.info_as_list(key)
        return np.expand_dims(lst, -1) if expand_dims else np.array(lst)

    @property
    def size(self) -> int:
        return len(self.transitions)

    def __getitem__(self, key):
        return self.transitions[key]

    def __setitem__(self, key, item):
        self.transitions[key] = item


class DeviceBatch(object):
    """A minibatch whose columns already sit in HBM (CUDA tensors), produced by ``memory.sample_batch``.

    columns: dict with keys ``'state:<key>'``, ``'next_state:<key>'``, ``'action'``, ``'reward'`` (float64),
    ``'game_over'`` (uint8), and the ``info`` entries (``'idx'`` int64 leaf / slot indices, ``'weight'`` float64
    importance weights, ``'weight32'`` the same rounded once to float32).
    """

    def __init__(self, columns: dict, size: int, lazy=None):
        """lazy(name) -> tensor: materialises a column the sampler did not stage (the fused image path hands the frames
        to the first convolution as operand planes and skips the uint8 copy; ``states()`` / ``column()`` gather it on
        demand from the drawn slots)."""
        self.columns = columns
        self._size = size
        self._lazy = lazy

    def column(self, name):
        if name not in self.columns and self._lazy is not None:
            self.columns[name] = self._lazy(name)
        return self.columns[name]

    @property
    def size(self) -> int:
        return self._size

    def _state_like(self, prefix, fetches, expand_dims):
        out = {}
        for key in fetches:
            name = prefix + key
            if name not in self.columns and self._lazy is not None:
                try:
                    self.column(name)
                except KeyError:
                    pass
            if name in self.columns:
                t = self.columns[name]
                out[key] = t.unsqueeze(-1) if expand_dims else t
        return out

    def states(self, fetches, expand_dims=False):
        return self._state_like("state:", fetches, expand_dims)

    def next_states(self, fetches, expand_dims=False):
        return self._state_like("next_state:", fetches, expand_dims)

    def _col(self, name, expand_dims):
        t = self.columns[name]
        return t.unsqueeze(-1) if expand_dims else t

    def actions(self, expand_dims=False):
        return self._col("action", expand_dims)

    def rewards(self, expand_dims=False):
        return self._col("reward", expand_dims)

    def game_overs(self, expand_dims=False):
        return self._col("game_over", expand_dims)

    def n_step_discounted_rewards(self, expand_dims=False):
        return self._col("n_step_discounted_rewards", expand_dims)

    def info(self, key, expand_dims=False):
        return self._col(key, expand_dims)

    def slice(self, start, end) -> None:
        self.columns = {k: v[start:end] for k, v in self.columns.items()}
        self._size = next(iter(self.columns.values())).shape[0]

    def to_transitions(self) -> List[Transition]:
        """Host materialisation (device -> host copy of every column); API-compatibility path only."""
        if self._lazy is not None:
            for name in getattr(self._lazy, "names", ()):
                self.column(name)
        host = {k: v.cpu().numpy() for k, v in self.columns.items()}
        out = []
        for i in range(self._size):
            state = {k[len("state:"):]: host[k][i] for k in host if k.startswith("state:")}
            nstate = {k[len("next_state:"):]: host[k][i] for k in host if k.startswith("next_state:")}
            action = host["action"][i]
            action = action.item() if action.ndim == 0 else action
            info = {}
            if "idx" in host:
                info["idx"] = int(host["idx"][i])
            if "weight" in host:
                info["weight"] = host["weight"][i]
            for k in host:
                if k.startswith("info:"):
                    info[k[len("info:"):]] = host[k][i]
            out.append(Transition(state=state, action=action, reward=float(host["reward"][i]), next_state=nstate,
                                  game_over=bool(host["game_over"][i]), info=info))
        return out
