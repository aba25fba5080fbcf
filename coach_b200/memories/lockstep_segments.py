"""On-policy segments of E environment streams stepped in lock step, on the device.  The rollout side of

  rl_coach/agents/policy_optimization_agent.py:85-135    segment cut every t_max steps or at the episode's end

shared by the agents that learn from such segments: N-step Q, A3C and Policy Gradients, on the common agent base
``coach_b200.agents.lockstep_agent``.  Each stream behaves like one asynchronous reference worker: it has its own cut
position and closes a segment when t_max (``num_steps_between_gradient_updates``) steps have passed since its last
cut, or on game_over.  All segments closed at one lock-step are learned in ONE learn step.

Device rollout buffer: ``depth`` slots per stream (default t_max), slot (t mod depth) * E + e for stream e at lock-step
t: a segment spans at most t_max consecutive steps and is consumed at the step it closes, so with depth = t_max a slot is
never overwritten while it is live.  A shallower ring (depth < t_max: whole episodes bounded by the environment's time
limit, A3C's Mujoco preset cuts every 10^7 steps) refuses a lock-step that would overwrite the first row of a segment
still open.
``observe`` stores one lock-step with one host-to-device copy per column and one ring scatter; ``gather`` copies the
closed segments' rows (and each segment's last s', the bootstrap state) into the learn buffers with ``cb200_gather``.

Learn steps run on 32-row buckets (padding rows carry no weight); ``run`` replays the step of every bucket of 128 rows
or more as one CUDA graph once it has run eagerly twice.
"""
import numpy as np
import torch

from coach_b200 import _lib
from coach_b200.utils import graph_capture

COLUMNS = ("state", "next_state", "action", "reward", "game_over")


def round32(n):
    return max(32, (int(n) + 31) // 32 * 32)


def bucket_rows(n):
    """a learn step's row bucket for n rows: n rounded up to 32 up to 256 rows, above that to a quarter of the power of
    two below n (256 -> 320 -> 384 -> 448 -> 512 -> 640 -> ...): at most 25 % padding, about 4 log2(rows / 256) + 8
    sizes"""
    n = round32(n)
    if n <= 256:
        return n
    step = 1 << ((n - 1).bit_length() - 3)
    return -(-n // step) * step


class LockstepSegments(object):
    def __init__(self, lib, device, observation_shape, num_envs, t_max, action_dim=None, depth=None):
        """action_dim: the action column holds float32 [action_dim] vectors (continuous actions) instead of int64;
        depth: rows per stream of the rollout ring and the learn buffers (default t_max)"""
        self.lib = lib
        self.device = dev = torch.device(device)
        obs = tuple(observation_shape)
        self.num_envs = E = int(num_envs)
        self.t_max = int(t_max)
        self.depth = T = self.t_max if depth is None else int(depth)
        if E < 1 or self.t_max < 1 or T < 1:
            raise ValueError("num_envs, num_steps_between_gradient_updates and the ring depth must be >= 1")
        obs_dtype = torch.uint8 if len(obs) == 3 else torch.float32
        z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=dev)        # noqa: E731
        self.rollout = {"state": z((T * E,) + obs, obs_dtype), "next_state": z((T * E,) + obs, obs_dtype),
                        "action": z(T * E, torch.int64) if action_dim is None else
                        z((T * E, int(action_dim)), torch.float32), "reward": z(T * E, torch.float64),
                        "game_over": z(T * E, torch.uint8)}
        self._stage_dev = {k: torch.zeros((E,) + tuple(v.shape[1:]), dtype=v.dtype, device=dev)
                           for k, v in self.rollout.items()}
        pin = dev.type == "cuda"
        self._stage_host = {k: torch.zeros(v.shape, dtype=v.dtype, pin_memory=pin) for k, v in self._stage_dev.items()}
        self._stage_ev = None
        # learn buffers: at most E * depth rows close at one step
        self.max_rows = R = round32(E * T)
        self.learn = {k: z((R,) + tuple(v.shape[1:]), v.dtype) for k, v in self.rollout.items()}
        self.boot_states = z((E,) + obs, obs_dtype)
        self.idx_dev = z(R + E, torch.int64)                      # row slots | bootstrap slots
        self.seg_dev = z(2 * E, torch.int32)                      # offsets | lengths
        self._idx_host = torch.zeros(R + E, dtype=torch.int64, pin_memory=pin)
        self._seg_host = torch.zeros(2 * E, dtype=torch.int32, pin_memory=pin)
        self._tab_ev = None
        self._graphs = {}
        self._eager = {}
        self.graph_kernel_launches = 0
        # the per-stream cut state of policy_optimization_agent.py:85-135
        self.t = 0                                             # lock-steps observed
        self.episode_length = np.zeros(E, dtype=np.int64)
        self.last_gradient_update_step_idx = np.zeros(E, dtype=np.int64)
        self.complete = np.zeros(E, dtype=bool)
        self.segment_start = np.zeros(E, dtype=np.int64)       # lock-step of the open segment's first stored row
        self.learned_segments = []                             # (stream, start, end) of the last close()

    def seg_table(self):
        """(offsets, lengths) device pointers of the segment table: num_envs int32 slots each, 0 = unused"""
        return self.seg_dev.data_ptr(), self.seg_dev.data_ptr() + 4 * self.num_envs

    def observe(self, states, actions, rewards, next_states, game_overs):
        """one lock-step of the E streams (agent.py:905-975 observe, core_types.py:716-725 Episode.insert): host
        arrays [E, ...]"""
        E, T = self.num_envs, self.depth
        if T < self.t_max:
            held = np.minimum(self.episode_length - self.last_gradient_update_step_idx, self.t - self.segment_start)
            full = np.nonzero(held >= T)[0]
            if len(full):
                raise ValueError("stream(s) %s hold %d rows of a segment still open: the rollout ring's depth "
                                 "(max_episode_steps) is reached before num_steps_between_gradient_updates (%d)"
                                 % (full.tolist(), T, self.t_max))
        cols = {"state": states, "next_state": next_states, "action": actions, "reward": rewards,
                "game_over": game_overs}
        if self._stage_ev is not None:
            self._stage_ev.synchronize()                       # the previous step's copies have left the staging
        for k, v in cols.items():
            h = self._stage_host[k]
            h.numpy()[...] = np.asarray(v).reshape(h.shape)
            self._stage_dev[k].copy_(h, non_blocking=True)
        self._stage_ev = torch.cuda.Event()
        self._stage_ev.record()
        arr, n = _lib.make_columns((self.rollout[k].data_ptr(), self._stage_dev[k].data_ptr(),
                                    self.rollout[k][0].numel() * self.rollout[k].element_size()) for k in COLUMNS)
        _lib.check(self.lib.cb200_scatter_ring(arr, n, (self.t % T) * E, T * E, E, _lib.current_stream()))
        self.t += 1
        self.episode_length += 1
        self.complete |= np.asarray(game_overs).reshape(E).astype(bool)

    def close(self):
        """policy_optimization_agent.py:88-110 for every stream: (streams, rows) of the segments closed now"""
        passed = self.episode_length - self.last_gradient_update_step_idx
        closes = (passed >= self.t_max) | self.complete
        streams = np.nonzero(closes)[0]
        rows = np.minimum(passed, self.t - self.segment_start)[streams]
        self.learned_segments = [(int(e), int(self.last_gradient_update_step_idx[e]), int(self.episode_length[e]))
                                 for e in streams]
        self.last_gradient_update_step_idx[streams] = np.where(self.complete[streams], 0, self.episode_length[streams])
        self.episode_length[self.complete] = 0
        self.complete[:] = False
        self.segment_start[streams] = self.t
        keep = rows > 0
        return streams[keep], rows[keep]

    def tables(self, streams, rows, B=None):
        """the row-index and segment tables of the segments ``close`` returned, for a bucket of B rows (default: n
        rounded up to 32); returns B.  Only the slots a step of B rows reads are written and copied: the B row slots
        (padding rows read slot 0) and the bootstrap slots."""
        E, T, t_last = self.num_envs, self.depth, self.t - 1
        n = int(rows.sum())
        B = round32(n) if B is None else int(B)
        if B < n or B > self.max_rows:
            raise ValueError("a bucket of %d rows for %d rows (at most %d)" % (B, n, self.max_rows))
        offsets = np.concatenate([[0], np.cumsum(rows)[:-1]]).astype(np.int64)
        # row j of segment s is the lock-step t_last - rows[s] + 1 + j of its stream
        seg_of_row = np.repeat(np.arange(len(streams)), rows)
        j = np.arange(n) - offsets[seg_of_row]
        steps = t_last - rows[seg_of_row] + 1 + j
        if self._tab_ev is not None:
            self._tab_ev.synchronize()
        idx, seg = self._idx_host.numpy(), self._seg_host.numpy()
        R = self.max_rows
        idx[:n] = (steps % T) * E + streams[seg_of_row]
        idx[n:B] = 0
        idx[R:R + E] = 0
        idx[R:R + len(streams)] = (t_last % T) * E + streams
        seg[:] = 0
        seg[:len(streams)] = offsets
        seg[E:E + len(streams)] = rows
        self.idx_dev[:B].copy_(self._idx_host[:B], non_blocking=True)
        self.idx_dev[R:].copy_(self._idx_host[R:], non_blocking=True)
        self.seg_dev.copy_(self._seg_host, non_blocking=True)
        self._tab_ev = torch.cuda.Event()
        self._tab_ev.record()
        return B

    def load(self, batch, boot=True, B=None):
        """given segments, bypassing the rollout buffer: batch is a dict of host arrays states / next_states / actions
        / rewards / game_overs over the rows, and "lengths": the segments' lengths in row order (at most num_envs of
        them).  Fills the learn buffers, the bootstrap states (``boot``) and the segment table; returns the bucket's
        rows (B, default n rounded up to 32)."""
        lengths = np.asarray(batch["lengths"], dtype=np.int64)
        n, S = int(lengths.sum()), len(lengths)
        if S < 1 or S > self.num_envs or n > self.max_rows or (lengths < 1).any():
            raise ValueError("1..num_envs segments of >= 1 rows, at most num_envs * t_max rows in total")
        for k, key in (("state", "states"), ("next_state", "next_states"), ("action", "actions"),
                       ("reward", "rewards"), ("game_over", "game_overs")):
            self.learn[k][:n].copy_(torch.as_tensor(np.ascontiguousarray(batch[key])).reshape(
                self.learn[k][:n].shape))
        if boot:
            last = np.cumsum(lengths) - 1
            self.boot_states.zero_()
            self.boot_states[:S].copy_(torch.as_tensor(np.ascontiguousarray(np.asarray(batch["next_states"])[last]))
                                       .reshape(self.boot_states[:S].shape))
        seg = np.zeros(2 * self.num_envs, dtype=np.int32)
        seg[:S] = np.concatenate([[0], np.cumsum(lengths)[:-1]])
        seg[self.num_envs:self.num_envs + S] = lengths
        self.seg_dev.copy_(torch.from_numpy(seg))
        B = round32(n) if B is None else int(B)
        if B < n or B > self.max_rows:
            raise ValueError("a bucket of %d rows for %d rows (at most %d)" % (B, n, self.max_rows))
        return B

    def gather(self, B, keys, boot, stream):
        """rows of the closed segments (columns ``keys``) into the learn buffers, and with ``boot`` each segment's last
        s' into the bootstrap states"""
        arr, n = _lib.make_columns((self.rollout[k].data_ptr(), self.learn[k].data_ptr(),
                                    self.rollout[k][0].numel() * self.rollout[k].element_size()) for k in keys)
        _lib.check(self.lib.cb200_gather(arr, n, self.idx_dev.data_ptr(), B, stream))
        if boot:
            arr, n = _lib.make_columns([(self.rollout["next_state"].data_ptr(), self.boot_states.data_ptr(),
                                         self.boot_states[0].numel() * self.boot_states.element_size())])
            _lib.check(self.lib.cb200_gather(arr, n, self.idx_dev.data_ptr() + 8 * self.max_rows, self.num_envs,
                                             stream))

    def run(self, B, gather, step, graph_default):
        """runs ``step(B, gather)``: eagerly, or from 128 rows on (and when ``graph_default`` is on) as a CUDA graph of
        the bucket once it has run eagerly twice"""
        graph = gather and B >= 128 and self.device.type == "cuda" and graph_default
        if graph and self._eager.get(B, 0) >= 2:
            g = self._graphs.get(B)
            if g is None:
                c0 = self.lib.cb200_launch_count()
                g = torch.cuda.CUDAGraph()
                with graph_capture(g):
                    step(B, gather)
                g = self._graphs[B] = (g, int(self.lib.cb200_launch_count() - c0))
            g[0].replay()
            self.graph_kernel_launches += g[1]
        else:
            step(B, gather)
            self._eager[B] = self._eager.get(B, 0) + 1

    # ---- checkpoints (coach_b200/checkpoint.py) -------------------------------------------------------------------------
    def state(self):
        """every stream's cut position; the rows of open segments are not saved"""
        return {"t": int(self.t), "episode_length": self.episode_length.tolist(),
                "last_gradient_update_step_idx": self.last_gradient_update_step_idx.tolist(),
                "complete": self.complete.tolist()}

    def restore(self, state):
        self.t = int(state["t"])
        self.episode_length[:] = state["episode_length"]
        self.last_gradient_update_step_idx[:] = state["last_gradient_update_step_idx"]
        self.complete[:] = state["complete"]
        self.segment_start[:] = self.t                         # nothing of the open segments is in the buffer
