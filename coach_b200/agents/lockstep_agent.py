"""The part shared by the agents that learn from lock-step segments (coach_b200.memories.lockstep_segments): N-step Q,
A3C and Policy Gradients.  Every row bucket has its own forward / backward instance on the shared parameters, and its
step is gather -> operand planes -> bootstrap features -> features -> ``_launch_head`` -> backward ->
``_sink_gradients``; from 128 rows on it is replayed as one CUDA graph.
"""
from collections import namedtuple

import numpy as np
import torch

from coach_b200 import _lib
from coach_b200.architectures.layers import Workspace
from coach_b200.architectures.q_network import QNetworkDef
from coach_b200.agents.dqn_agent import DQNAgent, QNetworkWrapper
from coach_b200.base_parameters import middleware_units, scheme_layers
from coach_b200.memories.lockstep_segments import LockstepSegments

# a row bucket: the train-mode network on its rows, the bootstrap network or None, the head descriptor, its workspace
Bucket = namedtuple("Bucket", "online boot desc workspace")


class LockstepAgent(object):
    """Subclasses set ``head_desc_type``, ``head_error`` (the refusal of a network their head kernel cannot take),
    ``max_outputs``, ``graph_tuning`` (the CB200_* switch of the graph replay), ``gather_keys`` / ``gather_boot``, and
    define ``_fill_desc`` (their own descriptor fields; returns the workspace's floats) and ``_launch_head``."""
    max_outputs = 18
    is_on_policy = True

    def __init__(self, ap, parent, observation_shape, num_envs, device, seed, outputs, value_head=False,
                 action_dim=None, gaussian_policy=False, depth=None):
        """the constructor's common part; the subclass validates its parameters first.  outputs: the head's policy or
        Q outputs (value_head adds V's column; gaussian_policy: they are a mean and a std block); action_dim: float
        action vectors of that width (continuous actions); depth: the rollout ring's rows per stream (default t_max)"""
        net_params = ap.network_wrappers["main"]
        self.ap, self.parent = ap, parent
        self.lib = _lib.load()
        self.device = dev = torch.device(device if device is not None else "cuda")
        self.observation_shape = obs = tuple(observation_shape if observation_shape is not None
                                             else ap.observation_shape)
        self.num_envs = E = int(num_envs)
        self.t_max = int(ap.algorithm.num_steps_between_gradient_updates)
        emb = getattr(net_params, "input_embedders_parameters", {}).get("observation")
        scheme = getattr(getattr(net_params, "middleware_parameters", None), "scheme", "Medium")
        self.net_def = QNetworkDef(dev, obs, outputs, middleware_units=middleware_units(scheme),
                                   embedder_scheme=scheme_layers(getattr(emb, "scheme", "Medium")),
                                   value_head=value_head, gaussian_policy=gaussian_policy)
        gen = torch.Generator().manual_seed(int(seed)) if seed is not None else None
        self.net_def.store.init_glorot(gen)
        self.segments = sg = LockstepSegments(self.lib, dev, obs, E, self.t_max, action_dim, depth)
        self.learn = sg.learn
        # the shared parameters (online, target, Adam) and the acting path of the DQN agent.  The wrapper's own
        # bindings are the 32-row bucket.
        self.batch_buffers = {"state:observation": self.learn["state"][:32],
                              "next_state:observation": self.learn["next_state"][:32]}
        self.networks = {"main": QNetworkWrapper(self.lib, self.net_def, net_params, 32, self.batch_buffers, False,
                                                 dev)}
        self._buckets = {}
        self.loss_dev = torch.zeros(1, dtype=torch.float32, device=dev)
        self._fetch_host = torch.zeros(2, dtype=torch.float32, pin_memory=dev.type == "cuda")
        self._acting = {}
        # counters of agents/agent.py:112-135
        self.training_iteration = 0
        self.total_steps_counter = 0

    # ---- reference plumbing -------------------------------------------------------------------------------------------------
    def _join_optimizer(self):
        pass                                                   # the optimizer runs on the caller's stream

    @property
    def learned_segments(self):
        """(stream, start, end) of the segments the last train() step learned"""
        return self.segments.learned_segments

    @property
    def graph_kernel_launches(self):
        return self.segments.graph_kernel_launches

    def get_prediction(self, states):
        """the network's outputs for E states as a CUDA tensor [E, N] (persistent buffer, valid until the next call)"""
        return DQNAgent.get_all_q_values_for_states(self, states)

    def _stage(self, host, dev, values):
        """host draws -> the device buffer ``dev`` through the pinned ``host``; returns the device pointer"""
        torch.cuda.current_stream().synchronize()              # the previous call's copy has left the staging
        host.numpy()[...] = values.reshape(host.shape)
        dev.copy_(host, non_blocking=True)
        return dev.data_ptr()

    # ---- rollout ------------------------------------------------------------------------------------------------------------
    def observe_batch(self, states, actions, rewards, next_states, game_overs):
        """one lock-step of the E streams (agent.py:820-834 act's step count, :905-975 observe, core_types.py:716-725
        Episode.insert): host arrays [E, ...]"""
        self.segments.observe(states, actions, rewards, next_states, game_overs)
        self.total_steps_counter += 1

    # ---- the learn step -----------------------------------------------------------------------------------------------------
    def learn_from_batch(self, batch, fetch=True):
        """one learn step on given segments, bypassing the rollout buffer.  batch: dict of host arrays
        states / next_states / actions / rewards / game_overs over the rows, and "lengths": the segments' lengths in row
        order (at most num_envs of them).  Returns (loss, [loss], unclipped gradient norm) with fetch, else device
        scalars."""
        return self._learn(self.segments.load(batch, boot=self.gather_boot), False, fetch)

    def _bucket(self, B):
        """the learn step's bindings on B rows, built the first time"""
        bk = self._buckets.get(B)
        if bk is not None:
            return bk
        net = self.networks["main"]
        on = net.online_s if B == 32 else self.net_def.instantiate(self.lib, Workspace(self.device), B,
                                                                   self.learn["state"][:B], net.theta, net.store.grad,
                                                                   train=True)
        boot = self._boot_instance(B)
        head, outputs = on.trunk.layers[-1], self.net_def.num_actions
        if not (on.feature_head() and (boot is None or boot.feature_head()) and
                head.N == outputs + self.net_def.value_head and outputs <= self.max_outputs):
            raise ValueError(self.head_error)
        d = self.head_desc_type()
        d.seg_offsets, d.seg_lengths = self.segments.seg_table()
        d.segments, d.rows, d.features = self.num_envs, B, head.K
        d.loss = self.loss_dev.data_ptr()
        on.bind_head_grads(d)
        keep = torch.zeros(self._fill_desc(d, on, boot, B), dtype=torch.float32, device=self.device)
        d.workspace = keep.data_ptr()
        bk = self._buckets[B] = Bucket(on, boot, d, keep)
        return bk

    def _boot_instance(self, B):
        """the network whose features the head bootstraps from in a bucket of B rows, or None"""
        return None

    def _device_step(self, B, gather):
        st = _lib.current_stream()
        bk = self._bucket(B)
        if gather:
            self.segments.gather(B, self.gather_keys, self.gather_boot, st)
        if bk.online.theta_planes is not None and bk.online is not self.networks["main"].online_s:
            bk.online.theta_planes.refresh()                   # this bucket's operand planes of the current theta
        if bk.boot is not None:
            bk.boot.forward_features()
        bk.online.forward_features()
        self._launch_head(bk.desc, st)
        bk.online.backward_features()
        self._sink_gradients(st)

    def _sink_gradients(self, st):
        """global norm, clip by it, then the optimizer step"""
        lib, net = self.lib, self.networks["main"]
        _lib.check(lib.cb200_sumsq(net.store.grad.data_ptr(), net.store.size, net.sumsq.data_ptr(), net.ws.ptr(), st))
        clip = net.params.clip_gradients
        if clip is not None and clip != 0:
            if net.params.gradients_clipping_method != "ClipByGlobalNorm":
                raise NotImplementedError("only ClipByGlobalNorm is implemented on device")
            _lib.check(lib.cb200_clip_by_global_norm(net.store.grad.data_ptr(), net.store.size, net.sumsq.data_ptr(),
                                                     float(clip), st))
        net.apply_gradients(1.0)

    def _learn(self, B, gather, fetch):
        self.segments.run(B, gather, self._device_step, _lib.tune_default(self.graph_tuning, 1))
        if not fetch:
            return self.loss_dev if gather else (self.loss_dev, [self.loss_dev], self.networks["main"].sumsq)
        self._fetch_host[0:1].copy_(self.loss_dev, non_blocking=True)
        self._fetch_host[1:2].copy_(self.networks["main"].sumsq, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        loss = float(self._fetch_host[0])
        if gather:
            return loss
        return loss, [loss], float(np.sqrt(np.float32(self._fetch_host[1])))

    # ---- checkpoints (coach_b200/checkpoint.py) -------------------------------------------------------------------------
    def checkpoint_state(self):
        """every stream's cut position; the rows of open segments are not saved"""
        return self.segments.state()

    def restore_checkpoint_state(self, state):
        self.segments.restore(state)
