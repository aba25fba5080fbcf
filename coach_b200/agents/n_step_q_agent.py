"""N-step Q-learning on the GPU, E environment streams stepped in lock step.  Drop-in for

  rl_coach/agents/n_step_q_agent.py:34-153               parameters, learn_from_batch, train (target copy first)
  rl_coach/agents/policy_optimization_agent.py:85-135    segment cut every t_max steps or at the episode's end

Each stream behaves like one asynchronous reference worker: it has its own cut position and closes a segment when t_max
(``num_steps_between_gradient_updates``) steps have passed since its last cut, or on game_over.  At every lock-step
``train()`` all segments closed at that step are learned in ONE learn step whose gradient is the mean over those
segments of each segment's own gradient (the synchronous-training rule of
``scale_down_gradients_by_number_of_workers_for_sync_training``, one segment = one worker).  The target copy counts
lock-step steps (each stream's own steps); ``training_iteration`` counts learn steps.  With E = 1 this is the
reference schedule.

The rollout buffer, the cuts, the gather and the 32-row buckets with their CUDA graphs are
``coach_b200.memories.lockstep_segments``.

One learn step = gather -> target features of the bootstrap states (N-Step) or of every s' (1-Step) -> online features
-> ``cb200_nstep_q_head`` (Q, bootstrap max, the fp64 return recurrence, targets, loss, dL/dQ, the head's gradients and
dL/dh) -> backward -> TF-Adam.  Every 32-row bucket has its own forward / backward instance on the shared parameters.

Refused (ValueError): ``apply_gradients_every_x_episodes != 1`` (gradients are applied after every segment), a
``targets_horizon`` other than 'N-Step' / '1-Step' (the reference silently trains on zero loss then), a dueling head, and
more than one rank.  Checkpoints hold the networks, Adam and the counters, including every stream's cut position; the
rows of segments still open when the checkpoint is written are not saved: after a restore those segments are learned
from the rows observed since.
"""
import ctypes

import numpy as np
import torch

from coach_b200 import _lib, parallel
from coach_b200.agents.dqn_agent import DQNAgent, QNetworkWrapper
from coach_b200.architectures.layers import Workspace
from coach_b200.architectures.q_network import QNetworkDef
from coach_b200.base_parameters import (AgentParameters, AlgorithmParameters, EnvironmentSteps,
                                        InputEmbedderParameters, NetworkParameters, middleware_units, scheme_layers)
from coach_b200.exploration_policies.e_greedy import EGreedyParameters
from coach_b200.memories.lockstep_segments import LockstepSegments

HORIZONS = {"N-Step": _lib.NSTEP_NSTEP, "1-Step": _lib.NSTEP_ONESTEP}


class NStepQNetworkParameters(NetworkParameters):
    """n_step_q_agent.py:34-43"""

    def __init__(self):
        super().__init__()
        self.input_embedders_parameters = {'observation': InputEmbedderParameters()}
        self.heads_parameters = ["QHead"]
        self.optimizer_type = 'Adam'
        self.async_training = True
        self.shared_optimizer = True
        self.create_target_network = True


class NStepQAlgorithmParameters(AlgorithmParameters):
    """n_step_q_agent.py:46-73"""

    def __init__(self):
        super().__init__()
        self.num_steps_between_copying_online_weights_to_target = EnvironmentSteps(10000)
        self.apply_gradients_every_x_episodes = 1
        self.num_steps_between_gradient_updates = 5          # t_max
        self.targets_horizon = 'N-Step'


class NStepQAgentParameters(AgentParameters):
    """n_step_q_agent.py:76-85; the reference's SingleEpisodeBuffer is the agent's device rollout buffer"""

    def __init__(self):
        super().__init__(algorithm=NStepQAlgorithmParameters(), memory=None,
                         networks={"main": NStepQNetworkParameters()})
        self.exploration = EGreedyParameters()

    @property
    def path(self):
        return 'coach_b200.agents.n_step_q_agent:NStepQAgent'


class NStepQAgent(object):
    def __init__(self, agent_parameters, parent=None, observation_shape=None, num_actions=None, num_envs=1,
                 device=None, seed=None):
        self.ap = ap = agent_parameters
        alg, net_params = ap.algorithm, ap.network_wrappers["main"]
        if alg.apply_gradients_every_x_episodes != 1:
            raise ValueError("apply_gradients_every_x_episodes must be 1: gradients are applied after every segment")
        if alg.targets_horizon not in HORIZONS:
            raise ValueError("targets_horizon must be 'N-Step' or '1-Step', got %r (the reference would train on a "
                             "zero loss)" % (alg.targets_horizon,))
        if "DuelingQHead" in getattr(net_params, "heads_parameters", ["QHead"]):
            raise ValueError("NStepQAgent takes a plain QHead, not a dueling head")
        if parallel.is_distributed():
            raise ValueError("NStepQAgent runs on one rank")
        self.parent = parent
        self.lib = _lib.load()
        self.device = dev = torch.device(device if device is not None else "cuda")
        self.observation_shape = obs = tuple(observation_shape if observation_shape is not None
                                             else ap.observation_shape)
        self.num_actions = A = int(num_actions if num_actions is not None else ap.num_actions)
        self.num_envs = E = int(num_envs)
        self.t_max = int(alg.num_steps_between_gradient_updates)
        self.horizon = HORIZONS[alg.targets_horizon]
        emb = getattr(net_params, "input_embedders_parameters", {}).get("observation")
        scheme = getattr(getattr(net_params, "middleware_parameters", None), "scheme", "Medium")
        self.net_def = QNetworkDef(dev, obs, A, middleware_units=middleware_units(scheme),
                                   embedder_scheme=scheme_layers(getattr(emb, "scheme", "Medium")))
        gen = torch.Generator().manual_seed(int(seed)) if seed is not None else None
        self.net_def.store.init_glorot(gen)
        self.segments = sg = LockstepSegments(self.lib, dev, obs, E, self.t_max)
        self.learn, self.boot_states, self.max_rows = sg.learn, sg.boot_states, sg.max_rows
        # the shared parameters (online, target, Adam) and the acting path of the DQN agent.  The wrapper's own
        # bindings are the 32-row bucket.
        self.batch_buffers = {"state:observation": self.learn["state"][:32],
                              "next_state:observation": self.learn["next_state"][:32]}
        self.networks = {"main": QNetworkWrapper(self.lib, self.net_def, net_params, 32, self.batch_buffers, False,
                                                 dev)}
        net = self.networks["main"]
        net.sync()
        self.target_boot = None
        if self.horizon == _lib.NSTEP_NSTEP:
            self.target_boot = self.net_def.instantiate(self.lib, Workspace(dev), E, self.boot_states,
                                                        net.theta_target)
            net.add_planes(self.target_boot)
        self._buckets = {}
        self.loss_dev = torch.zeros(1, dtype=torch.float32, device=dev)
        self._fetch_host = torch.zeros(2, dtype=torch.float32, pin_memory=dev.type == "cuda")
        self._acting = {}
        # counters of agents/agent.py:112-135
        self.training_iteration = 0
        self.total_steps_counter = 0
        self.last_target_network_update_step = 0

    # ---- reference plumbing and the DQN agent's acting path -------------------------------------------------------------
    @property
    def is_on_policy(self) -> bool:
        return False

    _should_update_online_weights_to_target = DQNAgent._should_update_online_weights_to_target
    get_all_q_values_for_states = DQNAgent.get_all_q_values_for_states
    choose_actions = DQNAgent.choose_actions

    def _join_optimizer(self):
        pass                                                   # the optimizer runs on the caller's stream

    @property
    def learned_segments(self):
        """(stream, start, end) of the segments the last train() step learned"""
        return self.segments.learned_segments

    @property
    def graph_kernel_launches(self):
        return self.segments.graph_kernel_launches

    # ---- rollout ----------------------------------------------------------------------------------------------------------
    def observe_batch(self, states, actions, rewards, next_states, game_overs):
        """one lock-step of the E streams (agent.py:820-834 act's step count, :905-975 observe, core_types.py:716-725
        Episode.insert): host arrays [E, ...]"""
        self.segments.observe(states, actions, rewards, next_states, game_overs)
        self.total_steps_counter += 1

    def train(self, fetch=True):
        """n_step_q_agent.py:142-153 + policy_optimization_agent.py:85-135: target copy check first, then one learn step
        over the segments that closed.  Returns the loss (0 when no segment closed)."""
        net = self.networks["main"]
        if self._should_update_online_weights_to_target():
            net.update_target_network(self.ap.algorithm.rate_for_copying_weights_to_target)
        streams, rows = self.segments.close()
        if len(streams) == 0:
            return 0
        self.training_iteration += 1
        return self._learn(self.segments.tables(streams, rows), True, fetch)

    # ---- the learn step ---------------------------------------------------------------------------------------------------
    def learn_from_batch(self, batch, fetch=True):
        """one learn step on given segments, bypassing the rollout buffer.  batch: dict of host arrays
        states / next_states / actions / rewards / game_overs over the rows, and "lengths": the segments' lengths in row
        order (at most num_envs of them).  Returns (loss, [loss], unclipped gradient norm) with fetch, else device
        scalars."""
        B = self.segments.load(batch, boot=self.horizon == _lib.NSTEP_NSTEP)
        return self._learn(B, False, fetch)

    def _bucket(self, B):
        bk = self._buckets.get(B)
        if bk is not None:
            return bk
        lib, dev, net, nd = self.lib, self.device, self.networks["main"], self.net_def
        if B == 32:
            on = net.online_s
            tn = net.target_s2
        else:
            on = nd.instantiate(lib, Workspace(dev), B, self.learn["state"][:B], net.theta, net.store.grad, train=True)
            tn = None
            if self.horizon == _lib.NSTEP_ONESTEP:
                tn = nd.instantiate(lib, Workspace(dev), B, self.learn["next_state"][:B], net.theta_target)
                net.add_planes(tn)
        if self.horizon == _lib.NSTEP_NSTEP:
            tn = self.target_boot
        head = on.trunk.layers[-1]
        if not (not nd.dueling and len(on.trunk.layers) >= 2 and type(head).__name__ == "Dense" and
                head.K in (256, 512) and head.N == self.num_actions <= 18 and on.trunk.acts[-2] is not None and
                on.trunk.layers[-2].act == 1 and tn.trunk.acts[-2] is not None):
            raise ValueError("cb200_nstep_q_head needs a QHead of <= 18 actions on a 256- or 512-wide ReLU layer")
        store = net.store
        wname, bname = nd.trunk.names[-1]
        K, A, E = head.K, self.num_actions, self.num_envs
        d = _lib.NstepQHeadDesc()
        keep = torch.zeros(((E + 3) // 4) * 4 * (K * A + A + 1), dtype=torch.float32, device=dev)
        d.h_online, d.h_boot = on.trunk.acts[-2].data_ptr(), tn.trunk.acts[-2].data_ptr()
        d.w_target, d.b_target = store.view(net.theta_target, wname).data_ptr(), \
            store.view(net.theta_target, bname).data_ptr()
        d.w_online, d.b_online = store.view(net.theta, wname).data_ptr(), store.view(net.theta, bname).data_ptr()
        d.actions, d.rewards = self.learn["action"].data_ptr(), self.learn["reward"].data_ptr()
        d.game_overs = self.learn["game_over"].data_ptr()
        d.seg_offsets, d.seg_lengths = self.segments.seg_table()
        d.segments, d.rows = E, B
        d.discount = float(self.ap.algorithm.discount)
        d.horizon = self.horizon
        d.huber = 1 if net.params.replace_mse_with_huber_loss else 0
        d.features, d.n_actions = K, A
        d.q_online, d.dq, d.loss = on.q.data_ptr(), on.dq.data_ptr(), self.loss_dev.data_ptr()
        dz = on.trunk.dzs[-2]
        d.dh = dz.data_ptr() if dz is not None else None
        pl = on.trunk.dz_planes[-2]
        if pl is not None:
            d.dh_planes, d.dh_plane_stride = pl.ptr, pl.stride
        d.dw, d.db = store.view(store.grad, wname).data_ptr(), store.view(store.grad, bname).data_ptr()
        d.workspace = keep.data_ptr()
        bk = self._buckets[B] = (on, tn, d, keep)
        return bk

    def _device_step(self, B, gather):
        lib, st = self.lib, _lib.current_stream()
        net = self.networks["main"]
        on, tn, d, _ = self._bucket(B)
        if gather:
            keys = ("state", "action", "reward", "game_over") + \
                (("next_state",) if self.horizon == _lib.NSTEP_ONESTEP else ())
            self.segments.gather(B, keys, self.horizon == _lib.NSTEP_NSTEP, st)
        if on.theta_planes is not None and on is not net.online_s:
            on.theta_planes.refresh()                          # this bucket's operand planes of the current theta
        tn.forward_features()
        on.forward_features()
        _lib.check(lib.cb200_nstep_q_head(ctypes.byref(d), st))
        on.backward_features()
        _lib.check(lib.cb200_sumsq(net.store.grad.data_ptr(), net.store.size, net.sumsq.data_ptr(), net.ws.ptr(), st))
        clip = net.params.clip_gradients
        if clip is not None and clip != 0:
            if net.params.gradients_clipping_method != "ClipByGlobalNorm":
                raise NotImplementedError("only ClipByGlobalNorm is implemented on device")
            _lib.check(lib.cb200_clip_by_global_norm(net.store.grad.data_ptr(), net.store.size, net.sumsq.data_ptr(),
                                                     float(clip), st))
        net.apply_gradients(1.0)

    def _learn(self, B, gather, fetch):
        self.segments.run(B, gather, self._device_step, _lib.tune_default("nstep_graph", 1))
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
