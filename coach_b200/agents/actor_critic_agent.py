"""Actor-Critic (A3C) on the GPU, E environment streams stepped in lock step, discrete actions.  Drop-in for

  rl_coach/agents/actor_critic_agent.py:36-170          parameters, learn_from_batch (A_VALUE / GAE), get_prediction
  rl_coach/agents/policy_optimization_agent.py:85-185   segment cut every t_max steps or at the episode's end, acting
  rl_coach/exploration_policies/categorical.py:36-47    np.random.choice over the policy (training), argmax (evaluation)

The streams follow the N-step Q agent's lock-step semantics (coach_b200.memories.lockstep_segments: every stream is one
asynchronous reference worker; the segments closed at one lock-step are learned in ONE learn step whose gradient is the
mean of the segments' gradients).  With E = 1 this is the reference schedule.

One learn step = gather -> online features of each segment's last s' (the reference bootstraps with the online network;
there is no target network) -> online features of the rows -> ``cb200_actor_critic_head`` (V, the A_VALUE return or the
GAE recurrences, targets, advantages, softmax, the V / policy / entropy loss, a dense dL/dZ, the head's gradients and
dL/dh) -> backward -> global norm and clip -> TF-Adam.  Every 32-row bucket has its own forward / backward instance on
the shared parameters; from 128 rows on a bucket's step is replayed as one CUDA graph.

Acting: one forward pass of the E states, then ``cb200_categorical_act`` (the head's softmax, then np.random.choice's
inverse-cdf draw on uniforms drawn on the host with np.random.random_sample(E), or the first argmax in evaluation).

Refused (ValueError): a ``policy_gradient_rescaler`` other than A_VALUE / GAE (the reference only warns, then trains on
zero advantages), ``apply_gradients_every_x_episodes != 1``, a continuous action space, and more than one rank.
Checkpoints hold the network, Adam and the counters, including every stream's cut position; the rows of segments still
open when the checkpoint is written are not saved.
"""
import ctypes
from enum import Enum

import numpy as np
import torch

from coach_b200 import _lib, parallel
from coach_b200.agents.dqn_agent import DQNAgent, QNetworkWrapper
from coach_b200.architectures.layers import Workspace
from coach_b200.architectures.q_network import QNetworkDef
from coach_b200.base_parameters import (AgentParameters, AlgorithmParameters, InputEmbedderParameters,
                                        NetworkParameters, middleware_units, scheme_layers)
from coach_b200.memories.lockstep_segments import LockstepSegments


class PolicyGradientRescaler(Enum):
    """policy_optimization_agent.py:30-39"""
    TOTAL_RETURN = 0
    FUTURE_RETURN = 1
    FUTURE_RETURN_NORMALIZED_BY_EPISODE = 2
    FUTURE_RETURN_NORMALIZED_BY_TIMESTEP = 3
    Q_VALUE = 4
    A_VALUE = 5
    TD_RESIDUAL = 6
    DISCOUNTED_TD_RESIDUAL = 7
    GAE = 8


class ActorCriticAlgorithmParameters(AlgorithmParameters):
    """actor_critic_agent.py:36-64"""

    def __init__(self):
        super().__init__()
        self.policy_gradient_rescaler = PolicyGradientRescaler.A_VALUE
        self.apply_gradients_every_x_episodes = 5
        self.beta_entropy = 0
        self.num_steps_between_gradient_updates = 5000          # t_max
        self.gae_lambda = 0.96
        self.estimate_state_value_using_gae = False


class ActorCriticNetworkParameters(NetworkParameters):
    """actor_critic_agent.py:67-75: VHead (loss weight 0.5) and PolicyHead (loss weight 1.0) on the Medium network"""

    def __init__(self):
        super().__init__()
        self.input_embedders_parameters = {'observation': InputEmbedderParameters()}
        self.heads_parameters = ["VHead", "PolicyHead"]
        self.head_loss_weights = [0.5, 1.0]
        self.optimizer_type = 'Adam'
        self.clip_gradients = 40.0
        self.async_training = True


class CategoricalParameters(object):
    """exploration_policies/categorical.py:25-28"""

    @property
    def path(self):
        return 'rl_coach.exploration_policies.categorical:Categorical'


class ActorCriticAgentParameters(AgentParameters):
    """actor_critic_agent.py:78-88; the reference's SingleEpisodeBuffer is the agent's device rollout buffer"""

    def __init__(self):
        super().__init__(algorithm=ActorCriticAlgorithmParameters(), memory=None,
                         networks={"main": ActorCriticNetworkParameters()})
        self.exploration = CategoricalParameters()

    @property
    def path(self):
        return 'coach_b200.agents.actor_critic_agent:ActorCriticAgent'


MODES = {PolicyGradientRescaler.A_VALUE: _lib.AC_A_VALUE, PolicyGradientRescaler.GAE: _lib.AC_GAE}


class ActorCriticAgent(object):
    def __init__(self, agent_parameters, parent=None, observation_shape=None, num_actions=None, num_envs=1,
                 device=None, seed=None, action_dim=None):
        """num_actions: a discrete action space; action_dim (a continuous one, Mujoco_A3C) is refused"""
        self.ap = ap = agent_parameters
        alg, net_params = ap.algorithm, ap.network_wrappers["main"]
        if alg.policy_gradient_rescaler not in MODES:
            raise ValueError("policy_gradient_rescaler must be A_VALUE or GAE, got %s (the reference would train on "
                             "zero advantages)" % (alg.policy_gradient_rescaler,))
        if alg.apply_gradients_every_x_episodes != 1:
            raise ValueError("apply_gradients_every_x_episodes must be 1: gradients are applied after every segment "
                             "(the reference default is 5; CartPole_A3C and Atari_A3C set 1)")
        if action_dim is not None:
            raise ValueError("ActorCriticAgent takes a discrete action space; continuous actions are not implemented")
        if parallel.is_distributed():
            raise ValueError("ActorCriticAgent runs on one rank")
        self.parent = parent
        self.lib = _lib.load()
        self.device = dev = torch.device(device if device is not None else "cuda")
        self.observation_shape = obs = tuple(observation_shape if observation_shape is not None
                                             else ap.observation_shape)
        self.num_actions = A = int(num_actions if num_actions is not None else ap.num_actions)
        self.num_envs = E = int(num_envs)
        self.t_max = int(alg.num_steps_between_gradient_updates)
        self.mode = MODES[alg.policy_gradient_rescaler]
        if self.mode == _lib.AC_GAE and alg.estimate_state_value_using_gae:
            self.mode = _lib.AC_GAE_VALUE
        emb = getattr(net_params, "input_embedders_parameters", {}).get("observation")
        scheme = getattr(getattr(net_params, "middleware_parameters", None), "scheme", "Medium")
        self.net_def = QNetworkDef(dev, obs, A, middleware_units=middleware_units(scheme),
                                   embedder_scheme=scheme_layers(getattr(emb, "scheme", "Medium")), value_head=True)
        gen = torch.Generator().manual_seed(int(seed)) if seed is not None else None
        self.net_def.store.init_glorot(gen)
        self.segments = sg = LockstepSegments(self.lib, dev, obs, E, self.t_max)
        self.learn = sg.learn
        # the shared parameters (online, Adam); the wrapper's own bindings are the 32-row bucket
        self.batch_buffers = {"state:observation": self.learn["state"][:32],
                              "next_state:observation": self.learn["next_state"][:32]}
        self.networks = {"main": QNetworkWrapper(self.lib, self.net_def, net_params, 32, self.batch_buffers, False,
                                                 dev)}
        net = self.networks["main"]
        self.online_boot = self.net_def.instantiate(self.lib, Workspace(dev), E, sg.boot_states, net.theta)
        net.add_planes(self.online_boot)
        self._buckets = {}
        self.loss_dev = torch.zeros(1, dtype=torch.float32, device=dev)
        pin = dev.type == "cuda"
        self._fetch_host = torch.zeros(2, dtype=torch.float32, pin_memory=pin)
        self._acting = {}
        self._act_out = {}
        # counters of agents/agent.py:112-135
        self.training_iteration = 0
        self.total_steps_counter = 0

    # ---- reference plumbing -------------------------------------------------------------------------------------------------
    @property
    def is_on_policy(self) -> bool:
        return True

    def _join_optimizer(self):
        pass                                                   # the optimizer runs on the caller's stream

    @property
    def learned_segments(self):
        """(stream, start, end) of the segments the last train() step learned"""
        return self.segments.learned_segments

    @property
    def graph_kernel_launches(self):
        return self.segments.graph_kernel_launches

    # ---- acting -------------------------------------------------------------------------------------------------------------
    _forward_acting = DQNAgent.get_all_q_values_for_states

    def get_prediction(self, states):
        """actor_critic_agent.py:167-170 for E states: the network's outputs [E, 1 + A] (V | policy logits) as a CUDA
        tensor (persistent buffer, valid until the next call)"""
        return self._forward_acting(states)

    def choose_actions(self, states, evaluation=False, uniforms=None):
        """policy_optimization_agent.py:160-185 for E environments: p = softmax of the policy logits on the device,
        then Categorical.get_action: np.random.choice(A, p=p) per environment (training; ``uniforms`` [E], default
        np.random.random_sample(E), which draws what E successive choice calls draw) or the first argmax (evaluation).
        Returns (actions int64 [E], all_action_probabilities float32 [E, A]) as numpy arrays."""
        z = self.get_prediction(states)
        E, A = int(z.shape[0]), self.num_actions
        out = self._act_out.get(E)
        if out is None:
            pin = self.device.type == "cuda"
            out = self._act_out[E] = (torch.zeros(E, dtype=torch.int64, device=self.device),
                                      torch.zeros((E, A), dtype=torch.float32, device=self.device),
                                      torch.zeros(E, dtype=torch.float64, device=self.device),
                                      torch.zeros(E, dtype=torch.float64, pin_memory=pin))
        actions, probs, u_dev, u_host = out
        u_ptr = None
        if not evaluation:
            u = np.random.random_sample(E) if uniforms is None else np.asarray(uniforms, dtype=np.float64)
            torch.cuda.current_stream().synchronize()          # the previous call's copy has left the staging
            u_host.numpy()[:] = u.reshape(E)
            u_dev.copy_(u_host, non_blocking=True)
            u_ptr = u_dev.data_ptr()
        _lib.check(self.lib.cb200_categorical_act(z.data_ptr(), E, A, u_ptr, actions.data_ptr(), probs.data_ptr(),
                                                  _lib.current_stream()))
        return actions.cpu().numpy(), probs.cpu().numpy()

    # ---- rollout ------------------------------------------------------------------------------------------------------------
    def observe_batch(self, states, actions, rewards, next_states, game_overs):
        """one lock-step of the E streams (agent.py:820-834 act's step count, :905-975 observe, core_types.py:716-725
        Episode.insert): host arrays [E, ...]"""
        self.segments.observe(states, actions, rewards, next_states, game_overs)
        self.total_steps_counter += 1

    def train(self, fetch=True):
        """policy_optimization_agent.py:85-135: one learn step over the segments that closed.  Returns the loss (0 when
        no segment closed)."""
        streams, rows = self.segments.close()
        if len(streams) == 0:
            return 0
        self.training_iteration += 1
        return self._learn(self.segments.tables(streams, rows), True, fetch)

    # ---- the learn step -----------------------------------------------------------------------------------------------------
    def learn_from_batch(self, batch, fetch=True):
        """one learn step on given segments, bypassing the rollout buffer.  batch: dict of host arrays
        states / next_states / actions / rewards / game_overs over the rows, and "lengths": the segments' lengths in row
        order (at most num_envs of them).  Returns (loss, [loss], unclipped gradient norm) with fetch, else device
        scalars."""
        return self._learn(self.segments.load(batch), False, fetch)

    def _bucket(self, B):
        bk = self._buckets.get(B)
        if bk is not None:
            return bk
        lib, dev, net, nd = self.lib, self.device, self.networks["main"], self.net_def
        on = net.online_s if B == 32 else \
            nd.instantiate(lib, Workspace(dev), B, self.learn["state"][:B], net.theta, net.store.grad, train=True)
        head = on.trunk.layers[-1]
        A = self.num_actions
        if not (len(on.trunk.layers) >= 2 and head.K in (256, 512) and head.N == A + 1 and A <= 18 and
                on.trunk.acts[-2] is not None and on.trunk.layers[-2].act == 1):
            raise ValueError("cb200_actor_critic_head needs <= 18 actions on a 256- or 512-wide ReLU layer")
        store, p, alg = net.store, net.params, self.ap.algorithm
        wname, bname = nd.trunk.names[-1]
        K, N, E = head.K, A + 1, self.num_envs
        d = _lib.ActorCriticHeadDesc()
        keep = torch.zeros(((E + 3) // 4) * 4 * (K * N + N + 1), dtype=torch.float32, device=dev)
        d.h, d.h_boot = on.trunk.acts[-2].data_ptr(), self.online_boot.trunk.acts[-2].data_ptr()
        d.w, d.b = store.view(net.theta, wname).data_ptr(), store.view(net.theta, bname).data_ptr()
        d.actions, d.rewards = self.learn["action"].data_ptr(), self.learn["reward"].data_ptr()
        d.game_overs = self.learn["game_over"].data_ptr()
        d.seg_offsets, d.seg_lengths = self.segments.seg_table()
        d.segments, d.rows = E, B
        d.discount, d.gae_lambda = float(alg.discount), float(alg.gae_lambda)
        d.mode = self.mode
        d.huber = 1 if p.replace_mse_with_huber_loss else 0
        d.beta_entropy = float(alg.beta_entropy)
        d.v_weight, d.p_weight = (float(x) for x in getattr(p, "head_loss_weights", (0.5, 1.0)))
        d.features, d.n_actions = K, A
        d.z, d.loss = on.q.data_ptr(), self.loss_dev.data_ptr()
        dz = on.trunk.dzs[-2]
        d.dh = dz.data_ptr() if dz is not None else None
        pl = on.trunk.dz_planes[-2]
        if pl is not None:
            d.dh_planes, d.dh_plane_stride = pl.ptr, pl.stride
        d.dw, d.db = store.view(store.grad, wname).data_ptr(), store.view(store.grad, bname).data_ptr()
        d.workspace = keep.data_ptr()
        bk = self._buckets[B] = (on, d, keep)
        return bk

    def _device_step(self, B, gather):
        lib, st = self.lib, _lib.current_stream()
        net = self.networks["main"]
        on, d, _ = self._bucket(B)
        if gather:
            self.segments.gather(B, ("state", "action", "reward", "game_over"), True, st)
        if on.theta_planes is not None and on is not net.online_s:
            on.theta_planes.refresh()                          # this bucket's operand planes of the current theta
        self.online_boot.forward_features()
        on.forward_features()
        _lib.check(lib.cb200_actor_critic_head(ctypes.byref(d), st))
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
        self.segments.run(B, gather, self._device_step, _lib.tune_default("a3c_graph", 1))
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
