"""Actor-Critic (A3C) on the GPU, E environment streams stepped in lock step, discrete or bounded continuous actions.
Drop-in for

  rl_coach/agents/actor_critic_agent.py:36-186          parameters, learn_from_batch (A_VALUE / GAE), get_prediction
  rl_coach/agents/policy_optimization_agent.py:85-185   segment cut every t_max steps or at the episode's end, acting
  rl_coach/exploration_policies/categorical.py:36-47    np.random.choice over the policy (training), argmax (evaluation)
  rl_coach/exploration_policies/continuous_entropy.py   AdditiveNoise with the network's std: np.random.normal(mean,
                                                        std) (training), the mean (evaluation)

The streams follow the N-step Q agent's lock-step semantics (coach_b200.memories.lockstep_segments: every stream is one
asynchronous reference worker; the segments closed at one lock-step are learned in ONE learn step whose gradient is the
mean of the segments' gradients).  With E = 1 this is the reference schedule.

One learn step = gather -> online features of each segment's last s' (the reference bootstraps with the online network;
there is no target network) -> online features of the rows -> ``cb200_actor_critic_head`` (V, the A_VALUE return or the
GAE recurrences, targets, advantages, softmax, the V / policy / entropy loss, a dense dL/dZ, the head's gradients and
dL/dh) -> backward -> global norm and clip -> TF-Adam (coach_b200.agents.lockstep_agent).

Acting: one forward pass of the E states, then ``cb200_categorical_act`` (the head's softmax, then np.random.choice's
inverse-cdf draw on uniforms drawn on the host with np.random.random_sample(E), or the first argmax in evaluation).

Continuous actions (``action_dim`` with finite bounds; Mujoco_A3C): the head is ONE Dense(1 + 2D), V | fc_mean | fc_std,
mean = tanh(z) * max_abs_range and std = softplus(z) + eps, a MultivariateNormalDiag policy with its entropy term, learned
by ``cb200_actor_critic_gaussian_head`` (parallel over rows: segments are whole episodes of up to
``max_episode_steps`` rows when t_max is 10^7).  The rollout ring and the learn buffers hold min(t_max,
max_episode_steps) rows per stream, and learn steps run on PG's geometric row buckets.  Acting is
``cb200_gaussian_policy_act``: (double) mean + (double) std * n on host standard normals (np.random.standard_normal((E,
D)), what E successive np.random.normal calls draw) in training, the fp32 mean in evaluation; the noise schedule is
stepped E times per call (it does not change the action) and is checkpointed.

Refused (ValueError): a ``policy_gradient_rescaler`` other than A_VALUE / GAE (the reference only warns, then trains on
zero advantages), ``apply_gradients_every_x_episodes != 1``, more than one rank; for continuous actions missing or
infinite bounds, more than 17 action dimensions, a head layer other than 256 / 512 wide, an exploration other than
ContinuousEntropy, and a stream whose open segment fills the ring (max_episode_steps) without closing.
Checkpoints hold the network, Adam and the counters, including every stream's cut position; the rows of segments still
open when the checkpoint is written are not saved.
"""
import ctypes
from enum import Enum

import numpy as np
import torch

from coach_b200 import _lib, parallel
from coach_b200.agents.lockstep_agent import LockstepAgent
from coach_b200.architectures.layers import Workspace
from coach_b200.base_parameters import (AgentParameters, AlgorithmParameters, InputEmbedderParameters,
                                        NetworkParameters, middleware_units, scheme_layers)
from coach_b200.exploration_policies.additive_noise import ContinuousEntropyParameters
from coach_b200.memories.lockstep_segments import bucket_rows


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
        self.exploration = {"DiscreteActionSpace": CategoricalParameters(),
                            "BoxActionSpace": ContinuousEntropyParameters()}

    @property
    def path(self):
        return 'coach_b200.agents.actor_critic_agent:ActorCriticAgent'


MODES = {PolicyGradientRescaler.A_VALUE: _lib.AC_A_VALUE, PolicyGradientRescaler.GAE: _lib.AC_GAE}
MAX_ACTION_DIM = 17                                            # Humanoid: every mujoco_v2 level


def _head_features(net_params, observation_shape):
    """the width of the layer the head reads (None for a convolution map)"""
    scheme = getattr(getattr(net_params, "middleware_parameters", None), "scheme", "Medium")
    units = middleware_units(scheme) or ()
    if units:
        return int(units[-1])
    if len(tuple(observation_shape)) == 3:
        return None
    emb = scheme_layers(getattr(net_params.input_embedders_parameters.get("observation"), "scheme", "Medium"))
    return 256 if emb is None else int(emb[-1].units)


class ActorCriticAgent(LockstepAgent):
    head_desc_type = _lib.ActorCriticHeadDesc
    head_error = "cb200_actor_critic_head needs <= 18 actions on a 256- or 512-wide ReLU layer"
    graph_tuning = "a3c_graph"
    gather_keys, gather_boot = ("state", "action", "reward", "game_over"), True

    def __init__(self, agent_parameters, parent=None, observation_shape=None, num_actions=None, num_envs=1,
                 device=None, seed=None, action_dim=None, action_low=None, action_high=None, max_episode_steps=None):
        """num_actions: a discrete action space; or action_dim with the bounds action_low / action_high [action_dim]
        (a BoxActionSpace: gym's float32 arrays).  max_episode_steps: the environment's time limit (1000 for the
        mujoco_v2 levels); the rollout ring holds min(t_max, max_episode_steps) rows per stream."""
        ap = agent_parameters
        alg = ap.algorithm
        if alg.policy_gradient_rescaler not in MODES:
            raise ValueError("policy_gradient_rescaler must be A_VALUE or GAE, got %s (the reference would train on "
                             "zero advantages)" % (alg.policy_gradient_rescaler,))
        if alg.apply_gradients_every_x_episodes != 1:
            raise ValueError("apply_gradients_every_x_episodes must be 1: gradients are applied after every segment "
                             "(the reference default is 5; CartPole_A3C and Atari_A3C set 1)")
        if parallel.is_distributed():
            raise ValueError("ActorCriticAgent runs on one rank")
        self.continuous = action_dim is not None
        depth = None
        if self.continuous:
            self._check_continuous(ap, observation_shape, action_dim, action_low, action_high, max_episode_steps)
            self.action_dim = D = int(action_dim)
            self.num_actions = None
            self.max_outputs = 2 * D
            self.head_desc_type = _lib.ActorCriticGaussianHeadDesc
            self.head_error = "cb200_actor_critic_gaussian_head needs <= 17 action dimensions on a 256- or 512-wide " \
                              "ReLU layer"
            if max_episode_steps is not None:
                depth = min(int(alg.num_steps_between_gradient_updates), int(max_episode_steps))
            outputs = 2 * D
        else:
            self.num_actions = outputs = int(num_actions if num_actions is not None else ap.num_actions)
        self.mode = MODES[alg.policy_gradient_rescaler]
        if self.mode == _lib.AC_GAE and alg.estimate_state_value_using_gae:
            self.mode = _lib.AC_GAE_VALUE
        super().__init__(ap, parent, observation_shape, num_envs, device, seed, outputs, value_head=True,
                         action_dim=self.action_dim if self.continuous else None, gaussian_policy=self.continuous,
                         depth=depth)
        net = self.networks["main"]
        self.online_boot = self.net_def.instantiate(self.lib, Workspace(self.device), self.num_envs,
                                                    self.segments.boot_states, net.theta)
        net.add_planes(self.online_boot)
        self._act_out = {}
        if self.continuous:
            rng = np.maximum(np.abs(self.action_low), np.abs(self.action_high)).astype(np.float32).reshape(D)
            self.max_abs_range = torch.from_numpy(rng).to(self.device)

    def _check_continuous(self, ap, observation_shape, action_dim, action_low, action_high, max_episode_steps):
        """the continuous form's refusals, before anything touches the GPU"""
        if action_low is None or action_high is None:
            raise ValueError("continuous actions need the bounds action_low / action_high")
        self.action_low, self.action_high = np.asarray(action_low), np.asarray(action_high)
        if not (np.all(np.isfinite(self.action_low)) and np.all(np.isfinite(self.action_high))):
            raise ValueError("Additive noise exploration requires bounded actions")
        if not 1 <= int(action_dim) <= MAX_ACTION_DIM:
            raise ValueError("cb200_actor_critic_gaussian_head takes 1 .. %d action dimensions, got %d"
                             % (MAX_ACTION_DIM, int(action_dim)))
        obs = observation_shape if observation_shape is not None else ap.observation_shape
        K = _head_features(ap.network_wrappers["main"], obs)
        if K not in (256, 512):
            raise ValueError("cb200_actor_critic_gaussian_head needs a 256- or 512-wide head layer, got %s" % (K,))
        ex = ap.exploration["BoxActionSpace"] if isinstance(ap.exploration, dict) else ap.exploration
        if not isinstance(ex, ContinuousEntropyParameters):
            raise ValueError("continuous actions take ContinuousEntropy exploration (the std is the network's output), "
                             "got %s" % (type(ex).__name__,))
        self.noise_schedule = ex.noise_schedule
        if max_episode_steps is not None and int(max_episode_steps) < 1:
            raise ValueError("max_episode_steps must be >= 1")

    # ---- acting (get_prediction, actor_critic_agent.py:167-170: [E, 1 + A] outputs, V | policy logits) -----------------
    def choose_actions(self, states, evaluation=False, uniforms=None):
        """policy_optimization_agent.py:160-185 for E environments: p = softmax of the policy logits on the device,
        then Categorical.get_action: np.random.choice(A, p=p) per environment (training; ``uniforms`` [E], default
        np.random.random_sample(E), which draws what E successive choice calls draw) or the first argmax (evaluation).
        Returns (actions int64 [E], all_action_probabilities float32 [E, A]) as numpy arrays.
        Continuous (``uniforms`` then holds the standard normals [E, D], default np.random.standard_normal((E, D))):
        see ``_choose_continuous``."""
        if self.continuous:
            return self._choose_continuous(states, evaluation, uniforms)
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
            u_ptr = self._stage(u_host, u_dev, u)
        _lib.check(self.lib.cb200_categorical_act(z.data_ptr(), E, A, u_ptr, actions.data_ptr(), probs.data_ptr(),
                                                  _lib.current_stream()))
        return actions.cpu().numpy(), probs.cpu().numpy()

    def _choose_continuous(self, states, evaluation, normals):
        """ContinuousEntropy.get_action([mean, std]) for E environments: mean = tanh(z) * range, std = softplus(z) + eps;
        in training np.random.normal(mean, std) = (double) mean + (double) std * n on the standard normals, and the
        noise schedule is stepped E times (as E successive get_action calls step it; it does not change the action); in
        evaluation the fp32 mean.  Returns (actions [E, D]: float64 in training, float32 in evaluation, means float32
        [E, D], stds float32 [E, D])."""
        z = self.get_prediction(states)
        E, D, dev = int(z.shape[0]), self.action_dim, self.device
        out = self._act_out.get(E)
        if out is None:
            pin = dev.type == "cuda"
            out = self._act_out[E] = dict(actions=torch.zeros((E, D), dtype=torch.float64, device=dev),
                                          means=torch.zeros((E, D), dtype=torch.float32, device=dev),
                                          stds=torch.zeros((E, D), dtype=torch.float32, device=dev),
                                          n_dev=torch.zeros((E, D), dtype=torch.float64, device=dev),
                                          n_host=torch.zeros((E, D), dtype=torch.float64, pin_memory=pin))
        n_ptr = None
        if not evaluation:
            n = np.random.standard_normal((E, D)) if normals is None else np.asarray(normals, dtype=np.float64)
            for _ in range(E):
                self.noise_schedule.step()
            n_ptr = self._stage(out["n_host"], out["n_dev"], n)
        _lib.check(self.lib.cb200_gaussian_policy_act(z.data_ptr(), E, D, self.max_abs_range.data_ptr(), n_ptr,
                                                      out["actions"].data_ptr(), out["means"].data_ptr(),
                                                      out["stds"].data_ptr(), _lib.current_stream()))
        means, stds = out["means"].cpu().numpy(), out["stds"].cpu().numpy()
        return (means.copy() if evaluation else out["actions"].cpu().numpy()), means, stds

    def train(self, fetch=True):
        """policy_optimization_agent.py:85-135: one learn step over the segments that closed.  Returns the loss (0 when
        no segment closed)."""
        streams, rows = self.segments.close()
        if len(streams) == 0:
            return 0
        self.training_iteration += 1
        B = self._bucket_for(int(rows.sum())) if self.continuous else None
        return self._learn(self.segments.tables(streams, rows, B), True, fetch)

    def learn_from_batch(self, batch, fetch=True):
        """LockstepAgent.learn_from_batch; the continuous head's steps run on bucket_rows buckets"""
        B = self._bucket_for(int(np.sum(batch["lengths"]))) if self.continuous else None
        return self._learn(self.segments.load(batch, boot=True, B=B), False, fetch)

    def _bucket_for(self, n):
        return min(bucket_rows(n), self.segments.max_rows)

    # ---- the learn step -----------------------------------------------------------------------------------------------------
    def _boot_instance(self, B):
        """the online network on the bootstrap states (the reference bootstraps with the online network)"""
        return self.online_boot

    def _fill_desc(self, d, on, boot, B):
        net, alg = self.networks["main"], self.ap.algorithm
        store, p = net.store, net.params
        wname, bname = self.net_def.trunk.names[-1]
        d.h, d.h_boot = on.trunk.acts[-2].data_ptr(), boot.trunk.acts[-2].data_ptr()
        d.w, d.b = store.view(net.theta, wname).data_ptr(), store.view(net.theta, bname).data_ptr()
        d.actions, d.rewards = self.learn["action"].data_ptr(), self.learn["reward"].data_ptr()
        d.game_overs = self.learn["game_over"].data_ptr()
        d.discount, d.gae_lambda = float(alg.discount), float(alg.gae_lambda)
        d.mode = self.mode
        d.huber = 1 if p.replace_mse_with_huber_loss else 0
        d.beta_entropy = float(alg.beta_entropy)
        d.v_weight, d.p_weight = (float(x) for x in getattr(p, "head_loss_weights", (0.5, 1.0)))
        d.z = on.q.data_ptr()
        K, E = d.features, self.num_envs
        if self.continuous:
            d.action_dim, d.max_abs_range = self.action_dim, self.max_abs_range.data_ptr()
            return _lib.acg_workspace_floats(B, E, K, self.action_dim)
        d.n_actions = self.num_actions
        N = self.num_actions + 1
        return ((E + 3) // 4) * 4 * (K * N + N + 1)

    def _launch_head(self, d, st):
        if self.continuous:
            _lib.check(self.lib.cb200_actor_critic_gaussian_head(ctypes.byref(d), st))
        else:
            _lib.check(self.lib.cb200_actor_critic_head(ctypes.byref(d), st))

    # ---- checkpoints (coach_b200/checkpoint.py) -------------------------------------------------------------------------
    def checkpoint_state(self):
        """every stream's cut position (and, for continuous actions, the noise schedule); the rows of open segments
        are not saved"""
        state = super().checkpoint_state()
        if self.continuous:
            state = dict(state, noise=float(self.noise_schedule.current_value))
        return state

    def restore_checkpoint_state(self, state):
        super().restore_checkpoint_state(state)
        if self.continuous:
            self.noise_schedule.current_value = state["noise"]
