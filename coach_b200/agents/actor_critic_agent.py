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
dL/dh) -> backward -> global norm and clip -> TF-Adam (coach_b200.agents.lockstep_agent).

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
from coach_b200.agents.lockstep_agent import LockstepAgent
from coach_b200.architectures.layers import Workspace
from coach_b200.base_parameters import (AgentParameters, AlgorithmParameters, InputEmbedderParameters,
                                        NetworkParameters)


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


class ActorCriticAgent(LockstepAgent):
    head_desc_type = _lib.ActorCriticHeadDesc
    head_error = "cb200_actor_critic_head needs <= 18 actions on a 256- or 512-wide ReLU layer"
    graph_tuning = "a3c_graph"
    gather_keys, gather_boot = ("state", "action", "reward", "game_over"), True

    def __init__(self, agent_parameters, parent=None, observation_shape=None, num_actions=None, num_envs=1,
                 device=None, seed=None, action_dim=None):
        """num_actions: a discrete action space; action_dim (a continuous one, Mujoco_A3C) is refused"""
        ap = agent_parameters
        alg = ap.algorithm
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
        self.num_actions = int(num_actions if num_actions is not None else ap.num_actions)
        self.mode = MODES[alg.policy_gradient_rescaler]
        if self.mode == _lib.AC_GAE and alg.estimate_state_value_using_gae:
            self.mode = _lib.AC_GAE_VALUE
        super().__init__(ap, parent, observation_shape, num_envs, device, seed, self.num_actions, value_head=True)
        net = self.networks["main"]
        self.online_boot = self.net_def.instantiate(self.lib, Workspace(self.device), self.num_envs,
                                                    self.segments.boot_states, net.theta)
        net.add_planes(self.online_boot)
        self._act_out = {}

    # ---- acting (get_prediction, actor_critic_agent.py:167-170: [E, 1 + A] outputs, V | policy logits) -----------------
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
            u_ptr = self._stage(u_host, u_dev, u)
        _lib.check(self.lib.cb200_categorical_act(z.data_ptr(), E, A, u_ptr, actions.data_ptr(), probs.data_ptr(),
                                                  _lib.current_stream()))
        return actions.cpu().numpy(), probs.cpu().numpy()

    def train(self, fetch=True):
        """policy_optimization_agent.py:85-135: one learn step over the segments that closed.  Returns the loss (0 when
        no segment closed)."""
        streams, rows = self.segments.close()
        if len(streams) == 0:
            return 0
        self.training_iteration += 1
        return self._learn(self.segments.tables(streams, rows), True, fetch)

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
        d.n_actions = self.num_actions
        d.z = on.q.data_ptr()
        K, N, E = d.features, self.num_actions + 1, self.num_envs
        return ((E + 3) // 4) * 4 * (K * N + N + 1)

    def _launch_head(self, d, st):
        _lib.check(self.lib.cb200_actor_critic_head(ctypes.byref(d), st))
