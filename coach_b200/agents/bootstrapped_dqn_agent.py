"""Bootstrapped DQN learn step and ensemble acting on the GPU.  Drop-in for

  rl_coach/agents/bootstrapped_dqn_agent.py:26-92      parameters, learn_from_batch, observe (bootstrap masks)
  rl_coach/architectures/tensorflow_components/general_network.py:304-325,352-360
                                                     head copies, gradient rescale, total loss = sum over heads

The step is the DDQN schedule of dqn_agent.DQNAgent -- replay sample + gather, the feature layers of target(s'),
online(s) and online(s'), one head launch, the backward pass below the head, Adam, the same CUDA graphs -- with the
fused DQN head replaced by the ensemble head (cb200_ensemble_head_fused): K Q heads on one feature layer, per-head
double-DQN targets where the transition's bootstrap mask is set, per-head losses, and the gradient into the features
scaled by r = 1 / K.  The masks are the replay column ``info:mask`` (uint8 [K] per transition).

The reference never updates PER priorities in this agent and never uses importance weights: a prioritized memory is
refused.  There is no unfused path: a network the fused head cannot take is refused too.
"""
import ctypes

import numpy as np
import torch

from coach_b200 import _lib
from coach_b200.agents.dqn_agent import DQNAgent, DQNAgentParameters, DQNNetworkParameters
from coach_b200.base_parameters import MiddlewareScheme
from coach_b200.exploration_policies.bootstrapped import BootstrappedParameters
from coach_b200.memories.prioritized_experience_replay import PrioritizedExperienceReplayParameters


def draw_bootstrap_masks(n, p, heads):
    """n sequential ``np.random.binomial(1, p, heads)`` calls (bootstrapped_dqn_agent.py:88-92) -> uint8 [n, heads]"""
    out = np.zeros((int(n), int(heads)), dtype=np.uint8)
    for i in range(int(n)):
        out[i] = np.random.binomial(1, p, int(heads))
    return out


class BootstrappedDQNNetworkParameters(DQNNetworkParameters):
    """bootstrapped_dqn_agent.py:26-30"""

    def __init__(self):
        super().__init__()
        self.num_output_head_copies = 10
        self.rescale_gradient_from_head_by_factor = 1.0 / self.num_output_head_copies


class BootstrappedDQNAgentParameters(DQNAgentParameters):
    """bootstrapped_dqn_agent.py:33-42: the DQN parameters (ExperienceReplay of 1M transitions, batch 32) with the
    Bootstrapped exploration and the head copies"""

    def __init__(self):
        super().__init__()
        self.exploration = BootstrappedParameters()
        self.network_wrappers = {"main": BootstrappedDQNNetworkParameters()}

    @property
    def path(self):
        return 'coach_b200.agents.bootstrapped_dqn_agent:BootstrappedDQNAgent'


class BootstrappedDQNAgent(DQNAgent):
    double_dqn = True          # bootstrapped_dqn_agent.py:65-70: the online network on s' selects each head's action

    def __init__(self, agent_parameters, parent=None, observation_shape=None, num_actions=None, device=None,
                 seed=None):
        ap = agent_parameters
        if isinstance(ap.memory, PrioritizedExperienceReplayParameters):
            raise NotImplementedError("BootstrappedDQNAgent with a prioritized replay: the reference agent never "
                                      "updates priorities (bootstrapped_dqn_agent.py:57-86) nor reads importance "
                                      "weights")
        net = ap.network_wrappers["main"]
        self.num_heads = int(net.num_output_head_copies)
        if int(ap.exploration.architecture_num_q_heads) != self.num_heads:
            raise ValueError("exploration.architecture_num_q_heads (%d) differs from the network's "
                             "num_output_head_copies (%d)" % (ap.exploration.architecture_num_q_heads, self.num_heads))
        A = int(num_actions if num_actions is not None else ap.num_actions)
        obs = tuple(observation_shape if observation_shape is not None else ap.observation_shape)
        scheme = getattr(getattr(net, "middleware_parameters", None), "scheme", MiddlewareScheme.Medium)
        if A > 8:
            raise NotImplementedError("the fused ensemble head takes at most 8 actions per head (got %d)" % A)
        if len(obs) == 3 and scheme == MiddlewareScheme.Empty:
            raise NotImplementedError("the fused ensemble head needs a 256- or 512-wide feature layer; "
                                      "MiddlewareScheme.Empty puts the heads on the conv map")
        if "DuelingQHead" in getattr(net, "heads_parameters", ["QHead"]):
            raise NotImplementedError("BootstrappedDQNAgent uses QHead copies")
        self.grad_rescale = float(net.rescale_gradient_from_head_by_factor)
        self.share_prob = float(ap.exploration.bootstrapped_data_sharing_probability)
        super().__init__(agent_parameters, parent, observation_shape, num_actions, device, seed)
        if self.head_desc is None:
            raise NotImplementedError("the fused ensemble head cannot take this network (feature layer of %s)"
                                      % (self.net_def.middleware_units or "the embedder",))
        K, dev = self.num_heads, self.device
        self.targets = torch.zeros((self.batch_size, K * self.num_actions), dtype=torch.float32, device=dev)
        self.losses_dev = torch.zeros(K, dtype=torch.float32, device=dev)
        self._losses_host = torch.zeros(K, dtype=torch.float32, pin_memory=dev.type == "cuda")
        self._act_heads = {}             # number of environments -> (int32 head indices, [E, A] values) on the device

    # ---- the hooks of DQNAgent -----------------------------------------------------------------------------------------
    def _head_kwargs(self):
        return dict(head_copies=self.num_heads, head_grad_rescale=self.grad_rescale)

    def _extra_columns(self):
        return {"info:mask": torch.zeros((self.batch_size, self.num_heads), dtype=torch.uint8, device=self.device)}

    def _head_fusable(self, net):
        return net.online_s.ensemble_fusable() and net.target_s2.ensemble_fusable() and \
            net.online_s2.ensemble_fusable()

    def _build_head_desc(self):
        net, B, A, H = self.networks["main"], self.batch_size, self.num_actions, self.num_heads
        store, on = net.store, net.online_s
        wname, bname = self.net_def.trunk.names[-1]
        F = on.trunk.layers[-1].K
        d = _lib.EnsembleHeadDesc()
        dev = self.device
        self._head_keep = [torch.zeros(((B + 15) // 16) * 8 * ((F + 1) * H * A + H), dtype=torch.float32, device=dev)]
        self.q_select = torch.zeros((B, H * A), dtype=torch.float32, device=dev)
        d.h_next, d.h_online = net.target_s2.trunk.acts[-2].data_ptr(), on.trunk.acts[-2].data_ptr()
        d.h_select = net.online_s2.trunk.acts[-2].data_ptr()
        d.w_target, d.b_target = store.view(net.theta_target, wname).data_ptr(), store.view(net.theta_target, bname).data_ptr()
        d.w_online, d.b_online = store.view(net.theta, wname).data_ptr(), store.view(net.theta, bname).data_ptr()
        d.discount = float(self.ap.algorithm.discount)
        d.huber = 1 if net.params.replace_mse_with_huber_loss else 0
        d.batch, d.features, d.heads, d.n_actions = B, F, H, A
        d.grad_rescale = self.grad_rescale
        d.q_online, d.dq = on.q.data_ptr(), on.dq.data_ptr()
        d.q_next, d.q_select = net.target_s2.q.data_ptr(), self.q_select.data_ptr()
        on.bind_head_grads(d)
        d.workspace = self._head_keep[0].data_ptr()
        self.head_desc = d

    # ---- bootstrap masks (bootstrapped_dqn_agent.py:88-92) --------------------------------------------------------------
    def draw_bootstrap_masks(self, n):
        """the masks ``observe`` attaches to n transitions, one ``np.random.binomial(1, p, K)`` call each, in order (the
        draw consumes numpy's global stream even at p = 1).  Returns uint8 [n, K], for ``info['mask']`` /
        the ``info:mask`` column of ``memory.store_columns``."""
        return draw_bootstrap_masks(n, self.share_prob, self.num_heads)

    # ---- the learn step ----------------------------------------------------------------------------------------------
    def _part_forward(self, cols, per_libm):
        """feature layers of the three bindings, then the ensemble head: Q values, masked per-head targets, per-head
        losses, dL/dQ and the head's backward pass (cb200_ensemble_head_fused)"""
        net, d = self.networks["main"], self.head_desc
        with self._side_fwd:
            net.target_s2.forward_features()
        net.online_s.forward_features()
        net.online_s2.forward_features()
        self._side_fwd.join()
        d.actions, d.rewards, d.game_overs = cols["action"].data_ptr(), cols["reward"].data_ptr(), \
            cols["game_over"].data_ptr()
        d.masks = cols["info:mask"].data_ptr()
        d.targets, d.losses, d.loss = self.targets.data_ptr(), self.losses_dev.data_ptr(), self.loss_dev.data_ptr()
        _lib.check(self.lib.cb200_ensemble_head_fused(ctypes.byref(d), _lib.current_stream()))
        self._loss_host.copy_(self.loss_dev, non_blocking=True)      # final here: train() reads it early
        self._losses_host.copy_(self.losses_dev, non_blocking=True)

    def learn_from_batch(self, batch, fetch=True):
        """bootstrapped_dqn_agent.py:57-86 -> (total_loss, [loss of each head], unclipped gradient norm)"""
        if "info:mask" not in batch.columns:
            raise ValueError("the batch carries no bootstrap masks (replay column 'info:mask')")
        total, _, gnorm = super().learn_from_batch(batch, fetch)
        if fetch:
            return total, [float(x) for x in self._losses_host.numpy()], gnorm
        return total, [self.losses_dev[k] for k in range(self.num_heads)], gnorm

    # ---- acting --------------------------------------------------------------------------------------------------------
    def get_all_q_values_for_states(self, states):
        """every head's Q-values for E states, one forward pass: a CUDA tensor [E, K, A] (valid until the next call)"""
        q = super().get_all_q_values_for_states(states)
        return q.view(q.shape[0], self.num_heads, self.num_actions)

    def choose_actions(self, states, exploration_policy):
        """value_optimization_agent.py:90-115 with BatchedBootstrapped / BatchedUCB for E environments: the forward pass
        and the ensemble values of the policy's mode on the device (cb200_ensemble_action_values), then the
        epsilon-greedy arithmetic on the [E, A] read-back.  Returns (actions int64 [E], values [E, A] numpy)."""
        q = self.get_all_q_values_for_states(states)
        E, A = q.shape[0], self.num_actions
        bufs = self._act_heads.get(E)
        if bufs is None:
            bufs = self._act_heads[E] = (torch.zeros(E, dtype=torch.int32, device=self.device),
                                         torch.zeros((E, A), dtype=torch.float32, device=self.device))
        heads, vals = bufs
        mode = exploration_policy.ensemble_mode()
        if mode == _lib.ENSEMBLE_SELECT:
            heads.copy_(torch.from_numpy(np.asarray(exploration_policy.selected_head, dtype=np.int32)))
        _lib.check(self.lib.cb200_ensemble_action_values(q.data_ptr(), E, self.num_heads, A, mode, heads.data_ptr(),
                                                         float(exploration_policy.lamb), vals.data_ptr(),
                                                         _lib.current_stream()))
        v = vals.cpu().numpy()
        actions, _ = exploration_policy.get_actions(v)
        return actions, v
