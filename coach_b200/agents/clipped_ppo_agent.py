"""Clipped PPO learn step on the GPU.  Drop-in for

  rl_coach/agents/clipped_ppo_agent.py:157-207   fill_advantages   (V(s) over the rollout, GAE per episode, standardise)
  rl_coach/agents/clipped_ppo_agent.py:209-308   train_network     (epochs x minibatches: old policy from the frozen
                                                                    target network, surrogate + value losses, Adam)
  rl_coach/agents/clipped_ppo_agent.py:314-344   train             (normalise observations, sync target, truncate to
                                                                    num_consecutive_playing_steps, shuffle, epochs)
  rl_coach/agents/actor_critic_agent.py:108-125  GAE

Network (presets/Mujoco_ClippedPPO.py:30-37, use_separate_networks_per_head): value net obs->64->64->1 and policy net
obs->64->64->A, tanh, plus the state-independent ``policy_log_std`` variable; variables in TF creation order inside
ONE flat buffer, the network wrapper ``_Net`` (``main``: target copy, device-state Adam), so both sub-networks share a
single gradient norm / Adam / all-reduce launch.

Each phase evaluates the old policy once for the whole rollout (the target network is frozen during ``train_network``
-- the reference recomputes identical values every minibatch, clipped_ppo_agent.py:238-240 TODO-perf) and stages the
rollout into persistent training columns and a persistent permutation, grown only when a phase needs more rows.  The
minibatch step (row gather through the permutation at a device-side cursor -> value fwd/bwd -> policy fwd -> PPO head ->
policy bwd -> global norm -> Adam with device-side step state -> loss accumulators -> cursor += B) has launch parameters
that never change, so it is a ``GraphedKernels``: captured once and replayed for every minibatch of every epoch and
phase, 0 host work per minibatch, and rebuilt only when the columns grow or its clip epsilon changes.

Discrete actions (``num_actions``; heads/ppo_head.py:100-116): the policy net ends in Dense(A) ``policy_fc`` (glorot,
zero bias, no log-std), the old policy is the target network's softmax and the head is cb200_ppo_categorical_head.  It
reads the clipping schedule's value from a device rescaler written at the start of each phase, so one graph follows a
moving schedule; the continuous head takes fp32(epsilon * value) as a launch argument, so a new value rebuilds its step.

Acting (clipped_ppo_agent.py:346-354): the pre-network filter without a statistics update, the policy net on the
device, then Categorical (cb200_policy_act: np.random.choice on host uniforms, or the first argmax in evaluation) or
AdditiveNoise on [mean, exp(log std)] (cb200_ppo_gaussian_act); the clipping schedule steps once per environment in
training and evaluation, as the reference steps it in every choose_action.
"""
import random

import numpy as np
import torch

from coach_b200 import _lib, parallel, rl_math
from coach_b200.agents.actor_critic_agent import CategoricalParameters
from coach_b200.agents.ddpg_agent import GraphedKernels, _Net
from coach_b200.architectures.layers import Dense, Workspace
from coach_b200.architectures.network import ParamStore, Sequential
from coach_b200.base_parameters import AgentParameters, AlgorithmParameters, EnvironmentSteps, NetworkParameters
from coach_b200.core_types import DeviceBatch
from coach_b200.exploration_policies.additive_noise import AdditiveNoiseParameters
from coach_b200.filters.filter import InputFilter, ObservationNormalizationFilter
from coach_b200.memories.episodic_experience_replay import EpisodicExperienceReplayParameters
from coach_b200.schedules import ConstantSchedule
from coach_b200.utils import dynamic_import_and_instantiate_module_from_params

# discrete actions: the categorical softmax and draw of cb200_policy_act (acting and the old policy) take 1 .. 18 actions,
# Atari's full action set; cb200_ppo_categorical_head itself takes up to 32
MAX_DISCRETE_ACTIONS = 18


class ClippedPPONetworkParameters(NetworkParameters):
    def __init__(self):
        super().__init__()
        self.batch_size = 64
        self.optimizer_type = 'Adam'
        self.clip_gradients = None
        self.use_separate_networks_per_head = True
        self.create_target_network = True
        # (learning rate, Adam epsilon / beta2 keep the NetworkParameters defaults like the reference class does; the
        # Mujoco preset sets 3e-4 / 1e-5 / 0.999: coach_b200/presets/Mujoco_ClippedPPO.py)
        self.hidden_units = 64


class ClippedPPOAlgorithmParameters(AlgorithmParameters):
    def __init__(self):
        super().__init__()
        self.gae_lambda = 0.95
        self.clip_likelihood_ratio_using_epsilon = 0.2
        self.estimate_state_value_using_gae = True
        self.beta_entropy = 0.01  # should be 0 for mujoco
        self.num_consecutive_playing_steps = EnvironmentSteps(2048)
        self.optimization_epochs = 10
        self.clipping_decay_schedule = ConstantSchedule(1)
        self.act_for_full_episodes = True
        self.update_pre_network_filters_state_on_train = True
        self.update_pre_network_filters_state_on_inference = False
        # the reference trains on dataset[:num_consecutive_playing_steps] only (clipped_ppo_agent.py:330-331); set to
        # False to train on the whole rollout (the 64-env synthetic configuration of BASELINE config 3)
        self.truncate_dataset_to_playing_steps = True


class ClippedPPOAgentParameters(AgentParameters):
    def __init__(self):
        super().__init__(algorithm=ClippedPPOAlgorithmParameters(), memory=EpisodicExperienceReplayParameters(),
                         networks={"main": ClippedPPONetworkParameters()})
        self.exploration = {"DiscreteActionSpace": CategoricalParameters(),
                            "BoxActionSpace": AdditiveNoiseParameters()}
        self.pre_network_filter = InputFilter()
        self.pre_network_filter.add_observation_filter('observation', 'normalize_observation',
                                                       ObservationNormalizationFilter(name='normalize_observation'))

    @property
    def path(self):
        return 'coach_b200.agents.clipped_ppo_agent:ClippedPPOAgent'


class PPONetworkDef(object):
    """flat parameter layout of the two sub-networks (general_network.py:244-349 creation order)"""

    def __init__(self, device, obs_dim, action_dim, hidden=64, discrete=False):
        """discrete: the policy net ends in the logits Dense(action_dim) (policy_fc) and has no log-std variable"""
        self.device = torch.device(device)
        self.D, self.A, self.Hd = int(obs_dim), int(action_dim), int(hidden)
        self.discrete = bool(discrete)
        s = self.store = ParamStore(self.device)
        self.v_seq = Sequential([Dense(self.D, hidden, "tanh"), Dense(hidden, hidden, "tanh"), Dense(hidden, 1, None)],
                                s, "main/online/network_0")
        s.add("main/online/network_0/gradients_from_head_0-0_rescalers", ())
        self.p_seq = Sequential([Dense(self.D, hidden, "tanh"), Dense(hidden, hidden, "tanh"),
                                 Dense(hidden, self.A, None)], s, "main/online/network_1")
        self.logstd_name = None if self.discrete else \
            s.add("main/online/network_1/ppo_head_0/policy_log_std", (self.A,))
        s.add("main/online/network_1/gradients_from_head_1-0_rescalers", ())
        s.finalize()

    def init(self, generator=None):
        self.store.init_glorot(generator)
        if self.discrete:
            return                                  # policy_fc: TF's default glorot kernel and zero bias (:109)
        self.store.view(self.store.theta, self.logstd_name).zero_()          # np.zeros((1, num_actions)), :129-133
        # policy mean layer: normalized_columns_initializer(0.01) (ppo_head.py:121, head.py:28-33)
        name = self.p_seq.names[2][0]
        w = torch.randn(self.Hd, self.A, generator=generator)
        w *= 0.01 / torch.sqrt((w * w).sum(dim=0, keepdim=True))
        self.store.view(self.store.theta, name).copy_(w)


class ClippedPPOAgent(object):
    def __init__(self, agent_parameters, parent=None, observation_dim=None, action_dim=None, device=None, seed=None,
                 num_actions=None, action_low=None, action_high=None):
        """num_actions: a discrete action space of that many actions; action_dim: a Box action space of that many
        dimensions.  Give exactly one.  action_low / action_high: the Box bounds (scalars or per dimension), needed only
        to act (AdditiveNoise refuses unbounded actions)."""
        self.ap = agent_parameters
        # ---- refusals, before anything touches the GPU ----
        if (num_actions is None) == (action_dim is None):
            raise ValueError("give exactly one of num_actions (discrete actions) or action_dim (continuous actions)")
        self.discrete = num_actions is not None
        if self.discrete:
            if not 1 <= int(num_actions) <= MAX_DISCRETE_ACTIONS:
                raise ValueError("discrete ClippedPPO takes 1 .. %d actions (the categorical acting and softmax code), "
                                 "got %d" % (MAX_DISCRETE_ACTIONS, num_actions))
            if parallel.world()[1] > 1:
                raise ValueError("discrete ClippedPPO runs on one rank")
        self.action_low = self.action_high = None
        if not self.discrete and action_low is not None and action_high is not None:
            self.action_low = np.broadcast_to(np.asarray(action_low, dtype=np.float64), (int(action_dim),))
            self.action_high = np.broadcast_to(np.asarray(action_high, dtype=np.float64), (int(action_dim),))
        ex = getattr(self.ap, "exploration", None)
        box = ex.get("BoxActionSpace") if isinstance(ex, dict) else ex
        self.noise_schedule = None if self.discrete else getattr(box, "noise_schedule", None)
        self.lib = _lib.load()
        self.device = torch.device(device if device is not None else "cuda")
        self.D, self.A = int(observation_dim), int(num_actions if self.discrete else action_dim)
        net_p = self.ap.network_wrappers["main"]
        self.B = int(net_p.batch_size)
        self.memory = dynamic_import_and_instantiate_module_from_params(
            self.ap.memory, extra_kwargs={"device": self.device, "discount": self.ap.algorithm.discount})
        self.pre_network_filter = self.ap.pre_network_filter
        if self.pre_network_filter is not None:
            self.pre_network_filter.set_device(self.device)
            for flt in self.pre_network_filter._observation_filters.values():
                for f in flt.values():
                    if hasattr(f, "set_shape"):
                        f.set_shape([self.D])
        self.net = PPONetworkDef(self.device, self.D, self.A, getattr(net_p, "hidden_units", 64), self.discrete)
        gen = torch.Generator().manual_seed(int(seed)) if seed is not None else None
        self.net.init(gen)
        st = self.net.store
        self.main = _Net(self.lib, st, net_p, self.device)
        # the captured minibatch step holds its workspace's pointer; rollout-sized and acting passes, which may grow
        # theirs, use another
        self.ws, self.ws_rollout = Workspace(self.device), Workspace(self.device)
        dev, B = self.device, self.B
        f32 = lambda *s: torch.zeros(s, dtype=torch.float32, device=dev)     # noqa: E731
        self.mb = self._columns(B)             # the minibatch the step gathers
        self.v_inst = self.net.v_seq.instantiate(self.lib, self.ws, B, self.mb["states"], st.theta, st.grad,
                                                 train=True)
        self.p_inst = self.net.p_seq.instantiate(self.lib, self.ws, B, self.mb["states"], st.theta, st.grad,
                                                 train=True)
        self.scalars = f32(5)
        self.v_loss = f32(1)
        self.v_acc, self.p_acc = f32(1), f32(1)       # one epoch's sums of the value loss and the policy loss
        self.cursor = torch.zeros(1, dtype=torch.int64, device=dev)
        # the clipping schedule's value as the discrete head reads it (fp32, written at the start of every phase)
        self.clip_rescaler = f32(1)
        self.clip_eps = None       # the head's fp32 clip epsilon launch argument, held by the step's graph
        self.graph_captures = 0
        self._step = None          # the minibatch step (GraphedKernels)
        self._rows = None          # persistent training columns (capacity, dict, permutation, argmax scratch)
        self._full = {}            # rollout-sized forward instances, keyed by N
        self._act = {}             # acting buffers, keyed by the number of environments
        self.training_iteration = 0
        self.total_steps_counter = 0
        self.last_training_phase_step = 0
        self.use_cuda_graph = True
        self.last_losses = None

    @property
    def is_on_policy(self) -> bool:
        return True

    def sync(self):
        """online -> target: the frozen "old policy" (network_wrapper.py:94-107, clipped_ppo_agent.py:326)"""
        self.main.sync()

    # ---- rollout-sized forward passes ------------------------------------------------------------------------------
    def _full_instances(self, N):
        if N not in self._full:
            st = self.net.store
            x = torch.zeros((N, self.D), dtype=torch.float32, device=self.device)
            v = self.net.v_seq.instantiate(self.lib, self.ws_rollout, N, x, st.theta)
            p_old = self.net.p_seq.instantiate(self.lib, self.ws_rollout, N, x, self.main.target)
            self._full = {N: (x, v, p_old)}           # keep only the latest size
        return self._full[N]

    def fill_advantages(self, states_norm, rewards, game_overs):
        """clipped_ppo_agent.py:157-207.  Returns (advantages fp64 standardised, value targets fp64, n_valid)."""
        N = states_norm.shape[0]
        x, v_full, _ = self._full_instances(N)
        x.copy_(states_norm)
        values = v_full.forward().reshape(-1)                                   # V(s_t), fp32
        return rl_math.fill_advantages(rewards, values, game_overs, self.ap.algorithm.discount,
                                       self.ap.algorithm.gae_lambda)

    # ---- training columns and one minibatch ----------------------------------------------------------------------
    def _columns(self, n):
        """n rows of what the minibatch step trains on: the actions (int64 [n] discrete, fp32 [n, A] continuous) and
        the old policy (the target network's probabilities or means, [n, A])"""
        f32 = lambda *s: torch.zeros(s, dtype=torch.float32, device=self.device)      # noqa: E731
        actions = torch.zeros(n, dtype=torch.int64, device=self.device) if self.discrete else f32(n, self.A)
        return dict(states=f32(n, self.D), actions=actions, advantages=f32(n), value_targets=f32(n, 1),
                    old_policy=f32(n, self.A))

    def _training_rows(self, n_rows):
        """the persistent training columns, the permutation of their rows and the argmax scratch of the old policy's
        softmax; grown when a phase trains on more rows, which rebuilds the minibatch step (its graph holds their
        pointers)"""
        if self._rows is None or self._rows[0] < n_rows:
            i64 = lambda: torch.zeros(n_rows, dtype=torch.int64, device=self.device)      # noqa: E731
            self._rows = (n_rows, self._columns(n_rows), i64(), i64())
            self._step = None
        return self._rows[1:]

    def _minibatch_kernels(self):
        """all launches of one minibatch step on the rows perm[cursor, cursor + B) of the training columns; parameters
        independent of the minibatch index"""
        lib, st = self.lib, _lib.current_stream()
        store, mb = self.main.store, self.mb
        alg, net_p = self.ap.algorithm, self.ap.network_wrappers["main"]
        _, cols, perm, _ = self._rows
        arr, cnt = _lib.make_columns([(cols[k].data_ptr(), t.data_ptr(), t.element_size() * int(np.prod(t.shape[1:])))
                                      for k, t in mb.items()])
        _lib.check(lib.cb200_gather_at(arr, cnt, perm.data_ptr(), self.cursor.data_ptr(), self.B, st))
        v = self.v_inst.forward()
        mu = self.p_inst.forward()
        # VHead: MSE(v, gae_based_value_target), loss weight 1 (v_head.py:41-44, head.py:172-177)
        _lib.check(lib.cb200_regression_head_loss_grad(v.data_ptr(), mb["value_targets"].data_ptr(), None,
                                                       self.B, 1, 0, 1.0, self.v_inst.d_out.data_ptr(),
                                                       self.v_loss.data_ptr(), st))
        if self.discrete:
            _lib.check(lib.cb200_ppo_categorical_head(mu.data_ptr(), mb["actions"].data_ptr(),
                                                      mb["old_policy"].data_ptr(), mb["advantages"].data_ptr(),
                                                      self.B, self.A, float(self.clip_eps),
                                                      self.clip_rescaler.data_ptr(), float(alg.beta_entropy),
                                                      self.p_inst.d_out.data_ptr(), self.scalars.data_ptr(), st))
        else:
            logstd = store.view(store.theta, self.net.logstd_name)
            old_logstd = store.view(self.main.target, self.net.logstd_name)
            d_logstd = store.view(store.grad, self.net.logstd_name)
            _lib.check(lib.cb200_ppo_continuous_head(mu.data_ptr(), logstd.data_ptr(), mb["actions"].data_ptr(),
                                                     mb["old_policy"].data_ptr(), old_logstd.data_ptr(),
                                                     mb["advantages"].data_ptr(), self.B, self.A,
                                                     float(self.clip_eps), float(alg.beta_entropy),
                                                     self.p_inst.d_out.data_ptr(), d_logstd.data_ptr(),
                                                     self.scalars.data_ptr(), st))
        self.v_inst.backward()
        self.p_inst.backward()
        self.main.apply(self.ws, ("ClipByGlobalNorm", net_p.clip_gradients) if net_p.clip_gradients else None)
        _lib.check(lib.cb200_axpby_2d(self.v_loss.data_ptr(), 1, 1, 1, 1.0, 1.0, self.v_acc.data_ptr(), 1, st))
        _lib.check(lib.cb200_axpby_2d(self.scalars.data_ptr(), 1, 1, 1, 1.0, 1.0, self.p_acc.data_ptr(), 1, st))
        _lib.check(lib.cb200_add_i64(self.cursor.data_ptr(), self.B, st))
        self.graph_captures += torch.cuda.is_current_stream_capturing()      # the step's graph is capturing this call

    def train_network(self, n_rows, epochs):
        """clipped_ppo_agent.py:209-308 on the first n_rows rows of the training columns.  Returns the mean [value loss,
        policy loss] of the last epoch as device tensors."""
        alg, B = self.ap.algorithm, self.B
        n_full = n_rows // B
        if n_rows % B:
            raise ValueError("the rollout length (%d) must be a multiple of the batch size (%d)" % (n_rows, B))
        # the clipping schedule's value: the discrete head reads it from the device rescaler, the continuous head takes
        # fp32(epsilon * value) as its launch argument.  The step's graph holds that argument, so a new value rebuilds
        # the step.
        value = float(alg.clipping_decay_schedule.current_value)
        self.clip_rescaler.fill_(value)
        clip_eps = np.float32(float(alg.clip_likelihood_ratio_using_epsilon) * (1.0 if self.discrete else value))
        if self._step is None or clip_eps != self.clip_eps:
            self.clip_eps = clip_eps
            self._step = GraphedKernels(self._minibatch_kernels, self.device)
            # several ranks run the step eagerly, their all-reduces outside any graph
            self._step.enabled &= self.use_cuda_graph and self.device.type == "cuda" and parallel.world()[1] == 1
        perm = self._rows[2]
        # one pinned row per epoch: an epoch's asynchronous copy may still be queued when the host shuffles the next
        perm_host = torch.zeros((epochs, n_rows), dtype=torch.int64, pin_memory=self.device.type == "cuda")
        order = list(range(n_rows))
        for epoch in range(epochs):
            random.shuffle(order)                                   # batch.shuffle(), core_types.py:452-468
            perm_host[epoch].copy_(torch.tensor(order, dtype=torch.int64))
            perm[:n_rows].copy_(perm_host[epoch], non_blocking=True)
            self.cursor.zero_()
            self.v_acc.zero_()
            self.p_acc.zero_()
            for _ in range(n_full):
                self._step()
        self.last_losses = (self.v_acc / n_full, self.p_acc / n_full)
        return self.last_losses

    # ---- driver ----------------------------------------------------------------------------------------------------
    def _should_train(self):
        steps = self.ap.algorithm.num_consecutive_playing_steps
        should = (self.total_steps_counter - self.last_training_phase_step) >= steps.num_steps
        should = should and self.memory.num_transitions_in_complete_episodes() > 0
        if should:
            self.last_training_phase_step = self.total_steps_counter
        return should

    def train(self):
        """clipped_ppo_agent.py:314-344"""
        if not self._should_train():
            return None
        alg = self.ap.algorithm
        batch = self.memory.transitions_batch()
        if self.pre_network_filter is not None:
            batch = self.pre_network_filter.filter(batch, deep_copy=False,
                                                   update_internal_state=alg.update_pre_network_filters_state_on_train)
        states = batch.states(["observation"])["observation"].to(torch.float32)
        actions = batch.actions().reshape((batch.size,) + self.mb["actions"].shape[1:])
        for _ in range(alg.num_consecutive_training_steps):
            self.sync()
            adv, tgt, n_valid = self.fill_advantages(states, batch.rewards(), batch.game_overs())
            n_rows = batch.size
            if alg.truncate_dataset_to_playing_steps:
                n_rows = min(n_rows, alg.num_consecutive_playing_steps.num_steps)
            if n_rows < self.B:
                raise ValueError("the rollout holds %d transitions, fewer than one minibatch of %d: nothing to train on "
                                 "(the reference would train on one partial minibatch)" % (n_rows, self.B))
            # whole minibatches only: the reference also trains on the partial tail batch (clipped_ppo_agent.py:225,
            # ceil(size / batch_size)); with the presets' 2048-step rollouts and batch 64 there is none
            n_rows = (n_rows // self.B) * self.B
            cols, _, argmax = self._training_rows(n_rows)
            _, _, p_old = self._full_instances(batch.size)
            old = p_old.forward()                                      # frozen target network, whole rollout at once
            if self.discrete:
                # the old policy's probabilities: the categorical softmax of the acting code (its argmax is not used)
                _lib.check(self.lib.cb200_policy_act(old.data_ptr(), n_rows, self.A, 0, None, None, None,
                                                     argmax.data_ptr(), cols["old_policy"].data_ptr(), None, None,
                                                     _lib.current_stream()))
            else:
                cols["old_policy"][:n_rows].copy_(old[:n_rows])
            cols["states"][:n_rows].copy_(states[:n_rows])
            cols["actions"][:n_rows].copy_(actions[:n_rows])
            cols["advantages"][:n_rows].copy_(adv[:n_rows])
            cols["value_targets"][:n_rows].copy_(tgt[:n_rows].reshape(-1, 1))
            self.train_network(n_rows, alg.optimization_epochs)
        self.memory.clean()                                            # post_training_commands :310-312
        self.training_iteration += 1
        return None

    # ---- acting ------------------------------------------------------------------------------------------------------
    def _act_buffers(self, E):
        if E not in self._act:
            dev, pin = self.device, self.device.type == "cuda"
            x = torch.zeros((E, self.D), dtype=torch.float32, device=dev)
            inst = self.net.p_seq.instantiate(self.lib, self.ws_rollout, E, x, self.net.store.theta)
            shape = (E,) if self.discrete else (E, self.A)
            self._act = {E: dict(x=x, inst=inst, actions=torch.zeros(E, dtype=torch.int64, device=dev),
                                 probs=torch.zeros((E, self.A), dtype=torch.float32, device=dev),
                                 cont=torch.zeros((E, self.A), dtype=torch.float64, device=dev),
                                 stds=torch.zeros((E, self.A), dtype=torch.float32, device=dev),
                                 d_dev=torch.zeros(shape, dtype=torch.float64, device=dev),
                                 d_host=torch.zeros(shape, dtype=torch.float64, pin_memory=pin))}
        return self._act[E]

    def choose_actions(self, states, evaluation=False, uniforms=None, normals=None):
        """clipped_ppo_agent.py:346-354 and policy_optimization_agent.py:160-185 for E environments.  The states pass
        the pre-network filter without a statistics update (update_pre_network_filters_state_on_inference False), and
        the clipping schedule is stepped E times, in training and evaluation.
        Discrete: Categorical.get_action on softmax(logits): np.random.choice(A, p) on ``uniforms`` [E] (default
        np.random.random_sample(E), what E successive choice calls draw) in training, the first argmax in evaluation.
        Returns (actions int64 [E], probabilities float32 [E, A]).
        Continuous: AdditiveNoise.get_action([mean, std]), std = exp(policy_log_std): np.random.normal(mean, std) =
        (double) mean + (double) std * n on ``normals`` [E, A] (default np.random.standard_normal((E, A))) in training,
        stepping the noise schedule E times; the fp32 mean in evaluation.  Returns (actions [E, A]: float64 in
        training, float32 in evaluation, means float32 [E, A], stds float32 [E, A])."""
        if not self.discrete and (self.action_low is None or not (np.all(np.isfinite(self.action_low)) and
                                                                  np.all(np.isfinite(self.action_high)))):
            raise ValueError("Additive noise exploration requires bounded actions: build the agent with finite "
                             "action_low / action_high")
        alg, A = self.ap.algorithm, self.A
        s = torch.as_tensor(np.asarray(states, dtype=np.float32)).reshape(-1, self.D)
        E = int(s.shape[0])
        buf = self._act_buffers(E)
        x = s.to(self.device)
        if self.pre_network_filter is not None:
            for flt in self.pre_network_filter._observation_filters.values():
                for f in flt.values():
                    x = f.filter(x, update_internal_state=alg.update_pre_network_filters_state_on_inference)
        buf["x"].copy_(x)
        z = buf["inst"].forward()
        for _ in range(E):
            alg.clipping_decay_schedule.step()
        d_ptr = None
        if not evaluation:
            if self.discrete:
                d = np.random.random_sample(E) if uniforms is None else np.asarray(uniforms, dtype=np.float64)
            else:
                d = np.random.standard_normal((E, A)) if normals is None else np.asarray(normals, dtype=np.float64)
                for _ in range(E):
                    self.noise_schedule.step()
            torch.cuda.current_stream().synchronize()            # the previous call's copy has left the staging
            buf["d_host"].numpy()[...] = d.reshape(buf["d_host"].shape)
            buf["d_dev"].copy_(buf["d_host"], non_blocking=True)
            d_ptr = buf["d_dev"].data_ptr()
        st = _lib.current_stream()
        if self.discrete:
            _lib.check(self.lib.cb200_policy_act(z.data_ptr(), E, A, 0, None, d_ptr, None, buf["actions"].data_ptr(),
                                                 buf["probs"].data_ptr(), None, None, st))
            return buf["actions"].cpu().numpy(), buf["probs"].cpu().numpy()
        logstd = self.net.store.view(self.net.store.theta, self.net.logstd_name)
        _lib.check(self.lib.cb200_ppo_gaussian_act(z.data_ptr(), logstd.data_ptr(), E, A, d_ptr,
                                                   buf["cont"].data_ptr(), buf["stds"].data_ptr(), st))
        means, stds = z.cpu().numpy().copy(), buf["stds"].cpu().numpy()
        return (means.copy() if evaluation else buf["cont"].cpu().numpy()), means, stds

    # ---- checkpoint host state ---------------------------------------------------------------------------------------
    def checkpoint_state(self):
        """the clipping schedule's value, and the noise schedule's for continuous actions (the network goes through the
        ``main`` checkpoint item)"""
        state = dict(clipping=float(self.ap.algorithm.clipping_decay_schedule.current_value))
        if not self.discrete:
            state["noise"] = float(self.noise_schedule.current_value)
        return state

    def restore_checkpoint_state(self, state):
        self.ap.algorithm.clipping_decay_schedule.current_value = state["clipping"]
        if "noise" in state:
            self.noise_schedule.current_value = state["noise"]
