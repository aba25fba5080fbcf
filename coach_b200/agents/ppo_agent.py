"""PPO (KL-penalty Proximal Policy Optimization) for continuous actions on the GPU.  Drop-in for

  rl_coach/agents/ppo_agent.py:40-133     PPOCritic/ActorNetworkParameters, PPOAlgorithmParameters, PPOAgentParameters
  rl_coach/agents/ppo_agent.py:156-195    fill_advantages   (V(s) from the critic before it trains, GAE per episode or
                                                              A_VALUE = R - V, standardised with np.std)
  rl_coach/agents/ppo_agent.py:197-327    train_value_network / train_policy_network (in-order minibatches, not shuffled)
  rl_coach/agents/ppo_agent.py:329-391    update_kl_coefficient / post_training_commands / train
  heads/ppo_head.py:52-144                the KL-penalty policy head (cb200_ppo_kl_head)
  heads/v_head.py                         the critic's V head: MSE on the Monte Carlo returns
  policy_optimization_agent.py:160-185    choose_action with AdditiveNoise on [mean, std] (cb200_ppo_gaussian_act)

Two separate networks, each with its own flat store, target buffer and device-state Adam (``_Net``):
  actor   obs -> Dense tanh -> Dense tanh -> Dense(A) policy mean (linear, normalized_columns(0.01)), plus the
          state-independent ``policy_log_std`` variable (zeros)
  critic  obs -> Dense tanh -> Dense tanh -> Dense(1) (normalized_columns(1.0))
with the preset's 64 / 64 or the reference defaults 256 (embedder Medium) / 512 (middleware Medium).

One training phase: sync both targets; V(s) over the rollout; advantages; the old policy's mean over the rollout from
the frozen actor target (once per phase: the reference recomputes the same values every minibatch); one critic epoch
and ten actor epochs of floor(N / B) in-order minibatches.  Each minibatch step (row gather at a device-side cursor ->
forward -> head -> backward -> global norm -> Adam -> cursor += B) has constant launch parameters, so the critic step
and the actor step are each captured once as a CUDA graph and replayed: no host work per minibatch.  The KL
coefficient lives in device memory, so the captured actor step reads the current value.  Each actor minibatch adds
its scalars (loss, KL, entropy, mean ratio, surrogate) to a device accumulator that is cleared per epoch; after the
last epoch one device-to-host read gives the KL mean that updates the coefficient.

A rollout of fewer than one minibatch of rows makes the reference fail; here ``train`` raises ValueError before any
network is touched.  Refused with ValueError when the agent is built, before anything touches the GPU: discrete
actions, unbounded actions, a clip epsilon (that is ClippedPPO), an optimizer other than Adam, a rescaler other than
GAE / A_VALUE, more than one rank, widths other than 64 / 64 and 256 / 512, actor and critic batch sizes that differ,
more than 32 action dimensions.
"""
import numpy as np
import torch

from coach_b200 import _lib, parallel, rl_math
from coach_b200.agents.actor_critic_agent import PolicyGradientRescaler
from coach_b200.agents.ddpg_agent import GraphedKernels, _Net
from coach_b200.architectures.layers import Dense, Workspace
from coach_b200.architectures.network import ParamStore, Sequential
from coach_b200.base_parameters import (AgentParameters, AlgorithmParameters, EnvironmentSteps,
                                        InputEmbedderParameters, MiddlewareParameters, NetworkParameters,
                                        middleware_units, scheme_layers)
from coach_b200.exploration_policies.additive_noise import AdditiveNoiseParameters
from coach_b200.memories.episodic_experience_replay import EpisodicExperienceReplayParameters
from coach_b200.utils import dynamic_import_and_instantiate_module_from_params

MAX_ACTION_DIM = 32                # cb200_ppo_kl_head: one lane per action dimension
WIDTHS = ((64, 64), (256, 512))    # (embedder, middleware): Mujoco_PPO, and the reference's Medium / Medium defaults
EPOCHS_CRITIC, EPOCHS_ACTOR = 1, 10     # ppo_agent.py:379-380


class PPOCriticNetworkParameters(NetworkParameters):
    """ppo_agent.py:40-49"""

    def __init__(self):
        super().__init__()
        self.input_embedders_parameters = {'observation': InputEmbedderParameters()}
        self.middleware_parameters = MiddlewareParameters()
        self.async_training = True
        self.l2_regularization = 0
        self.create_target_network = True
        self.batch_size = 128


class PPOActorNetworkParameters(NetworkParameters):
    """ppo_agent.py:52-62"""

    def __init__(self):
        super().__init__()
        self.input_embedders_parameters = {'observation': InputEmbedderParameters()}
        self.middleware_parameters = MiddlewareParameters()
        self.optimizer_type = 'Adam'
        self.async_training = True
        self.l2_regularization = 0
        self.create_target_network = True
        self.batch_size = 128


class PPOAlgorithmParameters(AlgorithmParameters):
    """ppo_agent.py:65-124"""

    def __init__(self):
        super().__init__()
        self.policy_gradient_rescaler = PolicyGradientRescaler.GAE
        self.gae_lambda = 0.96
        self.target_kl_divergence = 0.01
        self.initial_kl_coefficient = 1.0
        self.high_kl_penalty_coefficient = 1000
        self.clip_likelihood_ratio_using_epsilon = None
        self.value_targets_mix_fraction = 0.1
        self.estimate_state_value_using_gae = True
        self.use_kl_regularization = True
        self.beta_entropy = 0.01
        self.num_consecutive_playing_steps = EnvironmentSteps(5000)
        self.act_for_full_episodes = True


class PPOAgentParameters(AgentParameters):
    """ppo_agent.py:127-137 (continuous actions: AdditiveNoise acting on the head's [mean, std])"""

    def __init__(self):
        super().__init__(algorithm=PPOAlgorithmParameters(), memory=EpisodicExperienceReplayParameters(),
                         networks={"critic": PPOCriticNetworkParameters(), "actor": PPOActorNetworkParameters()})
        self.exploration = AdditiveNoiseParameters()

    @property
    def path(self):
        return 'coach_b200.agents.ppo_agent:PPOAgent'


def network_widths(net_p):
    """(embedder width, middleware width) of a PPO network's schemes; ValueError unless one of WIDTHS"""
    emb = scheme_layers(net_p.input_embedders_parameters['observation'].scheme)
    emb = (256,) if emb is None else tuple(int(d.units) for d in emb)
    mid = tuple(middleware_units(net_p.middleware_parameters.scheme))
    if len(emb) != 1 or len(mid) != 1 or (emb[0], mid[0]) not in WIDTHS:
        raise ValueError("PPO networks are one embedder and one middleware Dense layer of widths 64 / 64 or "
                         "256 / 512, got %s / %s" % (emb, mid))
    return emb[0], mid[0]


def _mlp(store, prefix, D, widths, out, head, std):
    """obs -> embedder Dense tanh -> middleware Dense tanh -> head Dense(out) (normalized_columns(std))"""
    e, m = widths
    seq = Sequential([Dense(D, e, "tanh")], store, prefix + "/observation")
    mid = Sequential([Dense(e, m, "tanh")], store, prefix + "/middleware_fc_embedder")
    top = Sequential([Dense(m, out, None)], store, prefix + "/" + head)
    seq.layers += mid.layers + top.layers
    seq.names += mid.names + top.names
    store.normalized_columns[top.names[0][0]] = [(0, out, std)]
    return seq


class PPOAgent(object):
    def __init__(self, agent_parameters, parent=None, observation_dim=None, action_dim=None, action_low=None,
                 action_high=None, device=None, seed=None, continuous_actions=True, use_cuda_graph=True):
        """action_low / action_high: the finite bounds of the Box action space (scalars or per dimension; AdditiveNoise
        refuses unbounded ones).  continuous_actions=False stands for a discrete action space, which is refused."""
        self.ap = ap = agent_parameters
        alg, a_p, c_p = ap.algorithm, ap.network_wrappers["actor"], ap.network_wrappers["critic"]
        # ---- refusals, before anything touches the GPU ----
        if not continuous_actions:
            raise ValueError("PPO on this GPU path supports continuous (Box) action spaces only")
        if action_low is None or action_high is None or \
                not (np.all(np.isfinite(action_low)) and np.all(np.isfinite(action_high))):
            raise ValueError("Additive noise exploration requires bounded actions")
        if not 1 <= int(action_dim) <= MAX_ACTION_DIM:
            raise ValueError("cb200_ppo_kl_head takes 1 .. %d action dimensions, got %d" % (MAX_ACTION_DIM, action_dim))
        if alg.clip_likelihood_ratio_using_epsilon is not None:
            raise ValueError("PPO uses the KL penalty: clip_likelihood_ratio_using_epsilon must be None "
                             "(the clipped objective is ClippedPPOAgent)")
        for name, p in (("actor", a_p), ("critic", c_p)):
            if p.optimizer_type != 'Adam':
                raise ValueError("the %s network's optimizer %r is not supported (Adam only)" % (name, p.optimizer_type))
        if alg.policy_gradient_rescaler not in (PolicyGradientRescaler.GAE, PolicyGradientRescaler.A_VALUE):
            raise ValueError("PPO advantages are GAE or A_VALUE, got %s" % (alg.policy_gradient_rescaler,))
        if parallel.world()[1] > 1:
            raise ValueError("PPO runs on one rank")
        self.widths = {"actor": network_widths(a_p), "critic": network_widths(c_p)}
        if int(a_p.batch_size) != int(c_p.batch_size):
            raise ValueError("actor and critic batch sizes differ (%d, %d)" % (a_p.batch_size, c_p.batch_size))
        self.D, self.A = D, A = int(observation_dim), int(action_dim)
        self.B = B = int(a_p.batch_size)
        self.action_low = np.broadcast_to(np.asarray(action_low, dtype=np.float64), (A,))
        self.action_high = np.broadcast_to(np.asarray(action_high, dtype=np.float64), (A,))
        self.noise_schedule = ap.exploration.noise_schedule

        self.lib = _lib.load()
        self.device = dev = torch.device(device if device is not None else "cuda")
        self.memory = dynamic_import_and_instantiate_module_from_params(
            ap.memory, extra_kwargs={"device": dev, "discount": alg.discount})
        gen = torch.Generator().manual_seed(int(seed)) if seed is not None else None
        # ---- networks (TF creation order: critic first, ppo_agent.py:133) ----
        sc = ParamStore(dev)
        self.critic_seq = _mlp(sc, "critic/online/network_0", D, self.widths["critic"], 1, "v_values_head_0", 1.0)
        sc.finalize()
        sc.init_glorot(gen)
        sa = ParamStore(dev)
        self.actor_seq = _mlp(sa, "actor/online/network_0", D, self.widths["actor"], A, "ppo_head_0/policy_mean", 0.01)
        self.logstd_name = sa.add("actor/online/network_0/ppo_head_0/policy_log_std", (A,))   # zeros, :133-136
        sa.finalize()
        sa.init_glorot(gen)
        self.critic, self.actor = _Net(self.lib, sc, c_p, dev), _Net(self.lib, sa, a_p, dev)
        self.critic.sync()
        self.actor.sync()
        # the captured minibatch steps hold their workspace's pointer; rollout-sized and acting passes, which may grow
        # theirs, use another
        self.ws, self.ws_rollout = Workspace(dev), Workspace(dev)
        f32 = lambda *s: torch.zeros(s, dtype=torch.float32, device=dev)      # noqa: E731
        # the fp32 KL coefficient: device copy read by the captured actor step, host copy for the update rule
        self.kl_coefficient = np.float32(alg.initial_kl_coefficient)
        self.kl_coef = torch.tensor([float(self.kl_coefficient)], dtype=torch.float32, device=dev)
        # ---- minibatch step buffers and bindings (persistent: the captured graphs hold their pointers) ----
        self.mb = dict(states=f32(B, D), targets=f32(B, 1), actions=f32(B, A), advantages=f32(B), old_mu=f32(B, A))
        self.cursor = torch.zeros(1, dtype=torch.int64, device=dev)
        self.v_loss, self.v_acc = f32(1), f32(1)
        self.scalars, self.p_acc = f32(5), f32(5)
        self.critic_inst = self.critic_seq.instantiate(self.lib, self.ws, B, self.mb["states"], sc.theta, sc.grad,
                                                       train=True)
        self.actor_inst = self.actor_seq.instantiate(self.lib, self.ws, B, self.mb["states"], sa.theta, sa.grad,
                                                     train=True)
        self.use_cuda_graph = bool(use_cuda_graph)
        self._rows = None           # rollout-sized training columns (capacity, dict), see _training_columns
        self._full = {}             # rollout-sized forward instances, keyed by N
        self._act = {}              # acting buffers, keyed by the number of environments
        self.training_iteration = 0
        self.total_steps_counter = 0
        self.last_training_phase_step = 0
        self.last_losses = None
        self.last_kl_mean = None

    @property
    def is_on_policy(self) -> bool:
        return True

    # ---- acting ------------------------------------------------------------------------------------------------------------
    def _act_buffers(self, E):
        if E not in self._act:
            dev, pin = self.device, self.device.type == "cuda"
            x = torch.zeros((E, self.D), dtype=torch.float32, device=dev)
            inst = self.actor_seq.instantiate(self.lib, self.ws_rollout, E, x, self.actor.store.theta)
            self._act = {E: dict(x=x, inst=inst, actions=torch.zeros((E, self.A), dtype=torch.float64, device=dev),
                                 stds=torch.zeros((E, self.A), dtype=torch.float32, device=dev),
                                 n_dev=torch.zeros((E, self.A), dtype=torch.float64, device=dev),
                                 n_host=torch.zeros((E, self.A), dtype=torch.float64, pin_memory=pin))}
        return self._act[E]

    def choose_actions(self, states, evaluation=False, normals=None):
        """policy_optimization_agent.py:160-185 + AdditiveNoise.get_action([mean, std]) for E environments: the actor's
        mean and std = exp(policy_log_std); in training np.random.normal(mean, std) = (double) mean + (double) std * n
        on the standard normals ``normals`` [E, A] (default np.random.standard_normal((E, A)), what E successive normal
        calls draw), and the noise schedule is stepped E times; in evaluation the fp32 mean.  Returns (actions [E, A]:
        float64 in training, float32 in evaluation, means float32 [E, A], stds float32 [E, A])."""
        s = torch.as_tensor(np.asarray(states, dtype=np.float32)).reshape(-1, self.D)
        E, A = int(s.shape[0]), self.A
        buf = self._act_buffers(E)
        buf["x"].copy_(s)
        mean = buf["inst"].forward()
        n_ptr = None
        if not evaluation:
            n = np.random.standard_normal((E, A)) if normals is None else np.asarray(normals, dtype=np.float64)
            for _ in range(E):
                self.noise_schedule.step()
            torch.cuda.current_stream().synchronize()            # the previous call's copy has left the staging
            buf["n_host"].numpy()[...] = n.reshape(E, A)
            buf["n_dev"].copy_(buf["n_host"], non_blocking=True)
            n_ptr = buf["n_dev"].data_ptr()
        logstd = self.actor.store.view(self.actor.store.theta, self.logstd_name)
        _lib.check(self.lib.cb200_ppo_gaussian_act(mean.data_ptr(), logstd.data_ptr(), E, A, n_ptr,
                                                   buf["actions"].data_ptr(), buf["stds"].data_ptr(),
                                                   _lib.current_stream()))
        means, stds = mean.cpu().numpy().copy(), buf["stds"].cpu().numpy()
        return (means.copy() if evaluation else buf["actions"].cpu().numpy()), means, stds

    # ---- training phase --------------------------------------------------------------------------------------------------
    def sync(self):
        """actor target <- actor, critic target <- critic (ppo_agent.py:369-370): the old policy of the phase"""
        self.actor.sync()
        self.critic.sync()

    def _full_instances(self, N):
        if N not in self._full:
            x = torch.zeros((N, self.D), dtype=torch.float32, device=self.device)
            v = self.critic_seq.instantiate(self.lib, self.ws_rollout, N, x, self.critic.store.theta)
            p_old = self.actor_seq.instantiate(self.lib, self.ws_rollout, N, x, self.actor.target)
            self._full = {N: (x, v, p_old)}           # keep only the latest size
        return self._full[N]

    def fill_advantages(self, states, rewards, game_overs, returns):
        """ppo_agent.py:156-195 over the complete episodes (N rows, CUDA tensors): V(s) from the critic, then GAE per
        episode (zero bootstrap at each episode end) or A_VALUE = R - V in fp64, standardised with the population std
        over all N rows.  Returns (advantages fp64 [N], V(s) fp32 [N], old policy means fp32 [N, A])."""
        alg = self.ap.algorithm
        x, v_full, p_old = self._full_instances(states.shape[0])
        x.copy_(states)
        values = v_full.forward().reshape(-1)
        if alg.policy_gradient_rescaler == PolicyGradientRescaler.GAE:
            adv, _, _ = rl_math.fill_advantages(rewards, values, game_overs, alg.discount, alg.gae_lambda)
        else:
            adv = returns - values.to(torch.float64)
            rl_math.standardize_(adv)
        return adv, values, p_old.forward()

    def _training_columns(self, rows):
        """persistent rollout-sized columns the minibatch gathers read (their pointers are captured in the graphs);
        grown, and the graphs rebuilt, when a phase trains on more rows than they hold"""
        if self._rows is None or self._rows[0] < rows:
            f32 = lambda *s: torch.zeros(s, dtype=torch.float32, device=self.device)      # noqa: E731
            cols = dict(states=f32(rows, self.D), targets=f32(rows, 1), actions=f32(rows, self.A),
                        advantages=f32(rows), old_mu=f32(rows, self.A))
            self._rows = (rows, cols)
            enabled = self.use_cuda_graph and self.device.type == "cuda"
            self._critic_step = GraphedKernels(self._critic_kernels, self.device)
            self._actor_step = GraphedKernels(self._actor_kernels, self.device)
            self._critic_step.enabled = self._critic_step.enabled and enabled
            self._actor_step.enabled = self._actor_step.enabled and enabled
        return self._rows[1]

    def _gather(self, names):
        cols = self._rows[1]
        arr, cnt = _lib.make_columns([(cols[k].data_ptr(), self.mb[k].data_ptr(),
                                       self.mb[k].element_size() * int(np.prod(self.mb[k].shape[1:])))
                                      for k in names])
        _lib.check(self.lib.cb200_gather_at(arr, cnt, None, self.cursor.data_ptr(), self.B, _lib.current_stream()))

    def _critic_kernels(self):
        """one critic minibatch (train_value_network, ppo_agent.py:212-240): rows [cursor, cursor + B) of the states
        and Monte Carlo returns, VHead MSE (loss weight 1), backward, Adam"""
        st = _lib.current_stream()
        self._gather(("states", "targets"))
        v = self.critic_inst.forward()
        _lib.check(self.lib.cb200_regression_head_loss_grad(v.data_ptr(), self.mb["targets"].data_ptr(), None, self.B,
                                                            1, 0, 1.0, self.critic_inst.d_out.data_ptr(),
                                                            self.v_loss.data_ptr(), st))
        self.critic_inst.backward()
        self.critic.apply(self.ws)
        _lib.check(self.lib.cb200_axpby_2d(self.v_loss.data_ptr(), 1, 1, 1, 1.0, 1.0, self.v_acc.data_ptr(), 1, st))
        _lib.check(self.lib.cb200_add_i64(self.cursor.data_ptr(), self.B, st))

    def _actor_kernels(self):
        """one actor minibatch (train_policy_network, ppo_agent.py:260-301): rows [cursor, cursor + B) of the states,
        actions, advantages and old means, the KL-penalty head, backward, Adam; the head's scalars are added to the
        epoch accumulator"""
        st, alg, s = _lib.current_stream(), self.ap.algorithm, self.actor.store
        self._gather(("states", "actions", "advantages", "old_mu"))
        mu = self.actor_inst.forward()
        _lib.check(self.lib.cb200_ppo_kl_head(
            mu.data_ptr(), s.view(s.theta, self.logstd_name).data_ptr(), self.mb["actions"].data_ptr(),
            self.mb["old_mu"].data_ptr(), s.view(self.actor.target, self.logstd_name).data_ptr(),
            self.mb["advantages"].data_ptr(), self.B, self.A, self.kl_coef.data_ptr(),
            float(2 * alg.target_kl_divergence), float(alg.high_kl_penalty_coefficient),
            int(bool(alg.use_kl_regularization)), float(alg.beta_entropy), self.actor_inst.d_out.data_ptr(),
            s.view(s.grad, self.logstd_name).data_ptr(), self.scalars.data_ptr(), st))
        self.actor_inst.backward()
        self.actor.apply(self.ws)
        _lib.check(self.lib.cb200_axpby_2d(self.scalars.data_ptr(), 5, 1, 5, 1.0, 1.0, self.p_acc.data_ptr(), 5, st))
        _lib.check(self.lib.cb200_add_i64(self.cursor.data_ptr(), self.B, st))

    def train_phase(self, states, actions, rewards, game_overs, returns):
        """one PPO training phase on N rows of complete episodes (CUDA tensors: states fp32 [N, D], actions fp32 [N, A],
        rewards fp64 [N], game_overs uint8 [N], returns fp64 [N] Monte Carlo returns).  Returns the KL mean of the last
        actor epoch."""
        alg, B = self.ap.algorithm, self.B
        N = int(states.shape[0])
        n_mb = min(N, alg.num_consecutive_playing_steps.num_steps) // B
        if n_mb == 0:
            raise ValueError("the rollout holds %d transitions, fewer than one minibatch of %d: nothing to train on "
                             "(the reference fails here)" % (N, B))
        rows = n_mb * B
        self.sync()
        adv, _, old_mu = self.fill_advantages(states, rewards, game_overs, returns)
        cols = self._training_columns(rows)
        cols["states"][:rows].copy_(states[:rows])
        cols["actions"][:rows].copy_(actions[:rows])
        cols["targets"][:rows].copy_(returns[:rows].reshape(-1, 1))          # the float32 placeholder's rounding
        cols["advantages"][:rows].copy_(adv[:rows])
        cols["old_mu"][:rows].copy_(old_mu[:rows])
        self.cursor.zero_()
        self.v_acc.zero_()
        for _ in range(n_mb * EPOCHS_CRITIC):
            self._critic_step()
        for _ in range(EPOCHS_ACTOR):
            self.cursor.zero_()
            self.p_acc.zero_()
            for _ in range(n_mb):
                self._actor_step()
        acc = self.p_acc.cpu().numpy()                               # the phase's one device-to-host read
        self.last_losses = (float(self.v_acc.item()) / n_mb, acc / n_mb)
        self.last_kl_mean = float(acc[1]) / n_mb
        return self.last_kl_mean

    def update_kl_coefficient(self, kl_mean):
        """ppo_agent.py:329-353: x1.5 above 1.3 * target, /1.5 below 0.7 * target, stored as fp32"""
        target = self.ap.algorithm.target_kl_divergence
        k = np.float32(self.kl_coefficient)
        new = k
        if kl_mean > 1.3 * target:
            new *= 1.5
        elif kl_mean < 0.7 * target:
            new /= 1.5
        self.set_kl_coefficient(new)

    def set_kl_coefficient(self, value):
        self.kl_coefficient = np.float32(value)
        self.kl_coef.fill_(float(self.kl_coefficient))

    def _should_train(self):
        steps = self.ap.algorithm.num_consecutive_playing_steps
        should = (self.total_steps_counter - self.last_training_phase_step) >= steps.num_steps
        should = should and self.memory.num_transitions_in_complete_episodes() > 0
        if should:
            self.last_training_phase_step = self.total_steps_counter
        return should

    def train(self):
        """ppo_agent.py:362-391: a training phase over the replay's complete episodes once num_consecutive_playing_steps
        have been played, then the KL coefficient update and memory.clean()"""
        if not self._should_train():
            return None
        alg = self.ap.algorithm
        batch = self.memory.transitions_batch()
        if min(batch.size, alg.num_consecutive_playing_steps.num_steps) < self.B:
            raise ValueError("the rollout holds %d transitions, fewer than one minibatch of %d: nothing to train on "
                             "(the reference fails here)" % (batch.size, self.B))
        states = batch.states(["observation"])["observation"].to(torch.float32).reshape(batch.size, self.D)
        actions = batch.actions().to(torch.float32).reshape(batch.size, self.A)
        kl = None
        for _ in range(alg.num_consecutive_training_steps):
            kl = self.train_phase(states.contiguous(), actions.contiguous(), batch.rewards(), batch.game_overs(),
                                  batch.n_step_discounted_rewards())
        if alg.use_kl_regularization:
            self.update_kl_coefficient(kl)
        self.memory.clean()
        self.training_iteration += 1
        return self.last_losses

    # ---- checkpoint host state ---------------------------------------------------------------------------------------
    def checkpoint_state(self):
        """the KL coefficient and the noise schedule (both networks go through the actor / critic checkpoint items)"""
        return dict(kl_coefficient=float(self.kl_coefficient), noise=float(self.noise_schedule.current_value))

    def restore_checkpoint_state(self, state):
        self.set_kl_coefficient(state["kl_coefficient"])
        self.noise_schedule.current_value = state["noise"]
