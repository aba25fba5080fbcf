"""DDPG and TD3 learn steps on the GPU.  Drop-in for

  rl_coach/agents/ddpg_agent.py:137-195   DDPGAgent.learn_from_batch
  rl_coach/agents/td3_agent.py:148-209    TD3Agent.learn_from_batch (target policy smoothing, clipped double-Q,
                                          delayed actor update on mean(Q1))
  heads: ddpg_actor_head.py:46-63 (tanh * max_abs_range), ddpg_v_head.py:34 (output[1] = reduce_mean(Q)),
         td3_v_head.py:40-62 (two Q outputs, loss = sum_i mean((y - Q_i)^2), output[3] = reduce_mean(Q1))
  networks (presets/Mujoco_DDPG.py:24-28, presets/Mujoco_TD3.py:24-29):
    actor : obs -> Dense(400) relu -> Dense(300) relu -> Dense(A) tanh, * scale
    critic: DDPG: concat[action, Dense(400)(obs)] -> Dense(300) relu -> Dense(1)
            TD3 : concat[action, obs] -> 2 streams x (Dense(400) relu, Dense(300) relu) -> Dense(1) each
    (multi-input embedders are built in sorted name order and concatenated on the last axis, so the action comes
     first: general_network.py:252-279, SURVEY.md Q14)

Gradient conventions reproduced (SURVEY.md Q10): the actor update back-propagates
``-d mean_b(Q)/d a = -(1/B) dQ_i/da_i`` through the actor with NO further batch normalisation
(tensorflow_components/architecture.py:206-216); DDPG takes dQ/da from the critic BEFORE its update, TD3 after it;
both sum gradients over workers (``scale_down_gradients_by_number_of_workers_for_sync_training = False``).
"""
import numpy as np
import torch

from coach_b200 import _lib, parallel
from coach_b200.architectures.layers import Dense, Workspace
from coach_b200.architectures.network import ParamStore, Sequential
from coach_b200.base_parameters import (AgentParameters, AlgorithmParameters, EnvironmentSteps, NetworkParameters,
                                        TrainingSteps)
from coach_b200.memories.episodic_experience_replay import EpisodicExperienceReplayParameters
from coach_b200.utils import dynamic_import_and_instantiate_module_from_params, graph_capture

RELU, TANH = 1, 2


class DDPGCriticNetworkParameters(NetworkParameters):
    def __init__(self):
        super().__init__()
        self.batch_size = 64
        self.learning_rate = 0.001
        self.adam_optimizer_beta2 = 0.999
        self.optimizer_epsilon = 1e-8
        self.create_target_network = True
        self.scale_down_gradients_by_number_of_workers_for_sync_training = False


class DDPGActorNetworkParameters(NetworkParameters):
    def __init__(self):
        super().__init__()
        self.batch_size = 64
        self.learning_rate = 0.0001
        self.adam_optimizer_beta2 = 0.999
        self.optimizer_epsilon = 1e-8
        self.create_target_network = True
        self.scale_down_gradients_by_number_of_workers_for_sync_training = False


class DDPGAlgorithmParameters(AlgorithmParameters):
    def __init__(self):
        super().__init__()
        self.num_steps_between_copying_online_weights_to_target = EnvironmentSteps(1)
        self.rate_for_copying_weights_to_target = 0.001
        self.num_consecutive_playing_steps = EnvironmentSteps(1)
        self.action_penalty = 0
        self.clip_critic_targets = None
        self.use_non_zero_discount_for_terminal_states = False


class DDPGAgentParameters(AgentParameters):
    def __init__(self):
        super().__init__(algorithm=DDPGAlgorithmParameters(), memory=EpisodicExperienceReplayParameters(),
                         networks={"actor": DDPGActorNetworkParameters(), "critic": DDPGCriticNetworkParameters()})

    @property
    def path(self):
        return 'coach_b200.agents.ddpg_agent:DDPGAgent'


class TD3AlgorithmParameters(DDPGAlgorithmParameters):
    def __init__(self):
        super().__init__()
        self.rate_for_copying_weights_to_target = 0.005
        self.update_policy_every_x_episode_steps = 2
        self.num_steps_between_copying_online_weights_to_target = TrainingSteps(2)
        self.policy_noise = 0.2
        self.noise_clipping = 0.5
        self.num_q_networks = 2
        self.act_for_full_episodes = True


class TD3AgentParameters(AgentParameters):
    def __init__(self):
        actor, critic = DDPGActorNetworkParameters(), DDPGCriticNetworkParameters()
        actor.batch_size = critic.batch_size = 100
        actor.learning_rate = critic.learning_rate = 0.001
        super().__init__(algorithm=TD3AlgorithmParameters(), memory=EpisodicExperienceReplayParameters(),
                         networks={"actor": actor, "critic": critic})

    @property
    def path(self):
        return 'coach_b200.agents.ddpg_agent:TD3Agent'


class GraphedKernels(object):
    """A launch sequence with constant parameters and pointers, replayed as ONE CUDA graph from its third call on (the
    first two run eagerly: lazy module loading, workspace sizing).  The actor-critic learn steps are 80-150 launches of
    microsecond kernels; replayed as a graph they cost what the kernels cost, not what Python + ctypes cost per launch.
    With several ranks the sequence contains NCCL all-reduces, which are captured with it (measured at 2 GPUs: SAC
    1,383 -> 1,782 steps/s, TD3 2,031 steps/s); CB200_GRAPH_COLLECTIVES=0 keeps such sequences eager.  A process that
    captured collectives must destroy its agents (the graphs) before ``destroy_process_group()`` (bench.py: _finish)."""

    def __init__(self, fn, device):
        self.fn = fn
        self.enabled = bool(_lib.tune_default("ac_graph", 1)) and torch.device(device).type == "cuda" and \
            (not parallel.is_distributed() or bool(_lib.tune_default("graph_collectives", 1)))
        self.calls, self.graph, self.launches = 0, None, 0

    def __call__(self):
        if not self.enabled or self.calls < 2:
            self.calls += 1
            return self.fn()
        if self.graph is None:
            lib = _lib.load()
            torch.cuda.synchronize()
            c0 = lib.cb200_launch_count()
            g = torch.cuda.CUDAGraph()
            with graph_capture(g):
                self.fn()
            self.launches = int(lib.cb200_launch_count() - c0)
            self.graph = g
        self.graph.replay()


class _Net(object):
    """one Coach "network wrapper": flat store + target buffer + device-state Adam"""

    def __init__(self, lib, store, params, device):
        self.lib, self.store, self.params = lib, store, params
        self.target = store.new_buffer()
        self.adam_state = torch.tensor([params.adam_optimizer_beta1, params.adam_optimizer_beta2],
                                       dtype=torch.float32, device=device)
        self.sumsq = torch.zeros(1, dtype=torch.float32, device=device)

    def sync(self, rate=1.0):
        _lib.check(self.lib.cb200_polyak(self.target.data_ptr(), self.store.theta.data_ptr(), self.store.size,
                                         float(rate), _lib.current_stream()))

    def apply(self, ws, clip=None):
        """clip: None (no clipping) or (gradients_clipping_method, clip_gradients) with "ClipByValue" or
        "ClipByGlobalNorm": applied to this worker's gradients after their (unclipped) norm is taken and before the
        all-reduce (architecture.py:193-194, 237-245)"""
        st, s, p = _lib.current_stream(), self.store, self.params
        _lib.check(self.lib.cb200_sumsq(s.grad.data_ptr(), s.size, self.sumsq.data_ptr(), ws.ptr(), st))
        if clip is not None:
            method, c = clip
            if method == "ClipByValue":
                _lib.check(self.lib.cb200_clip_by_value(s.grad.data_ptr(), s.size, float(c), st))
            elif method == "ClipByGlobalNorm":
                _lib.check(self.lib.cb200_clip_by_global_norm(s.grad.data_ptr(), s.size, self.sumsq.data_ptr(),
                                                              float(c), st))
            else:
                raise NotImplementedError("gradient clipping method %r" % (method,))
        scaler = parallel.allreduce_gradients(s.grad, p.scale_down_gradients_by_number_of_workers_for_sync_training)
        if scaler != 1.0:
            _lib.check(self.lib.cb200_scale(s.grad.data_ptr(), s.size, float(scaler), st))
        _lib.check(self.lib.cb200_adam_tf_dev(s.theta.data_ptr(), s.m.data_ptr(), s.v.data_ptr(), s.grad.data_ptr(),
                                              s.size, float(p.learning_rate), float(p.adam_optimizer_beta1),
                                              float(p.adam_optimizer_beta2), float(p.optimizer_epsilon),
                                              self.adam_state.data_ptr(), st))


class _CriticBinding(object):
    """critic forward/backward on one (state input, action input, parameter buffer) triple"""

    def __init__(self, agent, theta, grad, train, need_action_grad):
        lib, ws, B, dev = agent.lib, agent.ws, agent.B, agent.device
        A, D = agent.A, agent.D
        self.agent = agent
        self.obs = torch.zeros((B, D), dtype=torch.float32, device=dev)
        self.act = torch.zeros((B, A), dtype=torch.float32, device=dev)
        self.embed = None
        X = D
        if agent.critic_embedder is not None:                        # DDPG: Dense(400) relu on the observation
            self.embed = agent.critic_embedder.instantiate(lib, ws, B, self.obs, theta, grad, train=train)
            X = agent.critic_embedder.layers[-1].N
        self.X = X
        self.cat = torch.zeros((B, A + X), dtype=torch.float32, device=dev)
        self.d_cat = torch.zeros((B, A + X), dtype=torch.float32, device=dev) if (train or need_action_grad) else None
        self.streams = []
        for k, seq in enumerate(agent.critic_streams):
            want_dx = (train and self.embed is not None) or (need_action_grad and k == 0)
            self.streams.append(seq.instantiate(lib, ws, B, self.cat, theta, grad, train=train or want_dx,
                                                need_input_grad=want_dx, input_act=0, dx_in=self.d_cat,
                                                dx_accumulate=(k > 0)))
        self.q = [s.out for s in self.streams]

    def forward(self, n_streams=None):
        lib, st, A, B = self.agent.lib, _lib.current_stream(), self.agent.A, self.agent.B
        ld = A + self.X
        _lib.check(lib.cb200_axpby_2d(self.act.data_ptr(), A, B, A, 1.0, 0.0, self.cat.data_ptr(), ld, st))
        if self.embed is not None:
            e = self.embed.forward()
            _lib.check(lib.cb200_axpby_2d(e.data_ptr(), self.X, B, self.X, 1.0, 0.0, self.cat.data_ptr() + 4 * A, ld,
                                          st))
        else:
            _lib.check(lib.cb200_axpby_2d(self.obs.data_ptr(), self.X, B, self.X, 1.0, 0.0,
                                          self.cat.data_ptr() + 4 * A, ld, st))
        for s in self.streams[:n_streams]:
            s.forward()
        return self.q

    def backward(self, weights=True, n_streams=None):
        """expects d(loss)/dQ_k in streams[k].d_out; leaves d(loss)/d[action, x] in d_cat"""
        lib, st, A, B = self.agent.lib, _lib.current_stream(), self.agent.A, self.agent.B
        for s in self.streams[:n_streams]:
            s.backward(weights)
        if self.embed is not None and weights:
            ld = A + self.X
            _lib.check(lib.cb200_act_backward(self.d_cat.data_ptr() + 4 * A, ld, self.embed.out.data_ptr(), self.X, B,
                                              self.X, RELU, self.embed.d_out.data_ptr(), self.X, st))
            self.embed.backward()


class DDPGAgent(object):
    twin = False

    def __init__(self, agent_parameters, parent=None, observation_dim=None, action_dim=None, action_scale=1.0,
                 action_low=None, action_high=None, device=None, seed=None):
        self.ap = agent_parameters
        self.lib = _lib.load()
        self.device = dev = torch.device(device if device is not None else "cuda")
        self.D, self.A = int(observation_dim), int(action_dim)
        self.scale = float(action_scale)
        self.action_low = float(action_low if action_low is not None else -self.scale)
        self.action_high = float(action_high if action_high is not None else self.scale)
        pa, pc = self.ap.network_wrappers["actor"], self.ap.network_wrappers["critic"]
        self.B = B = int(pc.batch_size)
        self.memory = dynamic_import_and_instantiate_module_from_params(
            self.ap.memory, extra_kwargs={"device": dev, "discount": self.ap.algorithm.discount})
        self.ws = Workspace(dev)
        D, A = self.D, self.A
        # ---- parameter layouts (TF creation order) ----
        sa = ParamStore(dev)
        self.actor_seq = Sequential([Dense(D, 400, "relu"), Dense(400, 300, "relu"), Dense(300, A, "tanh")], sa,
                                    "actor/online/network_0")
        sa.add("actor/online/network_0/gradients_from_head_0-0_rescalers", ())
        sa.finalize()
        sc = ParamStore(dev)
        if self.twin:
            self.critic_embedder = None
            self.critic_streams = [Sequential([Dense(A + D, 400, "relu"), Dense(400, 300, "relu")], sc,
                                              "critic/online/network_0/middleware_fc_embedder/stream_%d" % k)
                                   for k in range(2)]
            heads = [Sequential([Dense(300, 1, None)], sc, "critic/online/network_0/td3_v_values_head_0/q_output_%d"
                                % (k + 1)) for k in range(2)]
            # one chain per stream: middleware layers followed by that stream's head
            for k in range(2):
                self.critic_streams[k].layers += heads[k].layers
                self.critic_streams[k].names += heads[k].names
        else:
            self.critic_embedder = Sequential([Dense(D, 400, "relu")], sc, "critic/online/network_0/observation")
            self.critic_streams = [Sequential([Dense(A + 400, 300, "relu"), Dense(300, 1, None)], sc,
                                              "critic/online/network_0/middleware_and_head")]
        sc.add("critic/online/network_0/gradients_from_head_0-0_rescalers", ())
        sc.finalize()
        gen = torch.Generator().manual_seed(int(seed)) if seed is not None else None
        sa.init_glorot(gen)
        sc.init_glorot(gen)
        self.actor = _Net(self.lib, sa, pa, dev)
        self.critic = _Net(self.lib, sc, pc, dev)
        self.actor.sync()
        self.critic.sync()
        # ---- bindings ----
        f32 = lambda *s: torch.zeros(s, dtype=torch.float32, device=dev)      # noqa: E731
        self.batch_buffers = {"state:observation": f32(B, D), "next_state:observation": f32(B, D),
                              "action": f32(B, A), "reward": torch.zeros(B, dtype=torch.float64, device=dev),
                              "game_over": torch.zeros(B, dtype=torch.uint8, device=dev)}
        if hasattr(self.memory, "declare_schema") and self.memory.ring.specs is None:
            self.memory.declare_schema(self.batch_buffers)       # store(Transition) casts gym's float64 to these dtypes
        s, s2 = self.batch_buffers["state:observation"], self.batch_buffers["next_state:observation"]
        self.actor_target_s2 = self.actor_seq.instantiate(self.lib, self.ws, B, s2, self.actor.target)
        self.actor_online_s = self.actor_seq.instantiate(self.lib, self.ws, B, s, sa.theta, sa.grad, train=True)
        self.critic_target = _CriticBinding(self, self.critic.target, None, False, False)
        self.critic_train = _CriticBinding(self, sc.theta, sc.grad, True, False)
        self.critic_pi = _CriticBinding(self, sc.theta, sc.grad, False, True)
        self.td_targets = f32(B, 1)
        self.q_min = f32(B, 1)
        self.noise = torch.zeros((B, A), dtype=torch.float64, device=dev)
        self.loss_dev = [f32(1), f32(1)]
        self.training_iteration = 0
        self.total_steps_counter = 0
        self.last_training_phase_step = 0
        self.last_target_network_update_step = 0
        self._graph_step, self._graph_actor = None, None

    @property
    def is_on_policy(self) -> bool:
        return False

    # ---- pieces ------------------------------------------------------------------------------------------------------
    def _scaled_actions(self, y, dst):
        _lib.check(self.lib.cb200_axpby_2d(y.data_ptr(), self.A, self.B, self.A, self.scale, 0.0, dst.data_ptr(),
                                           self.A, _lib.current_stream()))

    def _td_targets(self, cols, q_next):
        alg = self.ap.algorithm
        clip = alg.clip_critic_targets
        _lib.check(self.lib.cb200_ac_td_targets(cols["reward"].data_ptr(), cols["game_over"].data_ptr(),
                                                q_next.data_ptr(), 1, self.B, float(alg.discount),
                                                int(bool(alg.use_non_zero_discount_for_terminal_states)),
                                                int(clip is not None and bool(clip)),
                                                float(clip[0]) if clip else 0.0, float(clip[1]) if clip else 0.0,
                                                self.td_targets.data_ptr(), _lib.current_stream()))

    def _action_gradients_into_actor(self):
        """critic.gradients_wrt_inputs[.]['action'] of mean_b Q(s, mu(s)) -> -grad as the actor's output gradient
        (ddpg_agent.py:168-186, td3_agent.py:191-201)"""
        lib, st, A, B = self.lib, _lib.current_stream(), self.A, self.B
        cp = self.critic_pi
        cp.obs.copy_(self.batch_buffers["state:observation"])
        self._scaled_actions(self.actor_online_s.out, cp.act)
        cp.forward(n_streams=1)
        cp.streams[0].d_out.fill_(1.0 / B)                                  # d mean_b(Q1) / dQ1_i
        cp.backward(weights=False, n_streams=1)
        # d(policy_mean) = -dQ/da ; policy_mean = scale * tanh(z)  ->  dz = -dQ/da * scale * (1 - y^2)
        ai = self.actor_online_s
        _lib.check(lib.cb200_axpby_2d(cp.d_cat.data_ptr(), A + cp.X, B, A, -self.scale, 0.0, ai.d_out.data_ptr(), A,
                                      st))
        _lib.check(lib.cb200_act_backward(ai.d_out.data_ptr(), A, ai.out.data_ptr(), A, B, A, TANH,
                                          ai.d_out.data_ptr(), A, st))
        ai.backward()
        self.actor.apply(self.ws)

    def _train_critic(self, cols):
        lib, st, B = self.lib, _lib.current_stream(), self.B
        ct = self.critic_train
        ct.obs.copy_(cols["state:observation"])
        ct.act.copy_(cols["action"].reshape(B, self.A))
        qs = ct.forward()
        for k, q in enumerate(qs):
            # VHead / TD3VHead: mean((target - Q_k)^2), summed over the heads (v_head.py:41-44, td3_v_head.py:55-62)
            _lib.check(lib.cb200_regression_head_loss_grad(q.data_ptr(), self.td_targets.data_ptr(), None, B, 1, 0, 1.0,
                                                           ct.streams[k].d_out.data_ptr(), self.loss_dev[k].data_ptr(),
                                                           st))
        ct.backward()
        self.critic.apply(self.ws)

    def _next_actions(self, cols):
        self.critic_target.obs.copy_(cols["next_state:observation"])
        self._scaled_actions(self.actor_target_s2.forward(), self.critic_target.act)

    # ---- learn_from_batch ----------------------------------------------------------------------------------------------
    def _stage(self, batch):
        """every column of a batch that does not already live in the agent's persistent buffers is copied there: the
        kernels (and their CUDA graph) only ever read the persistent buffers"""
        cols = batch.columns
        for k, buf in self.batch_buffers.items():
            if k in cols and cols[k].data_ptr() != buf.data_ptr():
                buf.copy_(cols[k].reshape(buf.shape))
        return self.batch_buffers

    def learn_from_batch(self, batch, fetch=True):
        self._stage(batch)
        if self._graph_step is None:
            self._graph_step = GraphedKernels(self._ddpg_kernels, self.device)
        self._graph_step()
        return self._result(fetch)

    def _ddpg_kernels(self):
        cols = self.batch_buffers
        self._next_actions(cols)                                            # actor target on s'
        self.actor_online_s.forward()                                       # actions_mean = actor online on s
        q_next = self.critic_target.forward()[0]
        self._td_targets(cols, q_next)
        self._action_gradients_into_actor_deferred = True
        # DDPG: dQ/da from the critic BEFORE its update, actor step after the critic step (ddpg_agent.py:168-193)
        lib, st, A, B = self.lib, _lib.current_stream(), self.A, self.B
        cp = self.critic_pi
        cp.obs.copy_(self.batch_buffers["state:observation"])
        self._scaled_actions(self.actor_online_s.out, cp.act)
        cp.forward(n_streams=1)
        cp.streams[0].d_out.fill_(1.0 / B)
        cp.backward(weights=False, n_streams=1)
        self._train_critic(cols)
        ai = self.actor_online_s
        _lib.check(lib.cb200_axpby_2d(cp.d_cat.data_ptr(), A + cp.X, B, A, -self.scale, 0.0, ai.d_out.data_ptr(), A,
                                      st))
        _lib.check(lib.cb200_act_backward(ai.d_out.data_ptr(), A, ai.out.data_ptr(), A, B, A, TANH,
                                          ai.d_out.data_ptr(), A, st))
        ai.backward()
        self.actor.apply(self.ws)

    def _result(self, fetch):
        loss = self.loss_dev[0] + self.loss_dev[1] if self.twin else self.loss_dev[0]
        if fetch:
            l = float(loss.item())
            return l, [l], float(torch.sqrt(self.critic.sumsq).item())
        return loss, [loss], self.critic.sumsq

    # ---- driver (agents/agent.py:701-784) ------------------------------------------------------------------------------
    def _should_update_online_weights_to_target(self):
        step_method = self.ap.algorithm.num_steps_between_copying_online_weights_to_target
        counter = self.training_iteration if step_method.__class__ == TrainingSteps else self.total_steps_counter
        should = (counter - self.last_target_network_update_step) >= step_method.num_steps
        if should:
            self.last_target_network_update_step = counter
        return should

    def sample_batch(self):
        return self.memory.sample_batch(self.B, out=self.batch_buffers)

    def train(self, fetch=True):
        loss = 0
        if self.memory.num_transitions_in_complete_episodes() < 1:
            return loss
        for _ in range(self.ap.algorithm.num_consecutive_training_steps):
            self.training_iteration += 1
            batch = self.sample_batch()
            total_loss, _, _ = self.learn_from_batch(batch, fetch=fetch)
            loss = loss + total_loss if fetch else total_loss
            if self._should_update_online_weights_to_target():
                rate = self.ap.algorithm.rate_for_copying_weights_to_target
                self.actor.sync(rate)
                self.critic.sync(rate)
        return loss


class TD3Agent(DDPGAgent):
    twin = True

    def learn_from_batch(self, batch, fetch=True, noise=None):
        """``noise``: optional [B, A] array standing in for np.random.normal(0, policy_noise) (td3_agent.py:162);
        by default it is drawn here from numpy's global generator, like the reference."""
        alg = self.ap.algorithm
        self._stage(batch)
        B, A = self.B, self.A
        if noise is None:
            noise = np.random.normal(0, alg.policy_noise, (B, A))
        self.noise.copy_(torch.as_tensor(np.asarray(noise, dtype=np.float64)))
        if self._graph_step is None:
            self._graph_step = GraphedKernels(self._td3_critic_kernels, self.device)
            self._graph_actor = GraphedKernels(self._action_gradients_into_actor, self.device)
        self._graph_step()
        if self.training_iteration % alg.update_policy_every_x_episode_steps == 0:
            self._graph_actor()                                             # with the UPDATED critic (:190-201)
        return self._result(fetch)

    def _td3_critic_kernels(self):
        alg, cols = self.ap.algorithm, self.batch_buffers
        lib, st, B, A = self.lib, _lib.current_stream(), self.B, self.A
        self._next_actions(cols)
        self.actor_online_s.forward()
        _lib.check(lib.cb200_td3_smooth_actions(self.critic_target.act.data_ptr(), self.noise.data_ptr(), B * A,
                                                float(alg.noise_clipping), self.action_low, self.action_high, st))
        q1, q2 = self.critic_target.forward()
        _lib.check(lib.cb200_min2(q1.data_ptr(), q2.data_ptr(), B, self.q_min.data_ptr(), st))   # output #2
        self._td_targets(cols, self.q_min)
        self._train_critic(cols)
