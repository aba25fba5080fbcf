"""Policy Gradients (REINFORCE) on the GPU, E environment streams stepped in lock step, discrete or bounded continuous
actions.  Drop-in for

  rl_coach/agents/policy_gradients_agent.py:30-86        parameters, learn_from_batch (the return rescalers)
  rl_coach/agents/policy_optimization_agent.py:58-135    update_episode_statistics, train: whole episodes, gradients
                                                         accumulated and applied once in every x episodes
  rl_coach/exploration_policies/categorical.py:36-47     np.random.choice over the policy (training), argmax (evaluation)
  rl_coach/exploration_policies/additive_noise.py        np.random.normal(mean, noise * (high - low)) / the mean

Semantics over E streams: the E streams act as ONE reference worker that sees their episodes in (lock-step, stream)
order -- the per-timestep return table, the episode counter and the gradient accumulator are that worker's state, so
unlike the A3C agent the streams are not separate workers.  At each lock-step the episodes that closed are taken in
stream order and cut into parts: a part ends where the episode counter reaches a multiple of
``apply_gradients_every_x_episodes``.  Each part is one learn step whose gradient (the sum of its episodes' gradients)
is added to the accumulator, followed by one TF-Adam step on the accumulator (then zeroed) when the part ended on a
multiple.  With E = 1 this is the reference schedule; with E > 1 it equals a sequential reference run over the episodes
in that order.

Whole episodes only: an episode that reaches ``num_steps_between_gradient_updates`` (t_max, 20000) steps without ending
raises ValueError at that lock-step, before anything is learned (the reference's partial-episode path recomputes
statistics over rows the rollout ring no longer holds).  The rollout ring and the learn buffers hold t_max rows per
stream: at E = 64 on CartPole 1.28 M rows of 49 bytes each (two 16-byte observations, action, reward, game_over), about
63 MB per buffer.

Restoring a checkpoint: the rows of the episodes still open when it was written are not saved, so each stream's open
episode is discarded -- not learned and not counted -- and the stream learns again from its next episode.  The
reference loses its open episode the same way (a restored worker starts a new one).

Learn steps run on row buckets: 32-row steps up to 256 rows, then four sizes per doubling (at most 25 % padding), which
bounds the number of per-bucket network instances and CUDA graphs to about 4 log2(rows / 256) + 8.

One learn step = gather -> online features of the rows -> ``cb200_nstep_returns`` (n_step -1) -> ``cb200_pg_targets``
(the rescaler, the device table of the timestep rescaler) -> ``cb200_policy_gradient_head`` -> backward ->
``cb200_axpby_2d`` into the accumulator (coach_b200.agents.lockstep_agent).  The apply decision stays on the host.

Refused (ValueError): a rescaler other than the four return-based ones, ``n_step != -1``, ``clip_gradients`` (the
reference clips each episode's gradient before accumulating it, which one backward pass over several episodes cannot
reproduce), more than one rank, and unbounded continuous actions.  Checkpoints hold the network, Adam, the episode
counter, the accumulator, the table, the noise schedule and every stream's cut position.
"""
import base64
import ctypes

import numpy as np
import torch

from coach_b200 import _lib, parallel
from coach_b200.agents.actor_critic_agent import CategoricalParameters, PolicyGradientRescaler
from coach_b200.agents.lockstep_agent import LockstepAgent
from coach_b200.base_parameters import AgentParameters, AlgorithmParameters, InputEmbedderParameters, NetworkParameters
from coach_b200.exploration_policies.additive_noise import AdditiveNoiseParameters
from coach_b200.memories.lockstep_segments import bucket_rows

__all__ = ["PolicyGradientRescaler", "PolicyGradientAlgorithmParameters", "PolicyGradientNetworkParameters",
           "AdditiveNoiseParameters", "PolicyGradientsAgentParameters", "PolicyGradientsAgent"]


class PolicyGradientAlgorithmParameters(AlgorithmParameters):
    """policy_gradients_agent.py:43-65"""

    def __init__(self):
        super().__init__()
        self.policy_gradient_rescaler = PolicyGradientRescaler.FUTURE_RETURN_NORMALIZED_BY_TIMESTEP
        self.apply_gradients_every_x_episodes = 5
        self.beta_entropy = 0
        self.num_steps_between_gradient_updates = 20000          # t_max


class PolicyGradientNetworkParameters(NetworkParameters):
    """policy_gradients_agent.py:34-40: the Medium embedder and FC middleware, one PolicyHead (loss weight 1.0)"""

    def __init__(self):
        super().__init__()
        self.input_embedders_parameters = {'observation': InputEmbedderParameters()}
        self.heads_parameters = ["PolicyHead"]
        self.head_loss_weights = [1.0]
        self.async_training = True


class PolicyGradientsAgentParameters(AgentParameters):
    """policy_gradients_agent.py:68-79; the reference's SingleEpisodeBuffer is the agent's device rollout buffer"""

    def __init__(self):
        super().__init__(algorithm=PolicyGradientAlgorithmParameters(), memory=None,
                         networks={"main": PolicyGradientNetworkParameters()})
        self.exploration = {"DiscreteActionSpace": CategoricalParameters(),
                            "BoxActionSpace": AdditiveNoiseParameters()}

    @property
    def path(self):
        return 'coach_b200.agents.policy_gradients_agent:PolicyGradientsAgent'


RESCALERS = {PolicyGradientRescaler.TOTAL_RETURN: _lib.PG_TOTAL_RETURN,
             PolicyGradientRescaler.FUTURE_RETURN: _lib.PG_FUTURE_RETURN,
             PolicyGradientRescaler.FUTURE_RETURN_NORMALIZED_BY_EPISODE: _lib.PG_NORMALIZED_BY_EPISODE,
             PolicyGradientRescaler.FUTURE_RETURN_NORMALIZED_BY_TIMESTEP: _lib.PG_NORMALIZED_BY_TIMESTEP}


def _pack(t):
    return base64.b64encode(t.detach().cpu().numpy().tobytes()).decode("ascii")


def _unpack(s, t):
    t.copy_(torch.from_numpy(np.frombuffer(base64.b64decode(s), dtype=t.cpu().numpy().dtype).copy()))


class PolicyGradientsAgent(LockstepAgent):
    head_desc_type = _lib.PolicyGradientHeadDesc
    head_error = ("cb200_policy_gradient_head needs <= 18 actions (<= 32 action dimensions) on a 256- or 512-wide ReLU "
                  "layer")
    graph_tuning = "pg_graph"
    gather_keys, gather_boot = ("state", "action", "reward"), False

    def __init__(self, agent_parameters, parent=None, observation_shape=None, num_actions=None, num_envs=1,
                 device=None, seed=None, action_dim=None, action_low=None, action_high=None):
        """num_actions: a discrete action space; or action_dim with the bounds action_low / action_high [action_dim]
        (a BoxActionSpace: gym's float32 arrays)"""
        ap = agent_parameters
        alg, net_params = ap.algorithm, ap.network_wrappers["main"]
        if alg.policy_gradient_rescaler not in RESCALERS:
            raise ValueError("policy_gradient_rescaler must be TOTAL_RETURN, FUTURE_RETURN or one of the two "
                             "FUTURE_RETURN_NORMALIZED rescalers, got %s" % (alg.policy_gradient_rescaler,))
        if getattr(alg, "n_step", -1) != -1:
            raise ValueError("n_step must be -1: the policy gradient learns from whole-episode returns")
        if net_params.clip_gradients is not None and net_params.clip_gradients != 0:
            raise ValueError("clip_gradients is not supported: the reference clips every episode's gradient before "
                             "accumulating it, which one backward pass over several episodes cannot reproduce")
        if parallel.is_distributed():
            raise ValueError("PolicyGradientsAgent runs on one rank")
        self.continuous = action_dim is not None
        self.max_outputs = 32 if self.continuous else 18
        if self.continuous:
            if action_low is None or action_high is None:
                raise ValueError("continuous actions need the bounds action_low / action_high")
            self.action_low, self.action_high = np.asarray(action_low), np.asarray(action_high)
            if not (np.all(np.isfinite(self.action_low)) and np.all(np.isfinite(self.action_high))):
                raise ValueError("Additive noise exploration requires bounded actions")
        elif num_actions is None and getattr(ap, "num_actions", None) is None:
            raise ValueError("give num_actions (discrete) or action_dim with its bounds (continuous)")
        self.num_outputs = N = int(action_dim) if self.continuous else \
            int(num_actions if num_actions is not None else ap.num_actions)
        self.num_actions = None if self.continuous else N
        self.every = int(alg.apply_gradients_every_x_episodes)
        if self.every < 1:
            raise ValueError("apply_gradients_every_x_episodes must be >= 1")
        self.rescaler = RESCALERS[alg.policy_gradient_rescaler]
        super().__init__(ap, parent, observation_shape, num_envs, device, seed, N,
                         action_dim=N if self.continuous else None)
        dev, E, sg = self.device, self.num_envs, self.segments
        self.accumulator = torch.zeros(self.net_def.store.size, dtype=torch.float32, device=dev)
        # the per-timestep running mean of update_episode_statistics (mean, count), over t_max timesteps
        self.table = torch.zeros((2, self.t_max), dtype=torch.float64, device=dev)
        # a part holds at most x whole episodes
        R = min(sg.max_rows, bucket_rows(self.every * self.t_max))
        self.returns = torch.zeros(R, dtype=torch.float64, device=dev)
        self.targets = torch.zeros(R, dtype=torch.float32, device=dev)
        self.ep_bounds = torch.zeros((2, R), dtype=torch.int64, device=dev)
        pin = dev.type == "cuda"
        self._ep_host = torch.zeros((2, R), dtype=torch.int64, pin_memory=pin)
        self._ep_ev = None
        if self.continuous:
            rng = np.maximum(np.abs(self.action_low), np.abs(self.action_high)).astype(np.float32).reshape(N)
            self.max_abs_range = torch.from_numpy(rng).to(dev)
            ex = ap.exploration["BoxActionSpace"] if isinstance(ap.exploration, dict) else ap.exploration
            self.noise_schedule = ex.noise_schedule
        self._act_out = {}
        self.current_episode = 0
        self.last_parts = []                                   # [(episodes, applied)] of the last train()
        self._learned = []
        # streams whose open episode was cut by a checkpoint restore: discarded until their next game_over
        self.discard = np.zeros(E, dtype=bool)

    @property
    def learned_segments(self):
        """(stream, start, end) of the episodes the last train() step learned"""
        return self._learned

    # ---- acting (get_prediction: [E, N] outputs, the logits or the pre-tanh means) ----------------------------------------
    def choose_actions(self, states, evaluation=False, draws=None):
        """policy_optimization_agent.py:143-160 for E environments.
        Discrete: Categorical.get_action per environment: np.random.choice(A, p=softmax) on ``draws`` [E] (default
        np.random.random_sample(E)) or the first argmax (evaluation); returns (actions int64 [E], probabilities
        float32 [E, A]).
        Continuous: AdditiveNoise.get_action: mean = tanh(z) * range; in training np.random.normal(mean, noise *
        (high - low)) with the standard normals ``draws`` [E, D] (default np.random.standard_normal((E, D)), which
        draws what E successive normal calls draw); environment e's noise is the schedule's value after e steps, as
        E successive get_action calls read it, and the schedule is stepped E times; in evaluation the fp32 mean.  Returns (actions [E, D]:
        float64 in training, float32 in evaluation, means float32 [E, D])."""
        z = self.get_prediction(states)
        E, N, dev = int(z.shape[0]), self.num_outputs, self.device
        out = self._act_out.get(E)
        if out is None:
            pin = dev.type == "cuda"
            shape = (E, N) if self.continuous else (E,)
            out = self._act_out[E] = dict(
                actions=torch.zeros(E, dtype=torch.int64, device=dev),
                probs=torch.zeros((E, N), dtype=torch.float32, device=dev),
                cont=torch.zeros((E, N), dtype=torch.float64, device=dev),
                d_dev=torch.zeros(shape, dtype=torch.float64, device=dev),
                d_host=torch.zeros(shape, dtype=torch.float64, pin_memory=pin),
                scale=torch.zeros((E, N), dtype=torch.float64, device=dev))
        d_ptr = None
        if not evaluation:
            if self.continuous:
                d = np.random.standard_normal((E, N)) if draws is None else np.asarray(draws, dtype=np.float64)
                scale = np.zeros((E, N))
                for e in range(E):
                    noise = self.noise_schedule.current_value
                    scale[e] = np.asarray(noise * (self.action_high - self.action_low), dtype=np.float64).reshape(N)
                    self.noise_schedule.step()
                out["scale"].copy_(torch.from_numpy(scale))
            else:
                d = np.random.random_sample(E) if draws is None else np.asarray(draws, dtype=np.float64)
            d_ptr = self._stage(out["d_host"], out["d_dev"], d)
        rng = self.max_abs_range.data_ptr() if self.continuous else None
        _lib.check(self.lib.cb200_policy_act(z.data_ptr(), E, N, int(self.continuous), rng, d_ptr,
                                             out["scale"].data_ptr(), out["actions"].data_ptr(),
                                             out["probs"].data_ptr(), out["cont"].data_ptr(), out["probs"].data_ptr(),
                                             _lib.current_stream()))
        if not self.continuous:
            return out["actions"].cpu().numpy(), out["probs"].cpu().numpy()
        means = out["probs"].cpu().numpy()
        return (means.copy() if evaluation else out["cont"].cpu().numpy()), means

    def train(self, fetch=True):
        """policy_optimization_agent.py:85-135 over the episodes that closed at this lock-step, cut into parts at the
        multiples of apply_gradients_every_x_episodes.  Returns the last part's loss (the sum of its episodes' mean
        losses; 0 when no episode closed)."""
        sg = self.segments
        passed = sg.episode_length - sg.last_gradient_update_step_idx
        over = (passed >= self.t_max) & ~sg.complete & ~self.discard
        if over.any():
            raise ValueError("stream(s) %s reached num_steps_between_gradient_updates (%d) without ending an episode: "
                             "the policy gradient agent learns whole episodes only"
                             % (np.nonzero(over)[0].tolist(), self.t_max))
        ended = sg.complete.copy()
        streams, rows = sg.close()
        keep = ~self.discard[streams]
        streams, rows = streams[keep], rows[keep]
        self._learned = [seg for seg in sg.learned_segments if seg[0] in set(streams.tolist())]
        self.discard &= ~ended
        self.last_parts = []
        if len(streams) == 0:
            return 0
        loss, lo = 0, 0
        for k in range(len(streams)):
            self.current_episode += 1
            apply = self.current_episode % self.every == 0
            if apply or k == len(streams) - 1:
                loss = self._learn_part(streams[lo:k + 1], rows[lo:k + 1], apply, fetch)
                self.last_parts.append((k + 1 - lo, apply))
                lo = k + 1
        self.training_iteration += len(streams)
        return loss

    def _learn_part(self, streams, rows, apply, fetch):
        sg = self.segments
        B = sg.tables(streams, rows, self._bucket_for(int(rows.sum())))
        self._episode_bounds(rows, B)
        return self._learn(B, True, apply, fetch)

    def _episode_bounds(self, rows, B):
        """[ep_start | ep_end] of every row for cb200_nstep_returns (padding rows: their own one-row episode)"""
        if self._ep_ev is not None:
            self._ep_ev.synchronize()
        h = self._ep_host.numpy()
        offsets = np.concatenate([[0], np.cumsum(rows)[:-1]]).astype(np.int64)
        n = int(np.sum(rows))
        h[0, :B] = np.arange(B)
        h[1, :B] = np.arange(1, B + 1)
        h[0, :n] = np.repeat(offsets, rows)
        h[1, :n] = np.repeat(offsets + rows, rows)
        for i in range(2):
            self.ep_bounds[i, :B].copy_(self._ep_host[i, :B], non_blocking=True)
        self._ep_ev = torch.cuda.Event()
        self._ep_ev.record()

    # ---- the learn step -----------------------------------------------------------------------------------------------------
    def learn_from_batch(self, batch, apply=True, fetch=True):
        """one learn step on given whole episodes, bypassing the rollout buffer: batch is a dict of host arrays
        states / actions / rewards over the rows and "lengths": the episodes' lengths in row order (at most num_envs
        of them); the gradient is accumulated, then applied (and the accumulator zeroed) with ``apply``.  Returns the
        loss (the sum of the episodes' mean losses)."""
        lengths = np.asarray(batch["lengths"], dtype=np.int64)
        full = dict(batch, next_states=batch["states"], game_overs=np.zeros(int(lengths.sum()), np.uint8))
        B = self.segments.load(full, boot=False, B=self._bucket_for(int(lengths.sum())))
        self._episode_bounds(lengths, B)
        return self._learn(B, False, apply, fetch)

    def _bucket_for(self, n):
        R = self.returns.numel()
        if n > R:
            raise ValueError("a learn step of %d rows exceeds the %d-row buffers" % (n, R))
        return min(bucket_rows(n), R)

    def _fill_desc(self, d, on, boot, B):
        net, store = self.networks["main"], self.net_def.store
        wname, bname = self.net_def.trunk.names[-1]
        d.h = on.trunk.acts[-2].data_ptr()
        d.w, d.b = store.view(net.theta, wname).data_ptr(), store.view(net.theta, bname).data_ptr()
        d.targets = self.targets.data_ptr()
        if self.continuous:
            d.cont_actions, d.max_abs_range = self.learn["action"].data_ptr(), self.max_abs_range.data_ptr()
        else:
            d.actions = self.learn["action"].data_ptr()
        N = self.num_outputs
        d.continuous, d.n_outputs = int(self.continuous), N
        d.beta_entropy = float(self.ap.algorithm.beta_entropy)
        d.z = on.q.data_ptr()
        return B * (N + 1) + (B + 63) // 64 * (d.features * N + N + 1)

    def _launch_head(self, d, st):
        lib = self.lib
        _lib.check(lib.cb200_nstep_returns(self.learn["reward"].data_ptr(), self.ep_bounds[0].data_ptr(),
                                           self.ep_bounds[1].data_ptr(), d.rows, float(self.ap.algorithm.discount), -1,
                                           self.returns.data_ptr(), st))
        off, ln = self.segments.seg_table()
        _lib.check(lib.cb200_pg_targets(self.returns.data_ptr(), off, ln, self.num_envs, d.rows, self.rescaler,
                                        self.table[0].data_ptr(), self.table[1].data_ptr(), self.t_max,
                                        self.targets.data_ptr(), None, None, st))
        _lib.check(lib.cb200_policy_gradient_head(ctypes.byref(d), st))

    def _sink_gradients(self, st):
        """the step's gradient is added to the accumulator"""
        store = self.net_def.store
        _lib.check(self.lib.cb200_axpby_2d(store.grad.data_ptr(), store.size, 1, store.size, 1.0, 1.0,
                                           self.accumulator.data_ptr(), store.size, st))

    def apply_and_reset_gradients(self):
        """architecture.py:469-521 apply_and_reset_gradients: one TF-Adam step on the accumulated sum, then zero it"""
        self.networks["main"].apply_gradients(1.0, self.accumulator)
        self.accumulator.zero_()

    def _learn(self, B, gather, apply, fetch):
        self.segments.run(B, gather, self._device_step, _lib.tune_default(self.graph_tuning, 1))
        if apply:
            self.apply_and_reset_gradients()
        if not fetch:
            return self.loss_dev
        self._fetch_host[0:1].copy_(self.loss_dev, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return float(self._fetch_host[0])

    # ---- checkpoints (coach_b200/checkpoint.py) -------------------------------------------------------------------------
    def checkpoint_state(self):
        """the episode counter, the gradient accumulator, the per-timestep table, the noise schedule and every
        stream's cut position; the rows of episodes still open are not saved (a restore discards those episodes)"""
        torch.cuda.current_stream().synchronize()
        state = {"segments": super().checkpoint_state(), "current_episode": int(self.current_episode),
                 "training_iteration": int(self.training_iteration),
                 "accumulator": _pack(self.accumulator), "table": _pack(self.table)}
        if self.continuous:
            state["noise"] = float(self.noise_schedule.current_value)
        return state

    def restore_checkpoint_state(self, state):
        super().restore_checkpoint_state(state["segments"])
        sg = self.segments
        # an episode open at the checkpoint (or one that ended but was not trained yet) has rows the checkpoint does
        # not hold: it is neither learned nor counted
        self.discard[:] = (sg.episode_length > 0) | sg.complete
        self.current_episode = int(state["current_episode"])
        self.training_iteration = int(state["training_iteration"])
        _unpack(state["accumulator"], self.accumulator)
        _unpack(state["table"], self.table.view(-1))
        if self.continuous:
            self.noise_schedule.current_value = state["noise"]
