"""NAF (Normalized Advantage Functions) learn step and acting on the GPU.  Drop-in for

  rl_coach/agents/naf_agent.py:80-131       NAFAgent.learn_from_batch / choose_action
  heads/naf_head.py:45-86                   NAFHead: V = Dense(1), mu = tanh(Dense(A)) * max_abs_range,
                                            l = Dense(A(A+1)/2) -> L (exponentiated diagonal), Q = V - 0.5 d^T L L^T d
  network (naf_agent.py:34-43, presets/Mujoco_NAF.py:22-26):
    obs -> embedder Dense(256) relu -> middleware Dense(512) relu -> the three head projections
    (Mujoco_NAF: Dense(200) / Dense(200), ClipByValue(1000))

One learn step, replayed as one CUDA graph: the target trunk and V projection on s', the TD targets
(cb200_ac_td_targets: the same numpy expression as DDPG's), the online trunk and the three projections on s, the fused
head (cb200_naf_head: loss and the gradients of all three projections), the backward pass, the norm of the unclipped
gradients, the clip (ClipByValue or ClipByGlobalNorm), the all-reduce and Adam.
"""
import ctypes

import numpy as np
import torch

from coach_b200 import _lib
from coach_b200.agents.ddpg_agent import DDPGAgent, GraphedKernels, _Net
from coach_b200.architectures.layers import Dense, Workspace
from coach_b200.architectures.network import ParamStore, Sequential
from coach_b200.base_parameters import (AgentParameters, AlgorithmParameters, EnvironmentSteps, MiddlewareScheme,
                                        NetworkParameters)
from coach_b200.exploration_policies.ou_process import OUProcessParameters
from coach_b200.memories.episodic_experience_replay import EpisodicExperienceReplayParameters
from coach_b200.memories.prioritized_experience_replay import PrioritizedExperienceReplay
from coach_b200.utils import dynamic_import_and_instantiate_module_from_params

RELU = 1
MAX_ACTIONS = 32                  # cb200_naf_head: one warp per sample, one lane per action


class NAFNetworkParameters(NetworkParameters):
    def __init__(self):
        super().__init__()
        self.learning_rate = 0.001
        self.create_target_network = True
        # the vector embedder's layer widths (InputEmbedderParameters scheme Medium = [Dense(256)],
        # embedders/vector_embedder.py:57-60); the middleware's come from middleware_parameters.scheme, a
        # MiddlewareScheme or a list of widths
        self.embedder_units = (256,)
        self.replace_mse_with_huber_loss = False


class NAFAlgorithmParameters(AlgorithmParameters):
    def __init__(self):
        super().__init__()
        self.num_consecutive_training_steps = 5
        self.num_steps_between_copying_online_weights_to_target = EnvironmentSteps(1)
        self.rate_for_copying_weights_to_target = 0.001


class NAFAgentParameters(AgentParameters):
    def __init__(self):
        super().__init__(algorithm=NAFAlgorithmParameters(), memory=EpisodicExperienceReplayParameters(),
                         networks={"main": NAFNetworkParameters()})
        self.exploration = OUProcessParameters()

    @property
    def path(self):
        return 'coach_b200.agents.naf_agent:NAFAgent'


def _units(scheme):
    if isinstance(scheme, (list, tuple)):
        return tuple(int(u) for u in scheme)
    return MiddlewareScheme.units[getattr(scheme, "value", scheme)]


class NAFAgent(object):
    def __init__(self, agent_parameters, parent=None, observation_dim=None, action_dim=None, action_low=None,
                 action_high=None, device=None, seed=None, continuous_actions=True):
        """action_low / action_high: scalars or per-dimension bounds of the (continuous) action space, default -1 / 1;
        mu is scaled by max(|low|, |high|) (BoxActionSpace.max_abs_range).  continuous_actions=False stands for a
        discrete action space, which NAF refuses (naf_head.py:33-34)."""
        self.ap = agent_parameters
        net_p = self.ap.network_wrappers["main"]
        if not continuous_actions:
            raise ValueError("NAF works only for continuous action spaces (BoxActionSpace)")
        self.D, self.A = D, A = int(observation_dim), int(action_dim)
        if not 1 <= A <= MAX_ACTIONS:
            raise ValueError("NAF: the fused head takes 1 .. %d action dimensions, not %d" % (MAX_ACTIONS, A))
        if net_p.clip_gradients and net_p.gradients_clipping_method not in ("ClipByValue", "ClipByGlobalNorm"):
            raise NotImplementedError("NAF: gradient clipping %r is not implemented (ClipByValue, ClipByGlobalNorm)"
                                      % (net_p.gradients_clipping_method,))
        self.lib = _lib.load()
        self.device = dev = torch.device(device if device is not None else "cuda")
        self.B = B = int(net_p.batch_size)
        self.memory = dynamic_import_and_instantiate_module_from_params(
            self.ap.memory, extra_kwargs={"device": dev, "discount": self.ap.algorithm.discount})
        if isinstance(self.memory, PrioritizedExperienceReplay):
            # the reference NAF agent neither applies importance weights nor updates priorities
            raise ValueError("NAF does not support a prioritized replay")
        low = np.broadcast_to(np.asarray(-1.0 if action_low is None else action_low, dtype=np.float64), (A,))
        high = np.broadcast_to(np.asarray(1.0 if action_high is None else action_high, dtype=np.float64), (A,))
        # max_abs_range is fp64 numpy; TensorFlow multiplies by it as an fp32 constant
        self.scale_host = np.maximum(np.abs(low), np.abs(high)).astype(np.float32)
        self.scale = torch.from_numpy(self.scale_host.copy()).to(dev)
        self.clip = (net_p.gradients_clipping_method, float(net_p.clip_gradients)) if net_p.clip_gradients else None
        self.ws = Workspace(dev)
        # ---- parameter layout (TF creation order: embedder, middleware, head V / mu_unscaled / l_vector, rescaler) ----
        st = ParamStore(dev)
        emb = tuple(int(u) for u in net_p.embedder_units)
        mid = _units(net_p.middleware_parameters.scheme)
        widths = (D,) + emb + mid
        layers = [Dense(widths[i], widths[i + 1], "relu") for i in range(len(widths) - 1)]
        pre = "main/online/network_0"
        self.trunk = Sequential(layers[:len(emb)], st, pre + "/observation")
        middleware = Sequential(layers[len(emb):], st, pre + "/middleware_fc_embedder")
        self.trunk.layers += middleware.layers
        self.trunk.names += middleware.names
        F = widths[-1]
        self.n_l = A * (A + 1) // 2
        head = pre + "/naf_q_values_head_0"
        self.v_seq = Sequential([Dense(F, 1, None)], st, head + "/V")
        self.mu_seq = Sequential([Dense(F, A, None)], st, head + "/mu_unscaled")
        self.l_seq = Sequential([Dense(F, self.n_l, None)], st, head + "/l_vector")
        st.add(pre + "/gradients_from_head_0-0_rescalers", ())
        st.finalize()
        gen = torch.Generator().manual_seed(int(seed)) if seed is not None else None
        st.init_glorot(gen)
        self.main = _Net(self.lib, st, net_p, dev)
        self.main.sync()
        # ---- bindings ----
        f32 = lambda *s: torch.zeros(s, dtype=torch.float32, device=dev)      # noqa: E731
        self.batch_buffers = {"state:observation": f32(B, D), "next_state:observation": f32(B, D),
                              "action": f32(B, A), "reward": torch.zeros(B, dtype=torch.float64, device=dev),
                              "game_over": torch.zeros(B, dtype=torch.uint8, device=dev)}
        if hasattr(self.memory, "declare_schema") and self.memory.ring.specs is None:
            self.memory.declare_schema(self.batch_buffers)
        s, s2 = self.batch_buffers["state:observation"], self.batch_buffers["next_state:observation"]
        lib, ws = self.lib, self.ws
        self.trunk_target = self.trunk.instantiate(lib, ws, B, s2, self.main.target)
        self.v_target = self.v_seq.instantiate(lib, ws, B, self.trunk_target.out, self.main.target)
        self.trunk_online = self.trunk.instantiate(lib, ws, B, s, st.theta, st.grad, train=True)
        # the three projections' input gradients add up in the trunk's last pre-activation gradient
        self.heads = [seq.instantiate(lib, ws, B, self.trunk_online.out, st.theta, st.grad, train=True,
                                      need_input_grad=True, input_act=RELU, dx_in=self.trunk_online.d_out,
                                      dx_accumulate=k > 0)
                      for k, seq in enumerate((self.v_seq, self.mu_seq, self.l_seq))]
        self.td_targets = f32(B, 1)
        self.mu, self.q, self.adv, self.loss = f32(B, A), f32(B), f32(B), f32(1)
        self.head_desc = self._desc(B, self.heads[0].out, self.heads[1].out, self.heads[2].out, self.mu, self.q,
                                    train=True)
        self.training_iteration = 0
        self.total_steps_counter = 0
        self.last_training_phase_step = 0
        self.last_target_network_update_step = 0
        self._graph_step = None
        self._acting = {}

    @property
    def is_on_policy(self) -> bool:
        return False

    def _desc(self, B, z_v, z_mu, l, mu, q, train):
        d = _lib.NafHeadDesc()
        d.z_v, d.z_mu, d.l, d.scale = _lib.ptr(z_v), z_mu.data_ptr(), _lib.ptr(l), self.scale.data_ptr()
        d.huber = int(bool(self.ap.network_wrappers["main"].replace_mse_with_huber_loss))
        d.batch, d.n_actions, d.ld_mu, d.ld_l, d.ld_actions = B, self.A, self.A, self.n_l, self.A
        d.mu, d.q = mu.data_ptr(), _lib.ptr(q)
        if train:
            d.actions, d.targets = self.batch_buffers["action"].data_ptr(), self.td_targets.data_ptr()
            d.loss, d.adv = self.loss.data_ptr(), self.adv.data_ptr()
            d.d_zv, d.d_zmu, d.d_l = (h.d_out.data_ptr() for h in self.heads)
        return d

    # ---- learn_from_batch (naf_agent.py:80-99) ----------------------------------------------------------------------
    def learn_from_batch(self, batch, fetch=True):
        cols = batch.columns
        for k, buf in self.batch_buffers.items():          # the kernels (and their CUDA graph) read the agent's buffers
            if k in cols and cols[k].data_ptr() != buf.data_ptr():
                buf.copy_(cols[k].reshape(buf.shape))
        if self._graph_step is None:
            self._graph_step = GraphedKernels(self._naf_kernels, self.device)
        self._graph_step()
        if fetch:
            l = float(self.loss.item())
            return l, [l], float(torch.sqrt(self.main.sumsq).item())
        return self.loss, [self.loss], self.main.sumsq

    def _naf_kernels(self):
        lib, st, B = self.lib, _lib.current_stream(), self.B
        cols = self.batch_buffers
        # V of the target network on s'; TD targets r + (1 - done) * discount * V' in fp64, fed as fp32
        self.trunk_target.forward()
        v_next = self.v_target.forward()
        _lib.check(lib.cb200_ac_td_targets(cols["reward"].data_ptr(), cols["game_over"].data_ptr(), v_next.data_ptr(),
                                           1, B, float(self.ap.algorithm.discount), 0, 0, 0.0, 0.0,
                                           self.td_targets.data_ptr(), st))
        # the online network with the batch actions as the head input
        self.trunk_online.forward()
        for h in self.heads:
            h.forward()
        _lib.check(lib.cb200_naf_head(ctypes.byref(self.head_desc), st))
        for h in self.heads:                       # V first: it writes the trunk gradient, the others add to it
            h.backward()
        self.trunk_online.backward()
        self.main.apply(self.ws, clip=self.clip)

    # ---- driver (agents/agent.py:701-765): DDPG's ----------------------------------------------------------------------
    _should_update_online_weights_to_target = DDPGAgent._should_update_online_weights_to_target
    sample_batch = DDPGAgent.sample_batch

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
                self.main.sync(self.ap.algorithm.rate_for_copying_weights_to_target)
        return loss

    # ---- acting (naf_agent.py:101-112) ------------------------------------------------------------------------------
    def _acting_binding(self, E):
        if E not in self._acting:
            dev, th = self.device, self.main.store.theta
            ws = Workspace(dev)
            obs = torch.zeros((E, self.D), dtype=torch.float32, device=dev)
            trunk = self.trunk.instantiate(self.lib, ws, E, obs, th)
            mu_proj = self.mu_seq.instantiate(self.lib, ws, E, trunk.out, th)
            mu = torch.zeros((E, self.A), dtype=torch.float32, device=dev)
            # acting mode: no V projection, no l projection; the head writes mu only
            desc = self._desc(E, None, mu_proj.out, None, mu, None, train=False)
            self._acting[E] = (obs, trunk, mu_proj, mu, desc)
        return self._acting[E]

    def policy_means(self, states):
        """mu of the online network for states [E, D] (the device tensor [E, A])"""
        states = torch.as_tensor(np.asarray(states, dtype=np.float32)) if not torch.is_tensor(states) else states
        obs, trunk, mu_proj, mu, desc = self._acting_binding(int(states.shape[0]))
        obs.copy_(states.reshape(obs.shape))
        trunk.forward()
        mu_proj.forward()
        _lib.check(self.lib.cb200_naf_head(ctypes.byref(desc), _lib.current_stream()))
        return mu

    def choose_actions(self, states, exploration_policy):
        """one batched forward of the online network's trunk and mu projection for E environments, then the
        exploration policy on the [E, A] means.  Returns (actions [E, A], mu [E, A]) as numpy arrays."""
        mu = self.policy_means(states).cpu().numpy()
        return exploration_policy.get_actions(mu), mu
