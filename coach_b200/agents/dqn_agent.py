"""DQN / DDQN / dueling-DDQN learn step on the GPU.  Drop-in for the replay -> learn_from_batch part of

  rl_coach/agents/agent.py:701-784                 Agent.train            (driver, target-network cadence)
  rl_coach/agents/dqn_agent.py:69-113              DQNAgent               (TD targets, PER update, train step)
  rl_coach/agents/ddqn_agent.py:38-43              DDQNAgent.select_actions
  rl_coach/agents/value_optimization_agent.py:74-80  priorities are updated with the PRE-update TD errors
  rl_coach/architectures/network_wrapper.py:109-203 + tensorflow_components/architecture.py:312-521,598-607
                                                   (accumulate_gradients / apply_gradients / set_weights)

One learn step = fused PER sample+gather (memory) -> target & online forward -> TD-target kernel -> Huber/MSE head
loss + its gradient -> backward -> global norm (+ clip) -> [NCCL all-reduce] -> TF-semantics Adam -> tree update.
The online forward on ``s`` is computed once: the reference runs it twice (once for the TD targets, once inside the
train op) with identical weights, hence identical values.

``learn_from_batch`` keeps the reference contract ``-> (total_loss, losses, unclipped_grads)``; pass ``fetch=False`` to
get device scalars instead of floats and avoid the host synchronisation.
"""
import numpy as np
import torch

from coach_b200 import _lib
from coach_b200.architectures import tiled as tl
from coach_b200.architectures.layers import NO_SIDE, SideStream, Workspace
from coach_b200.architectures.q_network import QNetworkDef
from coach_b200.base_parameters import (AgentParameters, AlgorithmParameters, EnvironmentSteps, MiddlewareScheme,
                                        NetworkParameters, TrainingSteps)
from coach_b200.memories.experience_replay import ExperienceReplayParameters
from coach_b200.memories.prioritized_experience_replay import PrioritizedExperienceReplay
from coach_b200.utils import dynamic_import_and_instantiate_module_from_params, graph_capture
from coach_b200 import parallel


class DQNAlgorithmParameters(AlgorithmParameters):
    def __init__(self):
        super().__init__()
        self.num_steps_between_copying_online_weights_to_target = EnvironmentSteps(10000)
        self.num_consecutive_playing_steps = EnvironmentSteps(4)
        self.discount = 0.99


class DQNNetworkParameters(NetworkParameters):
    def __init__(self):
        super().__init__()
        self.heads_parameters = ["QHead"]              # or ["DuelingQHead"]
        self.optimizer_type = 'Adam'
        self.batch_size = 32
        self.replace_mse_with_huber_loss = True
        self.create_target_network = True


class DQNAgentParameters(AgentParameters):
    def __init__(self):
        super().__init__(algorithm=DQNAlgorithmParameters(), memory=ExperienceReplayParameters(),
                         networks={"main": DQNNetworkParameters()})

    @property
    def path(self):
        return 'coach_b200.agents.dqn_agent:DQNAgent'


class DDQNAgentParameters(DQNAgentParameters):
    def __init__(self):
        super().__init__()
        self.algorithm.num_steps_between_copying_online_weights_to_target = EnvironmentSteps(30000)

    @property
    def path(self):
        return 'coach_b200.agents.dqn_agent:DDQNAgent'


class QNetworkWrapper(object):
    """online + target parameter buffers over one QNetworkDef (network_wrapper.py:31-116), with the forward bindings a
    DQN step needs: online(s) [training], target(s'), online(s') [DDQN], target(s) [PAL: ``target_s``]."""

    def __init__(self, lib, net_def, params: NetworkParameters, batch_size, batch_buffers, double_dqn, device,
                 input_planes=None, target_s=False):
        self.lib, self.net, self.params, self.B = lib, net_def, params, batch_size
        self.store = net_def.store
        self.ws = Workspace(device)
        self.ws_target = Workspace(device)        # the target network's passes may run on a side stream
        self.theta = self.store.theta
        self.theta_target = self.store.new_buffer() if params.create_target_network else None
        s, s2 = batch_buffers["state:observation"], batch_buffers["next_state:observation"]
        if input_planes is not None:         # fused input path: the replay hands over the s2d operand planes directly
            s, s2 = input_planes["state:observation"], input_planes["next_state:observation"]
        self.online_s = net_def.instantiate(lib, self.ws, batch_size, s, self.theta, self.store.grad, train=True)
        self.target_s2 = net_def.instantiate(lib, self.ws_target, batch_size, s2, self.theta_target) \
            if self.theta_target is not None else None
        self.online_s2 = net_def.instantiate(lib, self.ws, batch_size, s2, self.theta) if double_dqn else None
        # the target network over the same input as online_s (on the fused input path: the same s2d plane)
        self.target_s = net_def.instantiate(lib, self.ws_target, batch_size, s, self.theta_target) \
            if target_s and self.theta_target is not None else None
        self.sumsq = torch.zeros(1, dtype=torch.float32, device=device)
        self.has_target = self.theta_target is not None
        # Adam state: the fp32 running powers of TF's non-slot beta1 / beta2 power variables, kept on the device
        # so that the optimizer step has constant launch parameters and can be captured in a CUDA graph
        # (cb200_adam_tf_dev)
        self.adam_state = torch.tensor([params.adam_optimizer_beta1, params.adam_optimizer_beta2],
                                       dtype=torch.float32, device=device)
        # parameter planes (operands of the tensor-core GEMMs) are re-derived where the parameters are written, not in
        # every forward pass: the target network's once per target update instead of once per learn step
        self._planes = []
        for inst in (self.online_s, self.online_s2, self.target_s2, self.target_s):
            self.add_planes(inst)

    def add_planes(self, inst):
        """derives the operand planes of ``inst`` (a network instance over theta or theta_target) now and again
        whenever those parameters change"""
        if inst is not None and inst.theta_planes is not None:
            self._planes.append(inst.theta_planes)
            inst.theta_planes.refresh()

    def sync(self):
        """online -> target hard copy (network_wrapper.py:94-107)."""
        self.update_target_network(1.0)

    def update_target_network(self, rate=1.0):
        _lib.check(self.lib.cb200_polyak(self.theta_target.data_ptr(), self.theta.data_ptr(), self.store.size,
                                         float(rate), _lib.current_stream()))
        self.target_changed()

    def _refresh(self, theta):
        for tp in self._planes:
            if tp.theta.data_ptr() == theta.data_ptr():
                tp.refresh()

    def online_changed(self):
        """call after ANY write to ``theta`` other than apply_gradients (checkpoint load, manual edits)"""
        self._refresh(self.theta)

    def target_changed(self):
        """call after ANY write to ``theta_target`` other than update_target_network"""
        if self.theta_target is not None:
            self._refresh(self.theta_target)

    def apply_gradients(self, scaler=1.0, grad=None):
        """clip is applied by the caller (accumulate_gradients side in the reference); here: optional rescale,
        then the optimizer (architecture.py:469-521).  grad: the gradient buffer to apply, default ``store.grad``."""
        st = _lib.current_stream()
        n = self.store.size
        grad = self.store.grad if grad is None else grad
        if scaler != 1.0:
            _lib.check(self.lib.cb200_scale(grad.data_ptr(), n, float(scaler), st))
        p = self.params
        if p.optimizer_type != 'Adam':
            raise NotImplementedError("only the Adam optimizer of the DQN presets is implemented on device")
        _lib.check(self.lib.cb200_adam_tf_dev(self.theta.data_ptr(), self.store.m.data_ptr(), self.store.v.data_ptr(),
                                              grad.data_ptr(), n, float(p.learning_rate),
                                              float(p.adam_optimizer_beta1), float(p.adam_optimizer_beta2),
                                              float(p.optimizer_epsilon), self.adam_state.data_ptr(), st))
        self.online_changed()


class DQNAgent(object):
    double_dqn = False
    target_on_s = False        # PAL: the target network's Q values on s (QNetworkWrapper.target_s)

    def __init__(self, agent_parameters, parent=None, observation_shape=None, num_actions=None, device=None,
                 seed=None):
        self.ap = agent_parameters
        self.parent = parent
        self.lib = _lib.load()
        self.device = torch.device(device if device is not None else "cuda")
        self.observation_shape = tuple(observation_shape if observation_shape is not None
                                       else agent_parameters.observation_shape)
        self.num_actions = int(num_actions if num_actions is not None else agent_parameters.num_actions)
        net_params = self.ap.network_wrappers["main"]
        self.batch_size = int(net_params.batch_size)
        self.memory = dynamic_import_and_instantiate_module_from_params(self.ap.memory,
                                                                        extra_kwargs={"device": self.device})
        self.pre_network_filter = self.ap.pre_network_filter
        B, A, dev = self.batch_size, self.num_actions, self.device
        obs_dtype = torch.uint8 if len(self.observation_shape) == 3 else torch.float32
        # persistent minibatch buffers: the replay's gather writes straight into the first conv's input
        self.batch_buffers = {
            "state:observation": torch.zeros((B,) + self.observation_shape, dtype=obs_dtype, device=dev),
            "next_state:observation": torch.zeros((B,) + self.observation_shape, dtype=obs_dtype, device=dev),
            "action": torch.zeros(B, dtype=torch.int64, device=dev),
            "reward": torch.zeros(B, dtype=torch.float64, device=dev),
            "game_over": torch.zeros(B, dtype=torch.uint8, device=dev),
            "idx": torch.zeros(B, dtype=torch.int64, device=dev),
            "weight": torch.ones(B, dtype=torch.float64, device=dev),
            "weight32": torch.ones(B, dtype=torch.float32, device=dev),
        }
        extra = self._extra_columns()
        self.batch_buffers.update(extra)
        derived = self._memory_columns()
        self.batch_buffers.update(derived)
        # columns whose persistent buffers a batch must use for the CUDA-graph replay (fixed pointers in the graphs)
        self._own_columns = ("action", "reward", "game_over") + tuple(extra) + tuple(derived)
        # the ring's column layout = the agent's batch buffers, fixed before the first store: store(Transition) then
        # casts what the environment hands out (gym: float64) instead of the gather overrunning float32 buffers
        if hasattr(self.memory, "declare_schema") and self.memory.ring.specs is None:
            img = ("state:observation", "next_state:observation") if len(self.observation_shape) == 3 else ()
            self.memory.declare_schema({k: self.batch_buffers[k] for k in
                                        ("state:observation", "next_state:observation", "action", "reward",
                                         "game_over") + tuple(extra)}, image_columns=img)
        dueling = "DuelingQHead" in getattr(net_params, "heads_parameters", ["QHead"])
        gen = torch.Generator().manual_seed(int(seed)) if seed is not None else None
        scheme = getattr(getattr(net_params, "middleware_parameters", None), "scheme", MiddlewareScheme.Medium)
        self.head_outputs = self._head_outputs()      # width of the head's output layer (C51: actions x atoms)
        self.net_def = QNetworkDef(dev, self.observation_shape, self.head_outputs, dueling=dueling,
                                   middleware_units=MiddlewareScheme.units[getattr(scheme, "value", scheme)],
                                   **self._head_kwargs())
        self.net_def.store.init_glorot(gen)
        # Fused input path (image observations on the tensor-core path): the replay's sample kernel writes the
        # space-to-depth bf16 plane the first convolution contracts -- no staged uint8 copy, no conversion pass.
        self.s2d = None
        first = self.net_def.trunk.layers[0]
        if (self.net_def.is_image and B >= 128 and B % 32 == 0 and _lib.tune_default("gemm_tiled", 1) and
                _lib.tune_default("conv_s2d", 1) and _lib.tune_default("fused_input", 1) and
                first.KH % first.S == 0 and first.H % first.S == 0 and first.W % first.S == 0 and
                (first.S * first.C) % 8 == 0 and tl.channels_ok(first.S * first.S * first.C) and
                tl.width_ok(first.N)):
            H, W, C, S = first.H, first.W, first.C, first.S
            mk = lambda: tl.PlaneBuf((H // S) * (W // S) * B, S * S * C, dev, npix=(H // S) * (W // S), nplanes=1)  # noqa
            self.s2d = {"columns": {"state:observation": mk(), "next_state:observation": mk()},
                        "geometry": (H, W, C, S)}
        self.networks = {"main": QNetworkWrapper(self.lib, self.net_def, net_params, B, self.batch_buffers,
                                                 self.double_dqn, dev,
                                                 input_planes=self.s2d["columns"] if self.s2d else None,
                                                 target_s=self.target_on_s)}
        if self.networks["main"].has_target:
            self.networks["main"].sync()
        # plain Q head: head forward passes, TD targets, loss and the head's backward pass are ONE fused launch
        net = self.networks["main"]
        self.head_desc = None
        if _lib.tune_default("fused_head", 1) and dev.type == "cuda" and net.has_target and self._head_fusable(net):
            self._build_head_desc()
        self.targets = torch.zeros((B, self.head_outputs), dtype=torch.float32, device=dev)
        self.td_err = torch.zeros(B, dtype=torch.float64, device=dev)
        self.loss_dev = torch.zeros(1, dtype=torch.float32, device=dev)
        pin = dev.type == "cuda"
        self._td_host = torch.zeros(B, dtype=torch.float64, pin_memory=pin)
        self._pa_host = torch.zeros(B, dtype=torch.float64, pin_memory=pin)
        self._pr_host = torch.zeros(B, dtype=torch.float64, pin_memory=pin)
        self._pa_dev = torch.zeros(B, dtype=torch.float64, device=dev)
        self._pr_dev = torch.zeros(B, dtype=torch.float64, device=dev)
        self._fetch_host = torch.zeros(2, dtype=torch.float32, pin_memory=pin)
        self._loss_host = torch.zeros(1, dtype=torch.float32, pin_memory=pin)    # loss of the forward part (fused head)
        # CUDA graphs of the learn step (own minibatch buffers only), one per part: forward + TD targets | loss +
        # backward [+ norm + clip] | [norm +] Adam + plane refresh.  Every launch parameter of those kernels is constant
        # from step to step, so three graph launches replace ~45 kernel launches; the first steps run eagerly (they
        # build the TMA tensor maps, size the workspace and configure shared memory).
        self.use_graph = bool(_lib.tune_default("dqn_graph", 1)) and dev.type == "cuda" and B >= 128
        # two more CUDA streams per learn step: the target network's forward pass runs beside the online network's, the
        # weight-gradient GEMMs beside the data-gradient chain (layers.SideStream; parallel branches of the CUDA graphs)
        self._side_fwd = SideStream(dev)
        self._side_w = SideStream(dev)
        # the tree update of a step only needs the TD errors of its forward part: it runs beside the backward pass and
        # the optimizer; the next sample waits for it (sample_batch)
        self._side_upd = SideStream(dev)
        # ... and the optimizer part of a replayed step (Adam, plane refresh) runs on a fourth stream: the next step's
        # sample + gather does not depend on it and starts as soon as the backward pass (and the all-reduce) is done
        self._side_opt = SideStream(dev)
        if isinstance(self.memory, PrioritizedExperienceReplay):
            self.memory._update_side = self._side_upd          # every other tree access of the memory joins it first
        self._graphs = None                       # [(graph, kernels in it)] of the three parts, once captured
        self._acting = {}                         # number of environments -> (input buffer, forward-only online network)
        self._head_weights = None
        self._eager_steps = 0
        self.graph_kernel_launches = 0            # kernels executed through graph replays (bench.py gpu_launches)
        # counters of agents/agent.py:112-135
        self.training_iteration = 0
        self.total_steps_counter = 0
        self.last_target_network_update_step = 0
        self.last_training_phase_step = 0

    def _head_outputs(self):
        return self.num_actions

    def _head_kwargs(self):
        """extra QNetworkDef arguments of the head (Bootstrapped DQN: head copies)"""
        return {}

    def _extra_columns(self):
        """replay columns beyond the transition's five, as {name: persistent batch buffer} (Bootstrapped DQN: the
        bootstrap masks); they join the ring's schema and the own-buffer check of the CUDA-graph replay"""
        return {}

    def _memory_columns(self):
        """batch columns the memory derives itself rather than storing them (MMC / PAL: the episodic replay's Monte
        Carlo returns), as {name: persistent batch buffer}: sampled into and part of the own-buffer check of the
        CUDA-graph replay, but not ring columns"""
        return {}

    def _head_fusable(self, net):
        return (net.online_s.head_fusable() and net.target_s2.head_fusable() and
                (net.online_s2 is None or net.online_s2.head_fusable()) and
                (net.target_s is None or net.target_s.head_fusable()))

    # ---- reference plumbing ------------------------------------------------------------------------------------------
    @property
    def is_on_policy(self) -> bool:
        return False

    def call_memory(self, func, args=()):
        if not isinstance(args, tuple):
            args = (args,)
        return getattr(self.memory, func)(*args)

    def _should_update_online_weights_to_target(self):
        """agents/agent.py:640-660"""
        step_method = self.ap.algorithm.num_steps_between_copying_online_weights_to_target
        if step_method.__class__ == TrainingSteps:
            should = (self.training_iteration - self.last_target_network_update_step) >= step_method.num_steps
            if should:
                self.last_target_network_update_step = self.training_iteration
        elif step_method.__class__ == EnvironmentSteps:
            should = (self.total_steps_counter - self.last_target_network_update_step) >= step_method.num_steps
            if should:
                self.last_target_network_update_step = self.total_steps_counter
        else:
            raise ValueError("The num_steps_between_copying_online_weights_to_target parameter should be either "
                             "EnvironmentSteps or TrainingSteps. Instead it is {}".format(step_method.__class__))
        return should

    def _should_train(self):
        """agents/agent.py:662-699 for EnvironmentSteps-paced agents"""
        steps = self.ap.algorithm.num_consecutive_playing_steps
        should = (self.total_steps_counter - self.last_training_phase_step) >= steps.num_steps
        should = should and self.call_memory('num_transitions') > 0
        if should:
            self.last_training_phase_step = self.total_steps_counter
        return should

    def _build_head_desc(self):
        net, B, A = self.networks["main"], self.batch_size, self.num_actions
        store, on = net.store, net.online_s
        wname, bname = self.net_def.trunk.names[-1]
        K = on.trunk.layers[-1].K
        d = _lib.DqnHeadDesc()
        self._head_keep = [torch.zeros(((B + 15) // 16) * 8 * (K * A + A + 1), dtype=torch.float32, device=self.device)]
        d.h_next, d.h_online = net.target_s2.trunk.acts[-2].data_ptr(), on.trunk.acts[-2].data_ptr()
        d.h_select = net.online_s2.trunk.acts[-2].data_ptr() if net.online_s2 is not None else None
        d.w_target, d.b_target = store.view(net.theta_target, wname).data_ptr(), store.view(net.theta_target, bname).data_ptr()
        d.w_online, d.b_online = store.view(net.theta, wname).data_ptr(), store.view(net.theta, bname).data_ptr()
        d.discount = float(self.ap.algorithm.discount)
        d.huber = 1 if net.params.replace_mse_with_huber_loss else 0
        d.batch, d.features, d.n_actions = B, K, A
        d.q_online, d.dq = on.q.data_ptr(), on.dq.data_ptr()
        d.q_next = net.target_s2.q.data_ptr()
        on.bind_head_grads(d)
        d.workspace = self._head_keep[0].data_ptr()
        # descriptor field -> batch column, pointed at the step's batch before every head launch
        self._head_columns = {"actions": "action", "rewards": "reward", "game_overs": "game_over"}
        self.head_desc = d

    # ---- acting path (SURVEY.md 8f-4) --------------------------------------------------------------------------------
    def get_all_q_values_for_states(self, states):
        """value_optimization_agent.py:68-72 for a batch of E rollout shards: ONE forward pass of the online network on
        the device.  states: [E, *observation_shape] (uint8 frames / float vectors; host array or CUDA tensor).
        Returns the Q-values as a CUDA tensor [E, num_actions] (persistent buffer, valid until the next call)."""
        self._join_optimizer()
        x = torch.as_tensor(states)
        E = int(x.shape[0])
        inst = self._acting.get(E)
        if inst is None:
            net = self.networks["main"]
            buf = torch.zeros((E,) + self.observation_shape, dtype=self.batch_buffers["state:observation"].dtype,
                              device=self.device)
            # (own workspace: growing the learn step's would invalidate the pointers baked into its CUDA graphs)
            on = self.net_def.instantiate(self.lib, Workspace(self.device), E, buf, net.theta)
            net.add_planes(on)
            inst = self._acting[E] = (buf, on)
        buf, on = inst
        buf.copy_(x.reshape(buf.shape), non_blocking=True)
        return on.forward()

    def choose_actions(self, states, exploration_policy):
        """value_optimization_agent.py:90-128 for E environments stepped in lock-step: batched Q-values on the device,
        then the reference's epsilon-greedy arithmetic on the [E, A] read-back
        (exploration_policies/e_greedy.BatchedEGreedy).  Returns (actions int64 [E], action values [E, A] numpy)."""
        q = self.get_all_q_values_for_states(states).cpu().numpy()
        actions, _ = exploration_policy.get_actions(q)
        return actions, q

    # ---- the hot path ------------------------------------------------------------------------------------------------
    def sample_batch(self):
        """memory sample straight into the persistent minibatch buffers"""
        self._side_upd.join()                     # the previous step's priority update (side stream) comes first
        if self.s2d is not None:
            return self.memory.sample_batch(self.batch_size, out=self.batch_buffers, s2d=self.s2d)
        return self.memory.sample_batch(self.batch_size, out=self.batch_buffers)

    def _part_forward(self, cols, per_libm):
        """target / online forward passes, TD targets and errors (dqn_agent.py:87-103); kernels and one D2H copy"""
        lib, st = self.lib, _lib.current_stream()
        net = self.networks["main"]
        if self.head_desc is not None:
            # feature layers of the three bindings, then the fused head launch: Q values, TD targets / errors, head loss,
            # dL/dQ and the head's backward pass (cb200_dqn_head_fused)
            import ctypes
            d = self.head_desc
            with self._side_fwd:
                net.target_s2.forward_features()
                if net.target_s is not None:
                    net.target_s.forward_features()
            net.online_s.forward_features()
            if self.double_dqn:
                net.online_s2.forward_features()
            self._side_fwd.join()
            for field, name in self._head_columns.items():
                setattr(d, field, cols[name].data_ptr())
            d.weights = self._head_weights.data_ptr() if self._head_weights is not None else None
            d.targets, d.td_err, d.loss = self.targets.data_ptr(), self.td_err.data_ptr(), self.loss_dev.data_ptr()
            _lib.check(lib.cb200_dqn_head_fused(ctypes.byref(d), st))
            if per_libm:
                self._td_host.copy_(self.td_err, non_blocking=True)
            self._loss_host.copy_(self.loss_dev, non_blocking=True)   # the loss is final here: train() reads it early
            return
        with self._side_fwd:
            q_next = net.target_s2.forward()                      # dqn_agent.py:87-90
        q_online = net.online_s.forward()
        q_select = net.online_s2.forward() if self.double_dqn else q_next      # ddqn_agent.py:42-43
        self._side_fwd.join()
        self._head_targets(cols, q_next, q_select, q_online, st)
        if per_libm:
            self._td_host.copy_(self.td_err, non_blocking=True)

    def _head_targets(self, cols, q_next, q_select, q_online, st):
        """TD targets and the errors the memory is updated with (dqn_agent.py:87-103)"""
        _lib.check(self.lib.cb200_dqn_td_targets(q_next.data_ptr(), q_select.data_ptr(), q_online.data_ptr(),
                                                 cols["action"].data_ptr(), cols["reward"].data_ptr(),
                                                 cols["game_over"].data_ptr(), float(self.ap.algorithm.discount),
                                                 self.batch_size, self.num_actions, self.targets.data_ptr(),
                                                 self.td_err.data_ptr(), st))

    def _head_loss_grad(self, weights, st):
        """head loss and dL/d(head output) of the training network (heads/q_head.py, head.py:152-181)"""
        net = self.networks["main"]
        huber = 1 if net.params.replace_mse_with_huber_loss else 0
        _lib.check(self.lib.cb200_regression_head_loss_grad(net.online_s.q.data_ptr(), self.targets.data_ptr(),
                                                            weights.data_ptr() if weights is not None else None,
                                                            self.batch_size, self.num_actions, huber, 1.0,
                                                            net.online_s.dq.data_ptr(), self.loss_dev.data_ptr(), st))

    def _part_optimizer(self, scaler, with_norm):
        """[gradient norm beside] rescale + Adam + refresh of the parameter planes"""
        net = self.networks["main"]
        if with_norm:
            with self._side_w:
                _lib.check(self.lib.cb200_sumsq(net.store.grad.data_ptr(), net.store.size, net.sumsq.data_ptr(),
                                                net.ws.ptr(), _lib.current_stream()))
        net.apply_gradients(scaler)
        self._side_w.join()

    def _join_optimizer(self):
        """the optimizer part of the previous step (own stream) is ordered before whatever the current stream does next"""
        self._side_opt.join()

    def _part_backward(self, weights, with_norm):
        """head loss, backward pass [, global norm and clipping]"""
        lib, st = self.lib, _lib.current_stream()
        net = self.networks["main"]
        if self.head_desc is not None:
            # loss, dL/dQ and the head's gradients were produced by the fused head launch of the forward part
            net.online_s.backward_features(side=self._side_w)
        else:
            self._head_loss_grad(weights, st)
            net.online_s.backward(side=self._side_w)
        self._side_w.join()
        if not with_norm:
            return                                                # the norm is reduced beside the optimizer step
        n = net.store.size
        _lib.check(lib.cb200_sumsq(net.store.grad.data_ptr(), n, net.sumsq.data_ptr(), net.ws.ptr(), st))
        clip = net.params.clip_gradients
        if clip is not None and clip != 0:
            if net.params.gradients_clipping_method != "ClipByGlobalNorm":
                raise NotImplementedError("only ClipByGlobalNorm is implemented on device")
            _lib.check(lib.cb200_clip_by_global_norm(net.store.grad.data_ptr(), n, net.sumsq.data_ptr(), float(clip),
                                                     st))

    def _run(self, k, graph, part, *args):
        """part k of the learn step: its kernels launched one by one, or (graph) its CUDA graph, recorded the first
        time and replayed from then on"""
        if not graph:
            part(*args)
            return
        if len(self._graphs) == k:
            c0 = self.lib.cb200_launch_count()
            g = torch.cuda.CUDAGraph()
            with graph_capture(g):
                part(*args)
            self._graphs.append((g, int(self.lib.cb200_launch_count() - c0)))
        g, n = self._graphs[k]
        g.replay()
        self.graph_kernel_launches += n

    def learn_from_batch(self, batch, fetch=True):
        net = self.networks["main"]
        cols = batch.columns
        img = ("state:observation", "next_state:observation")
        own = all(cols[k].data_ptr() == self.batch_buffers[k].data_ptr() for k in self._own_columns)
        for k in img:
            if self.s2d is not None:
                if k in cols:      # a batch that carries uint8 frames (not sampled through the fused path): convert
                    H, W, C, S = self.s2d["geometry"]
                    x = cols[k].contiguous()
                    _lib.check(self.lib.cb200_u8_s2d_planes(x.data_ptr(), self.batch_size, H, W, C, S,
                                                            self.s2d["columns"][k].ptr, _lib.current_stream()))
                    own = False
            elif cols[k].data_ptr() != self.batch_buffers[k].data_ptr():
                self.batch_buffers[k].copy_(cols[k])             # foreign batch: stage it (device -> device)
                own = False
        # value_optimization_agent.py:74-80: priorities from the pre-update errors, weights from the batch
        per = isinstance(self.memory, PrioritizedExperienceReplay)
        weights = None
        if per:
            weights = cols["weight32"] if "weight32" in cols else cols["weight"].to(torch.float32)
            own = own and weights.data_ptr() == self.batch_buffers["weight32"].data_ptr()
        per_libm = per and self.memory.priority_mode == "libm"
        self._head_weights = weights
        graph = self.use_graph and own and self._eager_steps >= 2
        self._join_optimizer()             # the previous step's Adam / plane refresh (own stream) comes first
        if graph and self._graphs is None:
            self._graphs = []              # this step records the graphs of its parts
        # one rank and no clipping: the gradient norm is only reported, so a replayed step reduces it beside the
        # optimizer step, which runs on its own stream (ordered after the all-reduce, joined lazily).  Eager steps are
        # bound by host time, where those forks and joins cost more than they overlap (CartPole): they keep the norm
        # and the optimizer on the caller's stream.
        clip = net.params.clip_gradients
        norm_in_opt = graph and not parallel.is_distributed() and not (clip is not None and clip != 0)
        self._run(0, graph, self._part_forward, cols, per_libm)
        ev = None
        if per_libm:
            ev = torch.cuda.Event()
            ev.record()
        self._run(1, graph, self._part_backward, weights, not norm_in_opt)
        scaler = parallel.allreduce_gradients(net.store.grad,
                                              net.params.scale_down_gradients_by_number_of_workers_for_sync_training)
        with self._side_opt if graph else NO_SIDE:
            self._run(2, graph, self._part_optimizer, scaler, norm_in_opt)
        if not graph:
            self._eager_steps += 1
        if per:
            if ev is not None:
                ev.synchronize()                                  # GPU is busy with the backward pass meanwhile
                pa, pr = self.memory.host_priorities(self._td_host.numpy())
                self._pa_host.numpy()[:] = pa
                self._pr_host.numpy()[:] = pr
                with self._side_upd.after(ev):
                    self._pa_dev.copy_(self._pa_host, non_blocking=True)
                    self._pr_dev.copy_(self._pr_host, non_blocking=True)
                    self.memory.update_priorities_device(cols["idx"], self._pa_dev, self._pr_dev)
            else:
                self.memory.update_priorities(cols["idx"], self.td_err)
        if fetch == "loss" and self.head_desc is not None:
            # train(): only the loss goes back to the caller.  With the fused head it is final when the forward part is
            # (its D2H copy sits right behind the head launch), so the host returns while the backward pass, the tree
            # update and the optimizer are still running -- the next step's store() / sample preparation overlaps them.
            if ev is None:
                ev = torch.cuda.Event()
                ev.record()             # (no libm priorities: nothing waited for the forward part yet; conservative)
            ev.synchronize()
            loss = float(self._loss_host[0])
            return loss, [loss], None
        if fetch:
            # one synchronisation for both scalars (loss, squared gradient norm) through a pinned pair
            self._join_optimizer()      # the optimizer's stream (where the norm is reduced when nothing clips) too:
            self._side_upd.join()       # a fetched step is complete -- parameters and trees -- when this call returns
            self._fetch_host[0:1].copy_(self.loss_dev, non_blocking=True)
            self._fetch_host[1:2].copy_(net.sumsq, non_blocking=True)
            torch.cuda.current_stream().synchronize() if self.device.type == "cuda" else None
            loss = float(self._fetch_host[0])
            return loss, [loss], float(np.sqrt(np.float32(self._fetch_host[1])))
        return self.loss_dev, [self.loss_dev], net.sumsq

    def train(self, fetch=True):
        """agents/agent.py:701-784 (single-agent, non batch-RL branch)."""
        loss = 0
        if not self._should_train():
            return loss
        for _ in range(self.ap.algorithm.num_consecutive_training_steps):
            self.training_iteration += 1
            batch = self.sample_batch()
            total_loss, losses, unclipped_grads = self.learn_from_batch(batch, fetch="loss" if fetch else False)
            loss = loss + total_loss if fetch else total_loss
            net = self.networks["main"]
            if net.has_target and self._should_update_online_weights_to_target():
                self._join_optimizer()
                net.update_target_network(self.ap.algorithm.rate_for_copying_weights_to_target)
        return loss


class DDQNAgent(DQNAgent):
    double_dqn = True
