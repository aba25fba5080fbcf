"""N-step Q-learning on the GPU, E environment streams stepped in lock step.  Drop-in for

  rl_coach/agents/n_step_q_agent.py:34-153               parameters, learn_from_batch, train (target copy first)
  rl_coach/agents/policy_optimization_agent.py:85-135    segment cut every t_max steps or at the episode's end

Each stream behaves like one asynchronous reference worker: it has its own cut position and closes a segment when t_max
(``num_steps_between_gradient_updates``) steps have passed since its last cut, or on game_over.  At every lock-step
``train()`` all segments closed at that step are learned in ONE learn step whose gradient is the mean over those
segments of each segment's own gradient (the synchronous-training rule of
``scale_down_gradients_by_number_of_workers_for_sync_training``, one segment = one worker).  The target copy counts
lock-step steps (each stream's own steps); ``training_iteration`` counts learn steps.  With E = 1 this is the
reference schedule.

The rollout buffer, the cuts and the gather are ``coach_b200.memories.lockstep_segments``, the row buckets and the
learn step's skeleton ``coach_b200.agents.lockstep_agent``.  One learn step = gather -> target features of the bootstrap
states (N-Step) or of every s' (1-Step) -> online features -> ``cb200_nstep_q_head`` (Q, bootstrap max, the fp64
return recurrence, targets, loss, dL/dQ, the head's gradients and dL/dh) -> backward -> TF-Adam.

Refused (ValueError): ``apply_gradients_every_x_episodes != 1`` (gradients are applied after every segment), a
``targets_horizon`` other than 'N-Step' / '1-Step' (the reference silently trains on zero loss then), a dueling head, and
more than one rank.  Checkpoints hold the networks, Adam and the counters, including every stream's cut position; the
rows of segments still open when the checkpoint is written are not saved: after a restore those segments are learned
from the rows observed since.
"""
import ctypes

from coach_b200 import _lib, parallel
from coach_b200.agents.dqn_agent import DQNAgent
from coach_b200.agents.lockstep_agent import LockstepAgent
from coach_b200.architectures.layers import Workspace
from coach_b200.base_parameters import (AgentParameters, AlgorithmParameters, EnvironmentSteps,
                                        InputEmbedderParameters, NetworkParameters)
from coach_b200.exploration_policies.e_greedy import EGreedyParameters

HORIZONS = {"N-Step": _lib.NSTEP_NSTEP, "1-Step": _lib.NSTEP_ONESTEP}


class NStepQNetworkParameters(NetworkParameters):
    """n_step_q_agent.py:34-43"""

    def __init__(self):
        super().__init__()
        self.input_embedders_parameters = {'observation': InputEmbedderParameters()}
        self.heads_parameters = ["QHead"]
        self.optimizer_type = 'Adam'
        self.async_training = True
        self.shared_optimizer = True
        self.create_target_network = True


class NStepQAlgorithmParameters(AlgorithmParameters):
    """n_step_q_agent.py:46-73"""

    def __init__(self):
        super().__init__()
        self.num_steps_between_copying_online_weights_to_target = EnvironmentSteps(10000)
        self.apply_gradients_every_x_episodes = 1
        self.num_steps_between_gradient_updates = 5          # t_max
        self.targets_horizon = 'N-Step'


class NStepQAgentParameters(AgentParameters):
    """n_step_q_agent.py:76-85; the reference's SingleEpisodeBuffer is the agent's device rollout buffer"""

    def __init__(self):
        super().__init__(algorithm=NStepQAlgorithmParameters(), memory=None,
                         networks={"main": NStepQNetworkParameters()})
        self.exploration = EGreedyParameters()

    @property
    def path(self):
        return 'coach_b200.agents.n_step_q_agent:NStepQAgent'


class NStepQAgent(LockstepAgent):
    head_desc_type = _lib.NstepQHeadDesc
    head_error = "cb200_nstep_q_head needs a QHead of <= 18 actions on a 256- or 512-wide ReLU layer"
    graph_tuning = "nstep_graph"
    is_on_policy = False

    def __init__(self, agent_parameters, parent=None, observation_shape=None, num_actions=None, num_envs=1,
                 device=None, seed=None):
        ap = agent_parameters
        alg, net_params = ap.algorithm, ap.network_wrappers["main"]
        if alg.apply_gradients_every_x_episodes != 1:
            raise ValueError("apply_gradients_every_x_episodes must be 1: gradients are applied after every segment")
        if alg.targets_horizon not in HORIZONS:
            raise ValueError("targets_horizon must be 'N-Step' or '1-Step', got %r (the reference would train on a "
                             "zero loss)" % (alg.targets_horizon,))
        if "DuelingQHead" in getattr(net_params, "heads_parameters", ["QHead"]):
            raise ValueError("NStepQAgent takes a plain QHead, not a dueling head")
        if parallel.is_distributed():
            raise ValueError("NStepQAgent runs on one rank")
        self.num_actions = int(num_actions if num_actions is not None else ap.num_actions)
        self.horizon = HORIZONS[alg.targets_horizon]
        self.gather_keys = ("state", "action", "reward", "game_over") + \
            (("next_state",) if self.horizon == _lib.NSTEP_ONESTEP else ())
        self.gather_boot = self.horizon == _lib.NSTEP_NSTEP
        super().__init__(ap, parent, observation_shape, num_envs, device, seed, self.num_actions)
        net = self.networks["main"]
        net.sync()
        self.target_boot = None
        if self.horizon == _lib.NSTEP_NSTEP:
            self.target_boot = self.net_def.instantiate(self.lib, Workspace(self.device), self.num_envs,
                                                        self.segments.boot_states, net.theta_target)
            net.add_planes(self.target_boot)
        self.last_target_network_update_step = 0

    # ---- the DQN agent's acting path ----------------------------------------------------------------------------------------
    _should_update_online_weights_to_target = DQNAgent._should_update_online_weights_to_target
    get_all_q_values_for_states = DQNAgent.get_all_q_values_for_states
    choose_actions = DQNAgent.choose_actions

    def train(self, fetch=True):
        """n_step_q_agent.py:142-153 + policy_optimization_agent.py:85-135: target copy check first, then one learn step
        over the segments that closed.  Returns the loss (0 when no segment closed)."""
        net = self.networks["main"]
        if self._should_update_online_weights_to_target():
            net.update_target_network(self.ap.algorithm.rate_for_copying_weights_to_target)
        streams, rows = self.segments.close()
        if len(streams) == 0:
            return 0
        self.training_iteration += 1
        return self._learn(self.segments.tables(streams, rows), True, fetch)

    # ---- the learn step ---------------------------------------------------------------------------------------------------
    def _boot_instance(self, B):
        """the target network on the bootstrap states (N-Step) or on every row's s' (1-Step)"""
        net = self.networks["main"]
        if self.horizon == _lib.NSTEP_NSTEP:
            return self.target_boot
        if B == 32:
            return net.target_s2
        tn = self.net_def.instantiate(self.lib, Workspace(self.device), B, self.learn["next_state"][:B],
                                      net.theta_target)
        net.add_planes(tn)
        return tn

    def _fill_desc(self, d, on, tn, B):
        net, store, alg = self.networks["main"], self.net_def.store, self.ap.algorithm
        wname, bname = self.net_def.trunk.names[-1]
        d.h_online, d.h_boot = on.trunk.acts[-2].data_ptr(), tn.trunk.acts[-2].data_ptr()
        d.w_target, d.b_target = store.view(net.theta_target, wname).data_ptr(), \
            store.view(net.theta_target, bname).data_ptr()
        d.w_online, d.b_online = store.view(net.theta, wname).data_ptr(), store.view(net.theta, bname).data_ptr()
        d.actions, d.rewards = self.learn["action"].data_ptr(), self.learn["reward"].data_ptr()
        d.game_overs = self.learn["game_over"].data_ptr()
        d.discount = float(alg.discount)
        d.horizon = self.horizon
        d.huber = 1 if net.params.replace_mse_with_huber_loss else 0
        d.n_actions = self.num_actions
        d.q_online, d.dq = on.q.data_ptr(), on.dq.data_ptr()
        K, A, E = d.features, self.num_actions, self.num_envs
        return ((E + 3) // 4) * 4 * (K * A + A + 1)

    def _launch_head(self, d, st):
        _lib.check(self.lib.cb200_nstep_q_head(ctypes.byref(d), st))
