"""The plug points of INTEGRATION.md checked against what the UNMODIFIED reference exposes, recorded in
tests/golden/boundary.json by oracle/make_golden_boundary.py: the argument lists of its memory methods and of the PER
constructor, its Parameters defaults and its checkpoint-file conventions.  CPU only: nothing here launches a kernel --
the device classes are bound, resolved and type-checked, not run."""
import importlib
import inspect
import json
import os

import pytest


@pytest.fixture
def ref(golden_dir):
    with open(os.path.join(golden_dir, "boundary.json")) as f:
        return json.load(f)


def test_device_per_accepts_the_reference_constructor_and_resolves_from_its_path(ref):
    """the device PER accepts every constructor argument of the reference PER, and its Parameters.path is the string the
    reference's own loader (short_dynamic_import behind dynamic_import_and_instantiate_module_from_params,
    utils.py:389-404) was recorded resolving to the device class; the project's resolver agrees"""
    from coach_b200.memories import prioritized_experience_replay as dev
    from coach_b200.utils import short_dynamic_import
    params = dev.PrioritizedExperienceReplayParameters()
    rec = ref["per_path_resolution"]
    assert params.path == rec["path"]
    assert rec["resolved"] == "coach_b200.memories.prioritized_experience_replay:PrioritizedExperienceReplay"
    cls = short_dynamic_import(params.path)
    assert cls is dev.PrioritizedExperienceReplay
    ctor = set(inspect.getfullargspec(cls).args)
    assert set(ref["per_constructor_args"]) <= ctor, "device PER must accept every constructor argument of the reference PER"
    passed = {k for k in params.__dict__ if k in ctor}
    assert {"max_size", "alpha", "beta", "epsilon", "allow_duplicates_in_batch_sampling"} <= passed


@pytest.mark.parametrize("dev_path,ref_path,cls_name", [
    ("coach_b200.memories.experience_replay", "rl_coach.memories.non_episodic.experience_replay", "ExperienceReplay"),
    ("coach_b200.memories.prioritized_experience_replay", "rl_coach.memories.non_episodic.prioritized_experience_replay",
     "PrioritizedExperienceReplay"),
    ("coach_b200.memories.episodic_experience_replay", "rl_coach.memories.episodic.episodic_experience_replay",
     "EpisodicExperienceReplay"),
])
def test_memory_method_surface_covers_the_reference(ref, dev_path, ref_path, cls_name):
    """every public method of the reference memory that the replay -> learn path calls exists on the device class with
    the same leading arguments"""
    assert ref["memory_modules"][cls_name] == ref_path, "golden data recorded from another reference class"
    dcls = getattr(importlib.import_module(dev_path), cls_name)
    used = {"store", "sample", "num_transitions", "length", "clean", "freeze", "assert_not_frozen", "get_transition",
            "get", "remove_transition", "update_priorities", "store_episode", "num_complete_episodes",
            "num_transitions_in_complete_episodes", "verify_last_episode_is_closed", "mean_reward", "save",
            "load_pickled", "get_shuffled_training_data_generator"}
    methods = ref["memory_methods"][cls_name]
    assert {"store", "sample", "num_transitions"} <= set(methods)
    for name, ra in methods.items():
        if name not in used:
            continue
        assert hasattr(dcls, name), "%s.%s missing" % (cls_name, name)
        da = [a for a in inspect.getfullargspec(getattr(dcls, name)).args if a not in ("self", "lock")]
        assert da[:len(ra)] == ra or name in ("sample",), (cls_name, name, ra, da)


def test_parameter_defaults_match_the_reference(ref):
    """the Parameters classes carry the reference's defaults for every field they define (agents' algorithm / network
    parameters, memory parameters)"""
    from coach_b200.agents.categorical_dqn_agent import CategoricalDQNAgentParameters
    from coach_b200.agents.dqn_agent import DQNAgentParameters, DDQNAgentParameters
    from coach_b200.agents.clipped_ppo_agent import ClippedPPOAgentParameters
    from coach_b200.agents.ddpg_agent import DDPGAgentParameters, TD3AgentParameters
    from coach_b200.agents.soft_actor_critic_agent import SoftActorCriticAgentParameters

    def same(a, b):
        if b is None:
            return True                               # structured values (filters, lists of layer objects): not compared
        if "num_steps" in b:
            return type(a).__name__ == b["steps_type"] and a.num_steps == b["num_steps"]
        if "schedule_value" in b:
            return float(a.current_value) == b["schedule_value"]
        if "enum" in b:                               # enums of the reference are plain strings here
            return a == b["enum"] or getattr(a, "name", None) == b["enum"]
        if "tuple" in b:
            return tuple(a) == tuple(b["tuple"])
        return a == b["value"]

    own_only = {"hidden_units", "truncate_dataset_to_playing_steps", "middleware_parameters", "heads_parameters"}
    for mine in (DQNAgentParameters(), DDQNAgentParameters(), ClippedPPOAgentParameters(), DDPGAgentParameters(),
                 TD3AgentParameters(), SoftActorCriticAgentParameters(), CategoricalDQNAgentParameters()):
        r = ref["parameters"][type(mine).__name__]
        for k, v in vars(mine.algorithm).items():
            if k in own_only or k not in r["algorithm"]:
                continue
            assert same(v, r["algorithm"][k]), (type(mine).__name__, "algorithm", k, v, r["algorithm"][k])
        for net in mine.network_wrappers:
            for k, v in vars(mine.network_wrappers[net]).items():
                if k in own_only or k not in r["network_wrappers"][net]:
                    continue
                rv = r["network_wrappers"][net][k]
                assert same(v, rv), (type(mine).__name__, net, k, v, rv)
        assert type(mine.memory).__name__ == r["memory_class"], type(mine).__name__


def test_presets_define_the_five_baseline_configurations():
    """coach_b200/presets/*: agent parameters whose path strings resolve to the device classes"""
    from coach_b200.utils import short_dynamic_import
    for name in ("CartPole_DQN", "Atari_DQN_with_PER", "Atari_Dueling_DDQN_with_PER_OpenAI", "Mujoco_ClippedPPO",
                 "Mujoco_SAC", "Mujoco_TD3", "Atari_C51"):
        mod = importlib.import_module("coach_b200.presets." + name)
        ap = mod.agent_params
        assert short_dynamic_import(ap.path).__module__.startswith("coach_b200.agents")
        assert short_dynamic_import(ap.memory.path).__module__.startswith("coach_b200.memories")
    from coach_b200.presets import Atari_Dueling_DDQN_with_PER_OpenAI as p5
    from coach_b200.architectures.q_network import QNetworkDef
    from coach_b200.base_parameters import MiddlewareScheme
    net = p5.agent_params.network_wrappers["main"]
    qn = QNetworkDef("cpu", p5.observation_shape, p5.num_actions, dueling="DuelingQHead" in net.heads_parameters,
                     middleware_units=MiddlewareScheme.units[net.middleware_parameters.scheme])
    assert qn.store.num_params() - 1 == 3293863          # SURVEY section 8d, config 5 (+1: the rescaler scalar)


def test_checkpoint_names_and_state_file_interoperate_with_the_reference(ref, tmp_path):
    """coach_b200/checkpoint.py follows the reference's on-disk conventions (checkpoint.py:115-155, :247-273,
    graph_manager.py:630): the state file has the reference's name and the content its CheckpointStateFile writes, we
    read what the reference writes, and a half-written or foreign state file yields no checkpoint."""
    from coach_b200 import checkpoint as ck
    d = str(tmp_path)
    name = ck.checkpoint_name(7, 123456)
    assert name == "7_Step-123456.ckpt"                                   # '{}_Step-{}.ckpt' of graph_manager.py:630
    sf = ref["checkpoint_state_file"]
    assert ck.STATE_FILE == sf["name"]
    # what the reference's CheckpointStateFile(d).write(SingleCheckpoint(12, "12_Step-99.ckpt")) leaves on disk
    ck._write_state_file(d, ck.checkpoint_name(12, 99))
    with open(os.path.join(d, ck.STATE_FILE)) as f:
        assert f.read() == sf["content_for_12_Step-99"]
    with open(os.path.join(d, ck.STATE_FILE), "w") as f:
        f.write(sf["content_for_12_Step-99"])
    assert ck.read_state_file(d) == "12_Step-99.ckpt"
    # garbage in the state file: no checkpoint
    with open(os.path.join(d, ck.STATE_FILE), "w") as f:
        f.write("not a checkpoint")
    assert ck.read_state_file(d) is None
