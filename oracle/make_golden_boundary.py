"""Generates tests/golden/acting.npz and tests/golden/boundary.json from the UNMODIFIED reference (imported through
oracle/ref_loader.py): the actions its per-environment EGreedy objects select, the argument lists of its memory
methods, its Parameters defaults and its checkpoint-file conventions.  tests/test_acting.py and tests/test_boundary.py
replay them without the reference.

Run where the reference tree is present:   python -m oracle.make_golden_boundary
TEST INFRASTRUCTURE ONLY.
"""
import importlib
import inspect
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")

# the q-value stream of tests/test_acting.py
E, A, T = 5, 6, 40


def acting_q():
    rng = np.random.RandomState(0)
    q = rng.randn(T, E, A).astype(np.float32)
    q[3, 1, 2] = q[3, 1, 4] = q[3, 1].max() + 1.0            # exact ties: random tie-break consumes the stream
    q[7, 0] = 0.5
    return q


def golden_acting():
    from rl_coach.core_types import RunPhase as RefPhase
    from rl_coach.exploration_policies.e_greedy import EGreedy
    from rl_coach.schedules import LinearSchedule as RefLinear
    from rl_coach.spaces import DiscreteActionSpace
    q = acting_q()
    out = {}
    for phase in ("train", "test"):
        np.random.seed(11)
        refs = [EGreedy(DiscreteActionSpace(A), RefLinear(1.0, 0.1, 25), 0.05) for _ in range(E)]
        for p in refs:
            p.change_phase(RefPhase.TEST if phase == "test" else RefPhase.TRAIN)
        want = np.zeros((T, E), dtype=np.int64)
        for t in range(T):
            for e in range(E):
                want[t, e], _ = refs[e].get_action(q[t, e])
        out["actions_" + phase] = want
        out["epsilon_" + phase] = np.float64(refs[0].epsilon_schedule.current_value)
    np.savez_compressed(os.path.join(OUT, "acting.npz"), **out)


MEMORY_CLASSES = {"ExperienceReplay": "rl_coach.memories.non_episodic.experience_replay",
                  "PrioritizedExperienceReplay": "rl_coach.memories.non_episodic.prioritized_experience_replay",
                  "EpisodicExperienceReplay": "rl_coach.memories.episodic.episodic_experience_replay"}
PARAMETERS = {"DQNAgentParameters": "rl_coach.agents.dqn_agent", "DDQNAgentParameters": "rl_coach.agents.ddqn_agent",
              "ClippedPPOAgentParameters": "rl_coach.agents.clipped_ppo_agent",
              "DDPGAgentParameters": "rl_coach.agents.ddpg_agent", "TD3AgentParameters": "rl_coach.agents.td3_agent",
              "SoftActorCriticAgentParameters": "rl_coach.agents.soft_actor_critic_agent",
              "CategoricalDQNAgentParameters": "rl_coach.agents.categorical_dqn_agent"}


def comparable(v):
    """the form tests/test_boundary.py compares a default in (None: structured value, not compared)"""
    if hasattr(v, "num_steps"):
        return {"steps_type": type(v).__name__, "num_steps": v.num_steps}
    if hasattr(v, "current_value"):
        return {"schedule_value": float(v.current_value)}
    if hasattr(v, "name") and not isinstance(v, (int, float, str, bool)):
        return {"enum": v.name}
    if isinstance(v, (int, float, str, bool, type(None))):
        return {"value": v}
    if isinstance(v, tuple) and all(isinstance(x, (int, float, str, bool, type(None))) for x in v):
        return {"tuple": list(v)}
    return None


def golden_boundary():
    from rl_coach.checkpoint import CheckpointStateFile, SingleCheckpoint
    from rl_coach.memories.non_episodic.prioritized_experience_replay import PrioritizedExperienceReplay
    out = {"per_constructor_args": sorted(inspect.getfullargspec(PrioritizedExperienceReplay).args)}
    methods = {}
    for cls_name, mod in MEMORY_CLASSES.items():
        rcls = getattr(importlib.import_module(mod), cls_name)
        methods[cls_name] = {name: [a for a in inspect.getfullargspec(fn).args if a not in ("self", "lock")]
                             for name, fn in inspect.getmembers(rcls, inspect.isfunction)}
    out["memory_methods"] = methods
    out["memory_modules"] = dict(MEMORY_CLASSES)
    # what the reference's own loader (utils.py short_dynamic_import, used by
    # dynamic_import_and_instantiate_module_from_params) returns for the device PER's Parameters.path
    from rl_coach.utils import short_dynamic_import
    from coach_b200.memories.prioritized_experience_replay import PrioritizedExperienceReplayParameters
    path = PrioritizedExperienceReplayParameters().path
    cls = short_dynamic_import(path)
    out["per_path_resolution"] = {"path": path, "resolved": "%s:%s" % (cls.__module__, cls.__name__)}
    params = {}
    for cls_name, mod in PARAMETERS.items():
        ref = getattr(importlib.import_module(mod), cls_name)()
        rec = {"memory_class": type(ref.memory).__name__,
               "algorithm": {k: comparable(v) for k, v in vars(ref.algorithm).items()},
               "network_wrappers": {net: {k: comparable(v) for k, v in vars(w).items()}
                                    for net, w in ref.network_wrappers.items()}}
        params[cls_name] = rec
    out["parameters"] = params
    with tempfile.TemporaryDirectory() as d:
        CheckpointStateFile(d).write(SingleCheckpoint(12, "12_Step-99.ckpt"))
        with open(os.path.join(d, CheckpointStateFile.checkpoint_state_filename)) as f:
            out["checkpoint_state_file"] = {"name": CheckpointStateFile.checkpoint_state_filename,
                                            "content_for_12_Step-99": f.read()}
    with open(os.path.join(OUT, "boundary.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


def main():
    from oracle import ref_loader
    ref_loader.load()
    golden_acting()
    golden_boundary()


if __name__ == "__main__":
    main()
