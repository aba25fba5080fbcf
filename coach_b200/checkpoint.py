"""Checkpoint / restore of everything the replay -> learn path owns on the device (SURVEY.md section 8f-3):

  network parameters, target copies, Adam slots and step state     (reference: the TF Saver inside
                                                                     graph_managers/graph_manager.py:616-658)
  replay ring columns + cursor / count, PER trees, beta schedule    (memories/non_episodic/experience_replay.py:229-261
                                                                     pickles the transition list; a 59 GB ring is
                                                                     streamed to .npy column files instead)
  running observation statistics                                     (utilities/shared_running_stats.py:170-189: the
                                                                     reference's own pickle, same keys, same file name)
  agent counters

On-disk conventions follow the reference: a checkpoint is named ``<id>_Step-<env steps>.ckpt`` (graph_manager.py:630),
the directory's ``.coach_checkpoint`` file holds the name of the last COMPLETE checkpoint and is written last
(checkpoint.py:115-155, CheckpointStateFile), so a reader never sees a half-written one.  A restored agent continues
bit-identically (same losses, same sampled indices given the same host RNG state): tests/test_checkpoint_gpu.py.
"""
import json
import os
import pickle
import re

import numpy as np
import torch

STATE_FILE = ".coach_checkpoint"
_NAME = re.compile(r"^(\d+)_Step-(\d+)\.ckpt$")


def checkpoint_name(checkpoint_id: int, env_steps: int) -> str:
    return "{}_Step-{}.ckpt".format(int(checkpoint_id), int(env_steps))


def read_state_file(checkpoint_dir: str):
    """name of the last complete checkpoint in the directory, or None (CheckpointStateFile.read)"""
    path = os.path.join(checkpoint_dir, STATE_FILE)
    if not os.path.exists(path):
        return None
    with open(path, "r") as fd:
        name = fd.read(256).strip()
    return name if _NAME.match(name) else None


def _write_state_file(checkpoint_dir: str, name: str):
    tmp = os.path.join(checkpoint_dir, STATE_FILE + ".tmp")
    with open(tmp, "w") as fd:
        fd.write(name)
    os.replace(tmp, os.path.join(checkpoint_dir, STATE_FILE))


# ---- tensors <-> files ----------------------------------------------------------------------------------------------
def _save_tensor(path, t, rows=None, chunk_bytes=1 << 28):
    """device tensor -> .npy, streamed through host chunks (the ring columns are tens of GB)"""
    t = t if rows is None else t[:rows]
    arr = np.lib.format.open_memmap(path, mode="w+", dtype=np.dtype(str(t.dtype).replace("torch.", "")),
                                    shape=tuple(t.shape))
    if t.numel() == 0:
        del arr
        return
    flat_rows = t.shape[0] if t.dim() > 0 else 1
    per = max(1, int(chunk_bytes // max(1, t[0].numel() * t.element_size()))) if t.dim() > 0 else 1
    if t.dim() == 0:
        arr[...] = t.item()
    else:
        for lo in range(0, flat_rows, per):
            arr[lo:lo + per] = t[lo:lo + per].cpu().numpy()
    arr.flush()
    del arr


def _load_into(path, t, rows=None, chunk_bytes=1 << 28):
    arr = np.load(path, mmap_mode="r")
    dst = t if rows is None else t[:rows]
    if tuple(arr.shape) != tuple(dst.shape):
        raise ValueError("checkpoint tensor %s has shape %s, expected %s" % (path, arr.shape, tuple(dst.shape)))
    if dst.dim() == 0:
        dst.fill_(arr.item())
        return
    if dst.numel() == 0:                   # an empty replay (ClippedPPO right after a training phase) saves no rows
        return
    per = max(1, int(chunk_bytes // max(1, dst[0].numel() * dst.element_size())))
    for lo in range(0, dst.shape[0], per):
        dst[lo:lo + per].copy_(torch.from_numpy(np.ascontiguousarray(arr[lo:lo + per])))


# ---- pieces ---------------------------------------------------------------------------------------------------------
def _schedule_state(s):
    return {k: (float(v) if isinstance(v, (int, float, np.floating)) else v) for k, v in vars(s).items()}


def save_memory(mem, prefix):
    """ring columns (valid slots only), cursor / count, PER trees and scalars, episodic bookkeeping"""
    mem._flush()
    r = mem.ring
    meta = {"class": type(mem).__name__, "capacity": r.capacity, "cursor": r.cursor, "count": r.count, "specs": None}
    if r.specs is not None:
        meta["specs"] = [[name, list(sp.shape), str(sp.dtype)] for name, sp in r.specs.items()]
        rows = r.capacity if r.count == r.capacity else r.cursor          # before the first wrap only [0, cursor) is live
        meta["rows"] = rows
        for k, (name, _) in enumerate(r.specs.items()):
            _save_tensor("%s.ring%d.npy" % (prefix, k), r.columns[name], rows)
        if r.frames is not None:          # frame-deduplicated ring: the frame store and its cursor
            meta["frame_stack"] = {name: list(shape) for name, shape in r.stack_cols.items()}
            meta["frame_slack"], meta["frame_counter"] = r.frame_slack, int(r._fc)
            _save_tensor(prefix + ".frames.npy", r.frames, min(int(r._fc), r.frame_capacity))
            np.save(prefix + ".frame_min.npy", r._min_fc)
    if hasattr(mem, "sum_tree"):
        for tag in ("sum_tree", "min_tree", "max_tree"):
            _save_tensor("%s.%s.npy" % (prefix, tag), getattr(mem, tag))
        meta.update(maximal_priority=float(mem.maximal_priority), list_len=int(mem._list_len), alpha=float(mem.alpha),
                    epsilon=float(mem.epsilon), beta=_schedule_state(mem.beta), priority_mode=mem.priority_mode)
    if hasattr(mem, "episode_lengths"):
        meta.update(episode_lengths=[int(x) for x in mem.episode_lengths], open_len=int(mem._open_len))
        if mem._returns is not None:
            _save_tensor(prefix + ".returns.npy", mem._returns)
        if getattr(mem, "_bootstrap", None) is not None:
            _save_tensor(prefix + ".bootstrap.npy", mem._bootstrap)
    with open(prefix + ".memory.json", "w") as f:
        json.dump(meta, f)


def restore_memory(mem, prefix):
    from coach_b200.memories.device_ring import ColumnSpec
    from collections import OrderedDict
    with open(prefix + ".memory.json") as f:
        meta = json.load(f)
    if meta["class"] != type(mem).__name__ or meta["capacity"] != mem.ring.capacity:
        raise ValueError("checkpoint holds a %s of capacity %d, this memory is a %s of capacity %d"
                         % (meta["class"], meta["capacity"], type(mem).__name__, mem.ring.capacity))
    r = mem.ring
    r._pending = 0
    if meta["specs"] is not None:
        specs = OrderedDict((name, ColumnSpec(name, tuple(shape), np.dtype(dt))) for name, shape, dt in meta["specs"])
        if r.specs is None:
            if meta.get("frame_stack"):
                r.frame_slack = float(meta["frame_slack"])
                for name, shape in meta["frame_stack"].items():
                    r.stack_cols[name] = tuple(shape)
            r.set_schema(specs)
        elif [(n, s.shape, s.dtype) for n, s in r.specs.items()] != [(n, s.shape, s.dtype) for n, s in specs.items()]:
            raise ValueError("checkpoint column layout differs from this replay's")
        for k, name in enumerate(r.specs):
            _load_into("%s.ring%d.npy" % (prefix, k), r.columns[name], meta["rows"])
    r.cursor, r.count = int(meta["cursor"]), int(meta["count"])
    if meta.get("frame_stack"):
        if {k: tuple(v) for k, v in meta["frame_stack"].items()} != dict(r.stack_cols):
            raise ValueError("checkpoint holds a frame-deduplicated replay, this memory is laid out differently")
        r._fc, r._pending_frames = int(meta["frame_counter"]), 0
        r._recent.clear()                 # frame identities do not survive a restart: the next frames are stored anew
        _load_into(prefix + ".frames.npy", r.frames, min(r._fc, r.frame_capacity))
        r._min_fc[:] = np.load(prefix + ".frame_min.npy")
    if hasattr(mem, "sum_tree"):
        for tag in ("sum_tree", "min_tree", "max_tree"):
            _load_into("%s.%s.npy" % (prefix, tag), getattr(mem, tag))
        mem.maximal_priority = meta["maximal_priority"]
        mem._list_len = int(meta["list_len"])
        for k, v in meta["beta"].items():
            setattr(mem.beta, k, v)
    if hasattr(mem, "episode_lengths"):
        mem.episode_lengths = list(meta["episode_lengths"])
        mem._open_len = int(meta["open_len"])
        if os.path.exists(prefix + ".returns.npy"):
            if mem._returns is None:
                mem._returns = torch.zeros(r.capacity, dtype=torch.float64, device=mem.device)
            _load_into(prefix + ".returns.npy", mem._returns)
        if os.path.exists(prefix + ".bootstrap.npy"):
            if mem._bootstrap is None:
                mem._bootstrap = torch.zeros(r.capacity, dtype=torch.uint8, device=mem.device)
            _load_into(prefix + ".bootstrap.npy", mem._bootstrap)


def _network_items(agent):
    """(tag, ParamStore, extra tensors {name: tensor}, owner) for every network of an agent"""
    out = []
    nets = getattr(agent, "networks", None)
    if isinstance(nets, dict) and "main" in nets and hasattr(nets["main"], "store"):          # DQN family
        w = nets["main"]
        extra = {"adam_state": w.adam_state}
        if w.theta_target is not None:
            extra["target"] = w.theta_target
        out.append(("main", w.store, extra, w))
    for tag in ("main", "actor", "critic", "policy", "q", "v"):                               # _Net based agents
        net = getattr(agent, tag, None)
        if net is not None and hasattr(net, "store") and hasattr(net, "adam_state"):
            out.append((tag, net.store, {"adam_state": net.adam_state, "target": net.target}, net))
    return out


def save_checkpoint(agent, checkpoint_dir: str, checkpoint_id: int = 0, env_steps: int = None) -> str:
    """Writes one checkpoint of the agent (networks + optimizer + replay + filters + counters) and, last, the state
    file.  Returns the checkpoint name."""
    os.makedirs(checkpoint_dir, exist_ok=True)
    if torch.cuda.is_available():
        torch.cuda.synchronize()          # side streams of the learn step (optimizer, priority update) included
    env_steps = int(getattr(agent, "total_steps_counter", 0) if env_steps is None else env_steps)
    name = checkpoint_name(checkpoint_id, env_steps)
    prefix = os.path.join(checkpoint_dir, name)
    torch.cuda.synchronize() if torch.cuda.is_available() else None
    meta = {"agent": type(agent).__name__, "counters": {k: int(getattr(agent, k)) for k in
                                                        ("training_iteration", "total_steps_counter",
                                                         "last_target_network_update_step", "last_training_phase_step")
                                                        if hasattr(agent, k)}, "networks": {}}
    if hasattr(agent, "checkpoint_state"):                    # agent-specific host state (NStepQ: per-stream cuts)
        meta["agent_state"] = agent.checkpoint_state()
    for tag, store, extra, _ in _network_items(agent):
        base = "%s.net_%s" % (prefix, tag)
        for nm, t in (("theta", store.theta), ("m", store.m), ("v", store.v)):
            _save_tensor("%s.%s.npy" % (base, nm), t)
        for nm, t in extra.items():
            _save_tensor("%s.%s.npy" % (base, nm), t)
        meta["networks"][tag] = {"size": int(store.size), "entries": [[n, int(o), list(s)] for n, (o, s) in
                                                                      store.entries.items()],
                                 "extra": sorted(extra)}
    if getattr(agent, "memory", None) is not None and hasattr(agent.memory, "ring"):
        save_memory(agent.memory, prefix)
    flt = getattr(agent, "pre_network_filter", None)
    if flt is not None and hasattr(flt, "save_state_to_checkpoint"):
        flt.save_state_to_checkpoint(checkpoint_dir, name)
    with open(prefix + ".agent.json", "w") as f:
        json.dump(meta, f)
    _write_state_file(checkpoint_dir, name)          # last: marks the checkpoint complete
    return name


def restore_checkpoint(agent, checkpoint_dir: str, name: str = None) -> str:
    """Restores the named checkpoint (default: the one the state file points at) into an agent built with the same
    parameters.  Raises FileNotFoundError when the directory holds no complete checkpoint."""
    name = name or read_state_file(checkpoint_dir)
    if name is None:
        raise FileNotFoundError("no complete checkpoint in %s (%s missing or malformed)" % (checkpoint_dir, STATE_FILE))
    prefix = os.path.join(checkpoint_dir, name)
    if torch.cuda.is_available():
        torch.cuda.synchronize()          # nothing of a running learn step may still write what is restored here
    with open(prefix + ".agent.json") as f:
        meta = json.load(f)
    if meta["agent"] != type(agent).__name__:
        raise ValueError("checkpoint was written by a %s, this is a %s" % (meta["agent"], type(agent).__name__))
    for tag, store, extra, owner in _network_items(agent):
        m = meta["networks"][tag]
        if m["size"] != store.size or [e[0] for e in m["entries"]] != list(store.entries):
            raise ValueError("network %r: parameter layout differs from the checkpoint's" % tag)
        base = "%s.net_%s" % (prefix, tag)
        for nm, t in (("theta", store.theta), ("m", store.m), ("v", store.v)):
            _load_into("%s.%s.npy" % (base, nm), t)
        for nm, t in extra.items():
            _load_into("%s.%s.npy" % (base, nm), t)
        host = m.get("host")
        if host:
            # a DQN checkpoint written while eager agents kept their Adam powers on the host ({beta1 power, beta2
            # power}): only one of the two copies ever advanced (host: eager agent, device: CUDA-graph agent), and both
            # only decrease from the betas
            old = torch.tensor(list(host.values()), dtype=torch.float32)
            extra["adam_state"].copy_(torch.minimum(extra["adam_state"].cpu(), old))
        # operand planes / derived kernels follow the parameters
        for hook in ("online_changed", "target_changed"):
            if hasattr(owner, hook):
                getattr(owner, hook)()
    for k, v in meta["counters"].items():
        setattr(agent, k, v)
    if "agent_state" in meta:
        agent.restore_checkpoint_state(meta["agent_state"])
    if getattr(agent, "memory", None) is not None and hasattr(agent.memory, "ring") and \
            os.path.exists(prefix + ".memory.json"):
        restore_memory(agent.memory, prefix)
    flt = getattr(agent, "pre_network_filter", None)
    if flt is not None and hasattr(flt, "restore_state_from_checkpoint"):
        flt.restore_state_from_checkpoint(checkpoint_dir, name)
    # captured CUDA graphs hold no state of their own, but an agent that captured before the restore replays kernels
    # over the same (now restored) buffers: nothing to invalidate
    return name


# ---- running statistics in the reference's own on-disk format (shared_running_stats.py:170-189) ---------------------
def save_running_stats(stats, checkpoint_dir: str, checkpoint_prefix, extension="srs"):
    d = {"_mean": stats._mean.cpu().numpy(), "_std": stats._std.cpu().numpy(), "_count": stats._count,
         "_sum": stats._sum.cpu().numpy(), "_sum_squares": stats._sum_squares.cpu().numpy()}
    with open(os.path.join(checkpoint_dir, str(checkpoint_prefix) + "." + extension), "wb") as f:
        pickle.dump(d, f, pickle.HIGHEST_PROTOCOL)


def restore_running_stats(stats, checkpoint_dir: str, checkpoint_prefix, extension="srs"):
    path = os.path.join(checkpoint_dir, str(checkpoint_prefix) + "." + extension)
    if not os.path.exists(path):
        raise ValueError("Could not find NumpySharedRunningStats checkpoint file. ")
    with open(path, "rb") as f:
        d = pickle.load(f)
    for k in ("_mean", "_std", "_sum", "_sum_squares"):
        getattr(stats, k).copy_(torch.from_numpy(np.asarray(d[k], dtype=np.float64)).reshape(getattr(stats, k).shape))
    stats._count = d["_count"]
