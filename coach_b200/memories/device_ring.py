"""HBM-resident struct-of-arrays transition ring.

The reference keeps a Python ``list`` of ``Transition`` objects (memories/non_episodic/experience_replay.py:53,146)
and converts AoS -> SoA on every sample (core_types.py:488-623).  Here every transition field is one row-major
``[capacity, row_bytes]`` uint8 matrix in HBM ("column"); a sample is a row gather
(``cb200_gather`` / ``cb200_per_sample_gather``), an append is a row scatter (``cb200_scatter_ring``).

Layout for the Atari configuration (2^20 slots): state 28,224 B + next_state 28,224 B + action 8 B + reward 8 B +
game_over 1 B per slot = 59.2 GB, which fits the 80 GB of an H100.

Frame-deduplicated mode (``declare_schema(..., frame_stack=[...])``, SURVEY.md 8(f1)): a stacked image observation
[H, W, K] is K frames of which K-1 also belong to the neighbouring transitions -- the reference shares them by
reference through ``LazyStack`` (filters/observation/observation_stacking_filter.py:27-41).  Here every distinct frame
is stored ONCE in a frame store ``[frame_capacity, H * W]`` and the stacked columns hold int32 ``[capacity, K]`` frame
slots; the gather kernels assemble the last-axis stack (cb200_per_sample_gather_s2d / cb200_gather_stack).  Atari:
59.2 GB -> 9.3 GB for 2^20 transitions (frame_capacity = 1.25 x capacity), 5 frames read per sampled transition
instead of 8, one 7 KB frame per ``store`` over PCIe instead of 56 KB.

Columns
  ``state:<key>`` / ``next_state:<key>``  one per entry of the transition's state dict, dtype/shape as stored
  ``action``     int64 scalar (discrete) or float vector (continuous), as given
  ``reward``     float64 (the reference's rewards are Python floats, core_types.py:523)
  ``game_over``  uint8
  ``info:<key>`` ``transition.info[<key>]`` as declared (e.g. Bootstrapped DQN's ``info:mask``, uint8 [heads])
"""
from collections import OrderedDict

import numpy as np
import torch

from coach_b200 import _lib


def _ptr_of(p):
    return p.data_ptr() if torch.is_tensor(p) else p.ptr


class ColumnSpec(object):
    def __init__(self, name, shape, dtype):
        self.name = name
        self.shape = tuple(int(s) for s in shape)
        self.dtype = np.dtype(dtype)
        self.row_bytes = int(np.prod(self.shape, dtype=np.int64)) * self.dtype.itemsize if self.shape else \
            self.dtype.itemsize

    def torch_dtype(self):
        return {np.dtype(np.uint8): torch.uint8, np.dtype(np.int8): torch.int8, np.dtype(np.int32): torch.int32,
                np.dtype(np.int64): torch.int64, np.dtype(np.float32): torch.float32,
                np.dtype(np.float64): torch.float64, np.dtype(np.bool_): torch.uint8,
                np.dtype(np.float16): torch.float16, np.dtype(np.int16): torch.int16}[self.dtype]

    def __repr__(self):
        return "ColumnSpec(%s, %s, %s)" % (self.name, self.shape, self.dtype)


def schema_from_transition(t):
    """Column layout inferred from the first stored transition."""
    specs = OrderedDict()
    for prefix, d in (("state:", t.state), ("next_state:", t.next_state)):
        for key in sorted(d.keys()):
            a = np.asarray(d[key])
            specs[prefix + key] = ColumnSpec(prefix + key, a.shape, a.dtype)
    a = np.asarray(t.action)
    if a.dtype.kind in "iub":
        a = a.astype(np.int64)
    specs["action"] = ColumnSpec("action", a.shape, a.dtype)
    specs["reward"] = ColumnSpec("reward", (), np.float64)
    specs["game_over"] = ColumnSpec("game_over", (), np.uint8)
    return specs


class DeviceTransitionRing(object):
    """Owns the HBM columns plus a pinned host staging area so that single ``store(transition)`` calls are a memcpy
    into pinned memory and reach the GPU in batches (one H2D copy + one scatter kernel per column per flush)."""

    def __init__(self, capacity, device=None, stage_rows=256):
        self.capacity = int(capacity)
        self.device = torch.device(device if device is not None else "cuda")
        self.lib = _lib.load()
        self.specs = None
        self.columns = None          # name -> uint8 [capacity, row_bytes] on device
        self.stage_rows = int(stage_rows)
        self._table_cache = {}
        self._stage_host = None      # name -> pinned uint8 [stage_rows, row_bytes]
        self._stage_dev = None
        self._pending = 0
        self._flush_event = None     # H2D of the pinned stage still in flight?
        self.cursor = 0              # next slot to write
        self.count = 0               # valid slots (<= capacity)
        # frame-deduplicated mode
        self.stack_cols = OrderedDict()      # column name -> (H, W, K)
        self.frame_slack = 0.25
        self.frame_streams = 1               # interleaved episode streams (rollout shards) feeding store(): sizes the identity cache
        self.frames = None                   # uint8 [frame_capacity, H * W]
        self.frame_capacity = 0
        self._fc = 0                         # frames allocated so far (frame f lives in slot f % frame_capacity)
        self._pending_frames = 0
        self._recent = OrderedDict()         # id(frame array) -> (frame array, frame counter): identity cache
        self._min_fc = None                  # per transition slot: oldest frame counter it references

    # -- schema ----------------------------------------------------------------------------------------------------
    def set_schema(self, specs):
        if self.specs is not None:
            return
        self.specs = specs
        self.columns, self._stage_host, self._stage_dev = OrderedDict(), OrderedDict(), OrderedDict()
        self._stage_np = {}
        pin = self.device.type == "cuda"
        # staging area: ONE pinned record per staged transition (columns at 16-byte aligned offsets inside it), so a
        # flush is one H2D copy of the used prefix plus one scatter launch for all columns
        self._rec_off, off = {}, 0
        self._phys = {name: (4 * self.stack_cols[name][2] if name in self.stack_cols else sp.row_bytes)
                      for name, sp in specs.items()}      # bytes per ring row (stacked columns: K int32 frame slots)
        for name, sp in specs.items():
            self._rec_off[name] = off
            off = (off + self._phys[name] + 15) // 16 * 16
        self._rec_bytes = off
        self._stage_host_all = torch.zeros((self.stage_rows, self._rec_bytes), dtype=torch.uint8, pin_memory=pin)
        self._stage_dev_all = torch.empty((self.stage_rows, self._rec_bytes), dtype=torch.uint8, device=self.device)
        host_np = self._stage_host_all.numpy()
        for name, sp in specs.items():
            self.columns[name] = torch.empty((self.capacity, self._phys[name]), dtype=torch.uint8, device=self.device)
            o = self._rec_off[name]
            self._stage_np[name] = host_np[:, o:o + self._phys[name]]  # same memory, no per-store tensor objects
        self._flush_table = None
        if self.stack_cols:
            geo = set(self.stack_cols.values())
            if len(geo) != 1:
                raise ValueError("frame-deduplicated columns must share one [H, W, K] geometry: %s" % self.stack_cols)
            H, W, K = next(iter(geo))
            self.frame_bytes, self.stack_depth = H * W, K
            self.frame_capacity = int(self.capacity * (1.0 + self.frame_slack)) + 2 * K + 8
            self.frames = torch.empty((self.frame_capacity, self.frame_bytes), dtype=torch.uint8, device=self.device)
            self._frame_stage_rows = self.stage_rows + 2 * K * len(self.stack_cols)
            self._frame_stage_host = torch.zeros((self._frame_stage_rows, self.frame_bytes), dtype=torch.uint8,
                                                 pin_memory=pin)
            self._frame_stage_dev = torch.empty((self._frame_stage_rows, self.frame_bytes), dtype=torch.uint8,
                                                device=self.device)
            self._frame_stage_np = self._frame_stage_host.numpy()
            self._min_fc = np.zeros(self.capacity, dtype=np.int64)

    def declare_schema(self, columns, frame_stack=None, frame_slack=None, frame_streams=None):
        """Fix the column layout before the first store: {name: (shape, numpy dtype)} or {name: batch tensor [n, ...]}.
        ``store(Transition)`` then converts every field to the declared dtype (gym hands out float64 observations and
        actions where the networks -- and the agents' persistent batch buffers -- are float32).
        ``frame_stack``: names of uint8 [H, W, K] columns (stacked frames, last-axis) to keep frame-deduplicated;
        ``frame_streams``: how many episode streams (vectorised environments / rollout shards) call ``store`` in turn --
        the cache of recently seen frames is sized for that many (a frame that fell out of it is simply stored again)."""
        if self.specs is not None:
            raise RuntimeError("the replay already holds transitions; the schema is fixed")
        if frame_slack is not None:
            self.frame_slack = float(frame_slack)
        if frame_streams is not None:
            self.frame_streams = max(1, int(frame_streams))
        specs = OrderedDict()
        for name, v in columns.items():
            if torch.is_tensor(v):
                dt = np.dtype(str(v.dtype).replace("torch.", "")) if v.dtype != torch.bool else np.dtype(np.uint8)
                specs[name] = ColumnSpec(name, tuple(v.shape[1:]), dt)
            else:
                specs[name] = ColumnSpec(name, v[0], v[1])
        for need in ("action", "reward", "game_over"):
            if need not in specs:
                raise ValueError("schema lacks the %r column" % need)
        for name in (frame_stack or ()):
            sp = specs[name]
            if sp.dtype != np.uint8 or len(sp.shape) != 3:
                raise ValueError("frame-deduplicated column %r must be uint8 [H, W, K], got %s%s" % (name, sp.dtype, sp.shape))
            self.stack_cols[name] = sp.shape
        self.set_schema(specs)

    def hbm_bytes(self):
        n = 0 if self.columns is None else sum(c.numel() for c in self.columns.values())
        return n + (self.frames.numel() if self.frames is not None else 0)

    def frames_ptr(self):
        """device pointer of the frame store (None: the ring stores stacked observations verbatim)"""
        return self.frames.data_ptr() if self.frames is not None else None

    # -- frame store ---------------------------------------------------------------------------------------------------
    def _frame_slots(self, v, K, slot_row):
        """Resolves the K frames of one stacked observation to frame-store slots, staging the ones not seen before.
        ``v``: a LazyStack (reference or coach_b200: ``history`` list + ``axis``) whose frame OBJECTS are shared between
        neighbouring observations -- matched by identity -- or a plain [H, W, K] array, whose frames are matched by
        content against the most recent frames.  Returns the oldest frame counter referenced."""
        hist = getattr(v, "history", None)
        if hist is not None and hasattr(v, "axis"):
            if len(hist) != K or v.axis not in (-1, 2):
                raise ValueError("stacked observation must hold %d frames on the last axis" % K)
            frames, by_identity = hist, True
        else:
            a = np.asarray(v)
            if a.shape[-1] != K:
                raise ValueError("stacked observation has shape %s, expected %d frames on the last axis" % (a.shape, K))
            frames, by_identity = [a[..., c] for c in range(K)], False
        oldest = None
        for c, f in enumerate(frames):
            hit = self._recent.get(id(f))
            if hit is not None and hit[0] is not f:
                hit = None
            if hit is None and not by_identity:
                for r in reversed(self._recent.values()):
                    if r[0].shape == f.shape and np.array_equal(r[0], f):
                        hit = r
                        break
            if hit is None:
                fc = self._fc
                if self.count + self._pending > 0:
                    live = min(self.count + self._pending, self.capacity - 1)
                    oldest_slot = (self.cursor + self._pending - live) % self.capacity
                    if live > 0 and fc - self.frame_capacity >= self._min_fc[oldest_slot]:
                        raise RuntimeError(
                            "frame store exhausted: %d frame slots for %d transitions (episodes shorter than %.0f "
                            "steps on average?); raise frame_slack" % (self.frame_capacity, self.capacity,
                                                                       1.0 / max(self.frame_slack, 1e-9)))
                fa = np.asarray(f, dtype=np.uint8)
                if fa.size != self.frame_bytes:
                    raise ValueError("frame of %d bytes, the replay stores %d-byte frames" % (fa.size, self.frame_bytes))
                self._frame_stage_np[self._pending_frames] = fa.reshape(-1)
                self._pending_frames += 1
                self._fc += 1
                hit = (f if by_identity else np.array(fa), fc)
                self._recent[id(hit[0]) if not by_identity else id(f)] = hit
                while len(self._recent) > (4 * K + 8) * self.frame_streams:
                    self._recent.popitem(last=False)
            slot_row[c] = hit[1] % self.frame_capacity
            oldest = hit[1] if oldest is None else min(oldest, hit[1])
        return oldest

    # -- append ----------------------------------------------------------------------------------------------------
    def stage_transition(self, t):
        """Copies one transition into the pinned staging rows; returns True when the stage is full."""
        if self.specs is None:
            self.set_schema(schema_from_transition(t))
        r = self._pending
        if r == 0 and self._flush_event is not None:
            self._flush_event.synchronize()      # the previous flush's H2D must have drained the pinned rows
            self._flush_event = None
        oldest = None
        for name, sp in self.specs.items():
            if name in self.stack_cols:
                v = t.state[name[6:]] if name.startswith("state:") else t.next_state[name[11:]]
                o = self._frame_slots(v, sp.shape[2], self._stage_np[name][r].view(np.int32))
                oldest = o if oldest is None else min(oldest, o)
                continue
            if name.startswith("state:"):
                v = t.state[name[6:]]
            elif name.startswith("next_state:"):
                v = t.next_state[name[11:]]
            elif name == "action":
                v = t.action
            elif name == "reward":
                v = t.reward
            elif name == "game_over":
                v = t.game_over
            elif name.startswith("info:"):
                if name[5:] not in t.info:
                    raise ValueError("the replay stores column %r but the transition's info has no %r entry"
                                     % (name, name[5:]))
                v = t.info[name[5:]]
            else:
                raise ValueError("the replay stores column %r, which a Transition cannot supply" % name)
            a = np.asarray(v, dtype=sp.dtype, order='C')
            if a.shape != sp.shape:
                raise ValueError("transition field %s has shape %s, the replay was created with %s"
                                 % (name, a.shape, sp.shape))
            self._stage_np[name][r] = a.reshape(-1).view(np.uint8)
        if oldest is not None:
            self._min_fc[(self.cursor + r) % self.capacity] = oldest
        self._pending += 1
        if self.stack_cols and self._pending_frames + 2 * self.stack_depth * len(self.stack_cols) > self._frame_stage_rows:
            return True
        return self._pending >= min(self.stage_rows, self.capacity)

    def flush(self):
        """Moves the staged rows into the ring.  Returns (first_slot, n)."""
        n = self._pending
        if n == 0:
            return self.cursor, 0
        first = self.cursor
        nf = self._pending_frames
        if nf:
            # new frames: one H2D copy + one scatter into the frame store at the frame cursor (it wraps like the ring)
            self._frame_stage_dev[:nf].copy_(self._frame_stage_host[:nf], non_blocking=True)
            arr, cnt = _lib.make_columns([(self.frames.data_ptr(), self._frame_stage_dev.data_ptr(), self.frame_bytes)])
            _lib.check(self.lib.cb200_scatter_ring(arr, cnt, (self._fc - nf) % self.frame_capacity, self.frame_capacity,
                                                   nf, _lib.current_stream()))
            self._pending_frames = 0
        self._stage_dev_all[:n].copy_(self._stage_host_all[:n], non_blocking=True)
        if self._flush_table is None:
            base = self._stage_dev_all.data_ptr()
            pairs = [(self.columns[name].data_ptr(), base + self._rec_off[name], self._phys[name])
                     for name, sp in self.specs.items()]
            self._flush_table = [_lib.make_columns(pairs[k:k + _lib.CB200_MAX_COLUMNS])
                                 for k in range(0, len(pairs), _lib.CB200_MAX_COLUMNS)]
        for arr, cnt in self._flush_table:
            _lib.check(self.lib.cb200_scatter_ring_packed(arr, cnt, self._rec_bytes, self.cursor, self.capacity, n,
                                                          _lib.current_stream()))
        self.cursor = (self.cursor + n) % self.capacity
        self.count = min(self.count + n, self.capacity)
        self._pending = 0
        if self.device.type == "cuda":
            self._flush_event = torch.cuda.Event()
            self._flush_event.record()
        return first, n

    def append_columns(self, cols):
        """Bulk append of n transitions given as {column name: tensor/ndarray [n, ...]} (device tensors are used in
        place, host arrays go through one H2D copy).  Returns (first_slot, n)."""
        self.flush()
        n = None
        staged = {}
        for name, v in cols.items():
            tt = torch.as_tensor(v)
            staged[name] = tt
            if name == "frames":                    # frame-deduplicated bulk append: the distinct frames, any count
                continue
            n = tt.shape[0] if n is None else n
            if tt.shape[0] != n:
                raise ValueError("all columns must have the same number of rows")
        if self.specs is None:
            specs = OrderedDict()
            for name, tt in staged.items():
                dt = np.dtype(str(tt.dtype).replace("torch.", "")) if tt.dtype != torch.bool else np.dtype(np.uint8)
                specs[name] = ColumnSpec(name, tuple(tt.shape[1:]), dt)
            self.set_schema(specs)
        if set(staged) - {"frames"} != set(self.specs):
            raise ValueError("append_columns needs exactly the columns %s" % list(self.specs))
        if n > self.capacity:
            raise ValueError("cannot append more rows than the ring holds in one call")
        first = self.cursor
        pairs, keep = [], []
        if self.stack_cols:
            staged = self._append_frames(staged, n)
        for name, sp in self.specs.items():
            if name in self.stack_cols:
                tt = staged[name]                                  # int32 [n, K] frame slots (device)
                keep.append(tt)
                pairs.append((self.columns[name].data_ptr(), tt.data_ptr(), self._phys[name]))
                continue
            tt = staged[name].to(self.device, non_blocking=True).contiguous()
            tt = tt.view(torch.uint8).reshape(n, -1) if tt.dtype != torch.bool else tt.to(torch.uint8).reshape(n, -1)
            if tt.shape[1] != sp.row_bytes:
                raise ValueError("column %s: %d bytes per row, expected %d" % (name, tt.shape[1], sp.row_bytes))
            keep.append(tt)
            pairs.append((self.columns[name].data_ptr(), tt.data_ptr(), sp.row_bytes))
        self._scatter(pairs, n)
        return first, n

    def _append_frames(self, staged, n):
        """Bulk append in frame-deduplicated mode.  Either the stacked columns come as full [n, H, W, K] arrays -- every
        frame is then stored as a new one (no sharing can be inferred; tests and small fills) -- or the caller passes the
        distinct frames once, ``"frames"``: uint8 [nf, H, W], and int32 [n, K] indices into them for every stacked
        column (a recorded frame stream: bench.py's synthetic fill)."""
        K, dev = self.stack_depth, self.device
        staged = dict(staged)
        if "frames" in staged:
            frames = staged.pop("frames").to(dev).reshape(-1, self.frame_bytes).contiguous()
            rel = {name: staged[name].to(dev).to(torch.int64).reshape(n, K) for name in self.stack_cols}
            for name, r in rel.items():
                lo_i, hi_i = int(r.min()), int(r.max())
                if lo_i < 0 or hi_i >= frames.shape[0]:
                    raise ValueError("column %s: frame indices %d..%d outside the %d frames of this append"
                                     % (name, lo_i, hi_i, frames.shape[0]))
        else:
            parts, rel, base = [], {}, 0
            for name in self.stack_cols:
                x = staged[name].to(dev)
                if tuple(x.shape[1:]) != self.stack_cols[name]:
                    raise ValueError("column %s: shape %s, expected [n, %s]" % (name, tuple(x.shape), self.stack_cols[name]))
                parts.append(x.permute(0, 3, 1, 2).reshape(n * K, self.frame_bytes))
                rel[name] = base + torch.arange(n * K, device=dev, dtype=torch.int64).reshape(n, K)
                base += n * K
            frames = torch.cat(parts).contiguous()
        nf = int(frames.shape[0])
        if nf > self.frame_capacity:
            raise ValueError("%d frames in one append, the frame store holds %d" % (nf, self.frame_capacity))
        if self.count > 0:
            live = min(self.count, self.capacity - 1)
            if self._fc + nf - self.frame_capacity > self._min_fc[(self.cursor - live) % self.capacity] and \
                    n < self.capacity:
                raise RuntimeError("frame store exhausted by a bulk append: raise frame_slack")
        arr, cnt = _lib.make_columns([(self.frames.data_ptr(), frames.data_ptr(), self.frame_bytes)])
        _lib.check(self.lib.cb200_scatter_ring(arr, cnt, self._fc % self.frame_capacity, self.frame_capacity, nf,
                                               _lib.current_stream()))
        lo = None
        for name in self.stack_cols:
            cnt_abs = rel[name] + self._fc
            staged[name] = (cnt_abs % self.frame_capacity).to(torch.int32).contiguous()
            m = cnt_abs.min(dim=1).values
            lo = m if lo is None else torch.minimum(lo, m)
        slots = (self.cursor + np.arange(n)) % self.capacity
        self._min_fc[slots] = lo.cpu().numpy()
        self._fc += nf
        self._keep_frames = frames                 # alive until the scatter has run
        return staged

    def _scatter(self, pairs, n):
        for k in range(0, len(pairs), _lib.CB200_MAX_COLUMNS):
            arr, cnt = _lib.make_columns(pairs[k:k + _lib.CB200_MAX_COLUMNS])
            _lib.check(self.lib.cb200_scatter_ring(arr, cnt, self.cursor, self.capacity, n, _lib.current_stream()))
        self.cursor = (self.cursor + n) % self.capacity
        self.count = min(self.count + n, self.capacity)

    def clear(self):
        self.cursor = 0
        self.count = 0
        self._pending = 0
        self._fc = 0
        self._pending_frames = 0
        self._recent.clear()

    # -- gather ----------------------------------------------------------------------------------------------------
    def alloc_batch(self, n):
        """Output tensors for one minibatch: {column: typed tensor [n, *shape]}."""
        out = OrderedDict()
        for name, sp in self.specs.items():
            out[name] = torch.empty((n,) + sp.shape, dtype=sp.torch_dtype(), device=self.device)
        return out

    def column_table(self, out, n):
        """ctypes gather table for ``n`` rows into ``out``.  The kernels write ``n * row_bytes`` bytes per column: a
        destination of another dtype or size would be overrun (or read back reinterpreted), so every buffer is checked
        against the ring's schema -- once per buffer set, the agents sample into the same persistent buffers."""
        key = (int(n),) + tuple(out[name].data_ptr() for name in self.specs)
        hit = self._table_cache.get(key)
        if hit is None:
            for name, sp in self.specs.items():
                t = out[name]
                if not (t.is_cuda == (self.device.type == "cuda") and t.is_contiguous()):
                    raise ValueError("batch buffer %r must be a contiguous tensor on %s" % (name, self.device))
                if t.dtype != sp.torch_dtype() or t.numel() * t.element_size() != n * sp.row_bytes:
                    raise ValueError(
                        "batch buffer %r is %s%s but the replay stores %s%s per transition (%d rows): declare the "
                        "schema up front (memory.declare_schema) or store transitions in the agent's dtypes"
                        % (name, t.dtype, tuple(t.shape), sp.dtype, sp.shape, n))
            # (frame-deduplicated columns are assembled from the frame store: assemble_stacks)
            pairs = [(self.columns[name].data_ptr(), out[name].data_ptr(), sp.row_bytes)
                     for name, sp in self.specs.items() if name not in self.stack_cols]
            hit = self._table_cache[key] = _lib.make_columns(pairs)
            if len(self._table_cache) > 64:
                self._table_cache.clear()
                self._table_cache[key] = hit
        return hit

    def s2d_tables(self, s2d, out, n):
        """ctypes tables of the fused gather + space-to-depth launch (cb200_per_sample_gather_s2d / cb200_gather_s2d).
        s2d: {"columns": {ring column name: plane tensor / PlaneBuf}, "geometry": (H, W, C, S)}; every other column
        is copied into ``out``.  Returns (image table, n_image, small table, n_small, image names)."""
        key = ("s2d", int(n)) + tuple(_ptr_of(p) for p in s2d["columns"].values()) + \
            tuple(out[name].data_ptr() for name in self.specs if name not in s2d["columns"])
        hit = self._table_cache.get(key)
        if hit is None:
            H, W, C, S = s2d["geometry"]
            img, small = [], []
            for name, sp in self.specs.items():
                if name in s2d["columns"]:
                    if sp.dtype != np.uint8 or sp.row_bytes != H * W * C:
                        raise ValueError("column %r is %s%s, the fused image path needs uint8 [%d, %d, %d] frames"
                                         % (name, sp.dtype, sp.shape, H, W, C))
                    if bool(self.stack_cols) != (name in self.stack_cols):
                        raise ValueError("either all image columns of the fused path are frame-deduplicated or none")
                    img.append((self.columns[name].data_ptr(), _ptr_of(s2d["columns"][name]), self._phys[name]))
                else:
                    t = out[name]
                    if t.dtype != sp.torch_dtype() or t.numel() * t.element_size() != n * sp.row_bytes or \
                            not t.is_contiguous():
                        raise ValueError("batch buffer %r does not match the replay's %s%s" % (name, sp.dtype, sp.shape))
                    small.append((self.columns[name].data_ptr(), t.data_ptr(), sp.row_bytes))
            ia, ni = _lib.make_columns(img)
            sa, ns = _lib.make_columns(small)
            hit = self._table_cache[key] = (ia, ni, sa, ns)
        return hit

    def gather_column(self, name, idx):
        """one column of the given slots as a typed tensor (lazy materialisation of un-staged batch columns)"""
        sp = self.specs[name]
        n = idx.shape[0]
        out = torch.empty((n,) + sp.shape, dtype=sp.torch_dtype(), device=self.device)
        if name in self.stack_cols:
            self.assemble_stacks({name: out}, idx, n, names=(name,))
            return out
        arr, cnt = _lib.make_columns([(self.columns[name].data_ptr(), out.data_ptr(), sp.row_bytes)])
        _lib.check(self.lib.cb200_gather(arr, cnt, idx.data_ptr(), n, _lib.current_stream()))
        return out

    def gather(self, idx, out=None):
        """out[c][i] = column c of slot idx[i]; idx int64 CUDA tensor."""
        n = idx.shape[0]
        if out is None:
            out = self.alloc_batch(n)
        arr, cnt = self.column_table(out, n)
        _lib.check(self.lib.cb200_gather(arr, cnt, idx.data_ptr(), n, _lib.current_stream()))
        self.assemble_stacks(out, idx, n)
        return out

    def assemble_stacks(self, out, idx, n, names=None):
        """frame-deduplicated columns of the slots ``idx``: out[name][i] = np.stack(frames of slot idx[i], axis=-1)
        (observation_stacking_filter.py:37-41) through cb200_gather_stack; no-op for a verbatim ring"""
        for name in (names if names is not None else self.stack_cols):
            t = out[name]
            H, W, K = self.stack_cols[name]
            if t.dtype != torch.uint8 or t.numel() != n * H * W * K or not t.is_contiguous():
                raise ValueError("batch buffer %r must be a contiguous uint8 [%d, %d, %d, %d] tensor" % (name, n, H, W, K))
            _lib.check(self.lib.cb200_gather_stack(self.frames.data_ptr(), self.frame_bytes,
                                                   self.columns[name].data_ptr(), K, idx.data_ptr(), n, t.data_ptr(),
                                                   _lib.current_stream()))
