"""The batched gym surface every env family shares.

``BatchedVectorEnv`` is gymnasium's ``VectorEnv`` shape over ``num_envs`` roads that live in HBM: constructor checks,
``configure``, seeding (env ``i`` owns the numpy ``Generator(PCG64)`` a reference env seeded with
``seed + env_index_offset + i`` would own), ``reset`` / ``step`` with the three autoreset modes, action staging,
standalone observation plugins and ``state_dict``.  A family supplies its kernels through ``_step_kernels``,
``_device_reset`` and ``_observe_kernel``.  ``BatchedNetworkEnv`` adds what the general-network families
(roundabout, merge, two-way, u-turn, exit, intersection) share: the lane table on the device, the ``HwyNetState``
buffers, ``road_substeps`` and the numpy-exact host reset mode.

The env streams always live on the device as 5 words per env (state hi, lo, inc hi, lo, has_uint32 << 32 |
uinteger); a host reset borrows numpy generators for the envs it re-spawns and writes their words back.
"""
from __future__ import annotations

import ctypes as C
from typing import Any, Optional

import numpy as np
import torch

from ... import _native as N
from ...config import default_config


def pcg64_words(generators) -> np.ndarray:
    """The [5, n] uint64 words of numpy PCG64 generators (the layout of the device streams)."""
    words = np.zeros((5, len(generators)), dtype=np.uint64)
    m64 = (1 << 64) - 1
    for i, g in enumerate(generators):
        st = g.bit_generator.state
        s, inc = st["state"]["state"], st["state"]["inc"]
        words[:, i] = (s >> 64, s & m64, inc >> 64, inc & m64, (int(st["has_uint32"]) << 32) | int(st["uinteger"]))
    return words


def set_pcg64_words(generators, words) -> None:
    """Inverse of pcg64_words: generator i takes column i of the [5, n] words."""
    for g, w in zip(generators, np.asarray(words, dtype=np.uint64).T):
        g.bit_generator.state = {
            "bit_generator": "PCG64", "state": {"state": (int(w[0]) << 64) | int(w[1]), "inc": (int(w[2]) << 64) | int(w[3])},
            "has_uint32": int(w[4]) >> 32, "uinteger": int(w[4]) & 0xFFFFFFFF}


class BatchedVectorEnv:
    ENV_ID: str
    REWARD_NAMES: tuple
    META_FLAGS = ("crashed", "has_impact", "check_collisions")  # the meta-word flags of state_dict
    NEXT_STEP_REWINDS_RNG = False  # NextStep: the step kernel draws from the streams of envs it is about to reset
    metadata = {"render_modes": [], "autoreset_mode": "SameStep"}
    reset_mode = "device"
    _kernel_events = None  # bench.py hook: list of (start, end) CUDA events around the step kernels
    _rngs = None  # reset_mode="host": the numpy generators of the envs

    @classmethod
    def default_config(cls) -> dict:
        return default_config(cls.ENV_ID)

    def __init__(self, config: Optional[dict] = None, render_mode: Optional[str] = None, num_envs: int = 1,
                 device: Any = None, autoreset_mode: str = "SameStep", env_index_offset: int = 0) -> None:
        if render_mode is not None:
            raise NotImplementedError("rendering is out of scope of the accelerated path (render_mode=None)")
        if not torch.cuda.is_available():
            raise RuntimeError("highwayenv_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self.num_envs = int(num_envs)
        if self.num_envs < 1:
            raise ValueError("num_envs must be >= 1")
        self.device = torch.device(device if device is not None else "cuda")
        if self.device.type != "cuda":
            raise RuntimeError("highwayenv_b200 only runs on CUDA devices")
        if autoreset_mode not in ("SameStep", "NextStep", "Disabled"):
            raise ValueError(f"autoreset_mode {autoreset_mode!r} (SameStep, NextStep, Disabled)")
        self._lib = N.load()
        self.render_mode = None
        self.autoreset_mode = autoreset_mode
        self.env_index_offset = int(env_index_offset)
        self.config = self.default_config()
        self.configure(config)
        self._seeded = False
        self._autoreset_envs = None
        # the env streams as uint64 words, bit-cast; [5, num_envs] fits every configuration, so a re-allocation keeps
        # them: the reference's np_random survives a reset without a seed (abstract.py:219-249)
        self._rng = torch.zeros(5, self.num_envs, dtype=torch.int64, device=self.device)
        self.define_spaces()
        self._allocate()

    def configure(self, config: Optional[dict]) -> None:
        """Shallow update, as the reference (abstract.py:127-129)."""
        if config:
            self.config.update(config)

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def close(self) -> None:
        pass

    @property
    def unwrapped(self):
        return self

    def host_stepper(self):
        """Host-buffer stepping through one CUDA graph (envs/common/host_stepper.py)."""
        from .host_stepper import HostStepper

        return HostStepper(self)

    # ------------------------------------------------------------------ seeding
    def _seed_streams(self, seed) -> None:
        n = self.num_envs
        if seed is None:
            seeds = [int(s.generate_state(1)[0]) for s in np.random.SeedSequence().spawn(n)]
        elif isinstance(seed, (int, np.integer)):
            seeds = [int(seed) + self.env_index_offset + i for i in range(n)]
        else:
            seeds = [int(s) for s in seed]
            if len(seeds) != n:
                raise ValueError("seed sequence must have num_envs entries")
        generators = [np.random.Generator(np.random.PCG64(np.random.SeedSequence(s))) for s in seeds]
        self._rng.copy_(torch.from_numpy(pcg64_words(generators).view(np.int64)).to(self.device))
        if self.reset_mode == "host":
            self._rngs = generators
        self.np_random_seed = seeds
        self._seeded = True

    def rng_words(self) -> np.ndarray:
        """The env streams as [5][n] uint64 words (state hi, lo, inc hi, lo, has_uint32 << 32 | uinteger)."""
        return self._rng.cpu().numpy().view(np.uint64).copy()

    # ------------------------------------------------------------------ gym API
    def reset(self, *, seed=None, options: Optional[dict] = None):
        """Reset every env (or those set in ``options["reset_mask"]``); returns (obs, info)."""
        mask = None
        if options and options.get("reset_mask") is not None:
            mask = torch.as_tensor(options["reset_mask"])
            if tuple(mask.shape) != (self.num_envs,):
                raise ValueError("reset_mask must have shape (num_envs,)")
            mask = mask.to(device=self.device, dtype=torch.uint8).contiguous()
            self._mask_keepalive = mask
        if options and "config" in options:
            self.configure(options["config"])
            self.define_spaces()
            self._allocate()
        if seed is not None or not self._seeded:
            self._seed_streams(seed)
        self._autoreset_envs = None
        self._reset(mask)
        return self._out_obs(), self._reset_info()

    def _reset_info(self) -> dict:
        return {"speed": self._hs[:, 0, 1], "crashed": (self._meta[:, 0] & N.META_CRASHED) != 0}

    def _stage_actions(self, actions) -> torch.Tensor:
        """The actions as the kernels read them: a device tensor of the buffer's dtype and shape is used in place."""
        buf = self._action_buf
        table = getattr(self.action_type, "table", None)
        if table is not None:  # DiscreteAction (action.py:165-196): index -> (throttle, steering), then ContinuousAction
            if getattr(self, "_action_table", None) is None or self._action_table.device != buf.device:
                self._action_table = torch.from_numpy(table).to(buf.device)
            idx = actions if isinstance(actions, torch.Tensor) else torch.from_numpy(np.asarray(actions))
            idx = idx.to(device=buf.device, dtype=torch.long).reshape(-1)
            if idx.numel() != buf.shape[0]:
                raise ValueError("one action per env")
            # (the check reads the device: not under CUDA-graph capture — HostStepper checks its host array instead)
            if not torch.cuda.is_current_stream_capturing() and bool(((idx < 0) | (idx >= table.shape[0])).any()):
                raise IndexError("list index out of range")  # all_actions[action] in the reference
            torch.index_select(self._action_table, 0, idx, out=buf)
            return buf
        if isinstance(actions, torch.Tensor):
            if actions.device == buf.device and actions.dtype == buf.dtype and actions.is_contiguous() \
                    and actions.shape == buf.shape:
                return actions
            buf.copy_(actions.reshape(buf.shape), non_blocking=True)  # dtype / device conversion on the device
            return buf
        a = np.asarray(actions)
        buf.copy_(torch.from_numpy(np.ascontiguousarray(a.reshape(tuple(buf.shape)))).to(buf.dtype),
                  non_blocking=True)
        return buf

    def step(self, actions):
        """One policy step of all envs; device tensors as actions are used in place.  Returns the env's device
        buffers ``(obs, reward, terminated, truncated, info)``, which the next call reuses."""
        if not self._seeded:
            raise RuntimeError("call reset() before step()")
        act = self._stage_actions(actions)
        prev = self._autoreset_envs if self.autoreset_mode == "NextStep" else None
        rng_before = self._rng.clone() if prev is not None and self.NEXT_STEP_REWINDS_RNG else None
        kev = self._kernel_events
        if kev is not None:  # bench.py: CUDA events around the step kernel(s) alone
            kev.append((torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)))
            kev[-1][0].record(torch.cuda.current_stream(self.device))
        self._step_kernels(act)
        if kev is not None:
            kev[-1][1].record(torch.cuda.current_stream(self.device))
        info = self._step_info(act)
        if self._plugin_standalone:
            self._observe_plugin(self._obs)
        if self.autoreset_mode == "SameStep":
            self._same_step_autoreset(info)
        elif self.autoreset_mode == "NextStep":
            self._next_step_autoreset(prev, rng_before)
        return self._step_result(info)

    def _step_info(self, act) -> dict:
        """AbstractEnv._info (abstract.py:200-217): speed, crashed, action and the un-weighted reward terms."""
        return {"speed": self._info_speed, "crashed": self._info_crashed.view(torch.bool), "action": act,
                "rewards": {name: self._reward_terms[:, k] for k, name in enumerate(self.REWARD_NAMES)}}

    def _step_result(self, info):
        return (self._out_obs(), self._reward, self._terminated.view(torch.bool), self._truncated.view(torch.bool),
                info)

    def _same_step_autoreset(self, info) -> None:
        """Keep the observation as final_obs, re-spawn the finished envs, observe those again."""
        self._final_obs.copy_(self._obs)
        info["final_obs"] = self._final_obs
        self._device_reset(self._terminated.data_ptr(), self._truncated.data_ptr(), self._fused_out.data_ptr())
        if self._plugin_standalone:
            self._observe_plugin(self._obs, self._terminated, self._truncated)

    def _next_step_autoreset(self, prev, rng_before) -> None:
        """gymnasium AutoresetMode.NEXT_STEP (the vector default): an env that ended in the previous step is reset by
        this call instead of stepped — reset observation, reward 0, both flags False.  The step kernel has already
        advanced those envs; their state is replaced by the masked device reset, from the stream as it was when the
        episode ended."""
        if prev is not None:
            if rng_before is not None:
                self._rng.copy_(torch.where(prev.bool().unsqueeze(0), rng_before, self._rng))
            self._device_reset(prev.data_ptr(), None, self._fused_out.data_ptr())
            if self._plugin_standalone:
                self._observe_plugin(self._obs, prev)
            keep = prev == 0
            self._reward.mul_(keep)
            self._terminated.mul_(keep)
            self._truncated.mul_(keep)
        self._autoreset_envs = (self._terminated | self._truncated).contiguous()

    def observe(self) -> torch.Tensor:
        self._observe_kernel()
        if self._plugin_standalone:
            self._observe_plugin(self._obs)
        return self._out_obs()

    def to_finite_mdp(self):
        """AbstractEnv.to_finite_mdp() (envs/common/abstract.py:452-453) of every env, built on the device: the
        time-to-collision MDP of highwayenv_b200.planning.FiniteMdp (`.env(i)` gives env i as the reference's
        DeterministicMDP)."""
        from ...planning import to_finite_mdp

        return to_finite_mdp(self)

    def _observe_plugin(self, out, mask_a=None, mask_b=None) -> None:
        self.observation_type.observe(self, out, mask_a, mask_b)

    def _out_obs(self) -> torch.Tensor:
        if getattr(self.observation_type, "as_image", False):  # OccupancyGrid(as_image=True): uint8 (observation.py:336-338)
            return self._obs.to(torch.uint8)
        return self._obs

    # ------------------------------------------------------------------ cloning
    # tensors with a leading num_envs axis that copy_envs leaves alone: per-step outputs (a later call overwrites them
    # before it reads them), scratch and staging buffers
    ROW_EXCLUDE = frozenset({
        "_final_obs", "_fused_out", "_reward", "_terminated", "_truncated", "_info_speed", "_info_crashed",
        "_reward_terms", "_action_buf", "_mask_keepalive", "_agents_reward", "_agents_terminated"})

    def _env_rows(self) -> dict:
        """Every per-env tensor a later call reads, as name -> a [num_envs, ...] view: the state copy_envs copies.
        The streams are [5, num_envs] and appear transposed; the NextStep pending-reset flag appears once it exists."""
        n = self.num_envs
        rows = {"_pos": self._pos, "_hs": self._hs, "_tt": self._tt, "_imp": self._imp, "_delta": self._delta,
                "_meta": self._meta, "_speed_index": self._speed_index.view(n, -1), "_time": self._time,
                "_rng": self._rng.t(), "_obs": self._obs}
        if self._autoreset_envs is not None:
            rows["_autoreset_envs"] = self._autoreset_envs
        return rows

    def _row_layout(self) -> dict:
        rows = self._env_rows()
        rows.pop("_autoreset_envs", None)
        return {k: (tuple(t.shape[1:]), t.dtype) for k, t in rows.items()}

    def _row_copy_table(self, source) -> "C.Array":
        """The HwyRowCopy entries that copy rows of `source` into rows of this env (one per contiguous row buffer)."""
        dst_rows, src_rows = self._env_rows(), source._env_rows()
        if "_autoreset_envs" in dst_rows and "_autoreset_envs" not in src_rows:  # no reset pending in the source
            src_rows["_autoreset_envs"] = torch.zeros_like(dst_rows["_autoreset_envs"])
            self._flag_keepalive = src_rows["_autoreset_envs"]
        pairs = []
        for name, d in dst_rows.items():
            s = src_rows[name]
            if d.dim() == 2 and not (d.is_contiguous() and s.is_contiguous()):  # [n, k] views of [k, n]: per column
                pairs += [(s[:, j], d[:, j]) for j in range(d.shape[1])]
            else:
                pairs.append((s, d))
        table = (N.HwyRowCopy * len(pairs))()
        for e, (s, d) in zip(table, pairs):
            assert s.is_contiguous() and d.is_contiguous() and s[0].numel() == d[0].numel()
            e.src, e.dst, e.row_bytes = s.data_ptr(), d.data_ptr(), d[0].numel() * d.element_size()
        return table

    def _available_actions(self, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """DiscreteMetaAction.get_available_actions of every env on the device (hwy_available_actions): a bool mask
        [N, 5] over (LANE_LEFT, IDLE, LANE_RIGHT, FASTER, SLOWER), written into `out` (uint8 [N, 5]) when given."""
        if out is None:
            out = torch.empty(self.num_envs, 5, dtype=torch.uint8, device=self.device)
        view, graph = self._obs_view()
        with torch.cuda.device(self.device):
            N.check(self._lib.hwy_available_actions(graph, C.byref(view), int(self._params.n_target_speeds),
                                                    out.data_ptr(), self._stream()))
        return out.view(torch.bool)

    def _copy_rows(self, table, dst: torch.Tensor, src: torch.Tensor) -> None:
        """One hwy_copy_env_rows launch, without checks (dst, src: device int64 [n_pairs])."""
        if dst.numel() == 0:
            return
        with torch.cuda.device(self.device):
            N.check(self._lib.hwy_copy_env_rows(table, len(table), dst.data_ptr(), src.data_ptr(), dst.numel(),
                                                self._stream()))

    def _index_tensor(self, ids) -> torch.Tensor:
        t = ids if isinstance(ids, torch.Tensor) else torch.from_numpy(np.asarray(ids, dtype=np.int64))
        return t.to(device=self.device, dtype=torch.int64).reshape(-1).contiguous()

    def copy_envs(self, dst_ids, src_ids, source=None) -> None:
        """Copy the complete state of envs `src_ids` of `source` (default: this env) into envs `dst_ids` of this env.
        Afterwards env dst_ids[k] behaves as `copy.deepcopy` of env src_ids[k] would: the same future under the same
        actions, streams included.  One kernel launch; device int64 index tensors make it capturable in a CUDA graph.

        Raises before any launch when `source` has another class or layout (vehicles, slots, observation shape, traffic
        model, agents, device) or the index lists differ in length; outside stream capture also when an index is out
        of range, `dst_ids` repeats an env, or (within one env) an env is both a source and a destination.  A
        destination env never seeded is seeded first, as load_state_dict does."""
        source = self if source is None else source
        if type(source) is not type(self):
            raise TypeError(f"copy_envs from a {type(source).__name__} into a {type(self).__name__}")
        if not source._seeded:
            raise RuntimeError("call reset() on the source before copy_envs()")
        if source.device != self.device or source.V != self.V or source._row_layout() != self._row_layout() \
                or source.config.get("other_vehicles_type") != self.config.get("other_vehicles_type"):
            raise ValueError("copy_envs between envs of different layouts (vehicles, observation, traffic model, "
                             "agents or device)")
        dst, src = self._index_tensor(dst_ids), self._index_tensor(src_ids)
        if dst.numel() != src.numel():
            raise ValueError("dst_ids and src_ids must have the same length")
        if not torch.cuda.is_current_stream_capturing() and dst.numel():  # reads the indices: one host round trip
            d, s = dst.cpu().numpy(), src.cpu().numpy()
            if d.min() < 0 or d.max() >= self.num_envs or s.min() < 0 or s.max() >= source.num_envs:
                raise IndexError("env index out of range")
            if np.unique(d).size != d.size:
                raise ValueError("dst_ids repeats an env")
            if source is self and np.intersect1d(d, s).size:
                raise ValueError("an env is both a source and a destination")
        if not self._seeded:
            self._seed_streams(0)
        if self.autoreset_mode == "NextStep" and self._autoreset_envs is None:
            self._autoreset_envs = torch.zeros(self.num_envs, dtype=torch.uint8, device=self.device)
        self._copy_rows(self._row_copy_table(source), dst, src)

    # ------------------------------------------------------------------ state import / export
    def state_dict(self) -> dict:
        """Per-field numpy arrays [N, V] (the reference's per-vehicle attributes), speed index, clock and streams."""
        V = self.V
        pos, hs, tt, imp = (t[:, :V].cpu().numpy() for t in (self._pos, self._hs, self._tt, self._imp))
        sd = {"x": pos[..., 0].copy(), "y": pos[..., 1].copy(), "heading": hs[..., 0].copy(), "speed": hs[..., 1].copy(),
              "target_speed": tt[..., 0].copy(), "timer": tt[..., 1].copy(), "delta": self._delta[:, :V].cpu().numpy(),
              "impact_x": imp[..., 0].copy(), "impact_y": imp[..., 1].copy()}
        sd.update(N.unpack_meta(self._meta[:, :V].cpu().numpy(), self.META_FLAGS))
        sd["speed_index"] = self._speed_index.cpu().numpy()
        sd["time"] = self._time.cpu().numpy()
        sd["rng"] = self._rng.cpu().numpy().view(np.uint64)
        return sd

    def load_state_dict(self, sd: dict, env_ids=None) -> None:
        """Inverse of :meth:`state_dict` (how oracle / reference states are injected), for every env or the rows
        `env_ids`.  An env never seeded is first seeded as reset(seed=0) would; `sd["rng"]` then replaces the words."""
        n, V, dev = self.num_envs, self.V, self.device
        idx = slice(None) if env_ids is None else torch.from_numpy(np.asarray(env_ids, dtype=np.int64)).to(dev)
        pair = lambda a, b: torch.from_numpy(np.ascontiguousarray(  # noqa: E731
            np.stack([np.asarray(sd[a], dtype=np.float64), np.asarray(sd[b], dtype=np.float64)], axis=-1))).to(dev)
        self._pos[idx, :V] = pair("x", "y")
        self._hs[idx, :V] = pair("heading", "speed")
        self._tt[idx, :V] = pair("target_speed", "timer")
        self._imp[idx, :V] = pair("impact_x", "impact_y")
        self._delta[idx, :V] = torch.from_numpy(np.ascontiguousarray(sd["delta"], dtype=np.float64)).to(dev)
        self._meta[idx, :V] = torch.from_numpy(N.pack_meta(sd, self.META_FLAGS).reshape(-1, V)).to(dev)
        si = np.ascontiguousarray(sd["speed_index"], dtype=np.int32).reshape(-1, self._speed_index.numel() // n)
        self._speed_index.view(n, -1)[idx] = torch.from_numpy(si).to(dev)
        self._time[idx] = torch.from_numpy(np.asarray(sd["time"], dtype=np.float64).reshape(-1)).to(dev)
        if not self._seeded:
            self._seed_streams(0)
        if "rng" in sd:
            w = np.ascontiguousarray(sd["rng"], dtype=np.uint64).reshape(5, -1)
            self._rng[:, idx] = torch.from_numpy(w.view(np.int64)).to(dev)


class BatchedNetworkEnv(BatchedVectorEnv):
    """The general-network families: a lane table on the device (``_make_network``), the ``HwyNetState`` buffers,
    ``hwy_network_observe`` / ``hwy_network_substeps`` and two reset modes.

    * ``reset_mode="device"`` (default): the family's reset kernel re-spawns from the env streams; SameStep autoreset
      stays on the device.
    * ``reset_mode="host"``: the family's numpy spawn (``_reset_envs``, bit-identical to the reference) is uploaded;
      autoreset round-trips through the host."""

    SLOTS = N.HWY_NET_GROUP  # vehicle slots per env: 8 (one warp serves four envs) or 32 (HWY_NET_GROUP_LARGE)
    n_agents = 1
    multi_agent = False

    def __init__(self, config: Optional[dict] = None, render_mode: Optional[str] = None, num_envs: int = 1,
                 device: Any = None, autoreset_mode: str = "SameStep", env_index_offset: int = 0,
                 reset_mode: str = "device") -> None:
        if reset_mode not in ("device", "host"):
            raise ValueError("reset_mode must be 'device' or 'host'")
        if autoreset_mode == "NextStep" and reset_mode != "device":
            raise NotImplementedError("NextStep autoreset uses the device reset")
        self.reset_mode = reset_mode
        super().__init__(config=config, render_mode=render_mode, num_envs=num_envs, device=device,
                         autoreset_mode=autoreset_mode, env_index_offset=env_index_offset)

    _net = None

    @property
    def net(self):
        """The family's road network (_make_network, built at its first use) and, as _graph_dev, its device table."""
        if self._net is None:
            self._net = self._make_network()
            self._graph_dev = torch.from_numpy(
                np.frombuffer(bytes(self._net.to_struct()), dtype=np.uint8).copy()).to(self.device)
        return self._net

    def _allocate_network_state(self, vp: int, fused_out_cols: int = 5) -> N.HwyNetState:
        """The per-vehicle and per-env buffers every network kernel reads, and the HwyNetState pointing at them."""
        n, dev, A = self.num_envs, self.device, self.n_agents
        z = lambda *shape, dtype: torch.zeros(*shape, dtype=dtype, device=dev)  # noqa: E731
        self.vp = vp
        self._pos, self._hs, self._tt, self._imp = (z(n, vp, 2, dtype=torch.float64) for _ in range(4))
        self._delta = z(n, vp, dtype=torch.float64)
        self._meta = z(n, vp, dtype=torch.int32)
        self._route = z(n, vp, N.HWY_NET_MAX_ROUTE, dtype=torch.int32)
        self._route_len = z(n, vp, dtype=torch.int32)
        self._speed_index = z(n * A, dtype=torch.int32)
        self._time = z(n, dtype=torch.float64)
        self._obs = z(n, *self.obs_shape, dtype=torch.float32)
        self._final_obs = z(n, *self.obs_shape, dtype=torch.float32)
        # what the step / reset / observe kernels write: the observation itself, or a scratch row per agent when a
        # standalone plugin observes after them
        self._fused_out = z(n, A, fused_out_cols, dtype=torch.float32) if self._plugin_standalone else self._obs
        self._plugin_view = None
        self._reward = z(n, dtype=torch.float64)
        self._terminated, self._truncated = z(n, dtype=torch.uint8), z(n, dtype=torch.uint8)
        self._info_speed, self._info_crashed = z(n, dtype=torch.float64), z(n, dtype=torch.uint8)
        self._reward_terms = z(n, N.HWY_REWARD_TERMS, dtype=torch.float64)
        st = N.HwyNetState()
        st.n_envs, st.vp = n, vp
        st.pos, st.hs, st.tt, st.imp = (t.data_ptr() for t in (self._pos, self._hs, self._tt, self._imp))
        st.delta, st.meta = self._delta.data_ptr(), self._meta.data_ptr()
        st.route, st.route_len = self._route.data_ptr(), self._route_len.data_ptr()
        st.speed_index, st.time = self._speed_index.data_ptr(), self._time.data_ptr()
        st.reward_terms = self._reward_terms.data_ptr()
        self._state = st
        return st

    def _env_rows(self) -> dict:
        rows = super()._env_rows()
        rows.update({"_route": self._route, "_route_len": self._route_len})
        for name in ("_count", "_road_steps", "_overflow"):  # the 32-slot kernels' population and rule clock
            if getattr(self, name, None) is not None:
                rows[name] = getattr(self, name)
        return rows

    def _route_tables(self, destinations):
        """plan_route_to(lane, destination) (vehicle/controller.py:71-87) for every lane, on the device; returns the
        host copies."""
        table, lens = self.net.route_table(destinations)
        self._route_table = torch.from_numpy(table).to(self.device)
        self._route_table_len = torch.from_numpy(lens).to(self.device)
        return table, lens

    def _obs_view(self):
        """-> (HwyObsView of the current state, device pointer of the HwyNetGraph lane table)"""
        if self._plugin_view is None:
            v = N.HwyObsView()
            v.n_envs, v.vp, v.n_vehicles, v.n_agents = self.num_envs, self.vp, self.V, int(self._params.n_agents)
            v.pos, v.hs, v.meta = self._pos.data_ptr(), self._hs.data_ptr(), self._meta.data_ptr()
            cnt = getattr(self, "_count", None)
            v.count = None if cnt is None else cnt.data_ptr()
            v.route, v.route_len = self._route.data_ptr(), self._route_len.data_ptr()
            v.speed_index = self._speed_index.data_ptr()
            self._plugin_view = v
        return self._plugin_view, self._graph_dev.data_ptr()

    def _observe_kernel(self) -> None:
        with torch.cuda.device(self.device):
            N.check(self._lib.hwy_network_observe(C.byref(self._params), self._graph_dev.data_ptr(),
                                                  C.byref(self._state), self._fused_out.data_ptr(), self._stream()))

    def _reset(self, mask) -> None:
        if self.reset_mode == "device":
            self._device_reset(None if mask is None else mask.data_ptr(), None, None)
        else:
            ids = np.arange(self.num_envs) if mask is None else np.nonzero(mask.cpu().numpy())[0]
            if len(ids):
                self._host_reset(ids)
        self.observe()

    def _host_reset(self, ids: np.ndarray) -> None:
        """Re-spawn the envs `ids` with numpy from their streams (_reset_envs), then store the advanced streams."""
        generators = [self._rngs[e] for e in ids]
        set_pcg64_words(generators, self._rng.cpu().numpy().view(np.uint64)[:, ids])
        self._reset_envs(ids)
        idx = torch.from_numpy(np.asarray(ids, dtype=np.int64)).to(self.device)
        self._rng[:, idx] = torch.from_numpy(pcg64_words(generators).view(np.int64)).to(self.device)

    def _same_step_autoreset(self, info) -> None:
        if self.reset_mode == "device":
            return super()._same_step_autoreset(info)
        done = (self._terminated | self._truncated).cpu().numpy().astype(bool)
        if done.any():
            self._final_obs.copy_(self._obs)
            info["final_obs"] = self._final_obs
            self._host_reset(np.nonzero(done)[0])
            self.observe()

    def road_substeps(self, n_substeps: int) -> None:
        """The reference's operator seam (`AbstractEnv._simulate` without `action_type.act`, abstract.py:304-307):
        `n_substeps` x (`Road.act()`; `Road.step(1 / simulation_frequency)`, with the RegulatedRoad rules where the
        scenario has them) on the device state of every env and nothing else — no observation, reward, clock,
        population change or autoreset; the controlled vehicle acts like `ControlledVehicle.act(None)`."""
        if not self._seeded:
            raise RuntimeError("call reset() before road_substeps()")
        with torch.cuda.device(self.device):
            N.check(self._lib.hwy_network_substeps(C.byref(self._params), self._graph_dev.data_ptr(),
                                                   C.byref(self._state), None, int(n_substeps), self._stream()))
