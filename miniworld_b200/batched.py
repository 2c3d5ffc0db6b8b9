"""BatchedMiniWorld: N independent MiniWorld environments stepped by one C-ABI call.

This is the hot path of the package: `step(actions)` = K1 (physics / reward / auto-reset,
one warp per env) + K2 (first-person render, one block per env) through `mwb_step`.
Per-environment semantics are exactly those of the reference's `MiniWorldEnv.reset/step`
(miniworld.py:544-604, 670-730) plus the level's own `step()` rule, for every env:

  * env i seeded with `reset(seed=[...])` owns the numpy stream
    Generator(PCG64(SeedSequence(seed_i))), continued across unseeded resets;
  * levels with a fixed room layout (Hallway, OneRoom, FourRooms, PickupObjects) reset
    entirely on the device from the lowered `device_program` (csrc/reset.cuh);
  * levels whose topology is random per episode (Maze) generate worlds with the level's
    Python `_gen_world()` on the host (same numpy stream) and upload them (`mwb_set_world`);
  * `autoreset=True` gives Gymnasium "next-step" auto-reset: the step after a
    terminated|truncated step resets that env (action ignored, reward 0);
  * with several levels and `dynamic_levels=True`, an env's level can change at its resets:
    pending assignments (`set_env_level`) and device-side draws from `level_weights`.

Outputs are torch CUDA tensors by default (zero-copy from the kernels); `step_host`
performs the same step with pinned host buffers for callers that want numpy.
"""
import numpy as np

from . import pack
from .engine import (Engine, LEVEL_CAP, OP_PLACE, OP_PUT, PROTO_DTYPE, RULE_GOAL, RULE_NONE, RULE_HEALTH, RULE_PICKUP,
                     RULE_PUTNEXT, RULE_SIDEWALK, RULE_SIGN, generator_from_state, rng_state_of, RNG_DTYPE)
from .envs import LEVELS
from .program import ResetProgram


_RULES = {"goal": RULE_GOAL, "pickup": RULE_PICKUP, "sidewalk": RULE_SIDEWALK, "sign": RULE_SIGN, "health": RULE_HEALTH,
          "putnext": RULE_PUTNEXT, "none": RULE_NONE}


def _resolve_level(level):
    if isinstance(level, str):
        if level not in LEVELS:
            raise KeyError("unknown level id %r (known: %s)" % (level, ", ".join(sorted(LEVELS))))
        return LEVELS[level]
    return level


def _torch_stream(torch, device):
    """Handle of torch's current stream for mwb_step / mwb_render_obs.  torch's default stream is the legacy default
    stream (handle 0); a NULL stream argument means "the handle's own stream" to the C ABI, which would not be ordered
    after the torch kernels that produced the actions -- so the default stream is passed as cudaStreamLegacy (0x1)."""
    return torch.cuda.current_stream(device).cuda_stream or 1


_SPLITMIX_GAMMA = 0x9E3779B97F4A7C15
_M64 = (1 << 64) - 1


def _splitmix64_at(seed, k):
    z = (int(seed) + (int(k) + 1) * _SPLITMIX_GAMMA) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def sample_level(seed, global_env, draw, weights):
    """The level draw a reset makes (include/mwb.h, mwb_enable_level_changes), restated in numpy: the level env
    `global_env` draws for the `draw`-th time (0-based) under float32 `weights` [n_levels] and handle seed `seed`.
    Returns None when the weights do not sum to more than 0 (the env keeps its level, and no draw is counted)."""
    w = np.asarray(weights, np.float32)
    w = np.where(w > 0, w, np.float32(0))               # NaN and negative weights count as 0
    total = np.float32(0)
    for x in w:
        total = np.float32(total + x)
    if not total > 0:
        return None
    k = ((int(global_env) & 0xFFFFFFFF) << 32) | (int(draw) & 0xFFFFFFFF)
    u24 = _splitmix64_at(int(seed) & _M64, k) >> 40
    target = np.float32(np.float32(u24) * np.float32(2.0 ** -24)) * total
    cdf, pick = np.float32(0), None
    for l, x in enumerate(w):
        if not x > 0:
            continue
        cdf = np.float32(cdf + x)
        pick = l
        if cdf > target:
            break
    return pick


def _definition_kwargs(kwargs, domain_rand):
    """Keyword arguments of a level's definition instance.  The level's own `domain_rand` wins; without one, the batch's
    `domain_rand` is the default.  The keyword is passed only when it is on, since Sign takes none (it fixes the flag
    off itself, like the reference).  The level's flag is then the `domain_rand` that instance ends up with."""
    kw = dict(kwargs or {})
    if domain_rand and "domain_rand" not in kw:
        kw["domain_rand"] = True
    return kw


class _LevelDef:
    """What the engine needs for one level: a single-level batch has one, a level table one per row."""
    rule = program = maze = maze_cdf = None
    num_placed = 0


def _define_level(level, kwargs, domain_rand, obs_width, obs_height):
    """Build `level`'s definition instance with `kwargs` and lower it: rule, reset program, Maze templates, geometry,
    capacities.  A level without a `device_rule` keeps `rule` None and is not lowered further (its batch rejects it).
    `program` is None when the level resets on the host: it has no `device_program`, or it is a Maze whose templates
    do not reproduce host-generated worlds (`maze_error` holds why)."""
    d = _LevelDef()
    d.cls = _resolve_level(level)
    d.name = level if isinstance(level, str) else level.__name__
    kw = _definition_kwargs(kwargs, domain_rand)
    d.pe = pe = d.cls(device=None, obs_width=obs_width, obs_height=obs_height, **kw)
    d.domain_rand = bool(pe.domain_rand)                 # the level's flag decides (its kwargs may set it)
    rule = getattr(pe, "device_rule", None)
    if rule is None:
        return d
    d.rule = _RULES[rule[0]], rule[1]
    d.geometry = pack.pack_geometry(pe)
    d.max_episode_steps = int(min(pe.max_episode_steps, 2 ** 31 - 1))     # math.inf: never truncates
    d.device_info = dict(getattr(pe, "device_info", None) or {})
    d.device_obs_extra = dict(getattr(pe, "device_obs_extra", None) or {})
    d.uses_maze, d.maze_error = False, None
    if getattr(pe, "device_program", None) is not None:
        prog = ResetProgram()
        pe.device_program(prog)
        d.uses_maze = prog.uses_maze
        if prog.uses_maze:
            # per-episode topology on the device: only if the translated templates reproduce host-generated worlds
            # exactly; otherwise the level resets on the host
            from .maze_lowering import MazeTemplate
            try:
                tmpl = MazeTemplate(d.cls, **kw)
                tmpl.verify(seeds=(0,))
                d.maze, d.maze_cdf = tmpl, pack.room_cdf(pe.room_probs)
            except AssertionError as e:
                d.maze_error = e
        if d.maze_error is None:
            d.program, d.num_placed = prog, prog.num_placed
    slack = 8 if d.maze is not None else 0               # Maze levels: 8 quads and 8 segments of slack
    rooms, quads, segs = d.geometry
    d.caps = (len(rooms), len(quads) + slack, len(segs) + slack)
    return d


def _common(dicts):
    """The entries every dict has, with equal values."""
    return {k: v for k, v in dicts[0].items() if all(d.get(k) == v for d in dicts[1:])}


def default_env_level(num_envs, n_levels):
    """Level of each env when none is given: contiguous, near-equal blocks in the order the levels were listed (the
    first num_envs % n_levels levels get one env more)."""
    base, extra = divmod(int(num_envs), int(n_levels))
    return np.repeat(np.arange(n_levels, dtype=np.int32), [base + (1 if k < extra else 0) for k in range(n_levels)])


class BatchedMiniWorld:
    """`level`: a level id or class, or a sequence of them to run several levels side by side in one batch (multi-task
    or curriculum training; env i runs level `env_level[i]`).  With a sequence, `level_kwargs` may be a sequence
    aligned with it; the observation size, MSAA, auto-reset and action noise are per batch.
    Domain randomisation is per level: a level's kwargs may set `domain_rand`, and `domain_rand` here is the default
    for levels whose kwargs do not.  Rows of one level id that differ in the flag (or in `params` ranges) form a
    randomisation curriculum: an env's resets draw by the flag of the level it resets into.
    Sign (dict observation) cannot share a batch with other levels.  Maze-family levels can with
    `per_env_worlds=True`: each env then gets a world block of its own, which a reset at a Maze level fills with a
    fresh maze (about 123 KB per env with an 8 x 8 Maze in the table, plus about 204 KB per env of HBM triangle
    lists; about 18 KB per env when the largest maze is MazeS3).  Without a Maze level the flag changes nothing.

    `dynamic_levels=True` (with a sequence of levels) lets envs move between levels at their resets, never
    mid-episode: a pending assignment from `set_env_level` wins, otherwise the next level is drawn on the device from
    `level_weights` (all zero, the default, keeps every env on its level).  The draws are keyed by `level_seed` and
    the env's global index `env_offset + i` (ShardedMiniWorld sets the offset), not by the env's own numpy stream."""

    def __init__(self, level, num_envs, obs_width=80, obs_height=60, domain_rand=False, autoreset=True,
                 msaa_samples=8, device=0, want_depth=False, level_kwargs=None, obs_format="hwc", env_level=None,
                 dynamic_levels=False, level_seed=0, env_offset=0, per_env_worlds=False):
        self.num_envs = int(num_envs)
        self.obs_width, self.obs_height = int(obs_width), int(obs_height)
        self.domain_rand = bool(domain_rand)
        self.want_depth = bool(want_depth)
        self.device = int(device)
        self.dynamic_levels = bool(dynamic_levels)
        self.per_env_worlds = bool(per_env_worlds)
        table = isinstance(level, (list, tuple))
        if table:
            defs = self._init_levels(list(level), level_kwargs, env_level)
        else:
            if env_level is not None:
                raise ValueError("env_level assigns envs to levels: pass `level` as a sequence of levels")
            if self.dynamic_levels:
                raise ValueError("dynamic_levels moves envs between levels: pass `level` as a sequence of levels")
            if self.per_env_worlds:
                raise ValueError("per_env_worlds lets Maze levels join a level table: pass `level` as a sequence of "
                                 "levels (a single Maze level always has per-env worlds)")
            defs = self._init_level(level, level_kwargs)
        self._init_engine(defs, table, msaa_samples, autoreset)
        self._level_views = None
        if self.dynamic_levels:
            self.level_seed, self.env_offset = int(level_seed), int(env_offset)
            self.engine.enable_level_changes(self.level_seed, self.env_offset)
        # observation layout written by the render kernel: the reference's PyTorchObsWrapper ("cwh") and
        # GreyscaleWrapper ("grey") are fused into its epilogue instead of running as separate passes
        self.obs_format = obs_format
        N, H, W = self.num_envs, self.obs_height, self.obs_width
        self.obs_shape = {"hwc": (N, H, W, 3), "cwh": (N, 3, W, H), "grey": (N, H, W, 1)}[obs_format]
        self.obs_dtype = np.float64 if obs_format == "grey" else np.uint8
        if obs_format != "hwc":
            self.engine.set_obs_format(obs_format)
        self._seeded = False
        self._torch = None
        self._bufs = None

    def _init_level(self, level, level_kwargs):
        d = _define_level(level, level_kwargs, self.domain_rand, self.obs_width, self.obs_height)
        if d.rule is None:
            raise TypeError("%s has no `device_rule`; use world.MiniWorldEnv (single env) for levels whose "
                            "step() rule is not lowered" % d.cls.__name__)
        self.level_cls, self.level_kwargs, self.proto_env = d.cls, dict(level_kwargs or {}), d.pe
        self.domain_rand = d.domain_rand
        self.max_episode_steps = d.pe.max_episode_steps
        self.level_ids = [level]
        self._env_level = np.zeros(self.num_envs, np.int32)
        return [d]

    def _init_levels(self, levels, level_kwargs, env_level):
        """Several levels in one handle: every level needs a device reset program, and Maze-family levels need
        per-env worlds and templates that reproduce host-generated mazes (a table has no host resets)."""
        n = len(levels)
        if n == 0:
            raise ValueError("empty level list")
        if level_kwargs is None or isinstance(level_kwargs, dict):
            kwargs = [dict(level_kwargs or {}) for _ in range(n)]
        else:
            kwargs = [dict(k or {}) for k in level_kwargs]
            if len(kwargs) != n:
                raise ValueError("level_kwargs has %d entries for %d levels" % (len(kwargs), n))
        if n > LEVEL_CAP:
            raise ValueError("at most %d levels per batch, got %d" % (LEVEL_CAP, n))
        if env_level is None:
            env_level = default_env_level(self.num_envs, n)
        env_level = np.asarray(env_level)
        if env_level.shape != (self.num_envs,) or not np.issubdtype(env_level.dtype, np.integer):
            raise ValueError("env_level must be an int array of shape (%d,), got %s %s" % (self.num_envs, env_level.dtype,
                                                                                     env_level.shape))
        if env_level.size and (env_level.min() < 0 or env_level.max() >= n):
            raise ValueError("env_level entries must lie in [0, %d)" % n)
        for lv in levels:
            _resolve_level(lv)                           # an unknown id fails before any level is built
        defs = []
        for lv, kw in zip(levels, kwargs):
            d = _define_level(lv, kw, self.domain_rand, self.obs_width, self.obs_height)
            if d.rule is None or (d.program is None and not d.uses_maze):
                raise ValueError("%s resets on the host only; a batch of several levels needs device reset programs"
                                 % d.name)
            if d.rule[0] == RULE_SIGN:
                raise ValueError("%s cannot share a batch with other levels: its observation is a dict" % d.name)
            if d.uses_maze and not self.per_env_worlds:
                raise ValueError("%s (Maze family) cannot share a batch with other levels: its geometry is per env "
                                 "(pass per_env_worlds=True to give every env a world of its own)" % d.name)
            if d.program is None:
                raise ValueError("%s: its maze templates do not reproduce host-generated worlds, and a level table "
                                 "cannot hold host-reset levels" % d.name) from d.maze_error
            defs.append(d)
        self.level_ids = [d.name for d in defs]
        self.level_cls, self.level_kwargs, self.proto_env = None, kwargs, None
        self.max_episode_steps = [d.pe.max_episode_steps for d in defs]     # per level
        self._env_level = env_level.astype(np.int32)
        return defs

    def _init_engine(self, defs, table, msaa_samples, autoreset):
        """Create the handle and program it in one of three ways: a single level that resets on the host (worlds
        uploaded per env at its resets), a single Maze level with device templates (a world per env, no shared
        template), or a level table through mwb_set_levels -- which is how every other single level is set up, as a
        table of one row.  Capacities are the maxima over the levels; level 0 fills mwb_create's rule fields."""
        d0 = defs[0]
        self.proto_envs = [d.pe for d in defs]
        largest = max(self.proto_envs, key=lambda pe: pe.action_space.n)
        self.action_space = self.single_action_space = largest.action_space
        self.single_observation_space = d0.pe.observation_space
        self.device_reset = all(d.program is not None for d in defs)
        self.program, self.maze_template = (None, None) if table else (d0.program, d0.maze)
        self.autoreset = bool(autoreset)
        if self.device_reset:
            caps = [max(c) for c in zip(*(d.caps for d in defs))]
            # exact: K2's shared-memory triangle capacity scales with max_ents
            max_ents = max([2] + [d.num_placed for d in defs])
        else:
            caps = [int(1.25 * len(g)) + 4 for g in d0.geometry]
            max_ents = 8
        self.engine = eng = Engine(self.num_envs, self.obs_width, self.obs_height, msaa_samples,
                                   shared_geometry=self.device_reset and self.maze_template is None,
                                   max_rooms=caps[0], max_quads=caps[1], max_segs=caps[2], max_ents=max_ents,
                                   rule=d0.rule, domain_rand=d0.domain_rand, max_episode_steps=d0.max_episode_steps,
                                   autoreset=self.autoreset and self.device_reset, device=self.device)
        eng.sync_assets()
        if not self.device_reset:
            eng.set_params(d0.pe.params)
            # host-reset levels: one worker env per slot keeps that env's RNG stream
            self._workers = [None] * self.num_envs
            self._host_done = np.zeros(self.num_envs, bool)
        elif self.maze_template is not None:
            eng.set_params(d0.pe.params)
            eng.set_protos(self.program.proto_array())
            eng.set_maze(self.maze_template, d0.maze_cdf)
            eng.set_program(self.program.op_array())
        else:
            rows, protos = [], []
            for d in defs:
                ops = d.program.op_array()
                moved = (ops["op"] == OP_PLACE) | (ops["op"] == OP_PUT)     # the ops whose `a` is a proto index
                ops["a"][moved] += len(protos)
                protos.extend(d.program.protos)
                rows.append(dict(rule=d.rule, max_episode_steps=d.max_episode_steps, params=d.pe.params,
                                 geometry=d.geometry, ops=ops, domain_rand=int(d.domain_rand)))
            eng.set_protos(np.array(protos, PROTO_DTYPE))
            eng.set_levels(rows, self._env_level)
            for lvl, d in enumerate(defs):
                if d.maze is not None:
                    eng.set_level_maze(lvl, d.maze, d.maze_cdf)
        # a level's `info` key / extra observation is returned only when every level defines it the same way
        self._device_info = _common([d.device_info for d in defs])
        self._device_obs_extra = _common([d.device_obs_extra for d in defs])

    # ------------------------------------------------------------------ buffers
    def _ensure_torch(self):
        if self._torch is None:
            import torch
            self._torch = torch
            dev = torch.device("cuda", self.device)
            N, H, W = self.num_envs, self.obs_height, self.obs_width
            self._bufs = dict(
                obs=torch.zeros(self.obs_shape, dtype=torch.float64 if self.obs_format == "grey" else torch.uint8, device=dev),
                depth=torch.zeros((N, H, W, 1), dtype=torch.float32, device=dev) if self.want_depth else None,
                reward=torch.zeros(N, dtype=torch.float64, device=dev),
                terminated=torch.zeros(N, dtype=torch.uint8, device=dev),
                truncated=torch.zeros(N, dtype=torch.uint8, device=dev),
                actions=torch.zeros(N, dtype=torch.int32, device=dev),
            )
            # bool views of the uint8 flag buffers the kernel writes (no per-step conversion kernels)
            self._bufs["term_view"] = self._bufs["terminated"].view(torch.bool)
            self._bufs["trunc_view"] = self._bufs["truncated"].view(torch.bool)
            self._info = {"depth": self._bufs["depth"]} if self.want_depth else {}
            # what the level's step() puts into `info` / the observation, read in place from the device state
            eng = self.engine
            self._info_views = {}
            for key, spec in self._device_info.items():
                if spec[0] == "counter":                   # CollectHealth: info["health"] (collecthealth.py:100)
                    self._info[key] = torch.as_tensor(eng.state_array("counter"), device=dev)
                elif spec[0] == "entity_pos":              # TMaze: info["goal_pos"] = self.box.pos (tmaze.py:89)
                    self._info_views[key] = (int(spec[1]), [torch.as_tensor(eng.state_array(n), device=dev)
                                                            for n in ("ent_x", "ent_y", "ent_z")])
            self._obs_dict = dict(self._device_obs_extra)
            if self.dynamic_levels:
                # the level of each env's current episode (after a terminating step still the one that just ended)
                self._info["level"] = self.level_tensor
        return self._torch

    # ------------------------------------------------------------------ level changes (dynamic_levels=True)
    def _views(self):
        """env_level / next_level / level_weights in place: torch CUDA tensors, or numpy arrays on the kernels' host
        build (whose state lives in host memory)."""
        if not self.dynamic_levels:
            raise RuntimeError("levels are fixed in this batch: construct it with dynamic_levels=True")
        if self._level_views is None:
            names = ("env_level", "next_level", "level_weights")
            if self.engine.host_memory:
                self._level_views = {n: self.engine.state_array(n) for n in names}
            else:
                import torch
                dev = torch.device("cuda", self.device)
                self._level_views = {n: torch.as_tensor(self.engine.state_array(n), device=dev) for n in names}
        return self._level_views

    @property
    def level_tensor(self):
        """int32 [N] view of each env's current level (changes only at the env's resets)."""
        return self._views()["env_level"]

    @property
    def level_weights(self):
        """float32 [n_levels] view of the level-sampling weights; update it in place (stream-ordered, no sync).
        Weights that are not > 0 count as 0; all zero keeps every env on its level at its resets."""
        return self._views()["level_weights"]

    def set_level_weights(self, weights):
        """Copy `weights` (sequence, numpy array or tensor of n_levels values) into `level_weights`."""
        view = self.level_weights
        n = len(self.level_ids)
        if tuple(np.shape(weights)) != (n,):
            raise ValueError("level weights must have shape (%d,), got %s" % (n, tuple(np.shape(weights))))
        if isinstance(view, np.ndarray):
            view[:] = np.asarray(weights.cpu() if hasattr(weights, "cpu") else weights, np.float32)
        else:
            torch = self._ensure_torch()
            view.copy_(torch.as_tensor(weights, dtype=torch.float32).to(view.device), non_blocking=False)

    def set_env_level(self, env_ids, levels):
        """Move the listed envs to `levels` (one level, or one per env) at their next reset; envs in mid-episode finish
        it on their current level.  An env listed more than once takes its last entry."""
        ids = np.atleast_1d(np.asarray(env_ids))
        lv = np.broadcast_to(np.asarray(levels), ids.shape) if np.ndim(levels) == 0 else np.asarray(levels)
        if lv.shape != ids.shape:
            raise ValueError("set_env_level: %d env ids but %d levels" % (ids.size, lv.size))
        if ids.size == 0:
            return
        if not (np.issubdtype(ids.dtype, np.integer) and np.issubdtype(lv.dtype, np.integer)):
            raise ValueError("set_env_level takes integer env ids and levels")
        if ids.min() < 0 or ids.max() >= self.num_envs:
            raise ValueError("env ids must lie in [0, %d)" % self.num_envs)
        if lv.min() < 0 or lv.max() >= len(self.level_ids):
            raise ValueError("levels must lie in [0, %d)" % len(self.level_ids))
        last = ids.size - 1 - np.unique(ids[::-1], return_index=True)[1]    # an env listed twice: its last entry wins
        ids, lv = ids[last], lv[last]
        view = self._views()["next_level"]
        if isinstance(view, np.ndarray):
            view[ids] = lv.astype(np.int32)
        else:
            import torch
            view[torch.as_tensor(ids.astype(np.int64), device=view.device)] = torch.as_tensor(
                lv.astype(np.int32), device=view.device)

    @property
    def env_level(self):
        """numpy int32 [N]: the level of each env.  With dynamic_levels it is a host copy of `level_tensor` and
        synchronises with the device (the current torch stream) to read it."""
        if not self.dynamic_levels:
            return self._env_level
        view = self.level_tensor
        return np.array(view) if isinstance(view, np.ndarray) else view.cpu().numpy()

    def _wrap(self, obs):
        """Observation / info as the level's own step() shapes them (Sign: {"obs", "goal"}, sign.py:176)."""
        torch = self._torch
        for key, (slot, xyz) in self._info_views.items():
            self._info[key] = torch.stack([a[slot] for a in xyz], dim=1)          # float64 [N, 3]
        if self._obs_dict:
            obs = dict({k: torch.full((self.num_envs,), int(v), dtype=torch.int64, device=obs.device)
                        for k, v in self._obs_dict.items()}, obs=obs)
        return obs

    # ------------------------------------------------------------------ reset
    def reset(self, seed=None, env_ids=None):
        """Reset all (or the listed) envs.  `seed`: int base (env i gets seed + i), a sequence
        of per-env seeds, or None to continue each env's stream.  Returns (obs, info)."""
        ids = np.arange(self.num_envs, dtype=np.int32) if env_ids is None else np.asarray(env_ids, np.int32)
        if seed is not None:
            seeds = [int(seed) + int(i) for i in ids] if np.isscalar(seed) else [int(s) for s in seed]
            assert len(seeds) == len(ids)
        else:
            seeds = None
            if not self._seeded:
                seeds = [int(s) for s in np.random.SeedSequence().generate_state(len(ids))]
        if self.device_reset:
            if seeds is not None:
                states = np.array([rng_state_of(s) for s in seeds], RNG_DTYPE)
                self.engine.seed(ids, states)
            self.engine.reset(None if env_ids is None else ids, stream=self._level_stream())
        else:
            self._host_reset(ids, seeds)
        self._seeded = True
        return self._wrap(self.render()), {}

    def _host_reset(self, ids, seeds, hold=False):
        """Host-side reset of the listed envs (levels without a device program).  The env's numpy
        stream is shared with the device: per-step domain-rand draws happen in K1, so the
        stream position is pulled from the device before `_gen_world()` runs on the host and
        pushed back afterwards."""
        worlds = []
        dev_rng = self.engine.get_state(rng=True)["rng"] if (self.domain_rand and self._seeded) else None
        for k, i in enumerate(ids):
            w = self._workers[i]
            if w is None:
                w = self._workers[i] = self.level_cls.__new__(self.level_cls)
                w.__dict__.update({k2: v for k2, v in self.proto_env.__dict__.items()
                                   if k2 not in ("_np_random", "agent", "entities", "rooms", "wall_segs")})
                w._np_random = None
            elif dev_rng is not None and (seeds is None):
                w._np_random = generator_from_state(dev_rng[i])
            w.reset(seed=None if seeds is None else seeds[k])
            worlds.append(pack.pack_world(w))
            worlds[-1]["hold"] = int(hold)
        # one proto table for the handle: per-env protos are identical for these levels
        self.engine.sync_assets()
        self.engine.set_protos(worlds[0]["protos"])
        self.engine.set_world(ids, worlds)
        if self.domain_rand:
            self.engine.seed(ids, np.array([rng_state_of(self._workers[i].np_random) for i in ids], RNG_DTYPE))

    # ------------------------------------------------------------------ step / render
    def step(self, actions):
        """actions: int tensor / array [N].  Returns (obs, reward, terminated, truncated, info)
        as torch CUDA tensors; obs is uint8 [N, H, W, 3] (and info['depth'] when want_depth)."""
        torch = self._ensure_torch()
        b = self._bufs
        if isinstance(actions, torch.Tensor) and actions.is_cuda and actions.dtype == torch.int32 and actions.is_contiguous():
            acts = actions                      # consumed in place by K1, no copy
        elif isinstance(actions, torch.Tensor):
            b["actions"].copy_(actions.to(torch.int32), non_blocking=True)
            acts = b["actions"]
        else:
            b["actions"].copy_(torch.as_tensor(np.asarray(actions, np.int32)), non_blocking=True)
            acts = b["actions"]
        stream = _torch_stream(torch, self.device)
        if not self.device_reset and self.autoreset and self._host_done.any():
            self._host_reset(np.nonzero(self._host_done)[0].astype(np.int32), None, hold=True)
            self._host_done[:] = False
        self.engine.step(acts, obs=b["obs"], depth=b["depth"], reward=b["reward"],
                         terminated=b["terminated"], truncated=b["truncated"], stream=stream)
        if not self.device_reset and self.autoreset:
            self._host_done = (b["terminated"] | b["truncated"]).bool().cpu().numpy()
        return self._wrap(b["obs"]), b["reward"], b["term_view"], b["trunc_view"], self._info

    def step_host(self, actions, out=None, render=True):
        """Same step with HOST buffers end to end (numpy in, numpy out): actions are copied
        host->device and obs / reward / flags device->host inside the call."""
        N, H, W = self.num_envs, self.obs_height, self.obs_width
        if out is None:
            out = dict(obs=np.zeros(self.obs_shape, self.obs_dtype), reward=np.zeros(N), terminated=np.zeros(N, np.uint8),
                       truncated=np.zeros(N, np.uint8),
                       depth=np.zeros((N, H, W, 1), np.float32) if self.want_depth else None)
        acts = np.ascontiguousarray(actions, np.int32)
        if not self.device_reset and self.autoreset and self._host_done.any():
            self._host_reset(np.nonzero(self._host_done)[0].astype(np.int32), None, hold=True)
            self._host_done[:] = False
        self.engine.step(acts, obs=out["obs"] if render else None, depth=out.get("depth") if render else None,
                         reward=out["reward"], terminated=out["terminated"], truncated=out["truncated"],
                         stream=self._level_stream())
        if not self.device_reset and self.autoreset:
            self._host_done = (out["terminated"] | out["truncated"]).astype(bool)
        return out

    def render(self):
        torch = self._ensure_torch()
        b = self._bufs
        stream = _torch_stream(torch, self.device)
        self.engine.render(obs=b["obs"], depth=b["depth"], stream=stream)
        return b["obs"]

    def render_depth(self):
        torch = self._ensure_torch()
        dev = torch.device("cuda", self.device)
        d = torch.zeros((self.num_envs, self.obs_height, self.obs_width, 1), dtype=torch.float32, device=dev)
        self.engine.render(depth=d, stream=_torch_stream(torch, self.device))
        return d

    def snapshot(self):
        """Checkpoint of all envs (numpy uint8 blob); `restore` resumes them bit for bit."""
        if not self.device_reset:
            raise TypeError("snapshot covers the device-resident state; host-reset levels keep RNG streams in Python")
        self._sync_level_writes()
        return self.engine.snapshot()

    def restore(self, blob):
        self._sync_level_writes()
        self.engine.restore(blob)
        self._seeded = True

    def _level_stream(self):
        """Stream for a call whose resets read next_level / level_weights: with level changes on, torch's current
        stream, so that the resets run behind the torch work that wrote those arrays (set_env_level, set_level_weights,
        in-place writes); otherwise None, the handle's own stream.  Calls with host outputs still return finished."""
        if self.dynamic_levels and not self.engine.host_memory:
            return _torch_stream(self._ensure_torch(), self.device)
        return None

    def _sync_level_writes(self):
        """Finish torch writes to next_level / level_weights before the handle's own stream reads or replaces them."""
        if self.dynamic_levels and not self.engine.host_memory:
            self._ensure_torch().cuda.current_stream(self.device).synchronize()

    def set_action_noise(self, prob=0.9, random_action=None):
        """Device-side StochasticActionWrapper (reference wrappers.py:49-71) for every env: the replacement draws
        come from each env's own numpy stream, in the order the wrapper would make them.  prob=None disables."""
        if not self.device_reset and prob is not None:
            raise TypeError("action noise needs the env streams on the device (levels with a device reset program)")
        self.engine.set_action_noise(prob, random_action)

    def render_top_view(self, render_agent=True, out=None):
        """Map view of every env in the observation layout -- uint8 [N, H, W, 3] by default (reference
        render_top_view, miniworld.py:1088-1175).
        Extents come from the level definition (all envs of a level share them; a batch of several levels needs
        levels with equal extents).  `out`: optional numpy array / CUDA tensor to fill; default a fresh CUDA tensor."""
        exts = [tuple(pe.top_view_extents(self.obs_width, self.obs_height)) for pe in self.proto_envs]
        if any(e != exts[0] for e in exts[1:]):
            raise ValueError("render_top_view needs one map extent for the whole batch; its levels' extents differ")
        ext = exts[0]
        if out is None:
            torch = self._ensure_torch()
            out = torch.zeros(self.obs_shape, dtype=torch.float64 if self.obs_format == "grey" else torch.uint8,
                              device=torch.device("cuda", self.device))      # same layout as the observations
        self.engine.render_top_view(ext, out, render_agent)
        return out

    def visible_ents(self, out=None):
        """uint32 [N]: bit e set iff entity-list slot e of that env passes the reference's occlusion query
        (get_visible_ents, miniworld.py:1238-1333)."""
        if out is None:
            torch = self._ensure_torch()
            out = torch.zeros(self.num_envs, dtype=torch.int32, device=torch.device("cuda", self.device))
        self.engine.visible_ents(out)
        return out

    # ------------------------------------------------------------------ state views
    def get_state(self, **kw):
        return self.engine.get_state(**kw)

    def np_random(self, i):
        """numpy Generator positioned where env i's device stream currently is."""
        return generator_from_state(self.engine.get_state(rng=True)["rng"][i])

    def close(self):
        self.engine.close()
