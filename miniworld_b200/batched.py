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
    pending assignments (`set_env_level`) and device-side draws from `level_weights`;
  * with `episode_seeds=True`, an env's next reset can start from a chosen seed (`next_seed`, `set_env_seed`),
    seeded on the device as `reset(seed=s)` would, and `info["seed"]` names the seed of each running episode;
  * with `maze_layouts=True`, an env's next reset at a Maze level can build a maze written into a device tensor
    (`next_maze`, `set_env_maze`), and `info["maze"]` holds the layout of each running episode;
  * with `start_poses=True`, an env's next reset can place the agent and the entities at poses written into device
    tensors (`next_pose`, `set_env_pose`), and `info["start"]` holds where each running episode's agent started;
  * with `reset_draws=True`, an env's next reset can take designed outcomes of its level's reset draws (object kinds and
    colours, box sizes, goal sides, headings) written into a device tensor (`next_draws`, `set_env_draws`), and
    `info["draws"]` holds the outcome of every draw of each running episode;
  * with `env_params=True`, an env's next episode can run on DomainParams of its own, (default, min, max) rows written
    into a device tensor (`next_params`, `set_env_param`), and `info["params"]` holds the rows of each running episode;
  * with `state_bank=K`, envs can be saved into K device-side records (`save_states`) and an env's next reset can load
    one (`next_state`, `set_env_state`), and `info["state"]` names the record each running episode was loaded from;
  * with `goal_distance=True`, every step and reset leaves each env's geodesic distance to its goal (`goal_dist`), an
    expert action (`expert_action`) and its episode's shortest path (`episode_shortest`) on the device.

Outputs are torch CUDA tensors by default (zero-copy from the kernels); `step_host`
performs the same step with pinned host buffers for callers that want numpy.
"""
from collections import namedtuple

import numpy as np

from . import pack
from .engine import (ENV_PARAM_ROWS, Engine, GOAL_GRID_DTYPE, LEVEL_CAP, LOWERED_PARAMS, OP_PLACE, OP_PUT, PARAMS_COLUMN, PROTO_DTYPE, RULE_GOAL,
                     RULE_NONE, RULE_HEALTH, RULE_PICKUP, RULE_PUTNEXT, RULE_SIDEWALK, RULE_SIGN, generator_from_state,
                     rng_state_of, RNG_DTYPE)
from .envs import LEVELS
from .params import DomainParams
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


# The run-time modes, in the order the constructor turns them on (the state bank last: its record layout depends on the
# other modes).  `flag`: the constructor argument and attribute (Engine.enable_<flag> turns the mode on, except
# enable_level_changes); `arrays`: the state arrays it adds, whose accessors raise RuntimeError(`missing`) on a batch
# without it; `host_reset`: the TypeError of a batch without device resets (None where an earlier check refuses
# one: level changes need a sequence of levels, maze layouts device Maze templates); `info`: (key, array) pairs.
_Mode = namedtuple("_Mode", "flag arrays missing host_reset info")
_MODES = (
    _Mode("dynamic_levels", ("env_level", "next_level", "level_weights"),
          "levels are fixed in this batch: construct it with dynamic_levels=True", None, [("level", "env_level")]),
    _Mode("episode_seeds", ("next_seed", "episode_seed"),
          "this batch has no episode seeds: construct it with episode_seeds=True",
          "episode seeds are taken by device resets; host-reset levels keep RNG streams in Python",
          [("seed", "episode_seed")]),
    _Mode("maze_layouts", ("next_maze", "next_maze_cells", "maze_pending", "episode_maze"),
          "this batch has no maze layouts: construct it with maze_layouts=True", None, [("maze", "episode_maze")]),
    _Mode("start_poses", ("next_pose", "next_agent_pose", "pose_pending", "episode_start"),
          "this batch has no start poses: construct it with start_poses=True",
          "start poses are taken by device resets; host-reset levels place entities in Python "
          "(reset(options={\"poses\": ...}) of the level itself)", [("start", "episode_start")]),
    _Mode("reset_draws", ("next_draws", "draws_pending", "episode_draws"),
          "this batch has no reset draws: construct it with reset_draws=True",
          "reset draws are taken by device resets; host-reset levels draw in Python "
          "(reset(options={\"draws\": ...}) of the level itself)", [("draws", "episode_draws")]),
    _Mode("env_params", ("next_params", "params_pending", "episode_params"),
          "this batch has no env params: construct it with env_params=True",
          "env params are taken by device resets; host-reset levels draw their params in Python "
          "(reset(options={\"params\": ...}) of the level itself)", [("params", "episode_params")]),
    _Mode("goal_distance", ("goal_dist", "expert_action", "episode_shortest", "goal_field"),
          "this batch has no goal distance: construct it with goal_distance=True",
          "goal distance is built by device resets; host-reset levels build their worlds in Python "
          "(MiniWorldEnv.goal_distance() of the level itself)",
          [("goal_dist", "goal_dist"), ("shortest", "episode_shortest")]),
    _Mode("state_bank", ("next_state", "episode_state", "bank_level"),
          "this batch has no state bank: construct it with state_bank=K",
          "the state bank loads states at device resets; host-reset levels keep their worlds and RNG streams in Python",
          [("state", "episode_state")]),
)

# the flag a run-time array needs, and what its accessor raises on a batch built without it
_NEEDS = {name: (m.flag, RuntimeError, m.missing) for m in _MODES for name in m.arrays}
_NEEDS["level_params"] = ("device_reset", TypeError, "level params change at device resets; host-reset levels draw "
                          "theirs in Python (set them on the level's own DomainParams)")


class _Views(dict):
    """Array name -> in-place view of one handle's state array (Engine.ARRAYS) in its final shape: a torch CUDA tensor,
    or a numpy array on the kernels' host build (whose state lives in host memory).  A view is made at the first lookup
    of its name, which raises as _NEEDS says when the batch lacks the array's mode; later lookups are dict lookups."""

    def __init__(self, engine, device, flags, maze_shape):
        super().__init__()
        self._engine, self._device, self._flags, self._maze_shape = engine, device, flags, maze_shape

    def __missing__(self, name):
        need = _NEEDS.get(name)
        if need is not None and not self._flags[need[0]]:
            raise need[1](need[2])
        shape = (self._engine.N,) + self._maze_shape if name in ("next_maze", "episode_maze") else None
        view = self._engine.state_array(name, shape)
        if not self._engine.host_memory:
            import torch
            view = torch.as_tensor(view, device=torch.device("cuda", self._device))
        self[name] = view
        return view


def _host(a):
    """`a` as a numpy array, copied from a torch tensor first when it is one."""
    return np.asarray(a.cpu() if hasattr(a, "cpu") else a)


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
    the env's global index `env_offset + i` (ShardedMiniWorld sets the offset), not by the env's own numpy stream.

    A level's params (`level_kwargs` `params=`) are the initial content of a table that `set_level_param` /
    `set_level_params` rewrite while the batch runs (automatic domain randomisation), as the reference's
    `env.params.set(...)` does: step ranges apply from the next step, the rest from each env's next reset.

    `episode_seeds=True` (one level or a table; levels that reset on the device) decides which episode of its level an
    env plays, for level replay: a seed written to `next_seed[i]` (`set_env_seed`) is consumed by env i's next reset,
    the auto-reset inside `step` included, which then starts the stream `reset(seed=s)` would, built on the device.
    `episode_seed` / `info["seed"]` hold the seed each running episode started from, or -1 when the env continued its
    stream; after a terminating step they still name the episode that just ended.

    `maze_layouts=True` (a single Maze-family level, or a table with some) lets torch code design the mazes, for
    environment design (PAIRED, ACCEL): a layout written to `next_maze[i]` (uint8 [rows, cols], the maxima over the
    batch's Maze levels; bit 0 of cell (j, i) opens its wall to (j, i + 1), bit 1 its wall to (j + 1, i)) with
    `maze_pending[i] = 1` is built by env i's next reset at a Maze level, the auto-reset inside `step` included, as
    `Maze.reset(options={"maze": layout, "goal_cell": g, "agent_cell": a})` builds it on the host; `next_maze_cells[i]`
    holds (g, a), flat cells j * cols + i where the goal box and the agent are placed, -1 for anywhere.  A reset at a
    level that is not a Maze leaves the layout pending.  `episode_maze` / `info["maze"]` hold the layout of every
    running episode, random carves included (zeros at other levels); after a terminating step they still name the
    episode that just ended.  Replaying a carve's recorded layout builds the same walls, but creates the connector rooms
    in another order than the carve did, so the episode's placement draws differ.  Each Maze level's capacities are
    sized for its all-open maze (c cells, E inner edges: c + E rooms, 6c + 2E quads, as against 2c - 1 and 8c - 2).

    `start_poses=True` (one level or a table; levels that reset on the device) decides where episodes start, for reverse
    and start-state curricula and goal placement: with `pose_pending[i]` set, env i's next reset at any level, the
    auto-reset inside `step` included, places the entity that fills slot e at `next_pose[i, e]` = (x, z, dir) and the
    agent at `next_agent_pose[i]`, as `reset(options={"poses": {e: (x, z, dir)}, "agent_pose": (x, z, dir)})` does on
    the host: the reference's `place_entity(pos=..., dir=...)` branch, without a search or a collision check.  A row
    applies when its x and z are finite (the rows start as NaN), its dir when that is finite (otherwise the level's dir,
    or a uniform draw).  The agent's row wins over the agent's slot row.  The reset clears `pose_pending` and leaves the
    rows as written.  A design that leaves a later searched placement of the same reset no free spot makes that search
    run forever, as it would in the reference.  `level_slots` names the slots each level fills.  `episode_start` / `info["start"]` hold the
    agent's (x, z, dir) at the start of every running episode, designed or drawn; after a terminating step they still
    name the episode that just ended.

    `reset_draws=True` (one level or a table; levels that reset on the device, one of them with a draw) decides what
    episodes contain, for environment design over object composition, goal-side balancing and size curricula.  A level's
    reset draws are the choices and uniforms its `_gen_world()` makes itself (not those inside place_entity), numbered
    0, 1, ... in call order; `draw_specs[level]` lists them (index, kind "choice" with n or "uniform" with lo and hi,
    label): Hallway's heading; TMaze's and YMaze's goal side and heading; PickupObjects' kind (0 Ball, 1 Box, 2 Key) and
    colour (index into COLOR_NAMES) per object; RoomObjects' Box, Ball and Key colours; PutNext's box size per colour.
    With `draws_pending[i]` set, env i's next reset at any level, the auto-reset inside `step` included, makes each draw d
    as usual and then replaces its result with `next_draws[i, d]` when that lies in the draw's support (a choice over n:
    an integer in [0, n); a uniform over [lo, hi]: finite, lo <= v <= hi), as `reset(options={"draws": {d: v}})` does on
    the host.  Otherwise (NaN, the rows' initial value, included) the drawn value stays, so the stream position never
    changes and a seed plus a design reproduces an episode.  The reset clears `draws_pending` and leaves the rows as
    written; rows beyond the level's draw count are ignored.  `episode_draws` / `info["draws"]` (float64 [N, D], D the
    largest draw count of the batch's levels) hold every draw's outcome of each running episode, NaN beyond its level's
    count; after a terminating step they still name the episode that just ended.  A designed start pose still wins for
    position and dir; a state-bank load leaves pending draws for the next reset that runs a program.

    `env_params=True` (one level or a table; levels that reset on the device) gives episodes DomainParams of their own,
    for automatic domain randomisation with per-env boundary sampling and for robustness sweeps over camera, lighting
    and dynamics.  A row is 22 element rows of float64 (default, min, max) in engine.LOWERED_PARAMS order, vector params
    expanded element by element; `param_rows` maps each param to its row index or slice.  With `params_pending[i]` set,
    env i's next reset at any level, the auto-reset inside `step` included, copies `next_params[i]` into
    `episode_params[i]` and clears the flag (the rows stay as written); any other reset that runs a program sets
    `episode_params[i]` to NaN.  The episode runs on its level's params merged element by element: the env's (min, max)
    when both are finite, else the level's range; the env's default when finite, else the level's.  The level's entries
    are read as they stand (forward_step, forward_drift and turn_step at every step, so `set_level_param` keeps reaching
    every entry an episode did not design), and max_forward_step follows a designed forward_step range.  Draw counts
    do not change (the level's `domain_rand` still decides whether draws are made), so a seed plus a row reproduces an
    episode, and (v, v, v) pins an element.  `episode_params` / `info["params"]` (float64 [N, 22, 3]) hold each running
    episode's row; after a terminating step they still name the episode that just ended.  A state-bank load leaves a
    pending row for the next reset that runs a program.  Memory: 1 057 B per env plus a 536 B merge scratch.

    `state_bank=K` (one level or a table; levels that reset on the device) keeps K records of env states on the device,
    for Go-Explore, backplay and branching rollouts: `save_states(env_ids, slots)` copies env env_ids[t] into slot
    slots[t] (entity list, counters, health, camera, lighting, colours, textures, the RNG stream, the level, the mode
    records and, at levels with per-env worlds, the world in use).  With `next_state[i] = s` (`set_env_state`), env i's
    next reset, the auto-reset inside `step` included, becomes slot s bit for bit instead of running the level's program,
    when the slot is filled and holds the env's level (any level with `dynamic_levels=True`); otherwise the entry is
    dropped and the reset runs as it would have.  The load consumes only `next_state`: a pending level, seed, layout or
    pose waits for the next reset that runs a program.  A loaded env continues exactly as the saved env would have,
    `step_count` included.  `episode_state` / `info["state"]` name the slot each running episode was loaded from, or -1;
    after a terminating step they still name the episode that just ended.  `bank_level` holds each slot's level (-1 =
    empty).  A record takes about 264 B + 68 B per entity slot + 12 B per room; at levels with per-env worlds it has
    room for one world block as well (about 123 KB for an 8 x 8 Maze), so 4096 slots of such a batch take over 0.5 GB.

    `goal_distance=True` (one level or a table; levels that reset on the device, one of them with a goal rule: Hallway,
    OneRoom, FourRooms, TMaze, YMaze, WallGap and the Maze family) gives the shortest path to the goal on the device, for
    SPL, shortest-path filters of environment design, distance-shaped rewards and imitation learning.  Each goal level
    gets a grid of 0.25 m over its rooms' bounding box (`goal_grids`, `grid_shape`); every reset, a state-bank load
    included, builds the env's distance field over it from the world it left (`goal_field`, uint16 [N, G] in units of
    0.05 m, node (k, l) at index l * nx + k, 0xFFFF unreachable), and after every step and reset `goal_dist` /
    `info["goal_dist"]` (float64 [N], metres) hold the agent's geodesic distance to the goal: 0 when it is near the goal,
    +inf when no free node near it reaches the goal, NaN at levels without a goal rule.  `expert_action` (int32 [N]) is
    the action along a shortest path (turn left, turn right or move forward; -1 where goal_dist is not finite), and
    `episode_shortest` / `info["shortest"]` the goal_dist right after the reset that started the running episode; after
    a terminating step it still names the episode that just ended.  navigation.py restates the definitions in numpy.
    Memory is 3 G + 21 bytes per env (G: the largest grid, 10 609 nodes for an 8 x 8 Maze)."""

    def __init__(self, level, num_envs, obs_width=80, obs_height=60, domain_rand=False, autoreset=True,
                 msaa_samples=8, device=0, want_depth=False, level_kwargs=None, obs_format="hwc", env_level=None,
                 dynamic_levels=False, level_seed=0, env_offset=0, per_env_worlds=False, episode_seeds=False,
                 maze_layouts=False, start_poses=False, state_bank=None, reset_draws=False, goal_distance=False,
                 env_params=False):
        given = locals()
        self.num_envs = int(num_envs)
        self.obs_width, self.obs_height = int(obs_width), int(obs_height)
        self.domain_rand = bool(domain_rand)
        self.want_depth = bool(want_depth)
        self.device = int(device)
        self.per_env_worlds = bool(per_env_worlds)
        if state_bank is not None and (isinstance(state_bank, bool) or not isinstance(state_bank, (int, np.integer))
                                       or state_bank < 1):
            raise ValueError("state_bank is a number of slots >= 1, got %r" % (state_bank,))
        self.bank_slots = int(state_bank or 0)
        for m in _MODES:
            setattr(self, m.flag, bool(given[m.flag]))
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
        if self.maze_layouts:
            self._size_for_layouts(defs)
        self._init_engine(defs, table, msaa_samples, autoreset)
        flags = {m.flag: getattr(self, m.flag) for m in _MODES}
        self._view_map = _Views(self.engine, self.device, dict(flags, device_reset=self.device_reset),
                                getattr(self, "maze_shape", None))
        for m in _MODES:
            if not flags[m.flag]:
                continue
            if m.host_reset is not None and not self.device_reset:
                self.engine.close()
                raise TypeError(m.host_reset)
            if m.flag == "dynamic_levels":
                self.level_seed, self.env_offset = int(level_seed), int(env_offset)
                self.engine.enable_level_changes(self.level_seed, self.env_offset)
            elif m.flag == "reset_draws" and not any(self.draw_specs):
                self.engine.close()
                raise ValueError("reset_draws needs a level with a reset draw; %s make none"
                                 % ", ".join(self.level_ids))
            elif m.flag == "goal_distance":
                self._enable_goal_distance(defs)
            elif m.flag == "state_bank":
                self.engine.enable_state_bank(self.bank_slots)
            else:
                getattr(self.engine, "enable_" + m.flag)()
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
        self._params_written = False

    def _enable_goal_distance(self, defs):
        """goal_distance=True: one grid per level from its definition instance (navigation.level_grid), goal slot -1 at
        levels without a goal rule."""
        from .navigation import level_grid
        grids = np.zeros(len(defs), GOAL_GRID_DTYPE)
        grids["goal_slot"] = -1
        for l, d in enumerate(defs):
            if d.rule[0] != RULE_GOAL:
                continue
            try:
                grids[l]["min_x"], grids[l]["min_z"], grids[l]["nx"], grids[l]["nz"] = level_grid(d.pe)
            except ValueError:
                self.engine.close()
                raise
            grids[l]["goal_slot"] = d.rule[1]
        if not (grids["goal_slot"] >= 0).any():
            self.engine.close()
            raise ValueError("goal_distance needs a level with a goal rule; %s have none" % ", ".join(map(str, self.level_ids)))
        self.goal_grids = grids
        self.engine.enable_goal_distance(grids)

    @property
    def grid_shape(self):
        """(nz, nx) of each level's goal grid, None at levels without a goal rule (goal_distance=True)."""
        self._views()["goal_dist"]                   # a batch without the mode raises
        return [(int(g["nz"]), int(g["nx"])) if g["goal_slot"] >= 0 else None for g in self.goal_grids]

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

    def _size_for_layouts(self, defs):
        """maze_layouts=True: every Maze level's capacities from its all-open maze (c cells, E inner edges: c + E rooms,
        6c + 2E quads, 4c segments), and the layout shape from the largest grid."""
        from .envs.maze import Maze
        mazes = [d for d in defs if d.uses_maze or issubclass(d.cls, Maze)]
        if not mazes:
            raise ValueError("maze_layouts needs a Maze-family level in the batch")
        for d in mazes:
            if d.maze is None:
                raise TypeError("%s: its maze templates do not reproduce host-generated worlds, so it resets on the host, "
                                "where designed layouts cannot reach it" % d.name) from d.maze_error
            R, C = d.maze.rows, d.maze.cols
            try:
                d.maze.verify_layouts([np.full((R, C), 3, np.uint8)])       # the all-open maze: every connector kind
            except AssertionError as err:
                raise TypeError("%s: its maze templates do not reproduce host-built designed layouts" % d.name) from err
            c, e = R * C, R * (C - 1) + (R - 1) * C
            d.caps = (max(d.caps[0], c + e), max(d.caps[1], 6 * c + 2 * e), max(d.caps[2], 4 * c))
        self.maze_shape = (max(d.maze.rows for d in mazes), max(d.maze.cols for d in mazes))

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
        # the entity-list slots each level's reset fills: kind, whether it is the agent, whether it takes a design
        self.level_slots = [[dict(slot=e, kind=k, agent=a, designable=ds) for e, (k, a, ds) in enumerate(d.program.slots)]
                            if d.program is not None else None for d in defs]
        # the reset draws of each level's program (reset_draws=True): index, kind, n or lo / hi, label
        self.draw_specs = [[dict(spec) for spec in d.program.draws] if d.program is not None else None for d in defs]
        self.program, self.maze_template = (None, None) if table else (d0.program, d0.maze)
        self.autoreset = bool(autoreset)
        if self.device_reset:
            caps = [max(c) for c in zip(*(d.caps for d in defs))]
            # exact: K2's shared-memory triangle capacity scales with max_ents
            max_ents = max([2] + [d.num_placed for d in defs])
        else:
            caps = [int(1.25 * len(g)) + 4 for g in d0.geometry]
            # room for the definition instance's entity list (CollectHealth: 18 kits and the agent) and a carried
            # object outside it
            max_ents = max(8, len(d0.pe.entities) + 1)
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
            self.proto_table = self.program.proto_array()
            eng.set_protos(self.proto_table)
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
            self.proto_table = np.array(protos, PROTO_DTYPE)
            eng.set_protos(self.proto_table)
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
            self._info_views = {}
            for key, spec in self._device_info.items():
                if spec[0] == "counter":                   # CollectHealth: info["health"] (collecthealth.py:100)
                    self._info[key] = self._views()["counter"]
                elif spec[0] == "entity_pos":              # TMaze: info["goal_pos"] = self.box.pos (tmaze.py:89)
                    self._info_views[key] = (int(spec[1]), [self._views()[n] for n in ("ent_x", "ent_y", "ent_z")])
            self._obs_dict = dict(self._device_obs_extra)
            # what each mode records of every env's current episode (after a terminating step still of the one that
            # just ended: its level, seed, maze, start pose, draws, shortest path and loaded slot), and goal_dist now
            for m in _MODES:
                if getattr(self, m.flag):
                    self._info.update((key, self._views()[name]) for key, name in m.info)
        return self._torch

    # ------------------------------------------------------------------ run-time arrays
    def _views(self):
        """The batch's state arrays by name, in place and in their final shapes (_Views)."""
        return self._view_map

    def _write_pending(self, what, ids, arrays):
        """The part set_env_level / set_env_seed / set_env_maze / set_env_pose / set_env_draws / set_env_param / set_env_state share: check the env ids `ids` (1-D
        integers in [0, N)), then write each (array name or view, values) of `arrays` at those envs -- values one per id
        (a numpy array, or a CUDA tensor) or one for all -- an env listed more than once taking its last entry.  On the host build the write is
        numpy's; on the device it is torch ops on the current stream, without a sync."""
        if not np.issubdtype(ids.dtype, np.integer) or ids.ndim != 1:
            raise ValueError("%s takes a 1-D sequence of integer env ids" % what)
        if ids.size and (ids.min() < 0 or ids.max() >= self.num_envs):
            raise ValueError("env ids must lie in [0, %d)" % self.num_envs)
        if ids.size == 0:
            return
        last = ids.size - 1 - np.unique(ids[::-1], return_index=True)[1]    # an env listed twice: its last entry wins
        if self.engine.host_memory:
            for name, vals in arrays:
                self._target(name)[ids[last]] = vals[last] if np.ndim(vals) else vals
            return
        import torch
        to_dev = lambda a: torch.as_tensor(a).to(torch.device("cuda", self.device), non_blocking=True)
        idx = to_dev(ids[last].astype(np.int64))
        for name, vals in arrays:
            if torch.is_tensor(vals):
                vals = vals[to_dev(last)] if vals.dim() else vals
            elif np.ndim(vals):
                vals = to_dev(np.ascontiguousarray(vals[last]))
            self._target(name)[idx] = vals

    def _target(self, name):
        return self._views()[name] if isinstance(name, str) else name

    # ------------------------------------------------------------------ level changes (dynamic_levels=True)
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
        if not np.issubdtype(lv.dtype, np.integer):
            raise ValueError("set_env_level takes integer env ids and levels")
        if lv.min() < 0 or lv.max() >= len(self.level_ids):
            raise ValueError("levels must lie in [0, %d)" % len(self.level_ids))
        self._write_pending("set_env_level", ids, [("next_level", lv.astype(np.int32))])

    @property
    def env_level(self):
        """numpy int32 [N]: the level of each env.  With dynamic_levels it is a host copy of `level_tensor` and
        synchronises with the device (the current torch stream) to read it."""
        if not self.dynamic_levels:
            return self._env_level
        view = self.level_tensor
        return np.array(view) if isinstance(view, np.ndarray) else view.cpu().numpy()

    # ------------------------------------------------------------------ episode seeds (episode_seeds=True)
    @property
    def next_seed(self):
        """int64 [N] view of the seed each env's next reset starts from; write it in place (stream-ordered, no sync).
        A negative entry means none: the env continues its stream.  The reset that takes an entry clears it to -1."""
        return self._views()["next_seed"]

    @property
    def episode_seed(self):
        """int64 [N] view of the seed each env's current episode started from, -1 when it continued its stream."""
        return self._views()["episode_seed"]

    def set_env_seed(self, env_ids, seeds):
        """Start the listed envs' next episodes from `seeds` (one seed, or one per env), as `reset(seed=s)` would; envs
        in mid-episode finish it first.  An env listed more than once takes its last entry.  `seeds` given as a CUDA
        tensor are written as they are (a negative entry means none); host values must lie in [0, 2**63)."""
        self._views()["next_seed"]                   # a batch without the mode raises before any input check
        ids = np.atleast_1d(_host(env_ids))
        if not (hasattr(seeds, "is_cuda") and seeds.is_cuda):
            seeds = self._host_seeds(seeds.cpu().numpy() if hasattr(seeds, "cpu") else seeds, ids.shape)
        elif seeds.dim() and tuple(seeds.shape) != ids.shape:
            raise ValueError("set_env_seed: %d env ids but %d seeds" % (ids.size, seeds.numel()))
        else:
            seeds = seeds.long()
        self._write_pending("set_env_seed", ids, [("next_seed", seeds)])

    @staticmethod
    def _host_seeds(seeds, shape):
        """Host seeds (an int, or one per env) as int64 of `shape`, checked to lie in [0, 2**63)."""
        arr = np.asarray(seeds)
        if arr.dtype.kind not in "iu":
            arr = np.array([int(v) for v in np.asarray(seeds, object).reshape(-1)], object).reshape(np.shape(seeds))
        if arr.size and (arr.min() < 0 or arr.max() >= 2 ** 63):
            raise ValueError("episode seeds must lie in [0, 2**63)")
        arr = arr.astype(np.int64)
        if np.ndim(seeds) == 0:
            return np.broadcast_to(arr.reshape(()), shape)
        if arr.shape != tuple(shape):
            raise ValueError("%d env ids but %d seeds" % (int(np.prod(shape)), arr.size))
        return arr

    # ------------------------------------------------------------------ maze layouts (maze_layouts=True)
    @property
    def next_maze(self):
        """uint8 [N, rows, cols] view of the layout each env's next reset at a Maze level builds once `maze_pending` is
        set; write it in place (stream-ordered, no sync)."""
        return self._views()["next_maze"]

    @property
    def next_maze_cells(self):
        """int32 [N, 2] view of (goal cell, agent cell) of each pending layout: j * cols + i, or -1 for anywhere."""
        return self._views()["next_maze_cells"]

    @property
    def maze_pending(self):
        """uint8 [N] view: nonzero when next_maze[i] waits for env i's next reset at a Maze level, which clears it."""
        return self._views()["maze_pending"]

    @property
    def episode_maze(self):
        """uint8 [N, rows, cols] view of the layout of each env's running episode (zeros at levels that are not Mazes)."""
        return self._views()["episode_maze"]

    def set_env_maze(self, env_ids, layouts, goal_cell=-1, agent_cell=-1):
        """Build the listed envs' next mazes from `layouts` (one uint8 [rows, cols] layout, or one per env) with the
        goal box in `goal_cell` and the agent in `agent_cell` (one flat cell j * cols + i, or one per env; -1 for
        anywhere); envs in mid-episode finish it first.  An env listed more than once takes its last entry.  The input
        is checked on the host, then written with torch ops on the current stream, without a sync."""
        self._views()["next_maze"]                   # a batch without the mode raises before any input check
        ids = np.atleast_1d(_host(env_ids))
        lay = _host(layouts)
        if not (np.issubdtype(lay.dtype, np.integer) or lay.dtype == np.bool_):
            raise ValueError("maze layouts are integer arrays (uint8), got %s" % lay.dtype)
        if lay.shape == self.maze_shape:
            lay = np.broadcast_to(lay, (ids.size,) + self.maze_shape)
        if lay.shape != (ids.size,) + self.maze_shape:
            raise ValueError("maze layouts must have shape %s or %s, got %s" % (self.maze_shape, (ids.size,) + self.maze_shape,
                                                                              lay.shape))
        if lay.size and (lay.min() < 0 or lay.max() > 3):
            raise ValueError("a maze layout sets only bits 0 (+x wall open) and 1 (+z wall open)")
        n_cells = self.maze_shape[0] * self.maze_shape[1]
        cells = []
        for name, c in (("goal_cell", goal_cell), ("agent_cell", agent_cell)):
            c = _host(c)
            if not np.issubdtype(c.dtype, np.integer) or c.ndim > 1 or (c.ndim == 1 and c.shape != ids.shape):
                raise ValueError("%s is one integer or one per env id" % name)
            if c.size and (c.min() < -1 or c.max() >= n_cells):
                raise ValueError("%s entries must lie in [-1, %d)" % (name, n_cells))
            cells.append(np.broadcast_to(c, ids.shape))
        both = np.stack(cells, axis=1).astype(np.int32)
        self._write_pending("set_env_maze", ids, [("next_maze", lay.astype(np.uint8, copy=False)),
                                                  ("next_maze_cells", both), ("maze_pending", 1)])

    # ------------------------------------------------------------------ start poses (start_poses=True)
    @property
    def next_pose(self):
        """float64 [N, max_ents, 3] view of the designed (x, z, dir) of each entity-list slot at each env's next reset
        with `pose_pending` set; write it in place (stream-ordered, no sync).  A row applies when x and z are finite."""
        return self._views()["next_pose"]

    @property
    def next_agent_pose(self):
        """float64 [N, 3] view of the designed (x, z, dir) of the agent at each env's next reset with `pose_pending`
        set, at every level; it wins over the agent's slot row of `next_pose`."""
        return self._views()["next_agent_pose"]

    @property
    def pose_pending(self):
        """uint8 [N] view: nonzero when the designed rows wait for env i's next reset, which clears it."""
        return self._views()["pose_pending"]

    @property
    def episode_start(self):
        """float64 [N, 3] view of the agent's (x, z, dir) at the start of each env's running episode."""
        return self._views()["episode_start"]

    def set_env_pose(self, env_ids, slot, x, z, dir=None):
        """Start the listed envs' next episodes with entity-list slot `slot` (an int in [0, max_ents), or "agent") at
        (x, z) facing `dir` (None: the level's dir, or a uniform draw); envs in mid-episode finish it first.  Values are
        one for all or one per env; an env listed more than once takes its last entry.  Sets `pose_pending`; rows
        written earlier stay.  Host values are checked (x and z finite); CUDA tensors are written as they are.  The
        write is numpy's on the host build, torch ops on the current stream without a sync on the device."""
        self._views()["next_pose"]                   # a batch without the mode raises before any input check
        ids = np.atleast_1d(_host(env_ids))
        if isinstance(slot, str) and slot == "agent":
            target = self.next_agent_pose
        elif isinstance(slot, (int, np.integer)) and not isinstance(slot, bool) and 0 <= slot < self.engine.max_ents:
            target = self.next_pose[:, int(slot)]
        else:
            raise ValueError("slot must be \"agent\" or an int in [0, %d), got %r" % (self.engine.max_ents, slot))
        comps, on_device = [], False
        for name, v in (("x", x), ("z", z), ("dir", np.nan if dir is None else dir)):
            if hasattr(v, "is_cuda") and v.is_cuda:
                on_device = True
                got = tuple(v.shape)
            else:
                v = np.asarray(_host(v), np.float64)
                got = v.shape
                if name != "dir" and not np.isfinite(v).all():
                    raise ValueError("set_env_pose: %s must be finite" % name)
            if got not in ((), ids.shape):
                raise ValueError("set_env_pose: %s is one value or one per env id (%d), got shape %s" % (name, ids.size, got))
            comps.append(v)
        if on_device:
            torch = self._ensure_torch()
            dev = torch.device("cuda", self.device)
            rows = torch.stack([torch.as_tensor(c, dtype=torch.float64).to(dev, non_blocking=True).expand(ids.shape)
                                for c in comps], dim=1)
        else:
            rows = np.stack([np.broadcast_to(c, ids.shape) for c in comps], axis=1)
        self._write_pending("set_env_pose", ids, [(target, rows), ("pose_pending", 1)])

    # ------------------------------------------------------------------ reset draws (reset_draws=True)
    @property
    def next_draws(self):
        """float64 [N, D] view of the designed outcome of each reset draw at each env's next reset with `draws_pending`
        set; write it in place (stream-ordered, no sync).  A value applies when it lies in the draw's support."""
        return self._views()["next_draws"]

    @property
    def draws_pending(self):
        """uint8 [N] view: nonzero when the designed draws wait for env i's next reset, which clears it."""
        return self._views()["draws_pending"]

    @property
    def episode_draws(self):
        """float64 [N, D] view of the outcome of each reset draw of each env's running episode, NaN beyond its level's
        draw count."""
        return self._views()["episode_draws"]

    def set_env_draws(self, env_ids, index, values):
        """Design draw `index` (an int in [0, D); `draw_specs` numbers each level's draws) of the listed envs' next
        episodes: `values` is one value for all or one per env (NaN: draw as usual); envs in mid-episode finish it
        first.  An env listed more than once takes its last entry.  Sets `draws_pending`; rows written earlier stay.
        Host values are checked to be real numbers; CUDA tensors are written as they are.  The write is numpy's on the
        host build, torch ops on the current stream without a sync on the device."""
        view = self._views()["next_draws"]           # a batch without the mode raises before any input check
        D = view.shape[1]
        if isinstance(index, bool) or not isinstance(index, (int, np.integer)) or not 0 <= index < D:
            raise ValueError("index must be an int in [0, %d), got %r" % (D, index))
        ids = np.atleast_1d(_host(env_ids))
        if hasattr(values, "is_cuda") and values.is_cuda:
            torch = self._ensure_torch()
            vals = values.to(torch.float64)
            got = tuple(vals.shape)
        else:
            vals = np.asarray(_host(values))
            if not (np.issubdtype(vals.dtype, np.floating) or np.issubdtype(vals.dtype, np.integer)):
                raise ValueError("set_env_draws: values are real numbers, got %s" % vals.dtype)
            vals = vals.astype(np.float64)
            got = vals.shape
        if got not in ((), ids.shape):
            raise ValueError("set_env_draws: values are one value or one per env id (%d), got shape %s" % (ids.size, got))
        self._write_pending("set_env_draws", ids, [(view[:, int(index)], vals), ("draws_pending", 1)])

    # ------------------------------------------------------------------ env params (env_params=True)
    param_rows = ENV_PARAM_ROWS

    @property
    def next_params(self):
        """float64 [N, 22, 3] view of the (default, min, max) rows each env's next episode runs with `params_pending`
        set (NaN: the level's); write it in place (stream-ordered, no sync).  `param_rows` names the rows."""
        return self._views()["next_params"]

    @property
    def params_pending(self):
        """uint8 [N] view: nonzero when next_params[i] waits for env i's next reset, which clears it."""
        return self._views()["params_pending"]

    @property
    def episode_params(self):
        """float64 [N, 22, 3] view of the rows of each env's running episode, all NaN when it runs its level's params."""
        return self._views()["episode_params"]

    def set_env_param(self, env_ids, name, default=None, min=None, max=None):
        """Design param `name` (one of engine.LOWERED_PARAMS, a float param) of the listed envs' next episodes: `default`,
        `min` and `max` are each a value of the param's shape (() or (3,)), or one per env id ([n, *shape]), as
        floats, sequences, numpy arrays or CUDA tensors; None writes NaN, the level's.  The range applies when both
        min and max are finite.  Envs in mid-episode finish it first; an env listed more than once takes its last entry.
        Sets `params_pending`; the other rows written earlier stay.  Host values are checked as DomainParams.set checks
        them (shapes, min <= default <= max where given); tensor values are not checked.  The write is numpy's on the
        host build, torch ops on the current stream on the device; env ids given as a CUDA tensor are read back to the
        host first (the duplicate and range checks run there), which synchronises."""
        view = self._views()["next_params"]          # a batch without the mode raises before any input check
        if name not in LOWERED_PARAMS:
            raise KeyError("%r is not a param the engine reads; these are: %s" % (name, ", ".join(LOWERED_PARAMS)))
        for level, pe in enumerate(self.proto_envs):
            if pe.params.params[name].type != "float":
                raise TypeError("%r of level %d is a %s param; only float params can be set"
                                % (name, level, pe.params.params[name].type))
        ids = np.atleast_1d(_host(env_ids))
        rows = self.param_rows[name]
        shape = (3,) if isinstance(rows, slice) else ()
        vals, host = {}, {}
        for key, v in (("default", default), ("min", min), ("max", max)):
            if v is None:
                vals[key] = float("nan")
                continue
            if hasattr(v, "is_cuda") and v.is_cuda:
                t = v.to(self._ensure_torch().float64)
                got = tuple(t.shape)
            else:
                a = np.asarray(_host(v))
                if a.dtype == object:                # None entries of a sequence: the level's
                    try:
                        a = a.astype(np.float64)
                    except (TypeError, ValueError):
                        pass
                if not (np.issubdtype(a.dtype, np.floating) or np.issubdtype(a.dtype, np.integer)):
                    raise ValueError("set_env_param: %s of %r is real numbers, got %s" % (key, name, a.dtype))
                t = host[key] = a.astype(np.float64)
                got = t.shape
            if got not in (shape, ids.shape + shape):
                raise ValueError("%s of %r must have shape %s or %s, got %s" % (key, name, shape, ids.shape + shape, got))
            vals[key] = t if got != shape else (np.broadcast_to(t, ids.shape + shape) if isinstance(t, np.ndarray)
                                                else t.expand(ids.shape + shape))
        for a, b in (("min", "default"), ("default", "max"), ("min", "max")):
            if a in host and b in host:
                lo, hi = np.broadcast_arrays(host[a], host[b])
                if not np.all((hi >= lo) | np.isnan(lo) | np.isnan(hi)):
                    raise ValueError("%r: %s %s is above %s %s" % (name, a, host[a], b, host[b]))
        self._write_pending("set_env_param", ids, [(view[:, rows, k], vals[key])
                                                   for k, key in enumerate(("default", "min", "max"))]
                            + [("params_pending", 1)])

    def set_env_params(self, env_ids, params):
        """Design every param of `params` (a DomainParams) that the engine reads for the listed envs' next episodes, as
        `set_env_param` does; entries the engine does not read are ignored."""
        for name in LOWERED_PARAMS:
            if name in params.params:
                p = params.params[name]
                self.set_env_param(env_ids, name, p.default, p.min, p.max)

    def get_env_params(self, env):
        """The DomainParams env `env`'s running episode runs on (synchronises with the device): its level's params as
        they stand now (get_level_params), merged with its `episode_params` row."""
        env = int(env)
        if not 0 <= env < self.num_envs:
            raise ValueError("env must lie in [0, %d), got %d" % (self.num_envs, env))
        self._sync_level_writes()
        row = _host(self.episode_params[env]).copy()
        level = int(_host(self._views()["env_level"])[env]) if self.dynamic_levels else int(self._env_level[env])
        out = self.get_level_params(level)
        for name in LOWERED_PARAMS:
            p, r = out.params[name], row[self.param_rows[name]]
            r = r.reshape(-1, 3)
            d, lo, hi = (np.array(p.default, float).reshape(-1), np.array(p.min, float).reshape(-1),
                         np.array(p.max, float).reshape(-1))
            rng = np.isfinite(r[:, 1]) & np.isfinite(r[:, 2])
            d = np.where(np.isfinite(r[:, 0]), r[:, 0], d)
            lo, hi = np.where(rng, r[:, 1], lo), np.where(rng, r[:, 2], hi)
            vals = [v if len(v) == 3 else float(v[0]) for v in (d, lo, hi)]
            out.params[name] = DomainParams.DomainParam(vals[0], vals[1], vals[2], "float")
        return out

    # ------------------------------------------------------------------ state bank (state_bank=K)
    @property
    def next_state(self):
        """int32 [N] view of the slot each env's next reset loads, -1 for none; write it in place (stream-ordered, no
        sync).  The reset that takes an entry clears it to -1, loaded or not."""
        return self._views()["next_state"]

    @property
    def episode_state(self):
        """int32 [N] view of the slot each env's running episode was loaded from, -1 when it ran the level's program."""
        return self._views()["episode_state"]

    @property
    def bank_level(self):
        """int32 [K] view of the level of the state each slot holds, -1 for an empty slot (read-only)."""
        return self._views()["bank_level"]

    # ------------------------------------------------------------------ goal distance (goal_distance=True)
    @property
    def goal_dist(self):
        """float64 [N] view of each agent's geodesic distance to its goal in metres after the last step or reset
        (read-only): 0 near the goal, +inf when unreachable, NaN at levels without a goal rule."""
        return self._views()["goal_dist"]

    @property
    def expert_action(self):
        """int32 [N] view of the action along a shortest path to the goal (0 turn left, 1 turn right, 2 move forward),
        -1 where goal_dist is not finite (read-only)."""
        return self._views()["expert_action"]

    @property
    def episode_shortest(self):
        """float64 [N] view of goal_dist right after the reset that started each env's running episode (read-only)."""
        return self._views()["episode_shortest"]

    @property
    def goal_field(self):
        """uint16 [N, G] view of each env's distance field in units of 0.05 m, 0xFFFF for unreachable and blocked
        nodes; env i's grid is goal_field[i, :nz * nx].reshape(nz, nx) with grid_shape[level] (read-only)."""
        return self._views()["goal_field"]

    def entity_xz(self, slot):
        """float64 [N, 2]: the (x, z) floor position of entity-list slot `slot` of every env, read from the device
        state by torch ops without a sync (a numpy array on the host build).  `level_slots` names each level's agent
        slot (FourRooms: 1)."""
        x, z = self._views()["ent_x"][slot], self._views()["ent_z"][slot]
        return np.stack([x, z], 1) if isinstance(x, np.ndarray) else self._ensure_torch().stack([x, z], 1)

    def _bank_ids(self, what, env_ids, slots, lo):
        """(env ids, slots) of save_states / set_env_state: host values as 1-D int64 numpy arrays, checked (env ids in
        [0, N), slots in [lo, K)); a CUDA tensor stays on the device, unchecked."""
        self._views()["next_state"]                  # a batch without the bank raises before any input check
        out = []
        for name, v, bound in (("env ids", env_ids, (0, self.num_envs)), ("slots", slots, (lo, self.bank_slots))):
            if hasattr(v, "is_cuda") and v.is_cuda:
                if v.dim() > 1 or v.dtype.is_floating_point or v.dtype == self._ensure_torch().bool:
                    raise ValueError("%s: %s are a 1-D integer tensor" % (what, name))
                out.append(v)
                continue
            a = np.atleast_1d(_host(v))
            if a.ndim != 1 or not (np.issubdtype(a.dtype, np.integer) or a.size == 0):
                raise ValueError("%s: %s are integers, one or a 1-D sequence" % (what, name))
            if a.size and (a.min() < bound[0] or a.max() >= bound[1]):
                raise ValueError("%s: %s must lie in [%d, %d)" % (what, name, bound[0], bound[1]))
            out.append(a.astype(np.int64))
        return out

    def save_states(self, env_ids, slots):
        """Copy env env_ids[t] into slot slots[t] (ints, numpy arrays or CUDA tensors of one length).  A slot named more
        than once keeps its last entry.  Host values are checked; CUDA tensors are taken as they are, entries out of
        range skipped on the device.  The copy is enqueued on torch's current stream without a sync (on the host build
        of the kernels it runs in the call)."""
        ids, sl = self._bank_ids("save_states", env_ids, slots, 0)
        if ids.shape[0] != sl.shape[0]:
            raise ValueError("save_states: %d env ids but %d slots" % (ids.shape[0], sl.shape[0]))
        if ids.shape[0] == 0:
            return
        if self.engine.host_memory:
            self.engine.save_states(ids.astype(np.int32), sl.astype(np.int32))
            return
        torch = self._ensure_torch()
        dev = torch.device("cuda", self.device)
        ids, sl = (torch.as_tensor(a).to(dev, torch.int32, non_blocking=True).contiguous() for a in (ids, sl))
        self.engine.save_states(ids, sl, stream=_torch_stream(torch, self.device))

    def set_env_state(self, env_ids, slots):
        """Start the listed envs' next episodes from `slots` (one slot, or one per env; -1 cancels a pending entry);
        envs in mid-episode finish it first.  An env listed more than once takes its last entry.  Host slots must lie
        in [-1, K); CUDA tensors are written as they are.  The write is numpy's on the host build, torch ops on the
        current stream without a sync on the device."""
        ids, sl = self._bank_ids("set_env_state", env_ids, slots, -1)
        if hasattr(ids, "is_cuda"):
            raise ValueError("set_env_state takes host env ids (write next_state in place for device ones)")
        if not hasattr(sl, "is_cuda"):
            if np.ndim(slots) == 0:
                sl = np.broadcast_to(sl, ids.shape)
            if sl.shape != ids.shape:
                raise ValueError("set_env_state: %d env ids but %d slots" % (ids.size, sl.size))
            sl = sl.astype(np.int32)
        elif sl.dim() and tuple(sl.shape) != ids.shape:
            raise ValueError("set_env_state: %d env ids but %d slots" % (ids.size, sl.numel()))
        else:
            sl = sl.to(self._ensure_torch().int32)
        self._write_pending("set_env_state", ids, [("next_state", sl)])

    # ------------------------------------------------------------------ level params at run time
    def set_level_param(self, level, name, default=None, min=None, max=None):
        """Change one DomainParams entry of level `level` while the batch runs (automatic domain randomisation).
        `name` is one of the twelve params the engine reads (engine.LOWERED_PARAMS) and must be a float param.  As
        with DomainParams.set, `min` and `max` default to `default`.  With `default` None the level keeps its default
        and `min` and `max` set the range (both or neither).  Values are floats, sequences, numpy arrays or CUDA
        tensors, of the param's shape (() or (3,)).
        The write is a few torch ops on the current stream, with no host sync.  The next `step` of every env at that
        level draws forward_step / forward_drift / turn_step from the new range, mid-episode included; everything
        else applies from each env's next reset, `max_forward_step` too (it follows forward_step's max).  The range
        is stored as min and max - min, computed in float64 as numpy's uniform() forms it.  Host values are checked
        as DomainParams.set checks them (shapes, min <= default <= max); tensor values are not checked."""
        if name not in LOWERED_PARAMS:
            raise KeyError("%r is not a param the engine reads; these are: %s" % (name, ", ".join(LOWERED_PARAMS)))
        n_levels = len(self.level_ids)
        if isinstance(level, bool) or not (isinstance(level, (int, np.integer)) and 0 <= int(level) < n_levels):
            raise ValueError("level must be an int in [0, %d), got %r" % (n_levels, level))
        level = int(level)
        view = self._views()["level_params"]
        p = self.proto_envs[level].params.params[name]
        if p.type != "float":
            raise TypeError("%r of level %d is a %s param; only float params can be set" % (name, level, p.type))
        if default is not None:
            min, max = default if min is None else min, default if max is None else max
        elif (min is None) != (max is None):
            raise ValueError("%r: without a default, give both min and max (or neither)" % name)
        given = {key: v for key, v in (("default", default), ("min", min), ("max", max)) if v is not None}
        shape = np.shape(p.default)
        for key, v in given.items():
            got = tuple(v.shape) if hasattr(v, "shape") else np.shape(v)
            if got != shape:
                raise ValueError("%s of %r must have shape %s, got %s" % (key, name, shape, got))
        host = {key: np.asarray(v, np.float64) for key, v in given.items() if not hasattr(v, "is_cuda")}
        for a, b in (("min", "default"), ("default", "max"), ("min", "max")):
            if a in host and b in host and not np.all(host[b] >= host[a]):
                raise ValueError("%r: %s %s is above %s %s" % (name, a, host[a], b, host[b]))
        if not given:
            return
        c, k = PARAMS_COLUMN[name], int(np.prod(shape, dtype=int))
        cols = {"default": slice(c, c + k), "min": slice(c + k, c + 2 * k)}
        if isinstance(view, np.ndarray):
            vals = {key: np.asarray(v.cpu() if hasattr(v, "cpu") else v, np.float64).reshape(k)
                    for key, v in given.items()}
            sub = np.subtract
        else:
            torch = self._ensure_torch()
            vals = {key: torch.as_tensor(v, dtype=torch.float64).to(view.device, non_blocking=True).reshape(k)
                    for key, v in given.items()}
            sub = torch.sub
            self._params_written = True
        for key in ("default", "min"):
            if key in vals:
                view[level, cols[key]] = vals[key]
        if "max" in vals:
            view[level, c + 2 * k:c + 3 * k] = sub(vals["max"], vals["min"])
            if name == "forward_step":
                view[level, PARAMS_COLUMN["max_forward_step"]] = vals["max"].reshape(())

    def set_level_params(self, level, params):
        """Write every param of `params` (a DomainParams) that the engine reads into level `level`, as
        `set_level_param` does; entries the engine does not read (bot_radius, tex_rand, ...) are ignored, as at
        construction."""
        for name in LOWERED_PARAMS:
            if name in params.params:
                p = params.params[name]
                self.set_level_param(level, name, p.default, p.min, p.max)

    def get_level_params(self, level):
        """Level `level`'s params as the device has them now, as a DomainParams (synchronises with the device).  The
        table holds min and max - min, so `max` is read back as min + (max - min), except forward_step's, which is
        max_forward_step.  The entries the engine does not read are the level's construction values."""
        view = self._views()["level_params"]
        row = np.array(view[level] if isinstance(view, np.ndarray) else view[level].cpu().numpy())
        out = DomainParams()
        out.params = dict(self.proto_envs[level].params.params)
        for name in LOWERED_PARAMS:
            c = PARAMS_COLUMN[name]
            k = int(np.prod(np.shape(out.params[name].default), dtype=int))
            lo = row[c + k:c + 2 * k]
            hi = row[PARAMS_COLUMN["max_forward_step"]:][:1] if name == "forward_step" else lo + row[c + 2 * k:c + 3 * k]
            vals = [row[c:c + k], lo, hi]
            vals = [np.array(v) if k == 3 else float(v[0]) for v in vals]
            out.params[name] = DomainParams.DomainParam(vals[0], vals[1], vals[2], "float")
        return out

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
        of per-env seeds, or None to continue each env's stream.  Returns (obs, info).
        With `episode_seeds=True`, `seed` may also be a CUDA int64 tensor (one seed per reset env): the seeds are
        queued in `next_seed` and the reset builds the streams on the device, without a sync.  Host seeds in
        [0, 2**63) go the same way, so that `episode_seed` records them; the streams are the same either way."""
        ids = np.arange(self.num_envs, dtype=np.int32) if env_ids is None else np.asarray(env_ids, np.int32)
        if self.episode_seeds and hasattr(seed, "is_cuda") and seed.is_cuda:
            if tuple(seed.shape) != ids.shape:
                raise ValueError("reset: %d envs but seeds of shape %s" % (ids.size, tuple(seed.shape)))
            self.set_env_seed(ids, seed)
            self.engine.reset(None if env_ids is None else ids, stream=self._level_stream())
            self._seeded = True
            return self._wrap(self.render()), {}
        if seed is not None:
            seeds = [int(seed) + int(i) for i in ids] if np.isscalar(seed) else [int(s) for s in seed]
            assert len(seeds) == len(ids)
        else:
            seeds = None
            if not self._seeded:
                seeds = [int(s) for s in np.random.SeedSequence().generate_state(len(ids))]
        if self.device_reset:
            if seeds is not None and self.episode_seeds and all(0 <= s < 2 ** 63 for s in seeds):
                self.set_env_seed(ids, seeds)
            elif seeds is not None:
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

    def _torch_writes(self):
        """True when torch work may write arrays the kernels read: next_level / level_weights (level changes on),
        next_seed (episode seeds on), the pending maze layouts (maze layouts on), the designed start poses (start poses
        on), the designed draws (reset draws on), the designed params (env params on), the pending slots (state bank on)
        or the params table (once set_level_param has written it)."""
        return ((self.dynamic_levels or self.episode_seeds or self.maze_layouts or self.start_poses
                 or self.reset_draws or self.env_params or self.state_bank or self._params_written)
                and not self.engine.host_memory)

    def _level_stream(self):
        """Stream for a call whose steps and resets read next_level / level_weights or the params table: when torch
        writes them, torch's current stream, so that the kernels run behind the torch work that wrote those arrays
        (set_env_level, set_level_weights, set_level_param, in-place writes); otherwise None, the handle's own stream.
        Calls with host outputs still return finished."""
        if self._torch_writes():
            return _torch_stream(self._ensure_torch(), self.device)
        return None

    def _sync_level_writes(self):
        """Finish torch writes to next_level / level_weights / the params table before the handle's own stream reads
        or replaces them."""
        if self._torch_writes():
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

    def visible_ents(self, out=None, poses=None):
        """uint32 [N]: bit e set iff entity-list slot e of that env passes the reference's occlusion query
        (get_visible_ents, miniworld.py:1238-1333).  With `poses` (float64 [N, 3] or [N, 7] rows as `render_views`
        takes them, a CUDA tensor or numpy array) the query runs from each env's designed camera as `render_views`
        defines it; a row that `render_views` skips leaves that env's entry of `out` as it is.  The reference's
        get_visible_ents always renders into obs_fb, so the query uses a 7-column row's camera attributes but the
        batch's own frame size and sample count."""
        if poses is not None:
            poses = self._view_rows("visible_ents", poses, single=True)
        if out is None:
            if self.engine.host_memory:
                out = np.zeros(self.num_envs, np.uint32)
            else:
                torch = self._ensure_torch()
                out = torch.zeros(self.num_envs, dtype=torch.int32, device=torch.device("cuda", self.device))
        stream = None if (self.engine.host_memory or poses is None) else _torch_stream(self._ensure_torch(), self.device)
        self.engine.visible_ents(out, stream=stream, poses=poses, row_width=3 if poses is None else poses.shape[-1])
        return out

    def _view_rows(self, what, poses, single=False):
        """Checked pose rows: a contiguous float64 CUDA tensor or numpy array [V, N, 3|7] (or [N, 3|7])."""
        if hasattr(poses, "is_cuda"):
            if poses.dtype != self._ensure_torch().float64:
                raise ValueError("%s: poses must be float64, not %s" % (what, poses.dtype))
            if not poses.is_cuda and not self.engine.host_memory:
                poses = poses.numpy()
            elif not poses.is_contiguous():
                poses = poses.contiguous()
        else:
            if np.asarray(poses).dtype != np.float64:
                raise ValueError("%s: poses must be float64, not %s" % (what, np.asarray(poses).dtype))
            poses = np.ascontiguousarray(poses)
        shape = tuple(poses.shape)
        ok = len(shape) == (2 if single else len(shape)) and len(shape) in (2, 3) and shape[-2] == self.num_envs and \
            shape[-1] in (3, 7)
        if not ok or (len(shape) == 3 and shape[0] <= 0):
            raise ValueError("%s: poses must have shape %s, not %s" % (
                what, "[N, 3] or [N, 7]" if single else "[V, N, 3|7] or [N, 3|7] with N = %d" % self.num_envs, shape))
        return poses

    def render_views(self, poses, render_agent=False, out=None, depth=None, size=None, samples=None):
        """Render every env from designed cameras (mwb_render_views_at).  `poses`: float64 [V, N, 3|7] or [N, 3|7]
        rows, a CUDA tensor or numpy array.  The view of env i from (x, z, dir) is what the reference's
        render_obs() / render_depth() return after agent.pos = (x, agent.pos[1], z), agent.dir = dir, nothing else
        changed (same entities, textures, light and the episode's camera parameters).  A 7-column row
        (x, z, dir, cam_height, cam_fwd_disp, cam_pitch, cam_fov_y) also sets those camera attributes; NaN in columns
        3-6 keeps the running episode's value, so an all-NaN 7-column row renders what its 3-column row does.
        `render_agent=True` also draws the agent's marker triangle at its real pose: a third-person view.
        A row is skipped when x, z or dir is not finite or |dir| >= 105414350 (beyond the range the glibc-exact sin /
        cos are validated for), and a 7-column row also when an intrinsic column is +-inf, a given cam_fov_y lies
        outside (0, 180) or a given |cam_pitch| >= 90.  A skipped row's frame (and depth) in that view is left as it is
        in `out` / `depth`.  No env state changes.
        `size` = (W, H) and `samples` (1, 4, 8 or 16) render as the reference does into FrameBuffer(W, H, samples);
        they default to the batch's observation size and sample count.
        Returns frames [V, N, *frame] (or [N, *frame]) in the batch's observation layout at that size -- `out` filled
        in place or a fresh zero tensor -- and, when `depth` is True or an array / tensor float32 [V, N, H, W, 1] (or
        [N, H, W, 1]) to fill, (frames, depth).  With CUDA tensors throughout the call runs on torch's current stream
        without a host sync."""
        poses = self._view_rows("render_views", poses)
        one = poses.ndim == 2 if isinstance(poses, np.ndarray) else poses.dim() == 2
        V = 1 if one else int(poses.shape[0])
        lead = () if one else (V,)
        if size is None:
            W, H = self.obs_width, self.obs_height
        else:
            if len(size) != 2 or not all(isinstance(v, (int, np.integer)) and not isinstance(v, bool) and v > 0
                                         for v in size):
                raise ValueError("render_views: size must be (width, height), two positive ints, not %r" % (size,))
            W, H = int(size[0]), int(size[1])
        if samples is None:
            samples = self.engine.cfg.msaa_samples
        elif isinstance(samples, bool) or samples not in (1, 4, 8, 16):
            raise ValueError("render_views: samples must be 1, 4, 8 or 16, not %r" % (samples,))
        N = self.num_envs
        obs_shape = {"hwc": (N, H, W, 3), "cwh": (N, 3, W, H), "grey": (N, H, W, 1)}[self.obs_format]
        host = self.engine.host_memory
        if out is None or depth is True:
            torch = None if host else self._ensure_torch()
            dev = None if host else torch.device("cuda", self.device)
            zeros = (lambda shape, dt: np.zeros(shape, dt)) if host else \
                (lambda shape, dt: torch.zeros(shape, dtype={np.uint8: torch.uint8, np.float64: torch.float64,
                                                             np.float32: torch.float32}[dt], device=dev))
            if out is None:
                out = zeros(lead + obs_shape, self.obs_dtype)
            if depth is True:
                depth = zeros(lead + (self.num_envs, H, W, 1), np.float32)
        for name, arr, shape, dt in (("out", out, lead + obs_shape, np.dtype(self.obs_dtype)),
                                     ("depth", depth, lead + (self.num_envs, H, W, 1), np.dtype(np.float32))):
            if arr is None or arr is False:
                continue
            adt = arr.dtype if isinstance(arr, np.ndarray) else np.dtype(str(arr.dtype).replace("torch.", ""))
            contig = arr.flags["C_CONTIGUOUS"] if isinstance(arr, np.ndarray) else arr.is_contiguous()
            if tuple(arr.shape) != shape or adt != dt or not contig:
                raise ValueError("render_views: %s must be a contiguous %s array of shape %s, not %s %s" % (
                    name, dt.name, shape, adt.name, tuple(arr.shape)))
        if depth is False:
            depth = None
        stream = None if host else _torch_stream(self._ensure_torch(), self.device)
        self.engine.render_views(poses, V, obs=out, depth=depth, render_agent=render_agent, stream=stream,
                                 row_width=poses.shape[-1], size=(W, H), samples=int(samples))
        return out if depth is None else (out, depth)

    # ------------------------------------------------------------------ state views
    def get_state(self, **kw):
        return self.engine.get_state(**kw)

    def np_random(self, i):
        """numpy Generator positioned where env i's device stream currently is."""
        return generator_from_state(self.engine.get_state(rng=True)["rng"][i])

    def close(self):
        self.engine.close()
