"""Rooms, procedural world generation and the single-environment drop-in class.

Host-side mirror of the reference's `miniworld/miniworld.py` public surface
(Room :122-434, MiniWorldEnv :437-1443): the level-building helpers (`add_rect_room`,
`add_room`, `connect_rooms`, `place_entity`, `place_agent`, `intersect`, `near`,
`_reward`, `_gen_world`), `reset`, `step`, `render_obs`, `render_depth` keep their names,
argument meaning and RNG call order, so the level definitions under `envs/` (and the
reference's own `miniworld/envs/*.py`) run on it unchanged.

What differs: nothing here talks to OpenGL.  `reset()` builds the world with numpy on the
host (exactly the reference's arithmetic, so poses / wall segments are bit-identical),
lowers it to the flat SoA of `pack.py`, and every `step()` / `render_obs()` executes on the
GPU through the C ABI in `engine.py` (kernels: csrc/physics.cuh, csrc/raster.cuh).  There
is no CPU physics or CPU renderer in this package: without the CUDA library the env can
only be constructed with `device=None`, which generates worlds but cannot step or render.

The many-environment fast path (device-side resets, lowered level rules) is
`batched.BatchedMiniWorld`; this class is the N = 1 compatibility view.
"""
import math
from enum import IntEnum

import numpy as np

from ._gym import gym, spaces
from .assets import Texture
from .entity import Agent, Entity
from .math import Y_VEC, intersect_circle_segs
from .params import DEFAULT_PARAMS, overlay_params

DEFAULT_WALL_HEIGHT = 2.74
TEX_DENSITY = 512   # texels per metre


def gen_texcs_wall(tex, min_x, min_y, width, height):
    """float32 texcoords of one wall quad, corner order (lo,lo) (lo,hi) (hi,hi) (hi,lo)."""
    xc, yc = TEX_DENSITY / tex.width, TEX_DENSITY / tex.height
    u0, u1 = min_x * xc, (min_x + width) * xc
    v0, v1 = min_y * yc, (min_y + height) * yc
    return np.array([[u0, v0], [u0, v1], [u1, v1], [u1, v0]], dtype=np.float32)


def gen_texcs_floor(tex, poss):
    """Floor / ceiling texcoords: world (x, z) scaled by texel density."""
    scale = np.array([TEX_DENSITY / tex.width, TEX_DENSITY / tex.height], dtype=float)
    return np.stack([poss[:, 0], poss[:, 2]], axis=1) * scale


class Room:
    """Convex room given by a counter-clockwise (seen from above) xz outline."""

    def __init__(self, outline, wall_height=DEFAULT_WALL_HEIGHT, floor_tex="floor_tiles_bw",
                 wall_tex="concrete", ceil_tex="concrete_tiles", no_ceiling=False):
        assert outline.ndim == 2 and outline.shape[1] == 2 and outline.shape[0] >= 3
        outline = np.insert(outline, 1, 0, axis=1)          # add y = 0
        self.num_walls = outline.shape[0]
        self.outline = outline
        xs, zs = outline[:, 0], outline[:, 2]
        self.min_x, self.max_x = xs.min(), xs.max()
        self.min_z, self.max_z = zs.min(), zs.max()
        self.mid_x = (self.max_x + self.min_x) / 2
        self.mid_z = (self.max_z + self.min_z) / 2
        self.area = (self.max_x - self.min_x) * (self.max_z - self.min_z)

        nxt = np.concatenate([outline[1:], np.expand_dims(outline[0], axis=0)], axis=0)
        dirs = nxt - outline
        self.edge_dirs = (dirs.T / np.linalg.norm(dirs, axis=1)).T
        norms = -np.cross(self.edge_dirs, Y_VEC)
        self.edge_norms = (norms.T / np.linalg.norm(norms, axis=1)).T

        self.wall_height = wall_height
        self.no_ceiling = no_ceiling
        self.wall_tex_name, self.floor_tex_name, self.ceil_tex_name = wall_tex, floor_tex, ceil_tex
        self.portals = [[] for _ in range(self.num_walls)]
        self.neighbors = []

    def add_portal(self, edge, start_pos=None, end_pos=None, min_x=None, max_x=None,
                   min_z=None, max_z=None, min_y=0, max_y=None):
        """Cut an opening into wall `edge`; extents along the wall, or via x / z ranges."""
        if max_y is None:
            max_y = self.wall_height
        assert edge <= self.num_walls and max_y > min_y
        p0 = self.outline[edge]
        p1 = self.outline[(edge + 1) % self.num_walls]
        e_len = np.linalg.norm(p1 - p0)
        e_dir = (p1 - p0) / e_len
        x0, _, z0 = p0
        x1, _, z1 = p1
        dx, _, dz = e_dir

        def span(lo, hi, origin, d):
            m0, m1 = (lo - origin) / d, (hi - origin) / d
            return (m1, m0) if m1 < m0 else (m0, m1)

        if min_x is not None:
            assert min_z is None and max_z is None and start_pos is None and end_pos is None
            assert x0 != x1
            start_pos, end_pos = span(min_x, max_x, x0, dx)
        elif min_z is not None:
            assert min_x is None and max_x is None and start_pos is None and end_pos is None
            assert z0 != z1
            start_pos, end_pos = span(min_z, max_z, z0, dz)
        else:
            assert min_x is None and max_x is None and min_z is None and max_z is None
        assert end_pos > start_pos
        assert start_pos >= 0 and end_pos <= e_len, "portal outside of wall extents"
        self.portals[edge].append({"start_pos": start_pos, "end_pos": end_pos, "min_y": min_y, "max_y": max_y})
        self.portals[edge].sort(key=lambda e: e["start_pos"])
        return start_pos, end_pos

    def point_inside(self, p):
        ap = p - self.outline
        return np.all(np.greater(np.sum(self.edge_norms * ap, axis=1), 0))

    def _gen_static_data(self, params, rng):
        """Wall quads / collision segments / texcoords for this room (reference :286-399)."""
        self.wall_tex = Texture.get(self.wall_tex_name, rng)
        self.floor_tex = Texture.get(self.floor_tex_name, rng)
        self.ceil_tex = Texture.get(self.ceil_tex_name, rng)

        self.floor_verts = self.outline
        self.floor_texcs = gen_texcs_floor(self.floor_tex, self.floor_verts)
        self.ceil_verts = np.flip(self.outline, axis=0) + self.wall_height * Y_VEC
        self.ceil_texcs = gen_texcs_floor(self.ceil_tex, self.ceil_verts)

        verts, norms, texcs, segs, uvm = [], [], [], [], []

        def emit(edge_p0, side_vec, seg_start, seg_end, min_y, max_y):
            if seg_end == seg_start or min_y == max_y:
                return
            s_p0 = edge_p0 + seg_start * side_vec
            s_p1 = edge_p0 + seg_end * side_vec
            if min_y == 0:                       # reaches the floor -> collidable
                segs.append(np.array([s_p1, s_p0]))
            verts.extend([s_p0 + min_y * Y_VEC, s_p0 + max_y * Y_VEC,
                          s_p1 + max_y * Y_VEC, s_p1 + min_y * Y_VEC])
            n = np.cross(s_p1 - s_p0, Y_VEC)
            n = -n / np.linalg.norm(n)
            norms.extend([n] * 4)
            w, h = seg_end - seg_start, max_y - min_y
            texcs.append(gen_texcs_wall(self.wall_tex, seg_start, min_y, w, h))
            # texel-density independent texcoords in metres (engine applies 512 / tex size)
            uvm.append(np.array([[seg_start, min_y], [seg_start, min_y + h],
                                 [seg_start + w, min_y + h], [seg_start + w, min_y]], dtype=float))

        for wi in range(self.num_walls):
            p0 = self.outline[wi, :]
            p1 = self.outline[(wi + 1) % self.num_walls, :]
            width = np.linalg.norm(p1 - p0)
            side = (p1 - p0) / width
            holes = self.portals[wi]
            emit(p0, side, 0, holes[0]["start_pos"] if holes else width, 0, self.wall_height)
            for hi, hole in enumerate(holes):
                a, b = hole["start_pos"], hole["end_pos"]
                emit(p0, side, a, b, 0, hole["min_y"])                      # below the opening
                emit(p0, side, a, b, hole["max_y"], self.wall_height)       # above it
                nxt = holes[hi + 1]["start_pos"] if hi < len(holes) - 1 else width
                emit(p0, side, b, nxt, 0, self.wall_height)                 # up to the next one

        self.wall_verts = np.array(verts)
        self.wall_norms = np.array(norms)
        self.wall_segs = np.array(segs) if segs else np.array([]).reshape(0, 2, 3)
        self.wall_texcs = np.concatenate(texcs) if texcs else np.array([]).reshape(0, 2)
        self.wall_uvm = np.concatenate(uvm) if uvm else np.zeros((0, 2))


class _DesignedDraws:
    """`np_random` while `_gen_world()` runs with designed reset draws (reset(options={"draws": {d: v}})): the draws the
    level makes itself -- choice(n), integers(low, high) and uniform(lo, hi) of one value, numbered 0, 1, ... in call
    order -- are made from the stream as usual, then draw d's result is replaced by design[d] when that lies in the
    draw's support (an integer in [low, high); a finite value in [lo, hi]).  `drawn` records every outcome.  Placement,
    texture and carve draws go to the stream itself (MiniWorldEnv._stream)."""

    def __init__(self, stream, design):
        self.stream, self.design, self.drawn = stream, design, []

    def __getattr__(self, name):
        return getattr(self.stream, name)

    def _take(self, v, ok):
        x = self.design.get(len(self.drawn))
        x = float(x) if x is not None else math.nan
        if ok(x):
            v = type(v)(x)
        self.drawn.append(float(v))
        return v

    def _integer(self, v, low, high):
        return self._take(v, lambda x: low <= x < high and x == math.floor(x))

    def choice(self, a, *args, **kw):
        v = self.stream.choice(a, *args, **kw)
        return self._integer(v, 0, int(a)) if isinstance(a, (int, np.integer)) and not args and not kw else v

    def integers(self, low, high=None, *args, **kw):
        v = self.stream.integers(low, high, *args, **kw)
        lo, hi = (0, low) if high is None else (low, high)
        return self._integer(v, lo, hi) if np.ndim(v) == 0 else v

    def uniform(self, low=0.0, high=1.0, *args, **kw):
        v = self.stream.uniform(low, high, *args, **kw)
        if np.ndim(v) or np.ndim(low) or np.ndim(high):
            return v
        return self._take(v, lambda x: math.isfinite(x) and low <= x <= high)


class MiniWorldEnv(gym.Env):
    """Single-environment MiniWorld with the reference's Gymnasium API, executed on the GPU."""

    metadata = {"render_modes": ["human", "rgb_array"], "render_fps": 30}

    class Actions(IntEnum):
        turn_left = 0
        turn_right = 1
        move_forward = 2
        move_back = 3
        pickup = 4
        drop = 5
        toggle = 6
        done = 7

    def __init__(self, max_episode_steps=1500, obs_width=80, obs_height=60, window_width=800,
                 window_height=600, params=DEFAULT_PARAMS, domain_rand=False, render_mode=None,
                 view="agent", device="cuda", msaa_samples=8):
        self.actions = MiniWorldEnv.Actions
        self.action_space = spaces.Discrete(len(self.actions))
        self.observation_space = spaces.Box(low=0, high=255, shape=(obs_height, obs_width, 3), dtype=np.uint8)
        self.reward_range = (-math.inf, math.inf)
        self.max_episode_steps = max_episode_steps
        self.params = params
        self.domain_rand = domain_rand
        self.render_mode = render_mode
        assert view in ["agent", "top"]
        self.view = view
        self.obs_width, self.obs_height = obs_width, obs_height
        self.window_width, self.window_height = window_width, window_height
        self.msaa_samples = msaa_samples
        self.vis_samples = 16 if msaa_samples == 8 else msaa_samples     # obs_fb 8 / vis_fb 16 like the reference
        self.device = device
        self._engine = None
        self._vis_engine = None
        self._view_engines = {}         # render_view at another (width, height, samples): one engine each
        self.reset()

    # ------------------------------------------------------------------ episode control

    def reset(self, *, seed=None, options=None):
        """New episode: regenerate the world (host), push it to the engine, render.  `options` may hold designed start
        poses: "poses" {slot: (x, z, dir)} for the place_entity calls that fill those entity-list slots and
        "agent_pose" (x, z, dir) for place_agent (see place_entity); Maze levels also read a designed layout.  "draws"
        {d: v} designs the level's reset draws, the choice / integers / uniform calls _gen_world() makes itself, numbered
        0, 1, ... in call order: each is made as usual, then replaced by v when v lies in its support (_DesignedDraws);
        `episode_draws` then lists every outcome.  Placement and texture draws are not reset draws.  "params"
        {name: (default, min, max)} runs the episode on a copy of the level's params overlaid element by element as
        BatchedMiniWorld(env_params=True) overlays them: a finite default replaces the level's, a finite (min, max)
        pair its range; None or NaN entries keep the level's.  The next reset without the option runs on the level's
        params again."""
        super().reset(seed=seed)
        overlay = getattr(self, "_params_overlay", None)
        if overlay is not None and self.params is overlay[1]:
            self.params = overlay[0]            # the level's params again
        self._params_overlay = None
        if options and "params" in options:
            self._params_overlay = (self.params, overlay_params(self.params, options["params"]))
            self.params = self._params_overlay[1]
        self.step_count = 0
        self.agent = Agent()
        self.entities = []
        self.rooms = []
        self.wall_segs = []
        self.reset_options = options        # what the level's _gen_world may read (Maze: a designed layout)
        self._goal_nav = None               # goal_distance()'s field of this episode, built on first use
        self._start_design = options if options and ("poses" in options or "agent_pose" in options) else None
        if options and "draws" in options:
            self._np_random = _DesignedDraws(self.np_random, dict(options["draws"]))
            try:
                self._gen_world()
            finally:
                self.episode_draws = self._np_random.drawn
                self._np_random = self._np_random.stream
        else:
            self._gen_world()
        self._start_design = None           # placements after the reset (CollectHealth's respawns) run as written

        rand = self.np_random if self.domain_rand else None
        self.params.sample_many(rand, self, ["sky_color", "light_pos", "light_color", "light_ambient"])
        self.max_forward_step = self.params.get_max("forward_step")
        for ent in self.entities:
            ent.randomize(self.params, rand)

        self.min_x = min(r.min_x for r in self.rooms)
        self.max_x = max(r.max_x for r in self.rooms)
        self.min_z = min(r.min_z for r in self.rooms)
        self.max_z = max(r.max_z for r in self.rooms)
        if len(self.wall_segs) == 0:
            self._gen_static_data()

        self._world_dirty = True
        obs = self.render_obs() if self.device is not None else None
        return obs, {}

    def step(self, action):
        """One action: physics on the GPU (csrc/physics.cuh), then render (csrc/raster.cuh)."""
        eng = self._require_engine()
        rand = self.np_random if self.domain_rand else None
        fwd_step = self.params.sample(rand, "forward_step")
        fwd_drift = self.params.sample(rand, "forward_drift")
        turn_step = self.params.sample(rand, "turn_step")
        self._push_world()
        obs = eng.step_single(int(action), float(fwd_step), float(fwd_drift), float(turn_step))
        self._pull_state()
        if self.step_count >= self.max_episode_steps:
            return obs, 0, False, True, {}
        return obs, 0, False, False, {}

    # ------------------------------------------------------------------ level building

    def add_rect_room(self, min_x, max_x, min_z, max_z, **kwargs):
        outline = np.array([[max_x, max_z], [max_x, min_z], [min_x, min_z], [min_x, max_z]])
        return self.add_room(outline=outline, **kwargs)

    def add_room(self, **kwargs):
        assert len(self.wall_segs) == 0, "cannot add rooms after static data is generated"
        room = Room(**kwargs)
        self.rooms.append(room)
        return room

    def connect_rooms(self, room_a, room_b, min_x=None, max_x=None, min_z=None, max_z=None, max_y=None):
        """Open facing walls of two rooms; insert a connector room when they do not touch."""
        pair = None
        for ia in range(room_a.num_walls):
            na = room_a.edge_norms[ia]
            for ib in range(room_b.num_walls):
                if np.dot(na, room_b.edge_norms[ib]) > -0.9:        # not facing each other
                    continue
                if np.dot(na, room_b.outline[ib] - room_a.outline[ia]) > 0.05:   # not touching
                    continue
                pair = (ia, ib)
                break
            if pair:
                break
        assert pair is not None, "matching edges not found in connect_rooms"
        ia, ib = pair
        kw = dict(min_x=min_x, max_x=max_x, min_z=min_z, max_z=max_z, max_y=max_y)
        start_a, end_a = room_a.add_portal(edge=ia, **kw)
        start_b, end_b = room_b.add_portal(edge=ib, **kw)
        a = room_a.outline[ia] + room_a.edge_dirs[ia] * start_a
        b = room_a.outline[ia] + room_a.edge_dirs[ia] * end_a
        c = room_b.outline[ib] + room_b.edge_dirs[ib] * start_b
        d = room_b.outline[ib] + room_b.edge_dirs[ib] * end_b
        if np.linalg.norm(a - d) < 0.001:
            return
        len_a, len_b = np.linalg.norm(b - a), np.linalg.norm(d - c)
        outline = np.stack([c, b, a, d])
        outline = np.stack([outline[:, 0], outline[:, 2]], axis=1)
        max_y = max_y if max_y is not None else room_a.wall_height
        link = Room(outline, wall_height=max_y, wall_tex=room_a.wall_tex_name,
                    floor_tex=room_a.floor_tex_name, ceil_tex=room_a.ceil_tex_name,
                    no_ceiling=room_a.no_ceiling)
        self.rooms.append(link)
        link.add_portal(1, start_pos=0, end_pos=len_a)
        link.add_portal(3, start_pos=0, end_pos=len_b)

    def place_entity(self, ent, room=None, pos=None, dir=None, min_x=None, max_x=None, min_z=None, max_z=None):
        """Rejection-sample a free spot for `ent` (RNG order as reference :839-909).
        During a reset with designed start poses, the call that fills entity-list slot e = len(self.entities) takes
        options["poses"][e], and the call for the agent takes options["agent_pose"] first, when its x and z are finite:
        it then runs the `pos=` branch with pos = [x, y, z] (y of the level's own pos, else 0) and the designed dir
        when finite, else the level's dir, else a uniform draw -- no room, search or collision check."""
        assert len(self.rooms) > 0, "create rooms before calling place_entity"
        assert ent.radius is not None, "entity must have physical size defined"
        if len(self.wall_segs) == 0:
            self._gen_static_data()
        design = self._designed_pose(ent)
        if design is not None:
            x, z, d = design
            pos = np.array([x, 0.0 if pos is None else float(pos[1]), z])
            dir = d if math.isfinite(d) else dir
        rng = self._stream()
        if pos is not None:
            ent.dir = dir if dir is not None else rng.uniform(-math.pi, math.pi)
            ent.pos = pos
            self.entities.append(ent)
            return ent
        while True:
            r = room if room else list(self.rooms)[rng.choice(len(list(self.rooms)), p=self.room_probs)]
            lx = r.min_x if min_x is None else min_x
            hx = r.max_x if max_x is None else max_x
            lz = r.min_z if min_z is None else min_z
            hz = r.max_z if max_z is None else max_z
            pos = rng.uniform(low=[lx - ent.radius, 0, lz - ent.radius], high=[hx + ent.radius, 0, hz + ent.radius])
            if not r.point_inside(pos):
                continue
            if self.intersect(ent, pos, ent.radius):
                continue
            ent.pos = pos
            ent.dir = dir if dir is not None else rng.uniform(-math.pi, math.pi)
            break
        self.entities.append(ent)
        return ent

    def _stream(self):
        """The env's numpy stream itself, for draws that are not reset draws (placement, textures, maze carving), also
        while a reset with designed draws runs."""
        rng = self.np_random
        return rng.stream if isinstance(rng, _DesignedDraws) else rng

    def _designed_pose(self, ent):
        """(x, z, dir) of the designed start pose that applies to placing `ent` now, or None."""
        design = getattr(self, "_start_design", None)
        if design is None:
            return None
        rows = [design.get("agent_pose")] if ent is self.agent else []
        rows.append((design.get("poses") or {}).get(len(self.entities)))
        for row in rows:
            if row is not None:
                x, z = float(row[0]), float(row[1])
                d = float(row[2]) if len(row) > 2 and row[2] is not None else math.nan
                if math.isfinite(x) and math.isfinite(z):
                    return x, z, d
        return None

    def place_agent(self, room=None, pos=None, dir=None, min_x=None, max_x=None, min_z=None, max_z=None):
        return self.place_entity(self.agent, room=room, pos=pos, dir=dir,
                                 min_x=min_x, max_x=max_x, min_z=min_z, max_z=max_z)

    def intersect(self, ent, pos, radius):
        """Host-side collision query (world generation and user code; stepping uses the GPU
        kernel).  Walls first -> True; else the first overlapping entity; else None."""
        px, _, pz = pos
        pos = np.array([px, 0, pz])
        if intersect_circle_segs(pos, radius, self.wall_segs):
            return True
        for other in self.entities:
            if other is ent:
                continue
            ox, _, oz = other.pos
            if np.linalg.norm(np.array([ox, 0, oz]) - pos) < radius + other.radius:
                return other
        return None

    def near(self, ent0, ent1=None):
        if ent1 is None:
            ent1 = self.agent
        dist = np.linalg.norm(ent0.pos - ent1.pos)
        return dist < ent0.radius + ent1.radius + 1.1 * self.max_forward_step

    def goal_distance(self):
        """The agent's geodesic distance to the goal in metres, as BatchedMiniWorld(goal_distance=True) computes it
        (navigation.py): 0 when near the goal, +inf when unreachable, NaN for a level without a goal rule."""
        return self._goal_query()[0]

    def expert_action(self):
        """The action along a shortest path to the goal (0 turn left, 1 turn right, 2 move forward), -1 where
        goal_distance() is not finite."""
        return self._goal_query()[1]

    def _goal_query(self):
        from . import navigation as nav
        rule = getattr(self, "device_rule", None)
        if rule is None or rule[0] != "goal":
            return math.nan, -1
        rooms, segs, ents, agent = nav.world_of(self)
        if self._goal_nav is None:     # the goal and the walls stay put during an episode of a goal level
            grid = nav.level_grid(self)
            cls = nav.node_classes(grid, rooms, segs, ents, agent, rule[1], self.max_forward_step)
            self._goal_nav = grid, cls, nav.distance_field(cls, grid[2], grid[3])
        grid, cls, field = self._goal_nav
        return nav.query(grid, field, cls, ents, agent, rule[1], self.max_forward_step, float(self.agent.dir),
                         float(self.params.params["turn_step"].default))

    def _load_tex(self, tex_name):
        rand = self.np_random if self.params.sample(self.np_random, "tex_rand") else None
        return Texture.get(tex_name, rand)

    def _gen_static_data(self):
        for room in self.rooms:
            room._gen_static_data(self.params, self._stream() if self.domain_rand else None)
        self.wall_segs = np.concatenate([r.wall_segs for r in self.rooms])
        self.room_probs = np.array([r.area for r in self.rooms], dtype=float)
        self.room_probs /= np.sum(self.room_probs)

    def _gen_world(self):
        raise NotImplementedError

    def _reward(self):
        return 1.0 - 0.2 * (self.step_count / self.max_episode_steps)

    def _get_carry_pos(self, agent_pos, ent):
        dist = self.agent.radius + ent.radius + self.max_forward_step
        pos = agent_pos + self.agent.dir_vec * 1.05 * dist
        y_pos = max(self.agent.cam_height - ent.height - 0.3, 0)
        return pos + Y_VEC * y_pos

    def move_agent(self, fwd_dist, fwd_drift):
        """Host-side move along the heading plus a sideways drift, refused (False) if the agent or the object it
        carries would touch a wall or another entity (reference miniworld.py:620-645).  `step()` performs the same
        move on the GPU (csrc/physics.cuh); this method is for level code and scripts that move the agent directly."""
        agent = self.agent
        target = agent.pos + agent.dir_vec * fwd_dist + agent.right_vec * fwd_drift
        if self.intersect(agent, target, agent.radius):
            return False
        held = agent.carrying
        if held:
            held_target = self._get_carry_pos(target, held)
            if self.intersect(held, held_target, held.radius):
                return False
            held.pos = held_target
        agent.pos = target
        self._world_dirty = True
        return True

    def turn_agent(self, turn_angle):
        """Host-side turn by `turn_angle` degrees; undone (False) if the carried object would collide at its new
        place in front of the agent (reference miniworld.py:647-668)."""
        agent = self.agent
        before = agent.dir
        agent.dir += turn_angle * (math.pi / 180)
        held = agent.carrying
        if held:
            held_target = self._get_carry_pos(agent.pos, held)
            if self.intersect(held, held_target, held.radius):
                agent.dir = before
                return False
            held.pos = held_target
            held.dir = agent.dir
        self._world_dirty = True
        return True

    # ------------------------------------------------------------------ GPU execution

    def _require_engine(self):
        if self.device is None:
            raise RuntimeError("MiniWorldEnv was built with device=None (world generation only); "
                               "stepping and rendering need the CUDA engine")
        if self._engine is None:
            from .engine import SingleEnvEngine
            self._engine = SingleEnvEngine(self.obs_width, self.obs_height, self.msaa_samples, self.device)
        return self._engine

    def _push_world(self):
        eng = self._require_engine()
        eng.push(self, full=self._world_dirty)
        self._world_dirty = False

    def _pull_state(self):
        self._engine.pull(self)

    def render_obs(self, frame_buffer=None):
        """First-person RGB observation uint8[H, W, 3] (row 0 = top)."""
        eng = self._require_engine()
        self._push_world()
        return eng.render(want_depth=False)[0]

    def render_depth(self, frame_buffer=None):
        """float32[H, W, 1] distance along the view axis in metres (sky = 100)."""
        eng = self._require_engine()
        self._push_world()
        return eng.render(want_depth=True)[1]

    def top_view_extents(self, fb_width, fb_height):
        """Scene extents of render_top_view after the aspect-ratio adjustment, float64 arithmetic of
        the reference (miniworld.py:1109-1133): (min_x, max_x, min_z, max_z)."""
        min_x, max_x = self.min_x - 1, self.max_x + 1
        min_z, max_z = self.min_z - 1, self.max_z + 1
        width, height = max_x - min_x, max_z - min_z
        aspect = width / height
        fb_aspect = fb_width / fb_height
        if aspect > fb_aspect:
            new_h = width / fb_aspect
            h_diff = new_h - height
            min_z -= h_diff / 2
            max_z += h_diff / 2
        elif aspect < fb_aspect:
            new_w = height * fb_aspect
            w_diff = new_w - width
            min_x -= w_diff / 2
            max_x += w_diff / 2
        return float(min_x), float(max_x), float(min_z), float(max_z)

    def render_top_view(self, frame_buffer=None, render_agent=True, return_scale=False):
        """Orthographic map of the whole level, uint8[H, W, 3] (reference miniworld.py:1088-1175).
        frame_buffer: None = observation size, "vis" = window size (the reference passes vis_fb)."""
        if frame_buffer == "vis":
            eng = self._require_vis_engine()
            eng.push(self, full=True)
        else:
            eng = self._require_engine()
            self._push_world()
        ext = self.top_view_extents(eng.W, eng.H)
        img = eng.render_top_view(ext, render_agent)
        if not return_scale:
            return img
        x_scale, z_scale = eng.W / (ext[1] - ext[0]), eng.H / (ext[3] - ext[2])
        return img, {"x_scale": x_scale, "z_scale": z_scale, "x_offset": int(0 - ext[0] * x_scale),
                     "z_offset": int(0 - ext[2] * z_scale)}

    def get_visible_ents(self):
        """Set of entities whose occlusion query passes from the agent's camera (reference
        miniworld.py:1238-1333: a 0.2 m box per entity against the rooms' depth)."""
        eng = self._require_engine()
        self._push_world()
        return {e for e in eng.visible_ents() if any(e is x for x in self.entities)}

    def render_view(self, x, z, dir, render_agent=False, cam_height=None, cam_fwd_disp=None, cam_pitch=None,
                    cam_fov_y=None, size=None, samples=None):
        """(rgb uint8[H, W, 3], depth float32[H, W, 1]) from a designed camera: what render_obs() / render_depth()
        return after agent.pos = (x, agent.pos[1], z), agent.dir = dir and each given camera attribute set, without
        changing the agent.  `size` = (W, H) and `samples` render as into FrameBuffer(W, H, samples); they default to
        the observation size and sample count.  `render_agent=True` also draws the agent's marker triangle at its real
        pose (a third-person view).  Raises ValueError on a row BatchedMiniWorld.render_views would skip."""
        intr = (cam_height, cam_fwd_disp, cam_pitch, cam_fov_y)
        given = [v for v in intr if v is not None]
        if not (math.isfinite(x) and math.isfinite(z) and abs(dir) < 105414350.0) or \
                any(math.isinf(v) for v in given) or \
                (cam_pitch is not None and not abs(cam_pitch) < 90) or \
                (cam_fov_y is not None and not 0 < cam_fov_y < 180):
            raise ValueError("render_view needs a finite x, z and |dir| < 105414350, finite camera attributes, "
                             "|cam_pitch| < 90 and 0 < cam_fov_y < 180, got (%r, %r, %r, %r, %r, %r, %r)" % (
                                 (x, z, dir) + intr))
        W, H = (self.obs_width, self.obs_height) if size is None else (int(size[0]), int(size[1]))
        S = self.msaa_samples if samples is None else int(samples)
        if W <= 0 or H <= 0 or S not in (1, 4, 8, 16):
            raise ValueError("render_view: size must be positive and samples 1, 4, 8 or 16, got %r, %r" % (size, samples))
        if (W, H, S) == (self.obs_width, self.obs_height, self.msaa_samples):
            eng = self._require_engine()
            self._push_world()
        else:
            # one cached engine per (size, samples), whose own frame is that size, as for the human view
            from .engine import SingleEnvEngine
            self._require_engine()          # refuses device=None
            eng = self._view_engines.get((W, H, S))
            if eng is None:
                eng = self._view_engines[(W, H, S)] = SingleEnvEngine(W, H, S, self.device)
            eng.push(self, full=True)
        row = (float(x), float(z), float(dir))
        if given:
            row += tuple(math.nan if v is None else float(v) for v in intr)
        return eng.render_view(row, render_agent)

    def _require_vis_engine(self):
        if self.device is None:
            raise RuntimeError("MiniWorldEnv was built with device=None (world generation only)")
        if self._vis_engine is None:
            from .engine import SingleEnvEngine
            # FrameBuffer(window_width, window_height, 16) (miniworld.py:518): the human-view buffer asks for 16 samples
            self._vis_engine = SingleEnvEngine(self.window_width, self.window_height, self.vis_samples, self.device)
        return self._vis_engine

    def render(self):
        """render_mode="rgb_array": the human-view frame at window_width x window_height (the
        reference's vis_fb image, miniworld.py:1340-1362) -- the agent's view, or the map when
        view="top".  16 samples per pixel like the reference's vis_fb (which takes what its GL driver grants);
        an explicit msaa_samples other than 8 applies to both buffers.  The interactive pyglet window (render_mode="human") is not part of this package."""
        if self.render_mode != "rgb_array":
            return None
        if self.view != "agent":
            return self.render_top_view("vis")
        eng = self._require_vis_engine()
        eng.push(self, full=True)
        return eng.render(want_depth=False)[0]

    def close(self):
        for name in ("_engine", "_vis_engine"):
            if getattr(self, name, None) is not None:
                getattr(self, name).close()
                setattr(self, name, None)
        for eng in self._view_engines.values():
            eng.close()
        self._view_engines = {}
