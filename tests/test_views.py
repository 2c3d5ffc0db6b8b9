"""Designed cameras (mwb_render_views / mwb_visible_ents_from, BatchedMiniWorld.render_views / visible_ents(poses=)):
rows equal to each agent's pose give render()'s frames, a twin batch whose agents were moved to the rows renders the
same frames and visibility masks, random rows match the pixel oracle, skipped rows leave their frames alone and no
call changes any env state.  CPU cases run the kernels' host build; `gpu` cases run libmwb.so on the device."""
import copy
import math

import numpy as np
import pytest

from level_parity import seed_reset

LEVEL_IDS = ["MiniWorld-CollectHealth-v0", "MiniWorld-FourRooms-v0", "MiniWorld-Hallway-v0", "MiniWorld-MazeS2-v0",
             "MiniWorld-MazeS3-v0", "MiniWorld-MazeS3Fast-v0", "MiniWorld-Maze-v0", "MiniWorld-OneRoom-v0",
             "MiniWorld-OneRoomS6-v0", "MiniWorld-OneRoomS6Fast-v0", "MiniWorld-PickupObjects-v0",
             "MiniWorld-PutNext-v0", "MiniWorld-RoomObjects-v0", "MiniWorld-Sidewalk-v0", "MiniWorld-Sign-v0",
             "MiniWorld-ThreeRooms-v0", "MiniWorld-TMaze-v0", "MiniWorld-TMazeLeft-v0", "MiniWorld-TMazeRight-v0",
             "MiniWorld-WallGap-v0", "MiniWorld-YMaze-v0", "MiniWorld-YMazeLeft-v0", "MiniWorld-YMazeRight-v0"]


def make(level, n, seed=5, steps=6, **kw):
    """A batch seeded env i = seed + i, advanced `steps` random steps (auto-reset on)."""
    from miniworld_b200.batched import BatchedMiniWorld
    env = BatchedMiniWorld(level, n, **kw)
    env._ctor = (level, n, kw)
    if env.device_reset:
        seed_reset(env, [seed + i for i in range(n)])
    else:
        env._host_reset(np.arange(n, dtype=np.int32), [seed + i for i in range(n)])
    env._seeded = True
    rs = np.random.default_rng(seed)
    for _ in range(steps):
        env.step_host(rs.integers(0, env.single_action_space.n, n).astype(np.int32), render=False)
    return env


def frames(env):
    """render() / render_depth() of every env through host buffers."""
    obs = np.zeros(env.obs_shape, env.obs_dtype)
    depth = np.zeros((env.num_envs, env.obs_height, env.obs_width, 1), np.float32)
    env.engine.render(obs=obs, depth=depth)
    return obs, depth


def agent_rows(env):
    st = env.get_state()
    return np.stack([st["agent_pos"][:, 0], st["agent_pos"][:, 2], st["agent_dir"]], 1).astype(np.float64)


def floor_rows(env, rs, n=None):
    """Random rows inside each env's level rooms (a random room, a random point of it, a random heading)."""
    rows = np.zeros((env.num_envs if n is None else n, 3))
    for i in range(rows.shape[0]):
        rooms = env.proto_envs[int(env.env_level[i])].rooms
        r = rooms[rs.integers(len(rooms))]
        rows[i] = room_point(r, rs) + (rs.uniform(-4, 4),)
    return rows


def room_point(r, rs):
    """A random (x, z) inside room `r`, away from its walls."""
    mx, mz = min(0.3, (r.max_x - r.min_x) / 4), min(0.3, (r.max_z - r.min_z) / 4)
    return rs.uniform(r.min_x + mx, r.max_x - mx), rs.uniform(r.min_z + mz, r.max_z - mz)


def twin_render(env, rows):
    """A second batch restored from env's snapshot with every agent moved to its row through the state views:
    (frames, depth, visibility mask) of its render() / visible_ents()."""
    from miniworld_b200.batched import BatchedMiniWorld
    level, n, kw = env._ctor
    twin = BatchedMiniWorld(level, n, **kw)
    twin.restore(env.snapshot())
    slots = twin.get_state()["agent_slot"]
    v = twin._views()
    for i, s in enumerate(slots):
        v["ent_x"][s, i], v["ent_z"][s, i], v["ent_dir"][s, i] = rows[i]
    obs, depth = frames(twin)
    mask = twin.visible_ents(out=np.zeros(env.num_envs, np.uint32))
    twin.close()
    return obs, depth, mask


# ---------------------------------------------------------------------------------------------------- CPU: identity
@pytest.mark.parametrize("level,dr", [(lv, dr) for lv in LEVEL_IDS for dr in (False, True)
                                      if not (dr and lv == "MiniWorld-Sign-v0")])     # Sign has no randomisation
def test_rows_at_the_agent_give_render(hostsim_path, level, dr):
    """Rows equal to each agent's own pose: render()'s frames and depth byte for byte, in a two-view call."""
    env = make(level, 3, domain_rand=dr)
    obs, depth = frames(env)
    rows = agent_rows(env)
    got, gd = env.render_views(np.stack([rows, rows]), depth=True)
    assert got.shape == (2,) + obs.shape and gd.shape == (2,) + depth.shape
    for v in range(2):
        assert np.array_equal(got[v], obs), (level, v)
        assert np.array_equal(gd[v], depth), (level, v)
    env.close()


@pytest.mark.parametrize("fmt,msaa", [("hwc", 16), ("cwh", 8), ("grey", 8), ("cwh", 16)])
def test_identity_formats_and_samples(hostsim_path, fmt, msaa):
    env = make("MiniWorld-PickupObjects-v0", 3, obs_format=fmt, msaa_samples=msaa, domain_rand=True)
    obs, depth = frames(env)
    got, gd = env.render_views(agent_rows(env), depth=True)
    assert np.array_equal(got, obs) and np.array_equal(gd, depth)
    env.close()


def test_identity_per_env_worlds_with_level_changes(hostsim_path):
    """A level table with the 8 x 8 Maze (per-env worlds, HBM triangle lists) whose envs change level at resets."""
    from miniworld_b200.batched import BatchedMiniWorld
    levels = ["MiniWorld-OneRoom-v0", "MiniWorld-MazeS3-v0", "MiniWorld-Maze-v0"]
    env = BatchedMiniWorld(levels, 6, env_level=[0, 1, 2, 0, 1, 2], dynamic_levels=True, level_seed=3,
                           per_env_worlds=True, domain_rand=True)
    seed_reset(env, list(range(6)))
    rs = np.random.default_rng(0)
    seen = set()
    for t in range(40):
        env.step_host(rs.integers(0, 3, 6).astype(np.int32), render=False)
        seen |= set(np.asarray(env.env_level).tolist())
        if t % 8 == 7:
            obs, depth = frames(env)
            got, gd = env.render_views(agent_rows(env), depth=True)
            assert np.array_equal(got, obs) and np.array_equal(gd, depth), t
    assert seen == {0, 1, 2}
    env.close()


# ---------------------------------------------------------------------------------------------------- CPU: twin
TWIN_LEVELS = ["MiniWorld-OneRoom-v0", "MiniWorld-FourRooms-v0", "MiniWorld-PickupObjects-v0", "MiniWorld-PutNext-v0",
               "MiniWorld-CollectHealth-v0", "MiniWorld-Sidewalk-v0", "MiniWorld-MazeS3-v0", "MiniWorld-TMaze-v0",
               "MiniWorld-RoomObjects-v0", "MiniWorld-ThreeRooms-v0"]


@pytest.mark.parametrize("level", TWIN_LEVELS)
def test_views_equal_a_twin_with_moved_agents(hostsim_path, level):
    """Mid-rollout states; random rows inside the level's rooms: render_views / visible_ents(poses=) equal the render()
    / visible_ents() of a twin batch whose agents were written to the rows."""
    env = make(level, 4, steps=25, domain_rand=True)
    rows = floor_rows(env, np.random.default_rng(7))
    want_obs, want_depth, want_mask = twin_render(env, rows)
    got, gd = env.render_views(rows, depth=True)
    assert np.array_equal(got, want_obs) and np.array_equal(gd, want_depth)
    assert np.array_equal(env.visible_ents(out=np.zeros(4, np.uint32), poses=rows), want_mask)
    env.close()


def test_twin_with_a_carried_object(hostsim_path):
    """PutNext with an object carried (picked up by a scripted walk): the carried object stays at its own pose."""
    env = make("MiniWorld-PutNext-v0", 4, steps=0)
    carried = 0
    rs = np.random.default_rng(1)
    for t in range(300):
        env.step_host(np.where(rs.random(4) < 0.3, 4, rs.integers(0, 3, 4)).astype(np.int32), render=False)
        if (env.get_state()["carrying"] >= 0).any():
            carried += 1
            if carried in (1, 5):
                rows = floor_rows(env, rs)
                want_obs, want_depth, want_mask = twin_render(env, rows)
                got, gd = env.render_views(rows, depth=True)
                assert np.array_equal(got, want_obs) and np.array_equal(gd, want_depth)
                assert np.array_equal(env.visible_ents(out=np.zeros(4, np.uint32), poses=rows), want_mask)
    assert carried >= 5
    env.close()


# ---------------------------------------------------------------------------------------------------- CPU: oracle
def oracle_view(softgl, env, ts, x, z, d, render_agent):
    """softgl's render of `env` with a copy of the agent at (x, z, d); the marker at the real agent's pose."""
    lst = softgl.draw_list(env, lambda tex: tex.tex_id, agent_marker=render_agent)
    moved = copy.copy(env)
    moved.agent = copy.copy(env.agent)
    moved.agent.pos = np.array([x, env.agent.pos[1], z])
    moved.agent.dir = d
    return softgl._run(moved, ts, lst, env.obs_width, env.obs_height, env.msaa_samples)


def oracle_visible(softgl, env, ts, x, z, d):
    """softgl's get_visible_ents of `env` with a copy of the agent at (x, z, d): the entity-list indices whose query
    box passes (the rooms and query boxes come from the real env, so the real agent is left out as the reference does)."""
    pos, nrm, uv, rgb, tx = softgl.draw_list(env, lambda tex: tex.tex_id, rooms_only=True)
    bpos, qid, ents = softgl._query_boxes(env)
    if len(qid) == 0:
        return set()
    nb = len(qid)
    lst = (np.concatenate([pos, bpos]).astype(np.float32), np.concatenate([nrm, np.tile(np.float32([0, 1, 0]), (nb, 3, 1))]),
           np.concatenate([uv, np.zeros((nb, 3, 2), np.float32)]), np.concatenate([rgb, np.ones((nb, 3, 3), np.float32)]),
           np.concatenate([tx, np.full(nb, -1, np.int32)]).astype(np.int32))
    lst = tuple(np.ascontiguousarray(a, np.int32 if a.dtype == np.int32 else np.float32) for a in lst)
    query = np.concatenate([np.full(len(tx), -1, np.int32), qid])
    flags = np.zeros(len(ents), np.uint8)
    moved = copy.copy(env)
    moved.agent = copy.copy(env.agent)
    moved.agent.pos = np.array([x, env.agent.pos[1], z])
    moved.agent.dir = d
    softgl._run(moved, ts, lst, env.obs_width, env.obs_height, env.msaa_samples, query=query, query_out=flags)
    return {env.entities.index(e) for e, f in zip(ents, flags) if f}


ACTIONS = [2, 2, 1, 2, 0, 2]


@pytest.mark.parametrize("level", ["MiniWorld-FourRooms-v0", "MiniWorld-PickupObjects-v0", "MiniWorld-Sidewalk-v0",
                                   "MiniWorld-MazeS3-v0"])
def test_random_rows_match_the_oracle(hostsim_path, softgl_lib, level):
    """The drop-in render_view from random rows, render_agent off and on, vs the pixel oracle (<= 1 LSB, depth
    identical); the batched render_views of the same episode equals the drop-in byte for byte, and its
    visible_ents(poses=) equals the oracle's occlusion queries from the row."""
    from miniworld_b200.assets import Texture
    from miniworld_b200.envs import LEVELS
    env = LEVELS[level]()
    env.reset(seed=11)
    batch = make(level, 1, seed=11, steps=0)
    for a in ACTIONS:
        env.step(a)
        batch.step_host(np.array([a], np.int32), render=False)
    assert np.array_equal(batch.get_state()["agent_pos"][0], env.agent.pos)
    ts = softgl_lib.TextureSet([t.texels for t in Texture.registry])
    rs = np.random.default_rng(2)
    for k in range(4):
        r = env.rooms[rs.integers(len(env.rooms))]
        (x, z), d = room_point(r, rs), rs.uniform(-4, 4)
        for ra in (False, True):
            rgb, depth = env.render_view(x, z, d, render_agent=ra)
            want, wd = oracle_view(softgl_lib, env, ts, x, z, d, ra)
            assert np.abs(rgb.astype(int) - want.astype(int)).max() <= 1, (k, ra)
            assert np.array_equal(depth, wd), (k, ra)
            got, gd = batch.render_views(np.array([[x, z, d]]), render_agent=ra, depth=True)
            assert np.array_equal(got[0], rgb) and np.array_equal(gd[0], depth), (k, ra)
        mask = int(batch.visible_ents(out=np.zeros(1, np.uint32), poses=np.array([[x, z, d]]))[0])
        assert {e for e in range(32) if (mask >> e) & 1} == oracle_visible(softgl_lib, env, ts, x, z, d), k
    ts.close()
    env.close()
    batch.close()


def test_marker_from_a_camera_above_the_agent(hostsim_path, softgl_lib):
    """cam_height lifted above the agent's 1.6 m: render_agent=True draws the marker (the frames differ from
    render_agent=False) and matches the oracle, which draws Agent.render()'s triangle at the real pose."""
    from miniworld_b200.assets import Texture
    from miniworld_b200.envs import LEVELS
    env = LEVELS["MiniWorld-OneRoom-v0"]()
    env.reset(seed=4)
    env.agent.cam_height = 2.5
    env._world_dirty = True
    ts = softgl_lib.TextureSet([t.texels for t in Texture.registry])
    a = env.agent
    changed = 0
    for back in (1.5, 2.5):              # the marker, 0.9 m below the eye, enters the 30-degree half FOV beyond 1.56 m
        x, z = a.pos[0] - back * math.cos(a.dir), a.pos[2] + back * math.sin(a.dir)
        plain, _ = env.render_view(x, z, a.dir)
        rgb, depth = env.render_view(x, z, a.dir, render_agent=True)
        want, wd = oracle_view(softgl_lib, env, ts, x, z, a.dir, True)
        assert np.abs(rgb.astype(int) - want.astype(int)).max() <= 1 and np.array_equal(depth, wd), back
        changed += int((plain != rgb).any(axis=-1).sum())
    assert changed > 0
    ts.close()
    env.close()
    # the batched path: the level's cam_height param above the agent, from the next reset on
    batch = make("MiniWorld-OneRoom-v0", 2, steps=0)
    batch.set_level_param(0, "cam_height", 2.5)
    seed_reset(batch, [4, 5])
    rows = agent_rows(batch)
    rows[:, 0] -= 2.5 * np.cos(rows[:, 2])
    rows[:, 1] += 2.5 * np.sin(rows[:, 2])
    assert (batch.get_state()["cam"][:, 0] == 2.5).all()
    plain = batch.render_views(rows)
    marked = batch.render_views(rows, render_agent=True)
    diff = (plain != marked).any(axis=-1)
    assert diff.sum(axis=(1, 2)).min() > 0
    assert (marked[diff][:, 0].astype(int) > marked[diff][:, 1:].max(axis=1)).all()       # the marker is red
    batch.close()


# ---------------------------------------------------------------------------------------------------- CPU: reference goldens
GOLDEN_VIEWS = ["oneroom", "fourrooms_dr", "pickup", "sidewalk", "mazes3"]


@pytest.mark.parametrize("name", GOLDEN_VIEWS)
def test_reference_view_goldens(hostsim_path, name):
    """tests/golden/views_*.npz (tools/gen_view_golden.py): what the unmodified reference's render_obs() /
    render_depth() / get_visible_ents() returned with its agent moved to rows inside the floor plan, at a wall, facing
    an entity and outside the floor plan, along a seeded rollout.  The batch replays the rollout and renders the same
    rows: frames within 1 LSB and mostly identical, depth and visibility identical."""
    import os
    from conftest import GOLDEN
    with np.load(os.path.join(GOLDEN, "views_%s.npz" % name)) as z:
        g = {k: z[k] for k in z.files}
    env = make(str(g["level"]), 1, seed=int(g["seed"]), steps=0, domain_rand=bool(g["domain_rand"]))
    rows = g["rows"].reshape(len(g["at"]), -1, 3)
    k = 0
    for t, a in enumerate(g["actions"]):
        env.step_host(np.array([a], np.int32), render=False)
        if t + 1 not in g["at"]:
            continue
        r = rows[k // rows.shape[1]]
        got, gd = env.render_views(np.ascontiguousarray(r[:, None, :]), depth=True)
        for j in range(len(r)):
            d = np.abs(got[j, 0].astype(int) - g["rgb"][k + j].astype(int))
            assert d.max() <= 1 and (d == 0).mean() > 0.99, (name, t, j)
            assert np.array_equal(gd[j, 0], g["depth"][k + j]), (name, t, j)
            mask = env.visible_ents(out=np.zeros(1, np.uint32), poses=np.ascontiguousarray(r[j:j + 1]))
            assert int(mask[0]) == int(g["vis"][k + j]), (name, t, j)
        k += len(r)
    assert k == len(g["rgb"])
    env.close()


# ---------------------------------------------------------------------------------------------------- CPU: skipped rows
def test_skipped_rows_leave_their_frames(hostsim_path):
    env = make("MiniWorld-FourRooms-v0", 4)
    rows = agent_rows(env)
    obs, depth = frames(env)
    poses = np.stack([rows, rows, rows])
    poses[0, 1, 0] = math.nan
    poses[1, 0, 2] = math.inf
    poses[1, 3, 1] = -math.inf
    poses[2, :, 0] = math.nan
    out = np.full((3,) + obs.shape, 77, np.uint8)
    d = np.full((3,) + depth.shape, -5.0, np.float32)
    env.render_views(poses, out=out, depth=d)
    for v in range(3):
        for i in range(4):
            skipped = not np.isfinite(poses[v, i]).all()
            assert np.array_equal(out[v, i], np.full_like(obs[i], 77) if skipped else obs[i]), (v, i)
            assert np.array_equal(d[v, i], np.full_like(depth[i], -5.0) if skipped else depth[i]), (v, i)
    mask = np.full(4, 0xABCD, np.uint32)
    env.visible_ents(out=mask, poses=poses[0])
    assert mask[1] == 0xABCD and np.array_equal(mask[[0, 2, 3]], env.visible_ents(out=np.zeros(4, np.uint32))[[0, 2, 3]])
    # an all-skipped call leaves out and depth untouched; with the default output the frames are zero
    out2, d2 = out.copy(), d.copy()
    env.render_views(np.full((3, 4, 3), math.nan), out=out2, depth=d2)
    assert np.array_equal(out2, out) and np.array_equal(d2, d)
    fresh, fd = env.render_views(np.full((4, 3), math.nan), depth=True)
    assert not fresh.any() and not fd.any()
    env.close()


def test_headings_beyond_the_exact_sin_cos_range_are_skipped(hostsim_path):
    """Headings the glibc-exact sin / cos are not validated for (|dir| >= 105414350), infinities and NaNs with any
    payload are skipped rows: no camera is evaluated and the frame, depth and mask stay as they were.  A heading just
    inside the range renders what a twin whose agent has that heading renders."""
    from miniworld_b200.envs import LEVELS
    env = make("MiniWorld-FourRooms-v0", 8)
    rows = agent_rows(env)
    bad = [1e300, -1e20, 105414350.0, -105414350.0, math.inf, -math.inf,
           np.uint64(0x7FF800000000FFFF).view(np.float64), np.uint64(0xFFFFFFFFFFFFFFFF).view(np.float64),
           np.uint64(0x7FF0000000000001).view(np.float64)]
    for j, d in enumerate(bad):
        poses = rows.copy()
        poses[:, 2] = d
        out = np.full((8, 60, 80, 3), 33, np.uint8)
        depth = np.full((8, 60, 80, 1), -1.0, np.float32)
        env.render_views(poses, out=out, depth=depth)
        assert (out == 33).all() and (depth == -1.0).all(), j
        mask = np.full(8, 7, np.uint32)
        env.visible_ents(out=mask, poses=poses)
        assert (mask == 7).all(), j
    inside = rows.copy()
    inside[:, 2] = 105414349.0
    want_obs, want_depth, want_mask = twin_render(env, inside)
    got, gd = env.render_views(inside, depth=True)
    assert np.array_equal(got, want_obs) and np.array_equal(gd, want_depth) and 0 < got.mean() < 255
    assert np.array_equal(env.visible_ents(out=np.zeros(8, np.uint32), poses=inside), want_mask)
    env.close()
    single = LEVELS["MiniWorld-OneRoom-v0"]()
    single.reset(seed=1)
    for row in ((1.0, 1.0, 1e300), (math.nan, 1.0, 0.0), (1.0, math.inf, 0.0)):
        with pytest.raises(ValueError, match="render_view"):
            single.render_view(*row)
    single.close()


# ---------------------------------------------------------------------------------------------------- CPU: no state change
def test_views_change_no_state(hostsim_path):
    """The snapshot is equal before and after a call; a 300-step rollout with render_views after every step equals a
    twin without it (state, streams, rewards, frames and depth)."""
    a = make("MiniWorld-PickupObjects-v0", 3, steps=0, domain_rand=True, want_depth=True)
    b = make("MiniWorld-PickupObjects-v0", 3, steps=0, domain_rand=True, want_depth=True)
    blob = a.snapshot()
    a.render_views(floor_rows(a, np.random.default_rng(0)), render_agent=True, depth=True)
    a.visible_ents(out=np.zeros(3, np.uint32), poses=floor_rows(a, np.random.default_rng(1)))
    assert np.array_equal(a.snapshot(), blob)
    rs = np.random.default_rng(3)
    vr = np.random.default_rng(4)
    for t in range(300):
        acts = rs.integers(0, 5, 3).astype(np.int32)
        oa, ob = a.step_host(acts), b.step_host(acts)
        a.render_views(np.stack([floor_rows(a, vr), agent_rows(a)]), render_agent=bool(t & 1), depth=True)
        for k in ("obs", "depth", "reward", "terminated", "truncated"):
            assert np.array_equal(oa[k], ob[k]), (t, k)
    assert np.array_equal(a.snapshot(), b.snapshot())
    sa, sb = a.get_state(rng=True), b.get_state(rng=True)
    assert all(np.array_equal(sa[k], sb[k]) for k in sa)
    a.close()
    b.close()


# ---------------------------------------------------------------------------------------------------- CPU: sharding
def _shard_worker(rank, port, lib, q):
    import os
    import torch.distributed as dist
    from miniworld_b200 import engine
    from miniworld_b200.dist import ShardedMiniWorld
    engine._override_library_for_tests(lib)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=2)
    env = ShardedMiniWorld("MiniWorld-FourRooms-v0", 5, dist=dist)
    env.local.engine.seed(np.arange(env.count), np.array([engine.rng_state_of(9 + env.start + k) for k in range(env.count)],
                                                         engine.RNG_DTYPE))
    env.local.engine.reset()
    rows = np.random.default_rng(0).uniform(1, 12, (2, 5, 3))
    out = env.render_views(np.ascontiguousarray(rows[:, env.start:env.start + env.count]),
                           out=np.zeros((2, env.count, 60, 80, 3), np.uint8))
    q.put((rank, out))
    dist.barrier()
    env.close()
    dist.destroy_process_group()


def test_sharded_views_equal_one_process(hostsim_path):
    import os
    import torch.multiprocessing as mp
    from miniworld_b200.batched import BatchedMiniWorld
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31000 + os.getpid() % 2000
    procs = [ctx.Process(target=_shard_worker, args=(r, port, hostsim_path, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=300) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
    one = BatchedMiniWorld("MiniWorld-FourRooms-v0", 5)
    seed_reset(one, [9 + i for i in range(5)])
    rows = np.random.default_rng(0).uniform(1, 12, (2, 5, 3))
    want = one.render_views(rows, out=np.zeros((2, 5, 60, 80, 3), np.uint8))
    assert np.array_equal(np.concatenate([got[0], got[1]], 1), want)
    one.close()


# ---------------------------------------------------------------------------------------------------- CPU: errors
def test_argument_errors(hostsim_path):
    from miniworld_b200.engine import EngineError
    env = make("MiniWorld-OneRoom-v0", 2, steps=0)
    rows = agent_rows(env)
    for bad, match in ((rows.astype(np.float32), "float64"), (rows[:1], "shape"), (rows[None, :, :2], "shape"),
                       (np.zeros((0, 2, 3)), "shape"), (np.zeros((2, 2, 2, 3)), "shape")):
        with pytest.raises(ValueError, match=match):
            env.render_views(bad)
    for out, match in ((np.zeros((2, 60, 80, 3), np.float64), "out"), (np.zeros((2, 3, 80, 60), np.uint8), "out"),
                       (np.zeros((2, 80, 60, 3), np.uint8)[:, ::-1], "out")):
        with pytest.raises(ValueError, match=match):
            env.render_views(rows, out=out)
    with pytest.raises(ValueError, match="depth"):
        env.render_views(rows, depth=np.zeros((2, 60, 80), np.float32))
    with pytest.raises(ValueError, match="shape"):
        env.visible_ents(out=np.zeros(2, np.uint32), poses=rows[None])
    eng, lib = env.engine, env.engine.lib
    obs = np.zeros((2, 60, 80, 3), np.uint8)
    for v in (0, -1):
        with pytest.raises(EngineError, match="views must be positive"):
            eng.render_views(rows, v, obs=obs)
    with pytest.raises(EngineError, match="null"):
        eng._check(lib.mwb_render_views(eng.h, None, 1, 0, obs.ctypes.data, None, None))
    with pytest.raises(EngineError, match="null"):
        eng._check(lib.mwb_render_views(eng.h, rows.ctypes.data, 1, 0, None, None, None))
    with pytest.raises(EngineError, match="null"):
        eng._check(lib.mwb_visible_ents_from(eng.h, None, np.zeros(2, np.uint32).ctypes.data, None))
    env.close()


# ---------------------------------------------------------------------------------------------------- GPU
def _gpu_batch(level, n, **kw):
    from miniworld_b200.batched import BatchedMiniWorld
    env = BatchedMiniWorld(level, n, **kw)
    env.reset(seed=0)
    import torch
    g = torch.Generator(device="cuda").manual_seed(1)
    for _ in range(8):
        env.step(torch.randint(0, 3, (n,), device="cuda", generator=g, dtype=torch.int32))
    return env


def _torch_rows(env):
    import torch
    st = env.get_state()
    return torch.tensor(np.stack([st["agent_pos"][:, 0], st["agent_pos"][:, 2], st["agent_dir"]], 1), device="cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("spec", ["MiniWorld-FourRooms-v0", "MiniWorld-PickupObjects-v0", "maze_table"])
def test_gpu_identity_at_scale(libmwb_path, spec):
    import torch
    kw = dict(per_env_worlds=True, env_level=np.arange(4096) % 2) if spec == "maze_table" else {}
    level = ["MiniWorld-FourRooms-v0", "MiniWorld-Maze-v0"] if spec == "maze_table" else spec
    env = _gpu_batch(level, 4096, want_depth=True, domain_rand=True, **kw)
    obs = env.render().clone()
    depth = env.render_depth()
    rows = _torch_rows(env)
    got, gd = env.render_views(torch.stack([rows, rows]), depth=True)
    torch.cuda.synchronize()
    assert torch.equal(got[0], obs) and torch.equal(got[1], obs)
    assert torch.equal(gd[0], depth) and torch.equal(gd[1], depth)
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("level", ["MiniWorld-FourRooms-v0", "MiniWorld-PickupObjects-v0", "MiniWorld-Sidewalk-v0"])
def test_gpu_random_rows_equal_the_host_build(libmwb_path, level):
    """The device's views from random rows (render_agent off and on) equal the host build's on a sample of envs."""
    import torch
    from miniworld_b200 import engine
    from miniworld_b200.batched import BatchedMiniWorld
    import subprocess, os
    n = 6
    dev = BatchedMiniWorld(level, n, domain_rand=True)
    seed_reset(dev, [40 + i for i in range(n)])
    rows = floor_rows(dev, np.random.default_rng(3))
    blob = dev.snapshot()
    want = [dev.render_views(torch.tensor(rows, device="cuda"), render_agent=ra, depth=True) for ra in (False, True)]
    want = [(o.cpu().numpy(), d.cpu().numpy()) for o, d in want]
    dev.close()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = subprocess.check_output([os.path.join(root, "tests", "hostsim", "build.sh")]).decode().strip().splitlines()[-1]
    engine._override_library_for_tests(lib)
    try:
        host = BatchedMiniWorld(level, n, domain_rand=True)
        host.restore(blob)
        for ra, (o, d) in zip((False, True), want):
            ho, hd = host.render_views(rows, render_agent=ra, depth=True)
            assert np.abs(ho.astype(int) - o.astype(int)).max() <= 1 and np.array_equal(hd, d), ra
        host.close()
    finally:
        engine._override_library_for_tests(None)


@pytest.mark.gpu
def test_gpu_imagenav_loop(libmwb_path):
    """The README loop: after every step the goal images of the reset envs equal a full render_views of those rows,
    and the other envs' images are unchanged."""
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    N = 4096
    envs = BatchedMiniWorld("MiniWorld-OneRoom-v0", num_envs=N)
    box = [s["slot"] for s in envs.level_slots[0] if not s["agent"]][0]
    goal_img = torch.zeros((N, 60, 80, 3), dtype=torch.uint8, device="cuda")
    nan = torch.full((N, 3), float("nan"), dtype=torch.float64, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(0)

    def goal_rows(which):
        xz = envs.entity_xz(box)
        a = torch.rand(N, device="cuda", dtype=torch.float64, generator=g) * 2 * math.pi
        eye = (xz + 1.5 * torch.stack([a.cos(), a.sin()], 1)).clamp(0.5, 9.5)
        d = xz - eye
        return torch.where(which[:, None], torch.cat([eye, torch.atan2(-d[:, 1], d[:, 0])[:, None]], 1), nan)

    envs.reset(seed=0)
    envs.render_views(goal_rows(torch.ones(N, dtype=torch.bool, device="cuda")), out=goal_img)
    resets = 0
    for t in range(30):
        _, _, term, trunc, _ = envs.step(torch.randint(0, 3, (N,), device="cuda", generator=g, dtype=torch.int32))
        done = term | trunc
        before = goal_img.clone()
        rows = goal_rows(done)
        envs.render_views(rows, out=goal_img)
        full = envs.render_views(torch.where(done[:, None], rows, nan))
        assert torch.equal(goal_img[done], full[done]) and torch.equal(goal_img[~done], before[~done]), t
        resets += int(done.sum())
    assert resets > 0
    envs.close()


@pytest.mark.gpu
def test_gpu_rows_from_a_busy_side_stream(libmwb_path):
    """Rows written by a slow torch kernel on a busy side stream, handed over by stream order, are read in order."""
    import torch
    env = _gpu_batch("MiniWorld-FourRooms-v0", 2048)
    obs = env.render().clone()
    rows = _torch_rows(env)
    side = torch.cuda.Stream()
    poses = torch.full_like(rows, float("nan"))
    with torch.cuda.stream(side):
        x = torch.randn(2048, 2048, device="cuda")
        for _ in range(20):
            x = x @ x / 2048.0                 # keeps the side stream busy
        poses.copy_(rows + 0.0 * x[:2048, :3].double().nan_to_num(0, 0, 0).clamp(0, 0))
    torch.cuda.current_stream().wait_stream(side)
    out = env.render_views(poses)
    torch.cuda.synchronize()
    assert torch.equal(out, obs)
    env.close()


@pytest.mark.gpu
def test_gpu_no_overflow_inside_the_floor_plan(libmwb_path):
    """mwb_overflow_count() is unchanged by views from rows inside every level's floor plan."""
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    for level in LEVEL_IDS:
        env = BatchedMiniWorld(level, 256)
        env.reset(seed=1)
        before = env.engine.overflow_count()
        rows = torch.tensor(floor_rows(env, np.random.default_rng(5)), device="cuda")
        env.render_views(torch.stack([rows, rows.flip(0)]), render_agent=True, depth=True)
        env.visible_ents(poses=rows)
        torch.cuda.synchronize()
        assert env.engine.overflow_count() == before, level
        env.close()


@pytest.mark.gpu
def test_gpu_views_change_no_state(libmwb_path):
    """A device rollout with render_views (and visible_ents(poses=)) after every step equals a twin that never calls
    them: observations, depth, rewards and flags every step, the snapshot at the end.  The device scratch the views
    overwrite (cam_trig, ent_cs, the mesh lists) is rebuilt by every render launch."""
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    N = 512
    a = BatchedMiniWorld("MiniWorld-PickupObjects-v0", N, domain_rand=True, want_depth=True)
    b = BatchedMiniWorld("MiniWorld-PickupObjects-v0", N, domain_rand=True, want_depth=True)
    a.reset(seed=3)
    b.reset(seed=3)
    g = torch.Generator(device="cuda").manual_seed(0)
    rs = np.random.default_rng(0)
    for t in range(150):
        acts = torch.randint(0, 5, (N,), device="cuda", generator=g, dtype=torch.int32)
        oa, ra, ta, ua, ia = a.step(acts)
        oa, ra, ta, ua, da = oa.clone(), ra.clone(), ta.clone(), ua.clone(), ia["depth"].clone()
        ob, rb, tb, ub, ib = b.step(acts)
        assert torch.equal(oa, ob) and torch.equal(da, ib["depth"]), t
        assert torch.equal(ra, rb) and torch.equal(ta, tb) and torch.equal(ua, ub), t
        rows = torch.tensor(floor_rows(a, rs), device="cuda")
        a.render_views(torch.stack([rows, rows.flip(0)]), render_agent=bool(t & 1), depth=True)
        a.visible_ents(poses=rows)
    torch.cuda.synchronize()
    assert np.array_equal(a.snapshot(), b.snapshot())
    a.close()
    b.close()
