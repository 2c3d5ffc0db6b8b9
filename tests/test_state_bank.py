"""State bank (mwb_enable_state_bank, BatchedMiniWorld(state_bank=K)): envs saved into device records and loaded at
resets.  The main oracle is a twin: batch A saves every env at step t and later loads a permutation of the slots, and a
twin B restored from A's snapshot at step t must equal A env for env (env i of A = env perm[i] of B) from the load on,
under the same actions.  CPU cases run the kernels' host build; `gpu` cases run libmwb.so on the device."""
import os

import numpy as np
import pytest

from level_parity import assert_env_equal, full_state, geometry_equal, seed_reset, short_level
from test_maze_layouts import host_array

MAZE_LEVELS = ("MiniWorld-MazeS2-v0", "MiniWorld-MazeS3-v0", "MiniWorld-Maze-v0")
TABLE = ["MiniWorld-OneRoom-v0", "MiniWorld-MazeS2-v0", "MiniWorld-MazeS3-v0", "MiniWorld-Maze-v0"]

# name -> (levels, BatchedMiniWorld keyword arguments); levels are truncated to short episodes so that the rollouts
# cross auto-resets
CASES = {
    "oneroom": ("MiniWorld-OneRoom-v0", {}),
    "fourrooms_dr": ("MiniWorld-FourRooms-v0", dict(domain_rand=True)),
    "pickup": ("MiniWorld-PickupObjects-v0", {}),
    "collecthealth": ("MiniWorld-CollectHealth-v0", {}),
    "putnext_dr": ("MiniWorld-PutNext-v0", dict(domain_rand=True)),
    "tmaze": ("MiniWorld-TMaze-v0", {}),
    "sign": ("MiniWorld-Sign-v0", {}),
    "mazes3": ("MiniWorld-MazeS3-v0", {}),
    "table": (TABLE, dict(per_env_worlds=True, dynamic_levels=True, level_seed=3)),
}


def short(levels, steps):
    return [short_level(lv, steps) for lv in levels] if isinstance(levels, list) else short_level(levels, steps)


def has_maze(levels):
    return any(lv in MAZE_LEVELS for lv in (levels if isinstance(levels, list) else [levels]))


def make(levels, n, kw, modes, slots, steps=12, **extra):
    from miniworld_b200.batched import BatchedMiniWorld
    mode_kw = dict(episode_seeds=True, start_poses=True, maze_layouts=has_maze(levels)) if modes else {}
    return BatchedMiniWorld(short(levels, steps), n, want_depth=True, state_bank=slots, **kw, **mode_kw, **extra)


def frames(env):
    """obs and depth of every env as the render kernel draws them now (numpy buffers: the host build)."""
    obs = np.zeros(env.obs_shape, env.obs_dtype)
    depth = np.zeros((env.num_envs, env.obs_height, env.obs_width, 1), np.float32)
    env.engine.render(obs=obs, depth=depth)
    return obs, depth


def mode_records(env):
    """The per-env records of the modes that are on: info["level" / "seed" / "maze" / "start"]."""
    out = {}
    if env.dynamic_levels:
        out["level"] = host_array(env.level_tensor)
    if env.episode_seeds:
        out["seed"] = host_array(env.episode_seed)
    if env.maze_layouts:
        out["maze"] = host_array(env.episode_maze)
    if env.start_poses:
        out["start"] = host_array(env.episode_start)
    return out


def assert_twins(a, b, perm, live, where, out_a=None, out_b=None):
    """Env i of `a` equals env perm[i] of `b` for every i in `live`: state, geometry, mode records and, given step
    outputs, rewards, flags, frames and depth."""
    sa, sb = full_state(a), full_state(b)
    ra, rb = mode_records(a), mode_records(b)
    for i in live:
        j = perm[i]
        assert_env_equal(sa, i, sb, j, (where, i))
        assert geometry_equal(a, i, b, j), (where, i)
        for key in ra:
            assert np.array_equal(ra[key][i], rb[key][j]), (where, i, key)
        if out_a is not None:
            for key in ("reward", "terminated", "truncated", "obs", "depth"):
                assert np.array_equal(out_a[key][i], out_b[key][j]), (where, i, key)
    assert a.engine.overflow_count() == 0 and b.engine.overflow_count() == 0


def twin_run(levels, kw, modes, n=6, t=9, k=7, after=26, seed=0):
    """The twin test on the host build (module docstring)."""
    rs = np.random.default_rng(seed)
    a = make(levels, n, kw, modes, n)
    b = make(levels, n, kw, modes, n)
    if modes:                                    # episode_seed then names each saved episode's seed
        a.set_env_seed(np.arange(n), 100 + np.arange(n))
        a.engine.reset()
    else:
        seed_reset(a, 100 + np.arange(n))
    nact = a.action_space.n
    acts = rs.integers(0, nact, size=(t + k + after, n), dtype=np.int32)
    out = None
    for s in range(t):
        out = a.step_host(acts[s], out, render=False)
    done = (out["terminated"] | out["truncated"]).astype(bool)      # these envs have needs_reset set
    blob = a.snapshot()
    a.save_states(np.arange(n), np.arange(n))
    for s in range(t, t + k):
        out = a.step_host(acts[s], out, render=False)
    perm = rs.permutation(n)
    a.set_env_state(np.arange(n), perm)
    a.engine.reset()
    assert np.array_equal(host_array(a.episode_state), perm) and (host_array(a.next_state) == -1).all()
    b.restore(blob)
    live = [i for i in range(n) if not done[perm[i]]]
    assert live
    fa, fb = frames(a), frames(b)
    for i in live:
        assert np.array_equal(fa[0][i], fb[0][perm[i]]) and np.array_equal(fa[1][i], fb[1][perm[i]]), i
    assert_twins(a, b, perm, live, "load")
    oa = ob = None
    inv = np.argsort(perm)
    for s in range(after):
        act = acts[t + k + s]
        act_b = np.empty_like(act)
        act_b[perm] = act                                          # env perm[i] of b takes env i's action
        render = s % 8 == 7
        oa = a.step_host(act, oa, render=render)
        ob = b.step_host(act_b, ob, render=render)
        assert_twins(a, b, perm, live, s, oa if render else None, ob if render else None)
        if not render:
            for key in ("reward", "terminated", "truncated"):
                assert np.array_equal(oa[key][live], ob[key][perm[live]]), (s, key)
    assert (oa["terminated"] | oa["truncated"]).any() or after > 20, inv
    a.close()
    b.close()


@pytest.mark.parametrize("modes", [False, True], ids=["modes_off", "modes_on"])
@pytest.mark.parametrize("case", list(CASES))
def test_twin_loads_equal_the_snapshot(hostsim_path, case, modes):
    levels, kw = CASES[case]
    twin_run(levels, kw, modes, seed=len(case))


def test_cross_level_load_adopts_the_level_without_a_draw(hostsim_path):
    """Level changes on: a load of another level's state adopts its level, makes no level draw, and leaves a pending
    level for the next program reset."""
    from miniworld_b200.batched import BatchedMiniWorld
    rows = ["MiniWorld-OneRoom-v0", "MiniWorld-FourRooms-v0"]
    mk = lambda: BatchedMiniWorld(rows, 4, env_level=[0, 0, 1, 1], dynamic_levels=True, level_seed=9, state_bank=3)
    a, c = mk(), mk()
    for e in (a, c):
        seed_reset(e, [11, 12, 13, 14])
        e.set_level_weights([1.0, 1.0])
    st = full_state(a)
    a.save_states([2], [1])
    a.set_env_level([0], [0])
    c.set_env_level([0], [0])
    a.set_env_state([0], 1)
    a.engine.reset([0])
    assert host_array(a.level_tensor)[0] == 1 and host_array(a._views()["next_level"])[0] == 0
    assert host_array(a.episode_state).tolist() == [1, -1, -1, -1]
    assert_env_equal(full_state(a), 0, st, 2, "load")
    assert geometry_equal(a, 0, a, 2)
    # the next program reset of env 0 takes the pending level, and its draw counter is where c's is (no draw made)
    from miniworld_b200.engine import RNG_DTYPE, rng_state_of

    def state(e):      # OneRoom's reset rewrites the texture row of its one room; the loaded FourRooms rows beyond stay
        st = full_state(e)
        st["room_tex"] = st["room_tex"][:, :1] if host_array(e.level_tensor)[0] == 0 else st["room_tex"]
        return st
    for e in (a, c):
        e.engine.seed([0], np.array([rng_state_of(99)], RNG_DTYPE))
        e.engine.reset([0])
        assert host_array(e.level_tensor)[0] == 0
    assert_env_equal(state(a), 0, state(c), 0, "pending level")
    for r in range(6):                                            # weighted draws: equal counters draw equal levels
        for e in (a, c):
            e.engine.reset([0])
        assert host_array(a.level_tensor)[0] == host_array(c.level_tensor)[0], r
        assert_env_equal(state(a), 0, state(c), 0, r)
    a.close()
    c.close()


def test_fallbacks_equal_a_reset_without_the_entry(hostsim_path):
    """Static table: another level's slot, an empty slot and a slot out of range fall back to the program reset."""
    from miniworld_b200.batched import BatchedMiniWorld
    rows = ["MiniWorld-OneRoom-v0", "MiniWorld-FourRooms-v0"]
    mk = lambda: BatchedMiniWorld(rows, 4, env_level=[0, 0, 1, 1], state_bank=4)
    a, c = mk(), mk()
    for e in (a, c):
        seed_reset(e, [21, 22, 23, 24])
    a.save_states([2], [0])                                       # slot 0: level 1
    nxt = a.next_state
    nxt[0], nxt[1], nxt[3] = 0, 3, 9                              # other level, empty slot, out of range
    a.engine.reset()
    c.engine.reset()
    assert host_array(a.episode_state).tolist() == [-1] * 4 and (host_array(a.next_state) == -1).all()
    sa, sc = full_state(a), full_state(c)
    for i in range(4):
        assert_env_equal(sa, i, sc, i, i)
    assert host_array(a.bank_level).tolist() == [1, -1, -1, -1]
    a.close()
    c.close()


def test_pending_inputs_survive_a_load(hostsim_path):
    """A pending seed, layout and pose stay pending through a load and are consumed by the next program reset."""
    from miniworld_b200.batched import BatchedMiniWorld
    from test_maze_layouts import spanning_tree
    mk = lambda bank: BatchedMiniWorld("MiniWorld-MazeS3-v0", 3, episode_seeds=True, maze_layouts=True,
                                       start_poses=True, state_bank=bank)
    a, d = mk(2), mk(2)
    for e in (a, d):
        seed_reset(e, [31, 32, 33])
    lay = spanning_tree(3, 3, np.random.default_rng(4))
    st = full_state(a)
    a.save_states([2], [1])
    for e in (a, d):
        e.set_env_seed([0], 77)
        e.set_env_maze([0], lay, goal_cell=4, agent_cell=0)
        e.set_env_pose([0], "agent", 1.5, 1.5, 0.25)
    a.set_env_state([0], 1)
    a.engine.reset([0])
    assert_env_equal(full_state(a), 0, st, 2, "load")
    assert host_array(a.next_seed)[0] == 77 and host_array(a.maze_pending)[0] == 1 and host_array(a.pose_pending)[0] == 1
    a.engine.reset([0])
    d.engine.reset([0])
    assert host_array(a.episode_state)[0] == -1 and host_array(a.episode_seed)[0] == 77
    assert_env_equal(full_state(a), 0, full_state(d), 0, "program")
    assert geometry_equal(a, 0, d, 0)
    for key, v in mode_records(d).items():
        assert np.array_equal(mode_records(a)[key][0], v[0]), key
    a.close()
    d.close()


@pytest.mark.parametrize("dynamic", [False, True])
def test_episode_state_follows_a_numpy_model(hostsim_path, dynamic):
    """next_state / episode_state / bank_level against a model over saves, loads, fallbacks and subset resets."""
    from miniworld_b200.batched import BatchedMiniWorld
    rows = ["MiniWorld-OneRoom-v0", "MiniWorld-FourRooms-v0"]
    N, K = 8, 5
    env = BatchedMiniWorld(rows, N, dynamic_levels=dynamic, state_bank=K)
    seed_reset(env, 40 + np.arange(N))
    rs = np.random.default_rng(7 + dynamic)
    lvl = env.env_level.copy()
    bank = np.full(K, -1)
    nxt, ep = np.full(N, -1), np.full(N, -1)
    for r in range(30):
        if r % 3 == 0:
            e, s = rs.integers(0, N, 3), rs.integers(0, K, 3)
            env.save_states(e, s)
            for ei, si in zip(e, s):
                bank[si] = lvl[ei]
        ids = rs.choice(N, rs.integers(1, N), replace=False)
        vals = rs.integers(-1, K + 2, ids.size)
        view = env.next_state
        view[ids] = vals
        nxt[ids] = vals
        reset = rs.choice(N, rs.integers(1, N + 1), replace=False)
        env.engine.reset(np.sort(reset))
        for i in reset:
            s = nxt[i]
            take = 0 <= s < K and bank[s] >= 0 and (bank[s] == lvl[i] or dynamic)
            ep[i] = s if take else -1
            if take:
                lvl[i] = bank[s]
            nxt[i] = -1
        assert np.array_equal(host_array(env.next_state), nxt), r
        assert np.array_equal(host_array(env.episode_state), ep), r
        assert np.array_equal(host_array(env.bank_level), bank), r
        assert np.array_equal(env.env_level, lvl), r
    env.close()


def test_repeated_slots_and_envs_take_the_last_entry(hostsim_path):
    from miniworld_b200.batched import BatchedMiniWorld
    env = BatchedMiniWorld("MiniWorld-PickupObjects-v0", 5, state_bank=3)
    seed_reset(env, 50 + np.arange(5))
    st = full_state(env)
    env.save_states([0, 1, 2, 3], [2, 2, 0, 2])                   # slot 2: env 3
    env.set_env_state([4, 4, 0], [1, 2, 0])                       # env 4: slot 2
    assert host_array(env.next_state).tolist() == [0, -1, -1, -1, 2]
    env.engine.reset([0, 4])
    sa = full_state(env)
    assert_env_equal(sa, 4, st, 3, "slot 2")
    assert_env_equal(sa, 0, st, 2, "slot 0")
    env.close()


def test_snapshots_within_and_across_modes(hostsim_path):
    import helpers
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import EngineError
    helpers.snapshot_roundtrip("MiniWorld-FourRooms-v0", hostsim_path, n=4, state_bank=3)
    a = BatchedMiniWorld("MiniWorld-FourRooms-v0", 4, state_bank=3)
    seed_reset(a, [1, 2, 3, 4])
    a.save_states([1, 3], [0, 2])
    a.set_env_state([0], 2)
    a.engine.reset([0])
    a.set_env_state([1, 2], [0, 1])
    blob = a.snapshot()
    assert blob[:4].tobytes() == b"mWBS"
    views = lambda e: [host_array(v).copy() for v in (e.bank_level, e.next_state, e.episode_state)]
    before = views(a)
    fresh = BatchedMiniWorld("MiniWorld-FourRooms-v0", 4, state_bank=3)
    fresh.restore(blob)
    for x, y in zip(before, views(fresh)):
        assert np.array_equal(x, y)
    a.engine.reset([1, 2])
    fresh.engine.reset([1, 2])
    sa, sf = full_state(a), full_state(fresh)
    for i in range(4):
        assert_env_equal(sa, i, sf, i, i)
    plain = BatchedMiniWorld("MiniWorld-FourRooms-v0", 4)
    blob_plain = plain.snapshot()
    assert blob_plain[:4].tobytes() == b"MWBS"
    with pytest.raises(EngineError, match="error -6"):
        plain.restore(blob)
    with pytest.raises(EngineError, match="error -6"):
        a.restore(blob_plain)
    other = BatchedMiniWorld("MiniWorld-FourRooms-v0", 4, state_bank=5)
    with pytest.raises(EngineError, match="error -1"):
        other.restore(blob)
    for e in (a, fresh, plain, other):
        e.close()


def test_blobs_without_the_bank_keep_their_size(hostsim_path):
    """A handle without the bank writes the blob it wrote before: its size is that of the sections it always had, and
    the bank's sections are exactly the records and the three arrays."""
    from miniworld_b200.batched import BatchedMiniWorld
    for levels, kw in (("MiniWorld-FourRooms-v0", {}), ("MiniWorld-MazeS3-v0", {}), (TABLE, dict(per_env_worlds=True))):
        plain = BatchedMiniWorld(levels, 3, **kw)
        on = BatchedMiniWorld(levels, 3, state_bank=2, **kw)
        p, b = plain.snapshot(), on.snapshot()
        rec = (b.size - p.size - 4 * (2 + 3 + 3)) / 2
        assert rec == int(rec) and rec % 16 == 0 and rec > 0, (levels, rec)
        assert p[:4].tobytes()[1:] == b[:4].tobytes()[1:] and p[:1].tobytes().upper() == b[:1].tobytes().upper()
        plain.close()
        on.close()


def test_errors(hostsim_path):
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import EngineError
    from miniworld_b200.envs import LEVELS
    host_only = type("HostOnlyRoom", (LEVELS["MiniWorld-OneRoom-v0"],), {"device_program": None})
    with pytest.raises(TypeError, match="host"):
        BatchedMiniWorld(host_only, 2, state_bank=2)
    for bad in (0, -3, True, 1.5):
        with pytest.raises(ValueError):
            BatchedMiniWorld("MiniWorld-OneRoom-v0", 2, state_bank=bad)
    env = BatchedMiniWorld("MiniWorld-OneRoom-v0", 4, state_bank=3)
    assert host_array(env.next_state).tolist() == [-1] * 4 and host_array(env.bank_level).tolist() == [-1] * 3
    for args in (([4], [0]), ([-1], [0]), ([0], [3]), ([0], [-1]), ([0, 1], [0]), ([0.5], [0]), ([[0]], [[0]])):
        with pytest.raises(ValueError):
            env.save_states(*args)
    for args in (([4], 0), ([0], 3), ([0], -2), ([0, 1], [0, 1, 2]), ([0.5], 0)):
        with pytest.raises(ValueError):
            env.set_env_state(*args)
    assert host_array(env.bank_level).tolist() == [-1] * 3 and host_array(env.next_state).tolist() == [-1] * 4
    eng = env.engine
    with pytest.raises(EngineError, match="error -6"):
        eng.enable_state_bank(2)                                  # already on
    for enable in (eng.enable_episode_seeds, eng.enable_start_poses, lambda: eng.enable_level_changes(0, 0)):
        with pytest.raises(EngineError, match="error -6"):
            enable()                                              # another mode after the bank
    env.close()
    off = BatchedMiniWorld("MiniWorld-OneRoom-v0", 2)
    with pytest.raises(EngineError, match="error -6"):
        off.engine.save_states(np.zeros(1, np.int32), np.zeros(1, np.int32))
    with pytest.raises(EngineError, match="error -1"):
        off.engine.enable_state_bank(0)
    for name in ("next_state", "episode_state", "bank_level"):
        with pytest.raises(EngineError, match="error -6"):
            off.engine.state_array(name)
        with pytest.raises(RuntimeError, match="state_bank=K"):
            getattr(off, name)
    off.close()
    host = BatchedMiniWorld(host_only, 2)
    with pytest.raises(EngineError, match="error -6"):
        host.engine.enable_state_bank(2)                          # host resets
    host.close()


# ------------------------------------------------------------------ sharding (gloo, host build)
def _sharded_worker(rank, world, port, hostsim, total, steps, q):
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    sys.path.insert(0, os.path.join(root, "tests"))
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from miniworld_b200 import engine
    from miniworld_b200.dist import ShardedMiniWorld
    engine._override_library_for_tests(hostsim)
    env = ShardedMiniWorld(short_level("MiniWorld-FourRooms-v0", 9), total, dist=dist, state_bank=4)
    q.put((rank, sharded_run(env.local, env.start, steps)))
    dist.barrier()
    dist.destroy_process_group()


def sharded_run(env, start, steps):
    """A Go-Explore-like schedule over global env ids, applied to the envs `env` holds ([start, start + N)): envs save
    into local slots and load them back; returns each step's rewards and agent poses of those envs."""
    n = env.num_envs
    seed_reset(env, 1000 + start + np.arange(n))
    rs = np.random.default_rng(5)
    out, rec = None, []
    for t in range(steps):
        acts = rs.integers(0, 3, size=64, dtype=np.int32)[start:start + n]
        if t % 4 == 1:
            env.save_states(np.arange(n) % n, np.arange(n) % 4)
        if t % 5 == 3:
            env.set_env_state(np.arange(n), (np.arange(n) + t) % 4)
        out = env.step_host(acts, out, render=False)
        rec.append((out["reward"].copy(), env.get_state()["agent_pos"].copy(), host_array(env.episode_state).copy()))
    return rec


def test_sharded_bank_equals_one_process(hostsim_path):
    """world_size 2 over gloo: each rank's bank is its own and ids are local; the ranks together equal one process
    whose halves run the same schedule on their own banks."""
    import torch.multiprocessing as mp
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200 import engine
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29800 + os.getpid() % 2000
    total, steps = 10, 24
    procs = [ctx.Process(target=_sharded_worker, args=(r, 2, port, engine._test_library, total, steps, q))
             for r in range(2)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=300) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, (start, n) in enumerate(((0, 5), (5, 5))):
        one = BatchedMiniWorld(short_level("MiniWorld-FourRooms-v0", 9), n, state_bank=4)
        want = sharded_run(one, start, steps)
        for t, (x, y) in enumerate(zip(want, got[rank])):
            for u, v in zip(x, y):
                assert np.array_equal(u, v), (rank, t)
        one.close()


# ------------------------------------------------------------------ GPU (libmwb.so)
def go_explore(envs, steps, seed, record=None):
    """The README's Go-Explore loop in torch ops, without a host round trip: the archive maps the cell of the agent's
    floor position (a 14 x 14 grid over FourRooms) to the slot of the same index, an env that reaches a cell whose slot
    is empty is saved there, and every done env gets a pending slot drawn uniformly from the filled ones.  With
    `record`, each step's (actions, slot each env was saved to or -1, done mask, pending slots) are appended as numpy
    arrays."""
    import torch
    dev = envs.next_state.device
    N = envs.num_envs
    g = torch.Generator(device=dev).manual_seed(seed)
    agent = [s["slot"] for s in envs.level_slots[0] if s["agent"]][0]
    G, lo, size = 14, -7.0, 1.0
    ids = torch.arange(N, device=dev)
    for t in range(steps):
        acts = torch.randint(0, 3, (N,), generator=g, device=dev, dtype=torch.int32)
        obs, rew, term, trunc, info = envs.step(acts)
        ij = ((envs.entity_xz(agent) - lo) / size).floor().long().clamp(0, G - 1)
        cell = ij[:, 0] * G + ij[:, 1]
        save = torch.where(envs.bank_level[cell] < 0, cell, -1)    # new cells; -1 entries are skipped
        envs.save_states(ids, save)
        done = term | trunc
        cdf = (envs.bank_level >= 0).long().cumsum(0)
        u = (torch.rand(N, generator=g, device=dev, dtype=torch.float64) * cdf[-1]).long()
        pick = torch.searchsorted(cdf, u, right=True).clamp(max=cdf.numel() - 1)    # a filled slot (empty bank: 0)
        envs.next_state.copy_(torch.where(done, pick, -1).int())
        if record is not None:
            record.append([v.cpu().numpy() for v in (acts, save, done, pick)])


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["fourrooms", "pickup", "table_maze8"])
def test_gpu_twin_4096(libmwb_path, case):
    """The twin test at 4096 envs on the device: frames and depth byte-identical, no capacity fault."""
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    levels, kw = {"fourrooms": ("MiniWorld-FourRooms-v0", dict(domain_rand=True)),
                  "pickup": ("MiniWorld-PickupObjects-v0", {}),
                  "table_maze8": (TABLE, dict(per_env_worlds=True, dynamic_levels=True, level_seed=3))}[case]
    N = 4096
    mk = lambda: BatchedMiniWorld(short(levels, 20), N, want_depth=True, state_bank=N, **kw)
    a, b = mk(), mk()
    a.reset(seed=1234)
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(3)
    nact = a.action_space.n
    acts = torch.randint(0, nact, (40, N), generator=g, device=dev, dtype=torch.int32)
    for t in range(9):
        _, _, term, trunc, _ = a.step(acts[t])
    done = (term | trunc).cpu().numpy()
    blob = a.snapshot()
    a.save_states(torch.arange(N, device=dev), torch.arange(N, device=dev))
    for t in range(9, 16):
        a.step(acts[t])
    perm = torch.randperm(N, generator=g, device=dev)
    a.next_state.copy_(perm.to(torch.int32))
    obs_a = a.reset()[0].clone()
    b.restore(blob)
    obs_b = b.render().clone()
    p = perm.cpu().numpy()
    live = torch.as_tensor(~done[p], device=dev)
    assert live.sum() > N // 2
    pt = perm.long()
    assert torch.equal(obs_a[live], obs_b[pt][live])
    assert torch.equal(a.episode_state.long(), pt)
    for t in range(16, 40):
        act_b = torch.empty_like(acts[t])
        act_b[pt] = acts[t]
        oa, ra, ta, ua, ia = a.step(acts[t])
        oa, da = oa.clone(), ia["depth"].clone()
        ob, rb, tb, ub, ib = b.step(act_b)
        assert torch.equal(oa[live], ob[pt][live]), t
        assert torch.equal(da[live], ib["depth"][pt][live]), t
        for x, y in ((ra, rb), (ta, tb), (ua, ub)):
            assert torch.equal(x[live], y[pt][live]), t
        if "level" in ia:
            assert torch.equal(ia["level"][live], ib["level"][pt][live]), t
    sa, sb = full_state(a), full_state(b)
    for i in np.nonzero(live.cpu().numpy())[0][:256]:
        assert_env_equal(sa, i, sb, p[i], i)
    assert a.engine.overflow_count() == 0 and b.engine.overflow_count() == 0
    a.close()
    b.close()


@pytest.mark.gpu
def test_gpu_go_explore_equals_the_host_build(libmwb_path, _hostsim_built):
    """The README's Go-Explore loop at 4096 envs in torch ops; the host build replays the same actions, saves and
    pending slots and must reach the same states."""
    from miniworld_b200 import engine
    from miniworld_b200.batched import BatchedMiniWorld
    N, steps = 4096, 30
    mk = lambda: BatchedMiniWorld(short_level("MiniWorld-FourRooms-v0", 20), N, state_bank=14 * 14)
    dev_env = mk()
    dev_env.reset(seed=77)
    rec = []
    go_explore(dev_env, steps, 5, record=rec)
    st_dev = full_state(dev_env)
    ep_dev = host_array(dev_env.episode_state)
    bank_dev = host_array(dev_env.bank_level)
    dev_env.close()
    engine._override_library_for_tests(_hostsim_built)
    try:
        host = mk()
        seed_reset(host, 77 + np.arange(N))
        out = None
        for acts, save, done, pick in rec:
            out = host.step_host(acts, out, render=False)
            assert np.array_equal(out["terminated"] | out["truncated"], done)
            keep = save >= 0
            host.save_states(np.nonzero(keep)[0], save[keep])
            host.next_state[:] = np.where(done, pick, -1)
        st_host = full_state(host)
        assert np.array_equal(host_array(host.episode_state), ep_dev)
        assert np.array_equal(host_array(host.bank_level), bank_dev)
        for i in range(N):
            assert_env_equal(st_dev, i, st_host, i, i)
        assert (ep_dev >= 0).any()
        host.close()
    finally:
        engine._override_library_for_tests(None)


@pytest.mark.gpu
def test_gpu_saves_and_pending_slots_behind_a_busy_stream(libmwb_path):
    """Saves from CUDA-tensor ids and slots and next_state writes, enqueued on a side stream behind a long kernel,
    run in stream order; reset() of a subset loads its pending slots."""
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    N = 1024
    env = BatchedMiniWorld("MiniWorld-PickupObjects-v0", N, state_bank=64)
    env.reset(seed=5)
    st = full_state(env)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)
        ids = torch.arange(64, device="cuda", dtype=torch.int32) * 3
        env.save_states(ids, torch.arange(64, device="cuda", dtype=torch.int32))
        env.next_state[:64] = torch.arange(63, -1, -1, device="cuda", dtype=torch.int32)
        env.reset(env_ids=np.arange(32))
    torch.cuda.synchronize()
    sa = full_state(env)
    ep = host_array(env.episode_state)
    assert ep[:32].tolist() == list(range(63, 31, -1)) and (ep[32:] == -1).all()
    assert host_array(env.next_state)[32:64].tolist() == list(range(31, -1, -1))
    for i in range(32):
        assert_env_equal(sa, i, st, 3 * (63 - i), i)
    assert host_array(env.bank_level).tolist() == [0] * 64
    env.close()
