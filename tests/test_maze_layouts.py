"""Maze layouts (mwb_enable_maze_layouts, BatchedMiniWorld(maze_layouts=True)): designed resets against the host's
Maze.reset(options={"maze": ...}) world field for field, rollouts against host-built followers, the layouts random
carves record, the four arrays across level changes, numpy's pairwise sum, snapshots, sharding and errors.  CPU cases
run the kernels' host build; `gpu` cases run libmwb.so on the device."""
import ctypes

import numpy as np
import pytest

from level_parity import assert_env_equal, full_state, seed_reset, short_level

LEVEL_CASES = [("MiniWorld-MazeS2-v0", {}), ("MiniWorld-MazeS3-v0", {}), ("MiniWorld-MazeS3Fast-v0", {}),
               ("MiniWorld-Maze-v0", {}), ("MiniWorld-Maze-v0", {"num_rows": 3, "num_cols": 5})]
LEVEL_IDS = ["mazes2", "mazes3", "mazes3fast", "maze8", "maze3x5"]


def host_array(view):
    return np.array(view) if isinstance(view, np.ndarray) else view.cpu().numpy()


def spanning_tree(R, C, rs):
    """A random spanning tree of the R x C grid (randomised Kruskal) as a layout."""
    parent = list(range(R * C))

    def find(a):
        while parent[a] != a:
            parent[a] = parent[parent[a]]
            a = parent[a]
        return a
    edges = [(j, i, 1) for j in range(R) for i in range(C - 1)] + [(j, i, 2) for j in range(R - 1) for i in range(C)]
    out = np.zeros((R, C), np.uint8)
    for k in rs.permutation(len(edges)):
        j, i, bit = edges[k]
        a, b = j * C + i, (j * C + i + 1) if bit == 1 else ((j + 1) * C + i)
        if find(a) != find(b):
            parent[find(a)] = find(b)
            out[j, i] |= bit
    return out


def layout_kinds(R, C, rs):
    """All closed, all open, a spanning tree, a random edge subset with loops, and a disconnected layout (a tree with
    one cell cut off).  Bits that point outside the grid are set too: the reset ignores them."""
    tree = spanning_tree(R, C, rs)
    cut = tree.copy()
    cut[R - 1, C - 1] = 0
    if C > 1:
        cut[R - 1, C - 2] &= 2
    if R > 1:
        cut[R - 2, C - 1] &= 1
    return {"closed": np.zeros((R, C), np.uint8), "open": np.full((R, C), 3, np.uint8), "tree": tree,
            "loops": rs.integers(0, 4, (R, C)).astype(np.uint8), "disconnected": cut}


def padded(layout, shape):
    out = np.zeros(shape, np.uint8)
    out[:layout.shape[0], :layout.shape[1]] = layout
    return out


def host_maze(level, kwargs, seed, layout=None, goal=-1, agent=-1, rng_state=None):
    """The host-built world: the level's drop-in class, reset(seed, options) (or its stream from `rng_state`)."""
    from miniworld_b200.engine import generator_from_state
    from miniworld_b200.envs import LEVELS
    cls = LEVELS[level] if isinstance(level, str) else level
    env = cls(device=None, **kwargs)
    options = None if layout is None else {"maze": layout, "goal_cell": goal, "agent_cell": agent}
    if rng_state is not None:
        env._np_random = generator_from_state(rng_state)
        env.reset(options=options)
    else:
        env.reset(seed=seed, options=options)
    return env


def assert_world_equals_host(env, i, host, where):
    """Env i of a batch equals a host-built world: geometry (rooms with their cdf, quads, segments), entities, agent
    pose, colours, sky and light, camera and the stream after the reset."""
    from miniworld_b200 import pack
    from miniworld_b200.engine import RNG_DTYPE, rng_state_of
    w = pack.pack_world(host)
    for got, want, name in zip(env.engine.get_geometry(i), (w["rooms"], w["quads"], w["segs"]), ("rooms", "quads", "segs")):
        assert len(got) == len(want), (where, name, len(got), len(want))
        for f in want.dtype.names:
            if f not in ("reserved", "tex_id"):
                assert np.array_equal(got[f], want[f]), (where, name, f)
    st = env.get_state(rng=True)
    assert np.array_equal(st["agent_pos"][i], host.agent.pos) and st["agent_dir"][i] == host.agent.dir, where
    live = [e for e in range(st["ents"].shape[1]) if st["ents"][i, e]["proto"] >= 0]
    assert len(live) == len(w["ents"]), where
    for e, want, ent in zip(live, w["ents"], w["slot_entities"]):
        for f in ("pos", "dir", "color") if hasattr(ent, "color_vec") else ("pos", "dir"):
            assert np.array_equal(st["ents"][i, e][f], want[f]), (where, e, f)
    assert np.array_equal(st["cam"][i], np.array(w["cam"], float)), (where, "cam")
    envp = np.concatenate([np.asarray(w[k], float) for k in ("sky_color", "light_pos", "light_color", "light_ambient")])
    assert np.array_equal(st["env_params"][i], envp), (where, "env_params")
    assert st["rng"][i] == np.array(rng_state_of(host.np_random), RNG_DTYPE), (where, "rng")


# ------------------------------------------------------------------ CPU (kernels' host build)
PAIRWISE_SUM_SRC = r"""
#include "miniworld_b200/csrc/maze.cuh"
struct ArrayAt {
  const double* a;
  double operator()(int k) const { return a[k]; }
};
extern "C" double pairwise_sum(const double* a, int n) { return np_pairwise_sum(ArrayAt{a}, n); }
"""


def test_pairwise_sum_equals_numpy(tmp_path):
    """numpy's pairwise summation (np.sum) as maze.cuh restates it for the per-env room cdf, compiled for the CPU like
    the kernels' host build, on random doubles of every length 1..800, which a sequential sum misses.  (The default
    room areas, 9 and 0.75, sum exactly in any order, so a level alone does not exercise the order.)"""
    import os
    import subprocess
    from conftest import ROOT
    src, lib_path = tmp_path / "pairwise_sum.cpp", tmp_path / "libpairwise_sum.so"
    src.write_text(PAIRWISE_SUM_SRC)
    subprocess.check_call(["g++", "-x", "c++", "-std=c++17", "-O2", "-ffp-contract=off", "-mfma", "-fPIC", "-shared",
                           "-DMWB_HOSTSIM", "-I", ROOT, "-o", str(lib_path), str(src)], cwd=os.fspath(tmp_path))
    lib = ctypes.CDLL(str(lib_path))
    lib.pairwise_sum.restype = ctypes.c_double
    lib.pairwise_sum.argtypes = [ctypes.c_void_p, ctypes.c_int]
    rs = np.random.default_rng(0)
    sequential_differs = 0
    for n in range(1, 801):
        for a in (rs.random(n), rs.standard_normal(n) * 10.0 ** rs.integers(-6, 6, n)):
            a = np.ascontiguousarray(a)
            assert lib.pairwise_sum(a.ctypes.data, n) == np.sum(a), n
            sequential_differs += float(np.cumsum(a)[-1]) != float(np.sum(a))
    assert sequential_differs > 100


@pytest.mark.parametrize("seeds", ["stream", "episode_seeds"])
@pytest.mark.parametrize("domain_rand", [False, True])
@pytest.mark.parametrize("level,kwargs", LEVEL_CASES, ids=LEVEL_IDS)
def test_designed_reset_equals_the_host_world(hostsim_path, level, kwargs, domain_rand, seeds):
    """Every layout kind, with given and random goal / agent cells: the device reset equals the host's
    Maze.reset(seed, options) field for field, and episode_maze is the layout masked to the grid."""
    from miniworld_b200.batched import BatchedMiniWorld
    kw = dict(kwargs, domain_rand=domain_rand)
    rs = np.random.default_rng(len(level) + 7 * domain_rand)
    from miniworld_b200.envs import LEVELS
    pe = LEVELS[level](device=None, **kwargs)
    R, C = pe.num_rows, pe.num_cols
    kinds = layout_kinds(R, C, rs)
    names = list(kinds)
    N = 2 * len(names)
    env = BatchedMiniWorld(level, N, level_kwargs=kw, maze_layouts=True, episode_seeds=seeds == "episode_seeds")
    lay = np.stack([kinds[names[i % len(names)]] for i in range(N)])
    goal = np.where(np.arange(N) % 2 == 0, rs.integers(0, R * C, N), -1)
    agent = np.where(np.arange(N) % 3 == 0, -1, rs.integers(0, R * C, N))
    env.set_env_maze(np.arange(N), lay, goal, agent)
    s = 300 + np.arange(N)
    if seeds == "episode_seeds":
        env.set_env_seed(np.arange(N), s)
        env.engine.reset()
    else:
        seed_reset(env, s)
    assert (host_array(env.maze_pending) == 0).all()
    rec = host_array(env.episode_maze)
    for i in range(N):
        masked = lay[i].copy()
        masked[:, C - 1] &= 2
        masked[R - 1, :] &= 1
        assert np.array_equal(rec[i], masked), (i, names[i % len(names)])
        host = host_maze(level, kw, int(s[i]), lay[i], int(goal[i]), int(agent[i]))
        assert_world_equals_host(env, i, host, (names[i % len(names)], i))
    assert env.engine.overflow_count() == 0
    env.close()


@pytest.mark.parametrize("level,kwargs", LEVEL_CASES, ids=LEVEL_IDS)
def test_random_carves_record_their_topology(hostsim_path, level, kwargs):
    """Without a pending layout the reset carves as before and episode_maze holds the carve's topology as a layout
    (MazeTemplate.topology_of of the host maze of the same seed); the world is the one a batch without the mode builds."""
    from miniworld_b200.batched import BatchedMiniWorld
    from level_parity import geometry_equal
    N = 4
    env = BatchedMiniWorld(level, N, level_kwargs=kwargs, maze_layouts=True)
    plain = BatchedMiniWorld(level, N, level_kwargs=kwargs)
    seed_reset(env, 40 + np.arange(N))
    seed_reset(plain, 40 + np.arange(N))
    tmpl = env.maze_template
    rec = host_array(env.episode_maze)
    sa, sb = full_state(env), full_state(plain)
    for i in range(N):
        host = host_maze(level, kwargs, 40 + i)
        assert np.array_equal(rec[i], padded(tmpl.layout_of(tmpl.topology_of(host)), env.maze_shape)), i
        assert_env_equal(sa, i, sb, i, i)
        assert geometry_equal(env, i, plain, i), i
    env.close()
    plain.close()


class _Designed:
    """Mixin of the host-reset follower class: each reset builds the next layout queued in `queue` (None: carve)."""
    queue = []
    device_program = None

    def reset(self, *, seed=None, options=None):
        nxt = type(self).queue.pop(0) if type(self).queue else None
        return super().reset(seed=seed, options=nxt if options is None else options)


@pytest.mark.parametrize("level,kwargs,steps", [("MiniWorld-MazeS2-v0", {}, 6), ("MiniWorld-MazeS3-v0", {"domain_rand": True}, 9),
                                                ("MiniWorld-Maze-v0", {"num_rows": 3, "num_cols": 5}, 8)],
                         ids=["mazes2", "mazes3_dr", "maze3x5"])
def test_rollout_equals_host_world_followers(hostsim_path, level, kwargs, steps):
    """300 steps with auto-resets.  Every step, some done envs get a designed layout (an edit of the layout they just
    played, from info["maze"]) and the others carve.  A host-reset batch whose envs build the same layouts with the
    level's own Python _gen_world follows: rewards and flags every step, frames and depth byte-identical every fifth
    step, and the whole state at the end."""
    from miniworld_b200.batched import BatchedMiniWorld
    base = short_level(level, steps)
    follower_cls = type("Designed" + base.__name__, (_Designed, base), {"queue": []})
    N, T = 6, 300
    a = BatchedMiniWorld(base, N, level_kwargs=kwargs, maze_layouts=True, want_depth=True)
    b = BatchedMiniWorld(follower_cls, N, level_kwargs=kwargs, want_depth=True)
    assert a.device_reset and not b.device_reset
    R, C = a.maze_shape
    rs = np.random.default_rng(11)
    first = [spanning_tree(R, C, rs) for _ in range(N)]
    a.set_env_maze(np.arange(N), np.stack(first), goal_cell=0, agent_cell=-1)
    follower_cls.queue[:] = [{"maze": x, "goal_cell": 0, "agent_cell": -1} for x in first]
    seed_reset(a, 70 + np.arange(N))
    b._host_reset(np.arange(N, dtype=np.int32), [70 + i for i in range(N)])   # reset(seed=...) without the render
    b._seeded = True
    oa = ob = None
    designed = 0
    for t in range(T):
        acts = rs.integers(0, a.action_space.n, N).astype(np.int32)
        render = t % 5 == 0
        oa, ob = a.step_host(acts, oa, render=render), b.step_host(acts, ob, render=render)
        for key in ("reward", "terminated", "truncated") + (("obs", "depth") if render else ()):
            assert np.array_equal(oa[key], ob[key]), (t, key)
        done = np.nonzero(oa["terminated"] | oa["truncated"])[0]
        ended = host_array(a.episode_maze)
        queue = []
        for i in done:                                   # ascending: the order the host batch resets them in
            if rs.random() < 0.7:
                lay = ended[i].copy()
                for _ in range(2):
                    lay[rs.integers(0, R), rs.integers(0, C)] ^= 1 << int(rs.integers(0, 2))
                g, ag = int(rs.integers(-1, R * C)), int(rs.integers(-1, R * C))
                a.set_env_maze([i], lay, g, ag)
                queue.append({"maze": lay, "goal_cell": g, "agent_cell": ag})
                designed += 1
            else:
                queue.append(None)
        follower_cls.queue[:] = queue
    assert designed > 30
    from miniworld_b200.engine import RNG_DTYPE, rng_state_of
    sa, sb = a.get_state(rng=True), b.get_state(rng=True)
    if not b.domain_rand:                                # without per-step draws host resets keep the streams in Python
        sb["rng"] = np.array([rng_state_of(w.np_random) for w in b._workers], RNG_DTYPE)
    for key in ("agent_pos", "agent_dir", "step_count", "rng", "cam", "env_params"):
        assert np.array_equal(sa[key], sb[key]), key
    E = sa["ents"].shape[1]                              # the host-reset batch has more (empty) entity slots
    assert (sb["ents"]["proto"][:, E:] < 0).all()
    for i in range(N):
        ea, eb = sa["ents"][i], sb["ents"][i][:E]
        live = ea["proto"] >= 0
        assert np.array_equal(live, eb["proto"] >= 0), i
        for f in ("pos", "dir"):
            assert np.array_equal(ea[f][live], eb[f][live]), (i, f)
        box = live.copy()
        box[sa["agent_slot"][i]] = False                 # the agent's colour is not part of either world
        assert np.array_equal(ea["color"][box], eb["color"][box]), i
    assert a.engine.overflow_count() == 0 and b.engine.overflow_count() == 0
    a.close()
    b.close()


def test_the_arrays_follow_a_numpy_model_across_level_changes(hostsim_path):
    """A table of Maze and non-Maze rows with level changes: writes to the pending arrays are consumed at Maze
    levels, masked to each level's grid, left pending at other levels (which record zeros), and carves record their
    topology; info["maze"] still names the episode that just ended."""
    from miniworld_b200.batched import BatchedMiniWorld
    rows = [short_level("MiniWorld-MazeS2-v0", 5), short_level("MiniWorld-Hallway-v0", 4),
            short_level("MiniWorld-MazeS3-v0", 6)]
    grids = [(2, 2), None, (3, 3)]
    N, T = 9, 150
    env = BatchedMiniWorld(rows, N, per_env_worlds=True, dynamic_levels=True, maze_layouts=True)
    assert env.maze_shape == (3, 3)
    seed_reset(env, 10 + np.arange(N))
    rs = np.random.default_rng(3)
    pend = np.zeros(N, np.uint8)
    nxt = np.zeros((N, 3, 3), np.uint8)
    level = env.env_level.copy()
    episode = host_array(env.episode_maze).copy()
    assert not episode[level == 1].any()
    out = None
    took = carved = parked = 0
    prev_done = np.zeros(N, bool)
    for t in range(T):
        ids = np.nonzero(rs.random(N) < 0.15)[0]
        if ids.size:
            lay = rs.integers(0, 4, (ids.size, 3, 3)).astype(np.uint8)
            env.set_env_maze(ids, lay, goal_cell=-1, agent_cell=-1)
            nxt[ids], pend[ids] = lay, 1
        moved = np.nonzero(rs.random(N) < 0.2)[0]
        new_levels = rs.integers(0, 3, moved.size)
        env.set_env_level(moved, new_levels)
        out = env.step_host(rs.integers(0, 3, N).astype(np.int32), out, render=False)
        rec = host_array(env.episode_maze)
        level_now = env.env_level.copy()
        for i in range(N):
            if not prev_done[i]:
                assert np.array_equal(rec[i], episode[i]), (t, i)        # no reset: the running episode's layout
                continue
            g = grids[level_now[i]]
            if g is None:
                assert not rec[i].any(), (t, i)
                parked += int(pend[i])
            elif pend[i]:
                want = np.zeros((3, 3), np.uint8)
                want[:g[0], :g[1]] = nxt[i][:g[0], :g[1]]
                want[:, g[1] - 1] &= 2
                want[g[0] - 1, :] &= 1
                assert np.array_equal(rec[i], want), (t, i)
                pend[i] = 0
                took += 1
            else:
                assert not rec[i][g[0]:, :].any() and not rec[i][:, g[1]:].any(), (t, i)
                assert np.count_nonzero(np.unpackbits(rec[i][:g[0], :g[1]])) == g[0] * g[1] - 1, (t, i)   # a tree
                carved += 1
        episode = rec.copy()
        assert np.array_equal(host_array(env.maze_pending), pend), t
        prev_done = (out["terminated"] | out["truncated"]).astype(bool)
    assert took > 20 and carved > 5 and parked > 5
    assert env.engine.overflow_count() == 0
    env.close()


def test_reset_and_episode_seeds_reproduce_a_designed_episode(hostsim_path):
    """A layout, its two cells and a seed give one episode, whichever env plays it and when."""
    from miniworld_b200.batched import BatchedMiniWorld
    env = BatchedMiniWorld("MiniWorld-MazeS3-v0", 4, domain_rand=True, maze_layouts=True, episode_seeds=True)
    rs = np.random.default_rng(1)
    lay = spanning_tree(3, 3, rs)
    seed_reset(env, [1, 2, 3, 4])
    for _ in range(7):
        env.step_host(rs.integers(0, 3, 4).astype(np.int32), render=False)
    env.set_env_maze([0, 3], lay, goal_cell=4, agent_cell=8)
    env.set_env_seed([0, 3], 99)
    env.engine.reset(np.array([0, 3], np.int32))
    st = full_state(env)
    assert_env_equal(st, 0, st, 3, "replay")
    assert_world_equals_host(env, 3, host_maze("MiniWorld-MazeS3-v0", {"domain_rand": True}, 99, lay, 4, 8), "host")
    env.close()


def test_snapshots_within_and_across_modes(hostsim_path):
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import EngineError
    rows = ["MiniWorld-MazeS2-v0", "MiniWorld-OneRoom-v0"]
    make = lambda layouts: BatchedMiniWorld(rows, 4, per_env_worlds=True, maze_layouts=layouts)
    a = make(True)
    seed_reset(a, [1, 2, 3, 4])
    a.set_env_maze([0, 1, 2], np.full((2, 2), 3, np.uint8), goal_cell=[3, -1, 0])
    blob = a.snapshot()
    st, pend, nxt, rec = full_state(a), host_array(a.maze_pending).copy(), host_array(a.next_maze).copy(), \
        host_array(a.episode_maze).copy()
    acts = np.ones(4, np.int32)
    for _ in range(12):
        a.step_host(acts, render=False)
    after = full_state(a), host_array(a.episode_maze).copy()
    a.restore(blob)
    assert np.array_equal(host_array(a.maze_pending), pend) and np.array_equal(host_array(a.next_maze), nxt)
    assert np.array_equal(host_array(a.episode_maze), rec)
    s2 = full_state(a)
    for i in range(4):
        assert_env_equal(st, i, s2, i, i)
    for _ in range(12):
        a.step_host(acts, render=False)
    for i in range(4):
        assert_env_equal(after[0], i, full_state(a), i, ("again", i))
    assert np.array_equal(host_array(a.episode_maze), after[1])
    b = make(False)
    plain = b.snapshot()
    assert plain[:4].tobytes() in (b"MWBW", b"MWBX")              # blobs without the mode keep their mark
    with pytest.raises(EngineError, match="error -6"):
        b.restore(blob)
    with pytest.raises(EngineError, match="error -6"):
        a.restore(plain)
    a.close()
    b.close()


def test_errors(hostsim_path):
    from miniworld_b200 import pack
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import Engine, EngineError
    from miniworld_b200.envs import LEVELS
    from miniworld_b200.maze_lowering import MazeTemplate
    from miniworld_b200.program import ResetProgram
    with pytest.raises(ValueError, match="Maze-family"):
        BatchedMiniWorld("MiniWorld-FourRooms-v0", 2, maze_layouts=True)
    host_only = type("HostOnlyMaze", (LEVELS["MiniWorld-MazeS2-v0"],), {"device_program": None})
    with pytest.raises(TypeError, match="host"):
        BatchedMiniWorld(host_only, 2, maze_layouts=True)         # a Maze that resets on the host
    with pytest.raises(TypeError, match="host"):
        BatchedMiniWorld("MiniWorld-Maze-v0", 2, level_kwargs={"room_size": 2.9}, maze_layouts=True)
    env = BatchedMiniWorld("MiniWorld-MazeS3-v0", 4, maze_layouts=True)
    with pytest.raises(EngineError, match="error -6"):
        env.engine.enable_maze_layouts()                          # already on
    for args in [([0], np.zeros((2, 3), np.uint8)), ([0], np.zeros((3, 3), np.float32)), ([0], np.full((3, 3), 4)),
                 ([0, 1], np.zeros((3, 3, 3), np.uint8)), ([4], np.zeros((3, 3), np.uint8)),
                 ([0], np.zeros((3, 3), np.uint8), 9), ([0], np.zeros((3, 3), np.uint8), -1, -2),
                 ([0, 1], np.zeros((3, 3), np.uint8), [1, 2, 3])]:
        with pytest.raises(ValueError):
            env.set_env_maze(*args)
    assert not host_array(env.maze_pending).any() and (host_array(env.next_maze_cells) == -1).all()
    env.set_env_maze([1, 2, 1], np.stack([np.full((3, 3), k, np.uint8) for k in (1, 2, 3)]), [4, 5, 6])
    assert host_array(env.next_maze)[1].max() == 3 and host_array(env.next_maze_cells)[1].tolist() == [6, -1]
    env.close()
    off = BatchedMiniWorld("MiniWorld-MazeS3-v0", 2)
    for name in ("next_maze", "next_maze_cells", "maze_pending", "episode_maze"):
        with pytest.raises(EngineError, match="error -6"):
            off.engine.state_array(name)
    with pytest.raises(RuntimeError):
        off.next_maze
    with pytest.raises(EngineError, match="error -5"):
        off.engine.enable_maze_layouts()                          # sized for trees only
    off.close()
    # the C ABI: no Maze level, too small for an all-open maze
    pe = LEVELS["MiniWorld-Hallway-v0"](device=None)
    prog = ResetProgram()
    pe.device_program(prog)
    lv = dict(rule=(1, 0), max_episode_steps=250, params=pe.params, geometry=pack.pack_geometry(pe), ops=prog.op_array())
    tmpl = MazeTemplate(LEVELS["MiniWorld-MazeS2-v0"])              # 4 cells, 4 edges: 8 rooms, 32 quads, 16 segments
    cdf = pack.room_cdf(LEVELS["MiniWorld-MazeS2-v0"](device=None).room_probs)
    def engine(**caps):
        eng = Engine(3, max_ents=2, **caps)
        eng.set_protos(prog.proto_array())
        eng.set_levels([lv, lv], [0, 1, 1])
        return eng
    tree = dict(max_rooms=7, max_quads=30, max_segs=16)
    eng = engine(**tree)
    with pytest.raises(EngineError, match="error -6"):
        eng.enable_maze_layouts()                                 # no Maze level
    eng.set_level_maze(1, tmpl, cdf)
    with pytest.raises(EngineError, match="error -5"):
        eng.enable_maze_layouts()                                 # sized for trees only
    eng.close()
    eng = engine(max_rooms=8, max_quads=32, max_segs=16)
    eng.set_level_maze(1, tmpl, cdf)
    eng.enable_maze_layouts()
    assert eng.state_array("next_maze").shape == (3, 4) and eng.state_array("next_maze_cells").shape == (3, 2)
    eng.close()


def _shard_worker(rank, port, hostsim, q):
    import os
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=2)
    from miniworld_b200 import engine
    from miniworld_b200.dist import ShardedMiniWorld
    engine._override_library_for_tests(hostsim)
    env = ShardedMiniWorld(short_level("MiniWorld-MazeS3-v0", 7), 7, dist=dist, maze_layouts=True)
    seed_reset(env.local, [1000 + env.start + k for k in range(env.count)])
    outs = shard_run(env.local, env.start, 40, 7, rank, lambda a: env.scatter_actions(a, like=torch.zeros(1)),
                     env.gather_to_root)
    if rank == 0:
        q.put(outs)
    dist.barrier()
    dist.destroy_process_group()


def shard_layouts(done, start, t):
    """Layouts the done envs of a shard starting at global env `start` get at step t (envs with (g + t) % 3 == 0 carve)."""
    g = start + np.arange(len(done))
    ids = np.nonzero(done & ((g + t) % 3 != 0))[0]
    return ids, np.stack([np.full((3, 3), (g[i] + t) % 4, np.uint8) for i in ids]) if ids.size else None


def shard_run(env, start, steps, total, rank=0, scatter=None, gather=None):
    import torch
    acts_all = np.random.default_rng(5).integers(0, 3, size=(steps, total), dtype=np.int32)
    outs, out = [], None
    for t in range(steps):
        acts = acts_all[t] if scatter is None else scatter(torch.as_tensor(acts_all[t]) if rank == 0 else None).numpy()
        out = env.step_host(acts, out, render=t == steps - 1)
        ids, lay = shard_layouts((out["terminated"] | out["truncated"]).astype(bool), start, t)
        if ids.size:
            env.set_env_maze(ids, lay, goal_cell=(start + ids) % 9)
        got = [out["obs"], out["reward"], np.array(env.episode_maze), np.array(env.maze_pending)]
        if gather is not None:
            got = [gather(torch.as_tensor(x)).numpy() if rank == 0 else gather(torch.as_tensor(x)) for x in got]
        outs.append([np.array(x) for x in got] if rank == 0 else None)
    return outs


def test_sharded_layout_writes_equal_one_process(hostsim_path):
    """Two gloo ranks that write their envs' layouts into their local batches equal one process: a layout belongs to an
    env, so no offset is involved."""
    import os
    import torch.multiprocessing as mp
    from miniworld_b200.batched import BatchedMiniWorld
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 37000 + os.getpid() % 2000
    procs = [ctx.Process(target=_shard_worker, args=(r, port, hostsim_path, q)) for r in range(2)]
    for p in procs:
        p.start()
    sharded = q.get(timeout=300)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    env = BatchedMiniWorld(short_level("MiniWorld-MazeS3-v0", 7), 7, maze_layouts=True)
    seed_reset(env, 1000 + np.arange(7))
    one = shard_run(env, 0, 40, 7)
    for t, (x, y) in enumerate(zip(one, sharded)):
        for k in (1, 2, 3):
            assert np.array_equal(x[k], y[k]), (t, k)
    assert np.array_equal(one[-1][0], sharded[-1][0]) and 0 < one[-1][0].mean() < 255
    env.close()


# ------------------------------------------------------------------ GPU (libmwb.so)
def accel_edit(torch, layouts, gen, flips=3):
    """ACCEL's edit in torch ops: flip `flips` random edge bits of every layout."""
    n, R, C = layouts.shape
    out = layouts.clone()
    for _ in range(flips):
        cell = torch.randint(0, R * C, (n,), device=layouts.device, generator=gen)
        bit = torch.randint(0, 2, (n,), device=layouts.device, generator=gen).to(torch.uint8)
        flat = out.view(n, R * C)
        flat[torch.arange(n, device=layouts.device), cell] ^= (1 << bit).to(torch.uint8)
    return out


@pytest.mark.gpu
def test_gpu_accel_loop_matches_the_host_build(libmwb_path):
    """4096 envs, 300 steps of an ACCEL loop in torch ops, never synchronising: the ended episodes' layouts
    (info["maze"]) are scored by return, the high-regret ones edited and written to next_maze / maze_pending of the
    done envs.  A sample of envs replays on the host build with the recorded actions and writes: flags, rewards and
    info["maze"] every step, state at the end, frames at three steps."""
    import subprocess
    import torch
    from conftest import ROOT
    from miniworld_b200 import engine
    from miniworld_b200.batched import BatchedMiniWorld
    level = short_level("MiniWorld-MazeS3-v0", 12)
    N, T = 4096, 300
    frames_at = (60, 180, T - 1)
    env = BatchedMiniWorld(level, N, domain_rand=True, maze_layouts=True)
    dev = torch.device("cuda")
    gen = torch.Generator(device="cuda")
    gen.manual_seed(3)
    env.reset(seed=500)
    ret = torch.zeros(N, dtype=torch.float64, device=dev)
    acts = torch.randint(0, 3, (T, N), dtype=torch.int32, device=dev, generator=gen)
    sample = np.sort(np.random.default_rng(4).choice(N, 64, replace=False))
    sample_t = torch.as_tensor(sample, device=dev)
    hist = {k: [] for k in ("maze", "cells", "pending", "rew", "te", "tr")}
    frames = {}
    for t in range(T):
        obs, rew, te, tr, info = env.step(acts[t])
        ret += rew
        done = te | tr
        regret = done & (ret < 0.5)                                 # unsolved levels: edit and replay them
        edited = accel_edit(torch, info["maze"], gen)
        env.next_maze.copy_(torch.where(regret[:, None, None], edited, env.next_maze))
        cells = torch.randint(-1, 9, (N, 2), dtype=torch.int32, device=dev, generator=gen)
        env.next_maze_cells.copy_(torch.where(regret[:, None], cells, env.next_maze_cells))
        env.maze_pending.copy_(torch.where(regret, torch.ones_like(env.maze_pending), env.maze_pending))
        ret[done] = 0
        for k, v in (("maze", info["maze"]), ("rew", rew), ("te", te), ("tr", tr), ("cells", env.next_maze_cells),
                     ("pending", env.maze_pending)):
            hist[k].append(v[sample_t].clone())
        hist.setdefault("next", []).append(env.next_maze[sample_t].clone())
        if t in frames_at:
            frames[t] = obs[sample_t].clone()
    final = full_state(env)
    hist = {k: torch.stack(v).cpu().numpy() for k, v in hist.items()}
    frames = {t: f.cpu().numpy() for t, f in frames.items()}
    assert env.engine.overflow_count() == 0
    assert hist["te"].sum() + hist["tr"].sum() > 1000 and hist["pending"].sum() > 100
    acts = acts.cpu().numpy()
    env.close()

    lib = subprocess.check_output([ROOT + "/tests/hostsim/build.sh"]).decode().strip().splitlines()[-1]
    engine._override_library_for_tests(lib)
    try:
        host = BatchedMiniWorld(level, len(sample), domain_rand=True, maze_layouts=True)
        seed_reset(host, 500 + sample)
        out = None
        for t in range(T):
            out = host.step_host(acts[t, sample], out, render=t in frames_at)
            assert np.array_equal(out["reward"], hist["rew"][t]), t
            assert np.array_equal(out["terminated"].astype(bool), hist["te"][t]), t
            assert np.array_equal(out["truncated"].astype(bool), hist["tr"][t]), t
            assert np.array_equal(host.episode_maze, hist["maze"][t]), t
            if t in frames_at:
                d = np.abs(out["obs"].astype(int) - frames[t].astype(int))
                assert d.max() <= 1 and 0 < frames[t].mean() < 255, (t, int(d.max()))
            host.next_maze[:] = hist["next"][t]
            host.next_maze_cells[:] = hist["cells"][t]
            host.maze_pending[:] = hist["pending"][t]
        st = full_state(host)
        for j, i in enumerate(sample):
            assert_env_equal(st, j, final, i, ("final", int(i)))
        host.close()
    finally:
        engine._override_library_for_tests(None)


@pytest.mark.gpu
@pytest.mark.parametrize("level,kind", [("MiniWorld-Maze-v0", "open"), ("MiniWorld-Maze-v0", "loops"),
                                        ("MiniWorld-MazeS3-v0", "tree"), ("MiniWorld-MazeS3-v0", "disconnected")])
def test_gpu_designed_frames_match_the_pixel_oracle(libmwb_path, softgl_lib, level, kind):
    """Frames of designed mazes against oracle/softgl.c rendering the host-built world (same state): the all-open 8 x 8
    maze's long sight lines put the most quads into K2's candidate lists, and no list overflows."""
    from test_render_paths import assert_matches, oracle_frame
    from miniworld_b200.batched import BatchedMiniWorld
    N = 24
    env = BatchedMiniWorld(level, N, maze_layouts=True, want_depth=True)
    R, C = env.maze_shape
    rs = np.random.default_rng(5)
    lay = np.stack([layout_kinds(R, C, rs)[kind] for _ in range(N)])
    env.set_env_maze(np.arange(N), lay, goal_cell=rs.integers(-1, R * C, N), agent_cell=-1)
    obs, _ = env.reset(seed=60)
    obs = obs.cpu().numpy()
    depth = env._bufs["depth"].cpu().numpy()
    assert env.engine.overflow_count() == 0
    st = env.get_state(rng=True)
    for i in range(N):
        host = host_maze(level, {}, 60 + i, lay[i], *[int(x) for x in host_array(env.next_maze_cells)[i]])
        assert np.array_equal(st["agent_pos"][i], host.agent.pos), i
        want_rgb, want_depth = oracle_frame(host, 80, 60, 8)
        assert_matches(obs[i], depth[i], want_rgb, want_depth, (kind, i))
    env.close()


@pytest.mark.gpu
def test_gpu_layouts_written_on_a_side_stream_behind_a_busy_stream(libmwb_path):
    """Layouts written on a side stream behind a long-running kernel are seen by the step (auto-reset) and the reset that
    run behind them on that stream: `a` writes and goes on at once, `b` waits for the device after the same write."""
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    N = 64
    level = short_level("MiniWorld-MazeS3-v0", 3)
    a, b = (BatchedMiniWorld(level, N, domain_rand=True, maze_layouts=True) for _ in range(2))
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        acts = torch.randint(0, 3, (N,), dtype=torch.int32, device="cuda")
        for e in (a, b):
            e.reset(seed=5)
            for _ in range(3):
                _, _, te, tr, _ = e.step(acts)
            done = te | tr
        assert int(done.sum()) > N // 2
        for k, call in enumerate(("step", "reset")):
            lay = torch.full((N, 3, 3), 3 - k, dtype=torch.uint8, device="cuda")
            b.next_maze.copy_(lay)
            b.maze_pending.fill_(1)
            torch.cuda.synchronize()
            torch.cuda._sleep(100_000_000)
            a.next_maze.copy_(lay)
            a.maze_pending.fill_(1)
            if call == "step":
                a.step(acts)
                b.step(acts)
            else:
                a.reset()
                b.reset()
            torch.cuda.synchronize()
            sa, sb = full_state(a), full_state(b)
            for i in range(N):
                assert_env_equal(sa, i, sb, i, call)
            took = done if call == "step" else torch.ones_like(done)
            assert torch.equal(a.episode_maze, b.episode_maze), call
            assert bool((a.maze_pending[took] == 0).all()) and bool((a.maze_pending[~took] == 1).all()), call
            assert bool((a.episode_maze[took].flatten(1).amax(1) > 0).all()), call
    a.close()
    b.close()


@pytest.mark.gpu
def test_gpu_reset_takes_pending_layouts(libmwb_path):
    """reset() builds the pending layouts, and equals the host build's reset of the same layouts and seeds."""
    from miniworld_b200.batched import BatchedMiniWorld
    N = 16
    env = BatchedMiniWorld("MiniWorld-MazeS3-v0", N, maze_layouts=True, domain_rand=True)
    rs = np.random.default_rng(2)
    lay = np.stack([spanning_tree(3, 3, rs) for _ in range(N)])
    env.set_env_maze(np.arange(N), lay, goal_cell=rs.integers(-1, 9, N), agent_cell=rs.integers(-1, 9, N))
    cells = host_array(env.next_maze_cells)
    env.reset(seed=80)
    assert not host_array(env.maze_pending).any() and np.array_equal(host_array(env.episode_maze), lay)
    for i in range(N):
        host = host_maze("MiniWorld-MazeS3-v0", {"domain_rand": True}, 80 + i, lay[i], int(cells[i, 0]), int(cells[i, 1]))
        assert_world_equals_host(env, i, host, i)
    env.close()
