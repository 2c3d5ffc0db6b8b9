"""Start poses (mwb_enable_start_poses, BatchedMiniWorld(start_poses=True)): designed resets against the host's
MiniWorldEnv.reset(options={"poses": ..., "agent_pose": ...}) world field for field, rollouts against host-reset
followers, the four arrays across level changes and subset resets, snapshots and errors.  CPU cases run the kernels'
host build; `gpu` cases run libmwb.so on the device."""
import math

import numpy as np
import pytest

from level_parity import assert_env_equal, full_state, seed_reset, short_level
from test_maze_layouts import assert_world_equals_host, host_array, spanning_tree

DEVICE_LEVELS = ["MiniWorld-CollectHealth-v0", "MiniWorld-FourRooms-v0", "MiniWorld-Hallway-v0", "MiniWorld-MazeS2-v0",
                 "MiniWorld-MazeS3-v0", "MiniWorld-MazeS3Fast-v0", "MiniWorld-Maze-v0", "MiniWorld-OneRoom-v0",
                 "MiniWorld-OneRoomS6-v0", "MiniWorld-OneRoomS6Fast-v0", "MiniWorld-PickupObjects-v0",
                 "MiniWorld-PutNext-v0", "MiniWorld-RoomObjects-v0", "MiniWorld-Sidewalk-v0", "MiniWorld-Sign-v0",
                 "MiniWorld-ThreeRooms-v0", "MiniWorld-TMaze-v0", "MiniWorld-TMazeLeft-v0", "MiniWorld-TMazeRight-v0",
                 "MiniWorld-WallGap-v0", "MiniWorld-YMaze-v0", "MiniWorld-YMazeLeft-v0", "MiniWorld-YMazeRight-v0"]


def host_env(level, kwargs, seed, options=None):
    from miniworld_b200.envs import LEVELS
    env = (LEVELS[level] if isinstance(level, str) else level)(device=None, **kwargs)
    env.reset(seed=seed, options=options)
    return env


def small_slots(level, kwargs, slots):
    """The designable non-agent slots whose entity is small enough that a design there never leaves a later searched
    placement without a free spot (Sidewalk's and WallGap's building covers the floor plan)."""
    pe = host_env(level, kwargs, 0)
    return [s["slot"] for s in slots if s["designable"] and not s["agent"] and pe.entities[s["slot"]].radius < 3]


def designs(level, kwargs, slots, rs):
    """One design per env: (poses {slot: (x, z, dir)}, agent_pose or None), covering agent only, the first slot only,
    every designable slot with dirs and with NaN dirs, the agent's slot row, non-finite x, a slot beyond the level's
    count and a pose far outside the floor plan."""
    pe = host_env(level, kwargs, 1)
    lo = np.array([min(r.min_x for r in pe.rooms), min(r.min_z for r in pe.rooms)])
    hi = np.array([max(r.max_x for r in pe.rooms), max(r.max_z for r in pe.rooms)])
    pose = lambda d=None: tuple(lo + rs.random(2) * (hi - lo)) + (rs.uniform(-3, 3) if d is None else d,)
    small = small_slots(level, kwargs, slots)
    agent = [s["slot"] for s in slots if s["agent"]][0]
    out = [({}, pose()),                                                     # agent only, dir given
           ({s: pose(math.nan) for s in small[:1]}, None),                  # first slot only, level / drawn dir
           ({s: pose() for s in small}, pose(math.nan)),                    # every slot, agent dir from the level
           ({s: pose(math.nan) for s in small}, None),
           ({agent: pose()}, None),                                          # the agent's slot row
           ({s: (math.nan, 1.0, 0.0) for s in small}, (math.inf, 2.0, 0.0)),   # non-finite x: as the level wrote it
           ({len(slots) + 2: pose()}, (hi[0] + 50.0, lo[1] - 40.0, 1.0))]   # beyond the count; outside the floor plan
    return out


def write_designs(env, ds):
    """In-place writes of every row as given (NaN and inf included), through numpy or torch."""
    if env.engine.host_memory:
        row = lambda p: np.asarray(p, np.float64)
    else:
        import torch
        row = lambda p: torch.tensor([float(v) for v in p], dtype=torch.float64, device=env.next_pose.device)
    for i, (poses, agent) in enumerate(ds):
        for s, p in poses.items():
            if s < env.engine.max_ents:
                env.next_pose[i, s] = row(p)
        if agent is not None:
            env.next_agent_pose[i] = row(agent)
        env.pose_pending[i] = 1


def options_of(poses, agent):
    return {"poses": dict(poses), **({} if agent is None else {"agent_pose": agent})}


@pytest.mark.parametrize("mode", ["plain", "dr", "dr_episode_seeds"])
@pytest.mark.parametrize("level", DEVICE_LEVELS)
def test_designed_resets_equal_the_host_world(hostsim_path, level, mode):
    """Every design kind: the device reset equals the host's reset(seed, options) field for field, episode_start is
    the agent's pose, and pose_pending is cleared while the rows stay."""
    from miniworld_b200.batched import BatchedMiniWorld
    kwargs = {} if level == "MiniWorld-Sign-v0" or mode == "plain" else {"domain_rand": True}
    rs = np.random.default_rng(len(level) + len(mode))
    probe = BatchedMiniWorld(level, 1, level_kwargs=kwargs, start_poses=True)
    slots = probe.level_slots[0]
    probe.close()
    ds = designs(level, kwargs, slots, rs)
    N = len(ds)
    env = BatchedMiniWorld(level, N, level_kwargs=kwargs, start_poses=True, episode_seeds=mode == "dr_episode_seeds")
    write_designs(env, ds)
    rows = host_array(env.next_pose).copy()
    s = 700 + np.arange(N)
    if mode == "dr_episode_seeds":
        env.set_env_seed(np.arange(N), s)
        env.engine.reset()
    else:
        seed_reset(env, s)
    assert not host_array(env.pose_pending).any() and np.array_equal(host_array(env.next_pose), rows, equal_nan=True)
    st = env.get_state()
    start = host_array(env.episode_start)
    for i, (poses, agent) in enumerate(ds):
        host = host_env(level, kwargs, int(s[i]), options_of(poses, agent))
        assert_world_equals_host(env, i, host, (level, mode, i))
        assert np.array_equal(start[i], [st["agent_pos"][i][0], st["agent_pos"][i][2], st["agent_dir"][i]]), i
    assert env.engine.overflow_count() == 0
    env.close()


def test_level_slots_name_what_each_reset_fills(hostsim_path):
    from miniworld_b200.batched import BatchedMiniWorld
    env = BatchedMiniWorld(["MiniWorld-FourRooms-v0", "MiniWorld-PickupObjects-v0"], 2, start_poses=True)
    four, pick = env.level_slots
    assert [(s["kind"], s["agent"], s["designable"]) for s in four] == [("Box", False, True), ("Agent", True, True)]
    assert pick[-1]["agent"] and all(not s["agent"] for s in pick[:-1]) and "Key" in pick[0]["kind"]
    env.close()
    sign = BatchedMiniWorld("MiniWorld-Sign-v0", 1, start_poses=True).level_slots[0]
    assert [s["designable"] for s in sign] == [True] * 6 + [False, True] and sign[6]["kind"] == "TextFrame"


@pytest.mark.parametrize("domain_rand", [False, True])
def test_designs_win_over_designed_maze_cells(hostsim_path, domain_rand):
    """A designed layout with goal and agent cells, and designed poses for the goal box, the agent or both."""
    from miniworld_b200.batched import BatchedMiniWorld
    kw = {"domain_rand": domain_rand}
    env = BatchedMiniWorld("MiniWorld-MazeS3-v0", 4, level_kwargs=kw, maze_layouts=True, start_poses=True)
    rs = np.random.default_rng(4)
    lay = np.stack([spanning_tree(3, 3, rs) for _ in range(4)])
    env.set_env_maze(np.arange(4), lay, goal_cell=[0, 4, 8, -1], agent_cell=[8, 0, 4, 2])
    ds = [({0: (5.0, 5.0, 0.3)}, None), ({}, (12.0, 2.0, math.nan)), ({0: (1.0, 1.0, math.nan)}, (20.0, 20.0, 1.0)),
          ({}, None)]
    write_designs(env, ds)
    cells = host_array(env.next_maze_cells)
    seed_reset(env, 90 + np.arange(4))
    for i, (poses, agent) in enumerate(ds):
        opts = dict(options_of(poses, agent), maze=lay[i], goal_cell=int(cells[i, 0]), agent_cell=int(cells[i, 1]))
        assert_world_equals_host(env, i, host_env("MiniWorld-MazeS3-v0", kw, 90 + i, opts), i)
    env.close()


class _Designed:
    """Mixin of the host-reset follower class: each reset takes the next options queued in `queue` (None: none)."""
    queue = []
    device_program = None

    def reset(self, *, seed=None, options=None):
        nxt = type(self).queue.pop(0) if type(self).queue else None
        return super().reset(seed=seed, options=nxt if options is None else options)


@pytest.mark.parametrize("level,kwargs,steps", [("MiniWorld-OneRoom-v0", {}, 8),
                                                ("MiniWorld-FourRooms-v0", {"domain_rand": True}, 10),
                                                ("MiniWorld-TMaze-v0", {}, 9)],
                         ids=["oneroom", "fourrooms_dr", "tmaze"])
def test_rollout_equals_host_world_followers(hostsim_path, level, kwargs, steps):
    """300 steps with auto-resets; every step numpy writes designs for some done envs.  A host-reset batch whose envs
    reset with the same options follows: rewards, flags, info["start"] every step, frames and depth byte-identical
    every fifth step."""
    from miniworld_b200.batched import BatchedMiniWorld
    base = short_level(level, steps)
    follower_cls = type("Designed" + base.__name__, (_Designed, base), {"queue": []})
    N, T = 6, 300
    a = BatchedMiniWorld(base, N, level_kwargs=kwargs, start_poses=True, want_depth=True)
    b = BatchedMiniWorld(follower_cls, N, level_kwargs=kwargs, want_depth=True)
    assert a.device_reset and not b.device_reset
    slots = a.level_slots[0]
    agent_slot = [s["slot"] for s in slots if s["agent"]][0]
    seed_reset(a, 70 + np.arange(N))
    b._host_reset(np.arange(N, dtype=np.int32), [70 + i for i in range(N)])
    b._seeded = True
    rs = np.random.default_rng(11)
    oa = ob = None
    designed = 0
    for t in range(T):
        acts = rs.integers(0, a.action_space.n, N).astype(np.int32)
        render = t % 5 == 0
        oa, ob = a.step_host(acts, oa, render=render), b.step_host(acts, ob, render=render)
        for key in ("reward", "terminated", "truncated") + (("obs", "depth") if render else ()):
            assert np.array_equal(oa[key], ob[key]), (t, key)
        st = b.get_state()
        start = host_array(a.episode_start)
        done = np.nonzero(oa["terminated"] | oa["truncated"])[0]
        queue = []
        a.next_pose[:] = np.nan                           # this step's designs only
        a.next_agent_pose[:] = np.nan
        for i in done:                                    # ascending: the order the host batch resets them in
            if rs.random() < 0.7:
                goal = (float(rs.uniform(1, 5)), float(rs.uniform(1, 5)), float(rs.choice([np.nan, 0.5])))
                agent = (float(rs.uniform(1, 5)), float(rs.uniform(1, 5)), float(rs.choice([np.nan, -1.0])))
                a.set_env_pose([i], 0, goal[0], goal[1], goal[2])
                a.set_env_pose([i], "agent", agent[0], agent[1], agent[2])
                queue.append({"poses": {0: goal}, "agent_pose": agent})
                designed += 1
            else:
                queue.append(None)
        follower_cls.queue[:] = queue
        for i in range(N):
            if st["step_count"][i] == 0 and t:            # reset inside this step: info["start"] is its pose
                assert np.array_equal(start[i], [st["agent_pos"][i][0], st["agent_pos"][i][2], st["agent_dir"][i]])
    assert designed > 30
    from miniworld_b200.engine import RNG_DTYPE, rng_state_of
    sa, sb = a.get_state(rng=True), b.get_state(rng=True)
    if not b.domain_rand:
        sb["rng"] = np.array([rng_state_of(w.np_random) for w in b._workers], RNG_DTYPE)
    for key in ("agent_pos", "agent_dir", "step_count", "rng", "cam", "env_params"):
        assert np.array_equal(sa[key], sb[key]), key
    assert agent_slot == sa["agent_slot"][0]
    a.close()
    b.close()


def test_the_arrays_follow_a_numpy_model_across_level_changes(hostsim_path):
    """A table with level changes: a pending design is consumed by the next reset at any level (subset resets
    included), the rows stay, slot rows land in the slot of the level the reset runs, the agent row reaches every
    level's agent, and episode_start names the running episode."""
    from miniworld_b200.batched import BatchedMiniWorld
    rows = [short_level("MiniWorld-OneRoom-v0", 5), short_level("MiniWorld-PickupObjects-v0", 4),
            short_level("MiniWorld-MazeS2-v0", 6)]
    N, T = 9, 150
    env = BatchedMiniWorld(rows, N, per_env_worlds=True, dynamic_levels=True, start_poses=True)
    seed_reset(env, 10 + np.arange(N))
    rs = np.random.default_rng(3)
    pend = np.zeros(N, np.uint8)
    agent_row = np.full((N, 3), np.nan)
    slot0 = np.full((N, 3), np.nan)
    out = None
    took = 0

    def check(reset, t):
        nonlocal took
        st = env.get_state()
        start = host_array(env.episode_start)
        for i in np.nonzero(reset)[0]:
            if pend[i]:
                a = st["agent_slot"][i]
                if np.isfinite(agent_row[i, 0]):
                    assert np.array_equal(start[i], agent_row[i]), (t, i)
                elif a == 0 and np.isfinite(slot0[i, 0]):
                    assert np.array_equal(start[i, :2], slot0[i, :2]), (t, i)
                if np.isfinite(slot0[i, 0]) and a != 0:
                    assert np.array_equal(st["ents"][i, 0]["pos"][[0, 2]], slot0[i, :2]), (t, i)
                pend[i] = 0
                took += 1
            assert np.array_equal(start[i], [st["agent_pos"][i][0], st["agent_pos"][i][2], st["agent_dir"][i]]), (t, i)
        assert np.array_equal(host_array(env.pose_pending), pend), t
        assert np.array_equal(host_array(env.next_agent_pose), agent_row, equal_nan=True), t
        assert np.array_equal(host_array(env.next_pose)[:, 0], slot0, equal_nan=True), t

    prev_done = np.zeros(N, bool)
    for t in range(T):
        ids = np.nonzero(rs.random(N) < 0.15)[0]
        if ids.size:
            xz = rs.uniform(1, 4, (ids.size, 2))
            if t % 2:
                env.set_env_pose(ids, "agent", xz[:, 0], xz[:, 1], 0.25)
                agent_row[ids] = np.c_[xz, np.full(ids.size, 0.25)]
            else:
                env.set_env_pose(ids, 0, xz[:, 0], xz[:, 1])
                slot0[ids] = np.c_[xz, np.full(ids.size, np.nan)]
            pend[ids] = 1
        if t % 37 == 5:                                   # a subset reset outside the step
            sub = np.array([1, 4], np.int32)
            env.engine.reset(sub)
            check(np.isin(np.arange(N), sub), t)
            prev_done[sub] = False                        # the step that follows is a real step
        env.set_env_level(np.nonzero(rs.random(N) < 0.2)[0], 0)
        out = env.step_host(rs.integers(0, 3, N).astype(np.int32), out, render=False)
        check(prev_done, t)
        prev_done = (out["terminated"] | out["truncated"]).astype(bool)
    assert took > 20
    env.close()


def test_snapshots_within_and_across_modes(hostsim_path):
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import EngineError
    make = lambda on: BatchedMiniWorld("MiniWorld-FourRooms-v0", 4, start_poses=on)
    a = make(True)
    seed_reset(a, [1, 2, 3, 4])
    a.set_env_pose([0, 2], "agent", 3.0, 4.0, 1.0)
    blob = a.snapshot()
    assert blob[:4].tobytes() == b"MwBS"
    st = full_state(a)
    arrays = [host_array(v).copy() for v in (a.next_pose, a.next_agent_pose, a.pose_pending, a.episode_start)]
    acts = np.full(4, 2, np.int32)
    for _ in range(12):
        a.step_host(acts, render=False)
    a.restore(blob)
    for want, v in zip(arrays, (a.next_pose, a.next_agent_pose, a.pose_pending, a.episode_start)):
        assert np.array_equal(host_array(v), want, equal_nan=True)
    for i in range(4):
        assert_env_equal(st, i, full_state(a), i, i)
    b = make(False)
    plain = b.snapshot()
    assert plain[:4].tobytes() == b"MWBS"                    # blobs without the mode keep their mark
    with pytest.raises(EngineError, match="error -6"):
        b.restore(blob)
    with pytest.raises(EngineError, match="error -6"):
        a.restore(plain)
    a.close()
    b.close()


def test_errors(hostsim_path):
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import EngineError
    from miniworld_b200.envs import LEVELS
    host_only = type("HostOnlyRoom", (LEVELS["MiniWorld-OneRoom-v0"],), {"device_program": None})
    with pytest.raises(TypeError, match="host"):
        BatchedMiniWorld(host_only, 2, start_poses=True)
    env = BatchedMiniWorld("MiniWorld-OneRoom-v0", 4, start_poses=True)
    assert env.next_pose.shape == (4, env.engine.max_ents, 3) and np.isnan(host_array(env.next_pose)).all()
    assert np.isnan(host_array(env.next_agent_pose)).all()
    with pytest.raises(EngineError, match="error -6"):
        env.engine.enable_start_poses()                          # already on
    for args in [([4], 0, 1.0, 1.0), ([-1], 0, 1.0, 1.0), ([0], 2, 1.0, 1.0), ([0], -1, 1.0, 1.0), ([0], True, 1.0, 1.0),
                 ([0], "goal", 1.0, 1.0), ([0], 0, np.nan, 1.0), ([0], 0, 1.0, np.inf), ([0, 1], 0, [1.0, 2.0, 3.0], 1.0),
                 ([0, 1], 0, 1.0, 1.0, [0.0]), ([[0, 1]], 0, 1.0, 1.0), ([0.5], 0, 1.0, 1.0)]:
        with pytest.raises(ValueError):
            env.set_env_pose(*args)
    assert not host_array(env.pose_pending).any() and np.isnan(host_array(env.next_pose)).all()
    env.set_env_pose([1, 2, 1], 0, [1.0, 2.0, 3.0], 4.0)
    assert host_array(env.next_pose)[1, 0].tolist()[:2] == [3.0, 4.0] and np.isnan(host_array(env.next_pose)[1, 0, 2])
    assert host_array(env.pose_pending).tolist() == [0, 1, 1, 0]
    env.close()
    off = BatchedMiniWorld("MiniWorld-OneRoom-v0", 2)
    for name in ("next_pose", "next_agent_pose", "pose_pending", "episode_start"):
        with pytest.raises(EngineError, match="error -6"):
            off.engine.state_array(name)
        with pytest.raises(RuntimeError, match="start_poses=True"):
            getattr(off, name)
    with pytest.raises(RuntimeError):
        off.set_env_pose([0], 0, 1.0, 1.0)
    off.close()


def test_append_only_slots_and_slots_beyond_the_count_ignore_their_design(hostsim_path):
    """Designs for Sign's and ThreeRooms' append-only frames (slots 6 and 2) are ignored, as the host's bare
    entities.append ignores them; so are a OneRoom env's rows beyond its two slots in a table whose other level fills
    more."""
    from miniworld_b200.batched import BatchedMiniWorld
    for level, frame in (("MiniWorld-Sign-v0", 6), ("MiniWorld-ThreeRooms-v0", 2)):
        env = BatchedMiniWorld(level, 2, start_poses=True)
        assert not env.level_slots[0][frame]["designable"]
        ds = [({frame: (3.0, 3.0, 0.5)}, None), ({frame: (3.0, 3.0, 0.5), 0: (2.0, 2.5, math.nan)}, (4.5, 5.0, 1.0))]
        write_designs(env, ds)
        seed_reset(env, [5, 6])
        plain = BatchedMiniWorld(level, 1)
        seed_reset(plain, [5])
        assert_env_equal(full_state(env), 0, full_state(plain), 0, (level, "frame design ignored"))
        for i, (poses, agent) in enumerate(ds):
            assert_world_equals_host(env, i, host_env(level, {}, 5 + i, options_of(poses, agent)), (level, i))
        env.close()
        plain.close()
    rows = ["MiniWorld-OneRoom-v0", "MiniWorld-ThreeRooms-v0"]
    env = BatchedMiniWorld(rows, 2, start_poses=True)
    E = env.engine.max_ents
    assert E > 2 and len(env.level_slots[0]) == 2
    beyond = ({e: (1.5, 1.0 + e, 0.25) for e in range(2, E)}, None)
    write_designs(env, [beyond, ({}, None)])
    seed_reset(env, [7, 8])
    assert_world_equals_host(env, 0, host_env("MiniWorld-OneRoom-v0", {}, 7, options_of(*beyond)), "beyond")
    plain = BatchedMiniWorld(rows, 2)
    seed_reset(plain, [7, 8])
    assert_env_equal(full_state(env), 0, full_state(plain), 0, "beyond the count")
    env.close()
    plain.close()


# reference goldens (oracle/gen_pose_golden.py): case -> (level, kwargs of the level)
POSE_CASES = {"oneroom": ("MiniWorld-OneRoom-v0", {}), "fourrooms_dr": ("MiniWorld-FourRooms-v0", {"domain_rand": True}),
              "tmaze": ("MiniWorld-TMaze-v0", {}), "pickup": ("MiniWorld-PickupObjects-v0", {}),
              "putnext_dr": ("MiniWorld-PutNext-v0", {"domain_rand": True}), "sidewalk": ("MiniWorld-Sidewalk-v0", {})}


def replay_pose_golden(case):
    """Replay golden `case` of the unmodified reference: before every reset (the seeded one and every auto-reset) the
    env's design for its next episode is written into next_pose / next_agent_pose / pose_pending, and every step the
    state, rewards, flags and stream equal the reference's, and episode_start its agent's pose at the episode's reset."""
    from conftest import golden
    from test_level_params import golden_mismatches
    from miniworld_b200.batched import BatchedMiniWorld
    g = golden("poses_" + case)
    level, kw = POSE_CASES[case]
    T, N = g["actions"].shape
    env = BatchedMiniWorld(short_level(level, int(g["episode_steps"])), N, level_kwargs=kw, start_poses=True)
    E = env.engine.max_ents
    assert np.isnan(g["design_pose"][:, :, E:]).all()       # the reference designs only slots the level fills
    if env.engine.host_memory:
        put = lambda view, ids, vals: view.__setitem__(ids, vals)
    else:
        import torch
        put = lambda view, ids, vals: view.__setitem__(torch.as_tensor(ids, device=view.device),
                                                       torch.as_tensor(np.ascontiguousarray(vals), device=view.device))

    def queue(ids, ep):
        put(env.next_pose, ids, g["design_pose"][ids, ep, :E])
        put(env.next_agent_pose, ids, g["design_agent"][ids, ep])
        put(env.pose_pending, ids, g["design_pending"][ids, ep].astype(np.uint8))

    ep = np.zeros(N, np.int64)
    queue(np.arange(N), ep)
    seed_reset(env, 1000 + np.arange(N))
    designed = 0
    out = None
    for t in range(T + 1):
        if t:
            out = env.step_host(g["actions"][t - 1], out, render=False)
        st = full_state(env)
        sub = None if out is None else {key: out[key] for key in ("reward", "terminated", "truncated")}
        bad = golden_mismatches(st, np.arange(N), g, t, sub)
        assert not bad, "%s row %d: %s" % (case, t, "; ".join(bad))
        assert np.array_equal(ep, g["episode"][t]), (case, t)
        reset = g["was_reset"][t]
        start = host_array(env.episode_start)
        want = np.stack([g["pos"][t, :, 0], g["pos"][t, :, 2], g["dir"][t]], 1)
        assert np.array_equal(start[reset], want[reset]), (case, t)
        designed += int(g["design_pending"][np.nonzero(reset)[0], ep[reset]].sum())
        if out is not None or t == 0:
            done = np.nonzero(g["terminated"][t] | g["truncated"][t])[0]
            if done.size:
                ep[done] += 1
                queue(done, ep[done])
    assert designed > 50 and env.engine.overflow_count() == 0
    env.close()


@pytest.mark.parametrize("case", sorted(POSE_CASES))
def test_designed_episodes_follow_the_reference(hostsim_path, case):
    replay_pose_golden(case)


def _shard_worker(rank, port, hostsim, q):
    import os
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=2)
    from miniworld_b200 import engine
    from miniworld_b200.dist import ShardedMiniWorld
    engine._override_library_for_tests(hostsim)
    env = ShardedMiniWorld(short_level("MiniWorld-FourRooms-v0", 7), 7, dist=dist, start_poses=True)
    seed_reset(env.local, [1000 + env.start + k for k in range(env.count)])
    outs = shard_run(env.local, env.start, 40, 7, rank, lambda a: env.scatter_actions(a, like=torch.zeros(1)),
                     env.gather_to_root)
    if rank == 0:
        q.put(outs)
    dist.barrier()
    dist.destroy_process_group()


def shard_run(env, start, steps, total, rank=0, scatter=None, gather=None):
    """Every step the done envs of a shard starting at global env `start` get designs keyed by their global index."""
    import torch
    acts_all = np.random.default_rng(5).integers(0, 3, size=(steps, total), dtype=np.int32)
    outs, out = [], None
    for t in range(steps):
        acts = acts_all[t] if scatter is None else scatter(torch.as_tensor(acts_all[t]) if rank == 0 else None).numpy()
        out = env.step_host(acts, out, render=t == steps - 1)
        done = np.nonzero((out["terminated"] | out["truncated"]).astype(bool))[0]
        g = start + done
        keep = done[(g + t) % 3 != 0]                   # the others are placed as the level writes it
        if keep.size:
            gk = start + keep
            env.set_env_pose(keep, "agent", -6.0 + (gk % 5) * 2.5, -5.0 + (t % 4) * 3.0, (gk + t) * 0.1)
            env.set_env_pose(keep, 0, 5.0 - (gk % 3), 4.0)
        got = [out["obs"], out["reward"], np.array(env.episode_start), np.array(env.pose_pending)]
        if gather is not None:
            got = [gather(torch.as_tensor(x)).numpy() if rank == 0 else gather(torch.as_tensor(x)) for x in got]
        outs.append([np.array(x) for x in got] if rank == 0 else None)
    return outs


def test_sharded_pose_writes_equal_one_process(hostsim_path):
    """Two gloo ranks that write their envs' designs into their local batches equal one process: a design belongs to
    an env, so each rank's arrays are its slice."""
    import os
    import torch.multiprocessing as mp
    from miniworld_b200.batched import BatchedMiniWorld
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 39000 + os.getpid() % 2000
    procs = [ctx.Process(target=_shard_worker, args=(r, port, hostsim_path, q)) for r in range(2)]
    for p in procs:
        p.start()
    sharded = q.get(timeout=300)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    env = BatchedMiniWorld(short_level("MiniWorld-FourRooms-v0", 7), 7, start_poses=True)
    seed_reset(env, 1000 + np.arange(7))
    one = shard_run(env, 0, 40, 7)
    for t, (x, y) in enumerate(zip(one, sharded)):
        for k in (1, 2, 3):
            assert np.array_equal(x[k], y[k]), (t, k)
    assert np.array_equal(one[-1][0], sharded[-1][0]) and 0 < one[-1][0].mean() < 255
    assert sum(int(x[3].sum()) for x in one) > 0          # designs were pending at some steps
    env.close()


# ------------------------------------------------------------------ GPU (libmwb.so)
@pytest.mark.gpu
def test_gpu_reverse_curriculum_matches_the_host_build(libmwb_path):
    """4096 OneRoom envs, 300 steps of a reverse curriculum in torch ops, never synchronising: every done env starts
    its next episode with the goal box at a fixed spot and the agent at a radius from it that widens with the success
    rate.  A sample of envs replays on the host build with the recorded actions and designs: flags, rewards and
    info["start"] every step, state at the end."""
    import subprocess
    import torch
    from conftest import ROOT
    from miniworld_b200 import engine
    from miniworld_b200.batched import BatchedMiniWorld
    level = short_level("MiniWorld-OneRoom-v0", 15)
    N, T = 4096, 300
    env = BatchedMiniWorld(level, N, start_poses=True)
    dev = torch.device("cuda")
    gen = torch.Generator(device="cuda")
    gen.manual_seed(3)
    env.reset(seed=500)
    radius = torch.full((N,), 0.5, dtype=torch.float64, device=dev)
    acts = torch.randint(0, 3, (T, N), dtype=torch.int32, device=dev, generator=gen)
    sample = np.sort(np.random.default_rng(4).choice(N, 64, replace=False))
    sample_t = torch.as_tensor(sample, device=dev)
    hist = {k: [] for k in ("start", "rew", "te", "tr", "pose", "agent", "pending")}
    goal = torch.tensor([7.0, 7.0], dtype=torch.float64, device=dev)
    for t in range(T):
        obs, rew, te, tr, info = env.step(acts[t])
        done = te | tr
        radius = torch.where(done & te, torch.clamp(radius + 0.25, max=6.0), radius)   # success: start further back
        ang = torch.rand(N, dtype=torch.float64, device=dev, generator=gen) * (2 * math.pi)
        xz = goal + radius[:, None] * torch.stack([torch.cos(ang), torch.sin(ang)], 1)
        xz = torch.clamp(xz, 0.5, 9.5)                # inside the 10 x 10 room
        d = done[:, None]
        env.next_pose[:, 0, :2] = torch.where(d, goal.expand(N, 2), env.next_pose[:, 0, :2])
        env.next_agent_pose[:, :2] = torch.where(d, xz, env.next_agent_pose[:, :2])
        env.pose_pending.copy_(torch.where(done, torch.ones_like(env.pose_pending), env.pose_pending))
        for k, v in (("start", info["start"]), ("rew", rew), ("te", te), ("tr", tr), ("pose", env.next_pose[:, 0]),
                     ("agent", env.next_agent_pose), ("pending", env.pose_pending)):
            hist[k].append(v[sample_t].clone())
    final = full_state(env)
    hist = {k: torch.stack(v).cpu().numpy() for k, v in hist.items()}
    assert hist["te"].sum() + hist["tr"].sum() > 1000 and hist["te"].sum() > 50
    acts = acts.cpu().numpy()
    env.close()

    lib = subprocess.check_output([ROOT + "/tests/hostsim/build.sh"]).decode().strip().splitlines()[-1]
    engine._override_library_for_tests(lib)
    try:
        host = BatchedMiniWorld(level, len(sample), start_poses=True)
        seed_reset(host, 500 + sample)
        out = None
        for t in range(T):
            out = host.step_host(acts[t, sample], out, render=False)
            assert np.array_equal(out["reward"], hist["rew"][t]), t
            assert np.array_equal(out["terminated"].astype(bool), hist["te"][t]), t
            assert np.array_equal(out["truncated"].astype(bool), hist["tr"][t]), t
            assert np.array_equal(host.episode_start, hist["start"][t]), t
            host.next_pose[:, 0] = hist["pose"][t]
            host.next_agent_pose[:] = hist["agent"][t]
            host.pose_pending[:] = hist["pending"][t]
        st = full_state(host)
        for j, i in enumerate(sample):
            assert_env_equal(st, j, final, i, ("final", int(i)))
        host.close()
    finally:
        engine._override_library_for_tests(None)


@pytest.mark.gpu
@pytest.mark.parametrize("level", ["MiniWorld-OneRoom-v0", "MiniWorld-FourRooms-v0", "MiniWorld-Sign-v0",
                                   "MiniWorld-PickupObjects-v0"])
def test_gpu_designed_frames_match_the_pixel_oracle(libmwb_path, softgl_lib, level):
    """Frames of designed starts (poses in and outside the floor plan, agents facing designed entities) against
    oracle/softgl.c rendering the host-built world, with no capacity fault."""
    from test_render_paths import assert_matches, oracle_frame
    from miniworld_b200.batched import BatchedMiniWorld
    rs = np.random.default_rng(5)
    probe = BatchedMiniWorld(level, 1, start_poses=True)
    slots = probe.level_slots[0]
    probe.close()
    ds = designs(level, {}, slots, rs) * 2
    N = len(ds)
    env = BatchedMiniWorld(level, N, start_poses=True, want_depth=True)
    write_designs(env, ds)
    obs, _ = env.reset(seed=60)
    obs = obs["obs"] if isinstance(obs, dict) else obs
    obs = obs.cpu().numpy()
    depth = env._bufs["depth"].cpu().numpy()
    assert env.engine.overflow_count() == 0
    st = env.get_state(rng=True)
    for i, (poses, agent) in enumerate(ds):
        host = host_env(level, {}, 60 + i, options_of(poses, agent))
        assert np.array_equal(st["agent_pos"][i], host.agent.pos), i
        want_rgb, want_depth = oracle_frame(host, 80, 60, 8)
        assert_matches(obs[i], depth[i], want_rgb, want_depth, (level, i))
    env.close()


@pytest.mark.gpu
def test_gpu_designs_written_on_a_side_stream_behind_a_busy_stream(libmwb_path):
    """Designs written on a side stream behind a long-running kernel are seen by the step (auto-reset) and the reset
    that run behind them on that stream: `a` writes and goes on at once, `b` waits for the device after the same
    write."""
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    N = 64
    level = short_level("MiniWorld-FourRooms-v0", 3)
    a, b = (BatchedMiniWorld(level, N, domain_rand=True, start_poses=True) for _ in range(2))
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
            pose = torch.tensor([2.0 + k, 3.0, 0.5], dtype=torch.float64, device="cuda")
            b.next_agent_pose.copy_(pose.expand(N, 3))
            b.pose_pending.fill_(1)
            torch.cuda.synchronize()
            torch.cuda._sleep(100_000_000)
            a.next_agent_pose.copy_(pose.expand(N, 3))
            a.pose_pending.fill_(1)
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
            assert torch.equal(a.episode_start, b.episode_start), call
            assert bool((a.pose_pending[took] == 0).all()) and bool((a.pose_pending[~took] == 1).all()), call
            assert bool((a.episode_start[took] == pose).all()), call
    a.close()
    b.close()


@pytest.mark.gpu
def test_gpu_reset_takes_pending_designs(libmwb_path):
    """reset() after set_env_pose places the designs, and equals the host build's reset of the same designs."""
    from miniworld_b200.batched import BatchedMiniWorld
    N = 16
    kw = {"domain_rand": True}
    env = BatchedMiniWorld("MiniWorld-FourRooms-v0", N, level_kwargs=kw, start_poses=True)
    rs = np.random.default_rng(2)
    goal = rs.uniform(-6, 6, (N, 2))
    agent = rs.uniform(-6, 6, (N, 2))
    env.set_env_pose(np.arange(N), 0, goal[:, 0], goal[:, 1])
    env.set_env_pose(np.arange(N)[::2], "agent", agent[::2, 0], agent[::2, 1], 1.5)
    env.reset(seed=80)
    assert not host_array(env.pose_pending).any()
    for i in range(N):
        opts = {"poses": {0: (goal[i, 0], goal[i, 1], math.nan)}}
        if i % 2 == 0:
            opts["agent_pose"] = (agent[i, 0], agent[i, 1], 1.5)
        assert_world_equals_host(env, i, host_env("MiniWorld-FourRooms-v0", kw, 80 + i, opts), i)
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(POSE_CASES))
def test_gpu_designed_episodes_follow_the_reference(libmwb_path, case):
    """The reference goldens replayed on the device, designs written with torch ops."""
    replay_pose_golden(case)
