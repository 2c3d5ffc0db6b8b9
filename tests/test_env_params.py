"""Env params (mwb_enable_env_params, BatchedMiniWorld(env_params=True)): an env whose episode runs a design against
the same env in a one-level batch whose level row is the merged row, the stream, mid-episode level writes, a numpy
model of the three arrays, goal distance, the drop-in reset option, snapshots, errors and a gloo shard.  CPU cases run
the kernels' host build; `gpu` cases run libmwb.so on the device."""
import math

import numpy as np
import pytest

from level_parity import assert_env_equal, full_state, seed_reset, short_level
from test_maze_layouts import host_array

E = 22
ROOM = "MiniWorld-OneRoom-v0"


def lowered_merge(level_row, design):
    """The numpy restatement of merge_env_params: the lowered level row (float64 [PARAMS_DOUBLES]) merged with a
    design ([22, 3] of (default, min, max), NaN = the level's)."""
    from miniworld_b200.engine import PARAMS_COLUMN
    out = np.array(level_row, np.float64)
    for e in range(E):
        w = (e // 3) * 9 + e % 3 if e < 15 else 45 + (e - 15) * 3
        s = 3 if e < 15 else 1
        d, lo, hi = design[e]
        if math.isfinite(d):
            out[w] = d
        if math.isfinite(lo) and math.isfinite(hi):
            out[w + s], out[w + 2 * s] = lo, np.subtract(hi, lo)
            if e == 15:
                out[PARAMS_COLUMN["max_forward_step"]] = hi
    return out


def designs(level_row, rs):
    """The design kinds: none, an all-NaN row, one scalar range, one vector element, defaults only, every element
    pinned at a boundary, ranges outside the level's, and min > max."""
    from miniworld_b200.engine import PARAMS_COLUMN
    lo = np.array([level_row[(e // 3) * 9 + 3 + e % 3] if e < 15 else level_row[45 + (e - 15) * 3 + 1] for e in range(E)])
    span = np.array([level_row[(e // 3) * 9 + 6 + e % 3] if e < 15 else level_row[45 + (e - 15) * 3 + 2]
                     for e in range(E)])
    hi = lo + span
    hi[15] = level_row[PARAMS_COLUMN["max_forward_step"]]
    nan = np.full((E, 3), np.nan)
    out = {"none": None, "nan": nan.copy()}
    d = nan.copy(); d[19, 1:] = (30.0, 120.0); out["scalar_range"] = d                       # cam_fov_y
    d = nan.copy(); d[4] = (3.0, 2.0, 4.0); out["vector_element"] = d                       # light_pos[1]
    d = nan.copy(); d[:, 0] = lo + rs.random(E) * span; out["defaults"] = d
    d = np.stack([np.where(rs.random(E) < 0.5, lo, hi)] * 3, axis=1); out["pinned"] = d
    d = nan.copy(); d[:, 1], d[:, 2] = lo - span, hi + span; d[15] = (0.25, 0.2, 0.3); d[20] = (2.5, 0.5, 3.0)
    out["outside"] = d
    d = nan.copy(); d[:, 1], d[:, 2] = hi, lo; d[15, 1:] = (0.2, 0.1); out["min_above_max"] = d
    return out


def write(view, i, vals):
    if isinstance(view, np.ndarray):
        view[i] = vals
    else:
        import torch
        view[i] = torch.as_tensor(np.ascontiguousarray(vals), device=view.device)


def _twin_run(level, dr, steps, seed0=700, render_every=25):
    """One batch of every design kind with env_params on (pending re-set every step, so every episode runs its design)
    against one one-env batch per design whose level row is the merged row."""
    from miniworld_b200.batched import BatchedMiniWorld
    kw = {"domain_rand": dr} if level != "MiniWorld-Sign-v0" else {}      # Sign fixes its own flag
    lv = short_level(level, 40)
    env = BatchedMiniWorld(lv, 8, env_params=True, want_depth=True, **kw)
    row0 = host_array(env._views()["level_params"])[0].copy()
    ds = designs(row0, np.random.default_rng(len(level) + dr))
    names = list(ds)
    N = len(names)
    env.close()
    env = BatchedMiniWorld(lv, N, env_params=True, want_depth=True, **kw)
    twins = []
    for i, n in enumerate(names):
        t = BatchedMiniWorld(lv, 1, want_depth=True, **kw)
        if ds[n] is not None:
            write(env.next_params, i, ds[n])
            write(t._views()["level_params"], 0, lowered_merge(row0, ds[n]))
        twins.append(t)
    pending = np.array([ds[n] is not None for n in names], np.uint8)
    write(env.params_pending, slice(None), pending)
    seeds = seed0 + np.arange(N)
    seed_reset(env, seeds)
    for i, t in enumerate(twins):
        seed_reset(t, seeds[i:i + 1])
    ep = host_array(env.episode_params)
    for i, n in enumerate(names):
        assert np.array_equal(ep[i], ds[n] if ds[n] is not None else np.full((E, 3), np.nan), equal_nan=True), n
    assert not host_array(env.params_pending).any()
    rs = np.random.default_rng(3)
    out, outs = None, [None] * N
    for step in range(steps):
        write(env.params_pending, slice(None), pending)
        acts = rs.integers(0, env.single_action_space.n, N).astype(np.int32)
        render = step % render_every == 0 or step == steps - 1
        out = env.step_host(acts, out, render=render)
        sa = full_state(env)
        for i, t in enumerate(twins):
            outs[i] = t.step_host(acts[i:i + 1], outs[i], render=render)
            for key in ("reward", "terminated", "truncated") + (("obs", "depth") if render else ()):
                assert np.array_equal(out[key][i], outs[i][key][0]), (level, dr, names[i], step, key)
            assert_env_equal(sa, i, full_state(t), 0, (level, dr, names[i], step))
    assert env.engine.overflow_count() == 0
    for t in twins:
        t.close()
    return env


@pytest.mark.parametrize("dr", [False, True], ids=["plain", "dr"])
@pytest.mark.parametrize("level", [
    "MiniWorld-CollectHealth-v0", "MiniWorld-FourRooms-v0", "MiniWorld-Hallway-v0", "MiniWorld-Maze-v0",
    "MiniWorld-MazeS2-v0", "MiniWorld-MazeS3-v0", "MiniWorld-MazeS3Fast-v0", "MiniWorld-MazeS8-v0",
    "MiniWorld-OneRoom-v0", "MiniWorld-OneRoomS6-v0", "MiniWorld-OneRoomS6Fast-v0", "MiniWorld-PickupObjects-v0",
    "MiniWorld-PutNext-v0", "MiniWorld-RoomObjects-v0", "MiniWorld-Sidewalk-v0", "MiniWorld-Sign-v0",
    "MiniWorld-TMaze-v0", "MiniWorld-TMazeLeft-v0", "MiniWorld-TMazeRight-v0", "MiniWorld-ThreeRooms-v0",
    "MiniWorld-WallGap-v0", "MiniWorld-YMaze-v0", "MiniWorld-YMazeLeft-v0", "MiniWorld-YMazeRight-v0"])
def test_designed_episode_equals_merged_level_row(hostsim_path, level, dr):
    """The central invariant: every design kind, through 300-step rollouts with auto-resets, equals a one-level batch
    whose level row is the merged row, field for field with frames and depth byte-identical.  Levels that reset on the
    host refuse the mode with TypeError."""
    from miniworld_b200.batched import BatchedMiniWorld
    if level == "MiniWorld-Sign-v0" and dr:
        pytest.skip("Sign fixes its own domain_rand flag")
    probe = BatchedMiniWorld(level, 1, domain_rand=dr)
    device = probe.device_reset
    probe.close()
    if not device:
        with pytest.raises(TypeError, match="env params are taken by device resets"):
            BatchedMiniWorld(level, 1, domain_rand=dr, env_params=True)
        return
    _twin_run(level, dr, 300).close()


def test_design_leaves_the_stream_where_an_undesigned_twin_is(hostsim_path):
    """A design changes no draw count: after the reset the stream is where an undesigned twin's is, with and without
    domain randomisation, for every design kind."""
    from miniworld_b200.batched import BatchedMiniWorld
    for dr in (False, True):
        for level in ("MiniWorld-FourRooms-v0", "MiniWorld-PickupObjects-v0"):
            a = BatchedMiniWorld(level, 8, domain_rand=dr, env_params=True)
            b = BatchedMiniWorld(level, 8, domain_rand=dr)
            row0 = host_array(a._views()["level_params"])[0]
            ds = [d for d in designs(row0, np.random.default_rng(1)).values() if d is not None]
            for i, d in enumerate(ds):
                write(a.next_params, i, d)
            write(a.params_pending, slice(None), np.ones(8, np.uint8))
            seed_reset(a, 50 + np.arange(8))
            seed_reset(b, 50 + np.arange(8))
            assert np.array_equal(full_state(a)["rng"], full_state(b)["rng"]), (level, dr)
            a.close()
            b.close()


def test_level_writes_reach_only_undesigned_entries(hostsim_path):
    """A set_level_param write mid-episode reaches, from the next step, the envs that left that entry NaN and not the
    envs that designed it."""
    from miniworld_b200.batched import BatchedMiniWorld
    N = 4
    env = BatchedMiniWorld(ROOM, N, env_params=True)
    env.set_env_param([1, 3], "forward_step", 0.3, 0.3, 0.3)
    env.set_env_param([2], "turn_step", 45.0)
    seed_reset(env, 10 + np.arange(N))
    env.set_level_param(0, "forward_step", 0.05)
    before = env.get_state()["agent_pos"].copy()
    env.step_host(np.full(N, 2, np.int32), render=False)      # move forward
    moved = np.linalg.norm(env.get_state()["agent_pos"] - before, axis=1)
    assert np.allclose(moved[[0, 2]], 0.05) and np.allclose(moved[[1, 3]], 0.3), moved
    d0 = env.get_state()["agent_dir"].copy()
    env.set_level_param(0, "turn_step", 5.0)
    env.step_host(np.zeros(N, np.int32), render=False)        # turn left
    turned = np.degrees(env.get_state()["agent_dir"] - d0)
    assert np.allclose(turned[[0, 1, 3]], 5.0) and np.allclose(turned[2], 45.0), turned
    p = env.get_env_params(2)
    assert p.params["turn_step"].default == 45.0 and p.params["forward_step"].default == 0.05
    assert env.get_env_params(1).params["forward_step"].max == 0.3
    env.close()


def test_model_of_the_arrays(hostsim_path):
    """A numpy model of next_params / params_pending / episode_params through auto-resets, subset resets, level changes
    in a per-env-worlds table with Maze rows, episode seeds, bank loads, and designs combined with start poses and
    reset draws."""
    from miniworld_b200.batched import BatchedMiniWorld
    rows = [short_level("MiniWorld-OneRoom-v0", 7), short_level("MiniWorld-MazeS2-v0", 9),
            short_level("MiniWorld-PickupObjects-v0", 5), short_level("MiniWorld-TMaze-v0", 6)]
    N = 12
    env = BatchedMiniWorld(rows, N, env_level=np.arange(N) % 4, dynamic_levels=True, per_env_worlds=True,
                           episode_seeds=True, start_poses=True, reset_draws=True, env_params=True, state_bank=4)
    rs = np.random.default_rng(9)
    nxt = np.full((N, E, 3), np.nan)
    pend = np.zeros(N, np.uint8)
    epi = np.full((N, E, 3), np.nan)
    saved = {}

    def design(ids):
        for i in ids:
            d = np.full((E, 3), np.nan)
            e = int(rs.integers(0, E))
            d[e] = (1.0 + i, 0.5 + i, 1.5 + i) if e >= 18 else (0.3, 0.2, 0.4)
            write(env.next_params, int(i), d)
            nxt[i] = d
        write(env.params_pending, np.asarray(ids), np.ones(len(ids), np.uint8))
        pend[np.asarray(ids)] = 1

    def program_reset(ids):
        for i in ids:
            epi[i] = nxt[i] if pend[i] else np.nan
            pend[i] = 0

    def check(where):
        assert np.array_equal(host_array(env.next_params), nxt, equal_nan=True), where
        assert np.array_equal(host_array(env.params_pending), pend), where
        assert np.array_equal(host_array(env.episode_params), epi, equal_nan=True), where

    check("start")
    design([0, 1, 2, 5])
    seed_reset(env, 30 + np.arange(N))
    program_reset(range(N))
    check("reset")
    design([3, 4])
    env.set_env_level([3], [1])
    env.set_env_seed([4], [77])
    env.set_env_pose([4], "agent", 1.5, 1.5, 0.0)
    env.set_env_draws([3, 4], 0, 1.0)
    env.engine.reset(np.array([3, 4], np.int32))
    program_reset([3, 4])
    check("subset reset")
    design([6, 7])
    env.save_states(np.array([6, 7], np.int32), np.array([0, 1], np.int32))
    saved = {0: epi[6].copy(), 1: epi[7].copy()}
    env.set_env_state([8, 9], [0, 1])
    design([8])
    out, done = None, np.zeros(N, bool)
    for t in range(60):
        # this step auto-resets the envs the last one ended: a bank load where a filled slot is pending (only next_state
        # is consumed), the level's program otherwise
        st = host_array(env.next_state).copy()
        out = env.step_host(rs.integers(0, 3, N).astype(np.int32), out, render=False)
        for i in np.nonzero(done)[0]:
            if st[i] >= 0:
                epi[i] = saved[int(st[i])]
            else:
                program_reset([i])
        done = (out["terminated"] | out["truncated"]).astype(bool)
        check(("step", t))
        if t % 3 == 0:
            design(rs.choice(N, 3, replace=False))
        if t == 20:
            env.set_env_state([10, 11], [1, 0])
    check("end")
    env.close()


def test_goal_distance_follows_the_merged_params(hostsim_path):
    """goal_dist and expert_action under a designed forward_step max and turn_step default equal the numpy mirror
    (MiniWorldEnv.goal_distance() / expert_action() of a drop-in env reset with the same params option)."""
    from miniworld_b200.batched import BatchedMiniWorld
    from test_start_poses import host_env
    level = "MiniWorld-FourRooms-v0"
    N = 4
    env = BatchedMiniWorld(level, N, goal_distance=True, env_params=True)
    opts = [{}, {"forward_step": (0.15, 0.1, 0.6)}, {"turn_step": (40.0, None, None)},
            {"forward_step": (0.2, 0.2, 1.0), "turn_step": (3.0, None, None)}]
    for i, o in enumerate(opts):
        for name, (d, lo, hi) in o.items():
            env.set_env_param([i], name, d, lo, hi)
    seed_reset(env, 60 + np.arange(N))
    gd, ex = host_array(env.goal_dist), host_array(env.expert_action)
    for i, o in enumerate(opts):
        host = host_env(level, {}, 60 + i, {"params": o} if o else None)
        assert host.max_forward_step == (o.get("forward_step", (0, 0, 0.17))[2])
        want_d, want_a = host.goal_distance(), host.expert_action()
        assert gd[i] == want_d and ex[i] == want_a, (i, gd[i], want_d, ex[i], want_a)
    env.close()


@pytest.mark.parametrize("dr", [False, True], ids=["plain", "dr"])
def test_drop_in_params_option(hostsim_path, dr):
    """MiniWorldEnv.reset(options={"params": ...}) builds the world the batched engine builds from the same design;
    the next reset without the option runs on the level's params again."""
    from miniworld_b200.batched import BatchedMiniWorld
    from test_maze_layouts import assert_world_equals_host
    from test_start_poses import host_env
    level = "MiniWorld-PickupObjects-v0"
    opt = {"cam_fov_y": (90.0, 80.0, 100.0), "light_pos": ([1.0, None, 0.5], [-1.0, 2.0, -1.0], [1.0, 6.0, 1.0]),
           "obj_color_bias": (None, [0.3, 0.3, 0.3], [0.3, 0.3, 0.3]), "cam_height": (2.5, 2.0, 3.0)}
    env = BatchedMiniWorld(level, 1, domain_rand=dr, env_params=True)
    for name, (d, lo, hi) in opt.items():
        env.set_env_param([0], name, d, lo, hi)
    seed_reset(env, [5])
    host = host_env(level, {"domain_rand": dr}, 5, {"params": opt})
    assert_world_equals_host(env, 0, host, dr)
    st = env.get_state()
    assert np.array_equal(st["cam"][0], [host.agent.cam_height, host.agent.cam_fwd_disp, host.agent.cam_pitch,
                                         host.agent.cam_fov_y])
    host.reset(seed=5)
    assert host.params is not None and host.params.params["cam_fov_y"].default == 60
    env.close()


def test_snapshots_round_trip_and_refuse_across_the_mode(hostsim_path):
    """A snapshot round trip restores the three arrays and the running episodes; restoring across the mode fails with
    MWB_ESTATE (error -6) and names the mode."""
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import EngineError
    N = 4
    a = BatchedMiniWorld("MiniWorld-FourRooms-v0", N, domain_rand=True, env_params=True)
    a.set_env_param(np.arange(N), "cam_fov_y", None, 30.0, 120.0)
    seed_reset(a, 3 + np.arange(N))
    a.set_env_param([1], "forward_step", 0.3, 0.3, 0.3)
    blob = a.snapshot()
    s0 = full_state(a)
    arrays = [host_array(v).copy() for v in (a.next_params, a.params_pending, a.episode_params)]
    acts = np.random.default_rng(2).integers(0, 3, (30, N)).astype(np.int32)
    outs = [a.step_host(x, render=False)["reward"].copy() for x in acts]
    end = full_state(a)
    a.restore(blob)
    for i in range(N):
        assert_env_equal(full_state(a), i, s0, i, i)
    for v, w in zip((a.next_params, a.params_pending, a.episode_params), arrays):
        assert np.array_equal(host_array(v), w, equal_nan=True)
    again = [a.step_host(x, render=False)["reward"].copy() for x in acts]
    assert all(np.array_equal(x, y) for x, y in zip(outs, again))
    for i in range(N):
        assert_env_equal(full_state(a), i, end, i, i)
    plain = BatchedMiniWorld("MiniWorld-FourRooms-v0", N, domain_rand=True)
    with pytest.raises(EngineError, match=r"error -6: .*env params on \(this one has"):
        plain.restore(blob)
    with pytest.raises(EngineError, match=r"error -6: .*goal distance off \(this one has .*env params on\)"):
        a.restore(plain.snapshot())
    a.close()
    plain.close()


def test_snapshot_blobs_without_the_mode_keep_their_layout(hostsim_path):
    """Handles without the mode write blobs of the sizes and marks they had: the mark has no env-params bit, and a
    handle with every other mode on restores its own blob."""
    from miniworld_b200.batched import BatchedMiniWorld
    env = BatchedMiniWorld(ROOM, 2, episode_seeds=True, start_poses=True, goal_distance=True, state_bank=2)
    blob = env.snapshot()
    assert not (int.from_bytes(blob[:4], "little") & 0x00800000)
    on = BatchedMiniWorld(ROOM, 2, episode_seeds=True, start_poses=True, goal_distance=True, env_params=True,
                          state_bank=2)
    on_blob = on.snapshot()
    assert int.from_bytes(on_blob[:4], "little") & 0x00800000
    # the mode adds its three arrays (2 envs) and 528 B to each of the 2 bank records
    assert len(on_blob) - len(blob) == 2 * (2 * 528 + 1) + 2 * 528
    env.restore(blob)
    env.close()
    on.close()


EXPECTED = {
    "already on": "libmwb error -6: env params are already on",
    "after the bank": "libmwb error -6: env params cannot be turned on once the state bank is on (its record layout "
                      "depends on it)",
    "array off": "libmwb error -6: env params are off (mwb_enable_env_params)",
    "accessor": "this batch has no env params: construct it with env_params=True",
}


def test_errors(hostsim_path):
    """Argument, ABI and mode errors: a second enable, enable after the state bank, the arrays of a handle without the
    mode, the accessors of a batch without it, the host-reset TypeError and set_env_param's checks."""
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import ENV_PARAM_ELEMS, EngineError, load_library
    import ctypes as C
    lib = load_library()
    assert lib.mwb_enable_env_params(None) == -1 and lib.mwb_last_error() == b"null handle"
    env = BatchedMiniWorld(ROOM, 3, env_params=True)
    with pytest.raises(EngineError) as e:
        env.engine.enable_env_params()
    assert str(e.value) == EXPECTED["already on"]
    assert env.next_params.shape == (3, ENV_PARAM_ELEMS, 3) and env.episode_params.shape == (3, 22, 3)
    assert env.params_pending.shape == (3,)
    assert np.isnan(host_array(env.next_params)).all() and np.isnan(host_array(env.episode_params)).all()
    with pytest.raises(KeyError):
        env.set_env_param([0], "bot_radius", 0.4)
    with pytest.raises(ValueError, match="shape"):
        env.set_env_param([0], "light_pos", 1.0)
    with pytest.raises(ValueError, match="shape"):
        env.set_env_param([0, 1], "cam_fov_y", [1.0, 2.0, 3.0])
    with pytest.raises(ValueError, match="above"):
        env.set_env_param([0], "cam_fov_y", 90.0, 100.0, 120.0)
    with pytest.raises(ValueError, match="above"):
        env.set_env_param([0], "cam_fov_y", None, 100.0, 90.0)
    with pytest.raises(ValueError, match="env ids"):
        env.set_env_param([3], "cam_fov_y", 90.0)
    with pytest.raises(ValueError, match="real numbers"):
        env.set_env_param([0], "cam_fov_y", "wide")
    assert not host_array(env.params_pending).any()
    env.set_env_param(np.array([0, 2]), "light_pos", [[1.0, 2.0, 3.0], [4.0, 5.0, 6.0]], None, None)
    got = host_array(env.next_params)
    assert np.array_equal(got[[0, 2], 3:6, 0], [[1, 2, 3], [4, 5, 6]]) and np.isnan(got[:, 3:6, 1:]).all()
    assert np.array_equal(host_array(env.params_pending), [1, 0, 1])
    env.close()
    plain = BatchedMiniWorld(ROOM, 2)
    for name in ("next_params", "params_pending", "episode_params"):
        with pytest.raises(RuntimeError) as e:
            getattr(plain, name)
        assert str(e.value) == EXPECTED["accessor"]
        with pytest.raises(EngineError) as e:
            plain.engine.state_array(name)
        assert str(e.value) == EXPECTED["array off"]
    with pytest.raises(RuntimeError):
        plain.set_env_param([0], "cam_fov_y", 90.0)
    plain.close()
    bank = BatchedMiniWorld(ROOM, 2, state_bank=2)
    with pytest.raises(EngineError) as e:
        bank.engine.enable_env_params()
    assert str(e.value) == EXPECTED["after the bank"]
    bank.close()


def test_sharded_equals_one_process(hostsim_path):
    """ShardedMiniWorld passes env_params on: a gloo world_size-2 run whose ranks design their slices with local ids
    equals one process."""
    import torch.multiprocessing as mp
    from miniworld_b200 import engine
    from miniworld_b200.batched import BatchedMiniWorld
    total, steps = 6, 30
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29650 + __import__("os").getpid() % 2000
    procs = [ctx.Process(target=_shard_worker, args=(r, port, engine._test_library, total, steps, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = sorted(q.get(timeout=300) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    env = BatchedMiniWorld(short_level("MiniWorld-FourRooms-v0", 9), total, domain_rand=True, env_params=True)
    _design_all(env, 0, total)
    seed_reset(env, 1000 + np.arange(total))
    acts = np.random.default_rng(5).integers(0, 3, (steps, total)).astype(np.int32)
    rew = []
    for t in range(steps):
        rew.append(env.step_host(acts[t], render=False)["reward"].copy())
    st = env.get_state()
    start = 0
    for rank, r_rew, pos, epi in got:
        n = len(pos)
        assert np.array_equal(np.array(rew)[:, start:start + n], r_rew)
        assert np.array_equal(st["agent_pos"][start:start + n], pos)
        assert np.array_equal(host_array(env.episode_params)[start:start + n], epi, equal_nan=True)
        start += n
    env.close()


def _design_all(env, start, count):
    """Global env g gets cam_fov_y default 40 + g and the forward_step range (0.1, 0.1 + 0.01 g)."""
    g = start + np.arange(count)
    env.set_env_param(np.arange(count), "cam_fov_y", 40.0 + g)
    env.set_env_param(np.arange(count), "forward_step", None, np.full(count, 0.1), 0.1 + 0.01 * g)


def _shard_worker(rank, port, hostsim, total, steps, q):
    import os
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    sys.path.insert(0, os.path.join(root, "tests"))
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=2)
    from miniworld_b200 import engine
    from miniworld_b200.dist import ShardedMiniWorld
    from level_parity import seed_reset as sr, short_level as sl
    engine._override_library_for_tests(hostsim)
    env = ShardedMiniWorld(sl("MiniWorld-FourRooms-v0", 9), total, dist=dist, domain_rand=True, env_params=True)
    _design_all(env.local, env.start, env.count)
    sr(env.local, [1000 + env.start + k for k in range(env.count)])
    acts = np.random.default_rng(5).integers(0, 3, (steps, total)).astype(np.int32)
    rew = [env.local.step_host(acts[t, env.start:env.start + env.count], render=False)["reward"].copy()
           for t in range(steps)]
    q.put((rank, np.array(rew), env.local.get_state()["agent_pos"].copy(), np.array(env.local.episode_params)))
    dist.barrier()
    dist.destroy_process_group()


# reference goldens (oracle/gen_env_params_golden.py): case -> (level, kwargs of the level)
GOLDEN_CASES = {"fourrooms_dr": ("MiniWorld-FourRooms-v0", {"domain_rand": True}), "oneroom": ("MiniWorld-OneRoom-v0", {}),
                "pickup_dr": ("MiniWorld-PickupObjects-v0", {"domain_rand": True}),
                "putnext_dr": ("MiniWorld-PutNext-v0", {"domain_rand": True}),
                "mazes3_dr": ("MiniWorld-MazeS3-v0", {"domain_rand": True})}


def replay_env_params_golden(case):
    """Replay golden `case` of the unmodified reference: before every reset (the seeded one and every auto-reset) the
    env's design for its next episode is written into next_params / params_pending, and at every row the state,
    rewards, flags and stream equal the reference's, episode_params holds the running episode's design (NaN when it
    ran its level's params), and at every reset the episode's max_forward_step (get_env_params) is the reference's."""
    from conftest import golden
    from test_level_params import golden_mismatches
    from miniworld_b200.batched import BatchedMiniWorld
    g = golden("envparams_" + case)
    level, kw = GOLDEN_CASES[case]
    T, N = g["actions"].shape
    env = BatchedMiniWorld(short_level(level, int(g["episode_steps"])), N, level_kwargs=kw, env_params=True)

    def queue(ids, ep):
        write(env.next_params, ids, g["design"][ids, ep])
        write(env.params_pending, ids, g["design_pending"][ids, ep].astype(np.uint8))

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
        pend = g["design_pending"][np.arange(N), ep]
        want = np.where(pend[:, None, None], g["design"][np.arange(N), ep], np.nan)
        assert np.array_equal(host_array(env.episode_params), want, equal_nan=True), (case, t)
        reset = np.nonzero(g["was_reset"][t])[0]
        for i in reset:
            assert env.get_env_params(int(i)).params["forward_step"].max == g["max_forward_step"][t, i], (case, t, i)
        designed += int(pend[reset].sum())
        if out is not None or t == 0:
            done = np.nonzero(g["terminated"][t] | g["truncated"][t])[0]
            if done.size:
                ep[done] += 1
                queue(done, ep[done])
    assert designed > 50 and env.engine.overflow_count() == 0
    env.close()


@pytest.mark.parametrize("case", sorted(GOLDEN_CASES))
def test_designed_params_follow_the_reference(hostsim_path, case):
    replay_env_params_golden(case)


# ------------------------------------------------------------------ GPU (libmwb.so)
@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(GOLDEN_CASES))
def test_gpu_designed_params_follow_the_reference(libmwb_path, case):
    """The reference goldens replayed on the device, designs written with torch ops."""
    replay_env_params_golden(case)


def adr_update(env, done, gen):
    """The README ADR step in torch ops: each done env pins one random element at its level's current lower or upper
    bound with probability 0.5, otherwise gets an all-NaN row; both set the pending flag."""
    import torch
    from miniworld_b200.engine import PARAMS_COLUMN
    n, dev = env.num_envs, done.device
    lp = env._views()["level_params"][0]
    e = torch.randint(0, E, (n,), device=dev, generator=gen)
    upper = torch.rand(n, device=dev, generator=gen) < 0.5
    probe = done & (torch.rand(n, device=dev, generator=gen) < 0.5)
    word = torch.where(e < 15, (e // 3) * 9 + e % 3, 45 + (e - 15) * 3)
    step = torch.where(e < 15, 3, 1)
    lo = lp[word + step]
    hi = torch.where(e == 15, lp[PARAMS_COLUMN["max_forward_step"]], lo + lp[word + 2 * step])
    row = torch.full((n, E, 3), float("nan"), dtype=torch.float64, device=dev)
    row[probe, e[probe]] = torch.where(upper, hi, lo)[probe].unsqueeze(1).expand(-1, 3)
    env.next_params[done] = row[done]
    env.params_pending[done] = 1


@pytest.mark.gpu
def test_gpu_adr_loop_matches_host_build(libmwb_path, _hostsim_built):
    """The README ADR loop at 4096 envs on the device, never synchronised: after every step info["params"] of each
    ended env equals the row that was pending at that episode's reset (NaN when none was), and a sample of envs
    replayed on the host build from the same seeds and designs ends in the same state."""
    import torch
    from miniworld_b200 import engine
    from miniworld_b200.batched import BatchedMiniWorld
    N, T = 4096, 60
    level = short_level("MiniWorld-FourRooms-v0", 15)
    env = BatchedMiniWorld(level, N, domain_rand=True, env_params=True)
    env.reset(seed=11)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(4)
    acts = torch.randint(0, 3, (T, N), dtype=torch.int32, device="cuda", generator=gen)
    pend = []
    # the row each env's running episode took: after the seeded reset all NaN (nothing was pending)
    cur = env.episode_params.clone()
    assert torch.isnan(cur).all()
    prev_done = torch.zeros(N, dtype=torch.bool, device="cuda")
    nxt, flag = env.next_params.clone(), env.params_pending.clone()
    mismatch, ended = torch.zeros((), dtype=torch.int64, device="cuda"), torch.zeros((), dtype=torch.int64, device="cuda")
    for t in range(T):
        obs, rew, te, tr, info = env.step(acts[t])
        # this step auto-reset the envs the last one ended: each took the row pending before the step, or NaN
        took = prev_done & (flag != 0)
        cur[prev_done] = torch.where(took[:, None, None], nxt, torch.full_like(nxt, float("nan")))[prev_done]
        done = te | tr
        same = (info["params"] == cur) | (torch.isnan(info["params"]) & torch.isnan(cur))
        mismatch += (~same.all(2).all(1) & done).sum()            # every ended episode names the row it ran
        ended += (done & torch.isfinite(cur).any(2).any(1)).sum()
        adr_update(env, done, gen)
        nxt, flag = env.next_params.clone(), env.params_pending.clone()
        pend.append((nxt, flag))
        prev_done = done
    final = env.get_state(rng=True)
    assert env.engine.overflow_count() == 0
    assert int(mismatch) == 0 and int(ended) > 1000, (int(mismatch), int(ended))
    sample = [0, 1, 777, 2048, 4095]
    acts_h = acts.cpu().numpy()
    pend_h = [(r.cpu().numpy()[sample], p.cpu().numpy()[sample]) for r, p in pend]
    env.close()
    engine._override_library_for_tests(_hostsim_built)
    try:
        host = BatchedMiniWorld(level, len(sample), domain_rand=True, env_params=True)
        seed_reset(host, [11 + i for i in sample])
        for t in range(T):
            host.step_host(acts_h[t, sample], render=False)
            write(host.next_params, slice(None), pend_h[t][0])
            write(host.params_pending, slice(None), pend_h[t][1])
        st = host.get_state(rng=True)
        for k, i in enumerate(sample):
            assert np.array_equal(st["agent_pos"][k], final["agent_pos"][i]), i
            assert np.array_equal(st["rng"][k], final["rng"][i]), i
            assert np.array_equal(st["cam"][k], final["cam"][i]), i
        host.close()
    finally:
        engine._override_library_for_tests(None)


@pytest.mark.gpu
def test_gpu_designs_from_a_busy_side_stream_reach_the_next_reset(libmwb_path):
    """Rows and flags written on a side stream behind a long kernel reach the reset enqueued on it; reset() with
    pending designs takes them."""
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    N = 1024
    env = BatchedMiniWorld("MiniWorld-OneRoom-v0", N, env_params=True)
    env.reset(seed=3)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        big = torch.rand(4096, 4096, device="cuda")
        for _ in range(20):
            big = big @ big / 4096.0
        fov = torch.linspace(30.0, 120.0, N, dtype=torch.float64, device="cuda")
        env.set_env_param(torch.arange(N, device="cuda"), "cam_fov_y", fov)
        env.set_env_param(np.arange(N), "cam_height", None, 0.5, 3.0)
        env.reset(seed=5)
        cam = env.get_state()["cam"]
    assert np.array_equal(cam[:, 3], fov.cpu().numpy())
    assert not env.params_pending.any()
    assert np.array_equal(env.episode_params[:, 19, 0].cpu().numpy(), fov.cpu().numpy())
    env.close()


@pytest.mark.gpu
def test_gpu_wide_cameras_render_against_the_oracle(libmwb_path, softgl_lib):
    """Wide designed cameras (cam_fov_y 30-120, cam_height 0.5-3 m) at every device-reset level: no capacity fault, and
    sampled frames match the pixel oracle within 1 LSB with identical depth."""
    import torch
    from miniworld_b200.assets import Texture
    from miniworld_b200.batched import BatchedMiniWorld
    from test_start_poses import host_env
    for level in ("MiniWorld-FourRooms-v0", "MiniWorld-PickupObjects-v0", "MiniWorld-MazeS3-v0",
                  "MiniWorld-Sidewalk-v0", "MiniWorld-CollectHealth-v0"):
        N = 512
        env = BatchedMiniWorld(level, N, want_depth=True, env_params=True)
        ts = softgl_lib.TextureSet([t.texels for t in Texture.registry])      # the textures the batch registered
        g = torch.arange(N, device="cuda", dtype=torch.float64)
        fov, height = 30.0 + 90.0 * (g % 16) / 15.0, 0.5 + 2.5 * (g // 16 % 32) / 31.0
        env.set_env_param(np.arange(N), "cam_fov_y", fov)
        env.set_env_param(np.arange(N), "cam_height", height)
        env.reset(seed=100)
        out = env.step_host(np.full(N, 2, np.int32))
        assert env.engine.overflow_count() == 0, level
        st = env.get_state()
        for i in (0, 15, 200, 511):
            ref = host_env(level, {}, 100 + i, {"params": {"cam_fov_y": (float(fov[i]), None, None),
                                                           "cam_height": (float(height[i]), None, None)}})
            ref.agent.pos, ref.agent.dir = st["agent_pos"][i], float(st["agent_dir"][i])
            rgb, depth = softgl_lib.render(ref, ts, lambda tex: tex.tex_id)
            assert np.abs(rgb.astype(int) - out["obs"][i].astype(int)).max() <= 1, (level, i)
            assert np.array_equal(depth, out["depth"][i]), (level, i)
        env.close()
