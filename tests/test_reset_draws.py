"""Reset draws (mwb_enable_reset_draws, BatchedMiniWorld(reset_draws=True)): designed resets against the host's
MiniWorldEnv.reset(options={"draws": ...}) world field for field, the reference goldens, rollouts against host-reset
followers, the three arrays across level changes, subset resets and bank loads, snapshots and errors.  CPU cases run
the kernels' host build; `gpu` cases run libmwb.so on the device."""
import math

import numpy as np
import pytest

from level_parity import assert_env_equal, full_state, seed_reset, short_level
from test_maze_layouts import assert_world_equals_host, host_array
from test_start_poses import _Designed, host_env

# every level with reset draws, with its draw count
DRAW_LEVELS = [("MiniWorld-Hallway-v0", {}, 1), ("MiniWorld-TMaze-v0", {}, 2), ("MiniWorld-TMazeLeft-v0", {}, 1),
               ("MiniWorld-TMazeRight-v0", {}, 1), ("MiniWorld-YMaze-v0", {}, 2), ("MiniWorld-YMazeLeft-v0", {}, 1),
               ("MiniWorld-YMazeRight-v0", {}, 1), ("MiniWorld-PickupObjects-v0", {}, 10),
               ("MiniWorld-PickupObjects-v0", {"num_objs": 2}, 4), ("MiniWorld-RoomObjects-v0", {}, 3),
               ("MiniWorld-PutNext-v0", {}, 6)]


def supports(spec, v):
    if spec["kind"] == "choice":
        return 0 <= v < spec["n"] and v == math.floor(v)
    return math.isfinite(v) and spec["lo"] <= v <= spec["hi"]


def in_support(spec, rs):
    return float(rs.integers(0, spec["n"])) if spec["kind"] == "choice" else float(rs.uniform(spec["lo"], spec["hi"]))


def designs(specs, rs):
    """One design {d: v} per env: none, every draw in support, one index, NaN everywhere, each out-of-support value of
    each draw (n, -1, 0.5 for a choice; below lo, above hi, +-inf for a uniform), the support's edges, and an index
    beyond the level's count."""
    out = [{}, {s["index"]: in_support(s, rs) for s in specs}, {specs[-1]["index"]: in_support(specs[-1], rs)},
           {s["index"]: math.nan for s in specs}]
    for s in specs:
        bad = [s["n"], -1.0, 0.5] if s["kind"] == "choice" else [s["lo"] - 1e-9, s["hi"] + 0.01, math.inf, -math.inf]
        edges = [float(s["n"] - 1), 0.0] if s["kind"] == "choice" else [s["lo"], s["hi"]]
        out += [{s["index"]: v} for v in bad + edges]
    out.append({len(specs) + 3: 0.0})
    return out


def draw_rows(ds, D):
    rows = np.full((len(ds), D), np.nan)
    for i, d in enumerate(ds):
        for k, v in d.items():
            if k < D:
                rows[i, k] = v
    return rows


def put(env, name, ids, vals):
    """view[ids] = vals through numpy on the host build, torch ops on the device."""
    view = getattr(env, name)
    if env.engine.host_memory:
        view[ids] = vals
    else:
        import torch
        view[torch.as_tensor(ids, device=view.device)] = torch.as_tensor(np.ascontiguousarray(vals), device=view.device)


def assert_kinds(env, i, host, where):
    """The entity kinds of env i (one-level batch) are the host world's."""
    ents = env.get_state()["ents"][i]
    kinds = [env.program.proto_kinds[p] for p in ents["proto"] if p >= 0]
    assert kinds == [type(e).__name__ for e in host.entities], where


@pytest.mark.parametrize("mode", ["plain", "dr", "dr_episode_seeds"])
@pytest.mark.parametrize("level,kwargs,count", DRAW_LEVELS,
                         ids=[lv + ("_2objs" if kw else "") for lv, kw, _ in DRAW_LEVELS])
def test_designed_resets_equal_the_host_world(hostsim_path, level, kwargs, count, mode):
    """Every design kind: the device reset equals the host's reset(seed, options={"draws": ...}) field for field,
    episode_draws equals the host's outcomes, designed where in support and drawn otherwise, and draws_pending is
    cleared while the rows stay."""
    from miniworld_b200.batched import BatchedMiniWorld
    kw = dict(kwargs, **({} if mode == "plain" else {"domain_rand": True}))
    rs = np.random.default_rng(len(level) + len(mode))
    probe = BatchedMiniWorld(level, 1, level_kwargs=kw, reset_draws=True)
    specs = probe.draw_specs[0]
    probe.close()
    assert [s["index"] for s in specs] == list(range(count)) and all(s["label"] for s in specs)
    ds = designs(specs, rs)
    N = len(ds)
    env = BatchedMiniWorld(level, N, level_kwargs=kw, reset_draws=True, episode_seeds=mode == "dr_episode_seeds")
    assert env.next_draws.shape == (N, count)
    put(env, "next_draws", np.arange(N), draw_rows(ds, count))
    put(env, "draws_pending", np.arange(N), np.ones(N, np.uint8))
    rows = host_array(env.next_draws).copy()
    s = 300 + np.arange(N)
    if mode == "dr_episode_seeds":
        env.set_env_seed(np.arange(N), s)
        env.engine.reset()
    else:
        seed_reset(env, s)
    assert not host_array(env.draws_pending).any() and np.array_equal(host_array(env.next_draws), rows, equal_nan=True)
    got = host_array(env.episode_draws)
    for i, d in enumerate(ds):
        host = host_env(level, kw, int(s[i]), {"draws": d})
        assert_world_equals_host(env, i, host, (level, mode, i))
        assert_kinds(env, i, host, (level, mode, i))
        assert np.array_equal(got[i], host.episode_draws), (i, got[i], host.episode_draws)
        for k, v in d.items():
            if k < count:
                assert got[i, k] == v if supports(specs[k], v) else got[i, k] != v, (i, k, v)
        assert all(supports(spec, got[i, k]) for k, spec in enumerate(specs)), i
    assert env.engine.overflow_count() == 0
    env.close()


def test_levels_without_draws_consume_the_flag(hostsim_path):
    """A table of draw levels and levels without draws, with level changes: a reset at a level without draws consumes
    the flag and records NaN; rows beyond a level's count are ignored; each reset reads the rows against the level it
    resolves to."""
    from miniworld_b200.batched import BatchedMiniWorld
    rows = ["MiniWorld-OneRoom-v0", "MiniWorld-TMaze-v0", "MiniWorld-PickupObjects-v0", "MiniWorld-FourRooms-v0"]
    N = 8
    env = BatchedMiniWorld(rows, N, dynamic_levels=True, reset_draws=True, env_level=np.arange(N) % 4)
    assert [len(s) for s in env.draw_specs] == [0, 2, 10, 0] and env.next_draws.shape == (N, 10)
    plain = BatchedMiniWorld(rows, N, dynamic_levels=True, env_level=np.arange(N) % 4)
    target = np.array([1, 0, 3, 2, 0, 1, 2, 3], np.int32)       # every env changes level at its reset
    design = np.tile([1.0, 0.25, 2.0, 3.0, 1.0, 6.0, 0.0, 1.0, 2.0, 5.0], (N, 1))
    put(env, "next_draws", np.arange(N), design)
    put(env, "draws_pending", np.arange(N), np.ones(N, np.uint8))
    for e in (env, plain):
        e.set_env_level(np.arange(N), target)
        seed_reset(e, 40 + np.arange(N))
    got = host_array(env.episode_draws)
    assert not host_array(env.draws_pending).any()
    for i in range(N):
        lv = rows[target[i]]
        n = len(env.draw_specs[target[i]])
        assert np.isnan(got[i, n:]).all(), i
        d = {k: design[i, k] for k in range(10)}
        host = host_env(lv, {}, 40 + i, {"draws": d})
        assert_world_equals_host(env, i, host, i)
        assert np.array_equal(got[i, :n], host.episode_draws), i
        if n == 0:
            assert_env_equal(full_state(env), i, full_state(plain), i, i)
    env.close()
    plain.close()


# reference goldens (oracle/gen_draws_golden.py): case -> (level, kwargs of the level)
DRAW_CASES = {"tmaze": ("MiniWorld-TMaze-v0", {}), "ymaze_dr": ("MiniWorld-YMaze-v0", {"domain_rand": True}),
              "pickup": ("MiniWorld-PickupObjects-v0", {}), "roomobjects": ("MiniWorld-RoomObjects-v0", {}),
              "putnext_dr": ("MiniWorld-PutNext-v0", {"domain_rand": True}), "hallway": ("MiniWorld-Hallway-v0", {})}


def replay_draw_golden(case):
    """Replay golden `case` of the unmodified reference: before every reset (the seeded one and every auto-reset) the
    env's design for its next episode is written into next_draws / draws_pending, and every step the state, rewards,
    flags and stream equal the reference's; at every reset episode_draws names the outcomes the design allows."""
    from conftest import golden
    from test_level_params import golden_mismatches
    from miniworld_b200.batched import BatchedMiniWorld
    g = golden("draws_" + case)
    level, kw = DRAW_CASES[case]
    T, N = g["actions"].shape
    env = BatchedMiniWorld(short_level(level, int(g["episode_steps"])), N, level_kwargs=kw, reset_draws=True)
    specs = env.draw_specs[0]
    assert g["design_draws"].shape[2] == len(specs)

    def queue(ids, ep):
        put(env, "next_draws", ids, g["design_draws"][ids, ep])
        put(env, "draws_pending", ids, g["design_pending"][ids, ep].astype(np.uint8))

    ep = np.zeros(N, np.int64)
    queue(np.arange(N), ep)
    seed_reset(env, 1000 + np.arange(N))
    designed = replaced = 0
    out = None
    for t in range(T + 1):
        if t:
            out = env.step_host(g["actions"][t - 1], out, render=False)
        st = full_state(env)
        sub = None if out is None else {key: out[key] for key in ("reward", "terminated", "truncated")}
        bad = golden_mismatches(st, np.arange(N), g, t, sub)
        assert not bad, "%s row %d: %s" % (case, t, "; ".join(bad))
        assert np.array_equal(ep, g["episode"][t]), (case, t)
        got = host_array(env.episode_draws)
        for i in np.nonzero(g["was_reset"][t])[0]:
            if g["design_pending"][i, ep[i]]:
                designed += 1
                for k, v in enumerate(g["design_draws"][i, ep[i]]):
                    if supports(specs[k], v):
                        assert got[i, k] == v, (case, t, i, k)
                        replaced += 1
            assert all(supports(specs[k], got[i, k]) for k in range(len(specs))), (case, t, i)
        if out is not None or t == 0:
            done = np.nonzero(g["terminated"][t] | g["truncated"][t])[0]
            if done.size:
                ep[done] += 1
                queue(done, ep[done])
    assert designed > 50 and replaced > 50 and env.engine.overflow_count() == 0
    env.close()


@pytest.mark.parametrize("case", sorted(DRAW_CASES))
def test_designed_episodes_follow_the_reference(hostsim_path, case):
    replay_draw_golden(case)


@pytest.mark.parametrize("level,kwargs,steps", [("MiniWorld-TMaze-v0", {}, 9),
                                                ("MiniWorld-YMaze-v0", {"domain_rand": True}, 8),
                                                ("MiniWorld-Hallway-v0", {}, 7)],
                         ids=["tmaze", "ymaze_dr", "hallway"])
def test_rollout_equals_host_world_followers(hostsim_path, level, kwargs, steps):
    """300 steps with auto-resets; every step numpy writes designs for some done envs.  A host-reset batch whose envs
    reset with the same options follows: rewards, flags and info["draws"] every step, frames and depth byte-identical
    every fifth step, state and stream at the end."""
    from miniworld_b200.batched import BatchedMiniWorld
    base = short_level(level, steps)
    follower_cls = type("Designed" + base.__name__, (_Designed, base), {"queue": []})
    N, T = 6, 300
    a = BatchedMiniWorld(base, N, level_kwargs=kwargs, reset_draws=True, want_depth=True)
    b = BatchedMiniWorld(follower_cls, N, level_kwargs=kwargs, want_depth=True)
    assert a.device_reset and not b.device_reset
    specs = a.draw_specs[0]
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
        for i in np.nonzero(b.get_state()["step_count"] == 0)[0]:
            if t and b._workers[i] is not None and hasattr(b._workers[i], "episode_draws"):
                assert np.array_equal(host_array(a.episode_draws)[i], b._workers[i].episode_draws), (t, i)
        done = np.nonzero(oa["terminated"] | oa["truncated"])[0]
        queue = []
        a.next_draws[:] = np.nan                          # this step's designs only
        for i in done:                                    # ascending: the order the host batch resets them in
            if rs.random() < 0.7:
                d = {s["index"]: in_support(s, rs) if rs.random() < 0.8 else math.nan for s in specs
                     if rs.random() < 0.6}
                for k, v in d.items():
                    a.set_env_draws([i], k, v)
                queue.append({"draws": d})
                designed += 1
            else:
                queue.append({"draws": {}})
        follower_cls.queue[:] = queue
    assert designed > 30
    from miniworld_b200.engine import RNG_DTYPE, rng_state_of
    sa, sb = a.get_state(rng=True), b.get_state(rng=True)
    if not b.domain_rand:
        sb["rng"] = np.array([rng_state_of(w.np_random) for w in b._workers], RNG_DTYPE)
    for key in ("agent_pos", "agent_dir", "step_count", "rng", "cam", "env_params"):
        assert np.array_equal(sa[key], sb[key]), key
    a.close()
    b.close()


def test_the_arrays_follow_a_numpy_model(hostsim_path):
    """A table with level changes and a state bank: a pending design is consumed by the next reset that runs a program
    at any level (auto-resets and subset resets included), the rows stay, a bank load leaves it pending and restores
    the saved episode's episode_draws, and episode_draws names the running episode."""
    from miniworld_b200.batched import BatchedMiniWorld
    rows = [short_level("MiniWorld-TMaze-v0", 5), short_level("MiniWorld-OneRoom-v0", 4),
            short_level("MiniWorld-PickupObjects-v0", 6)]
    N, T = 9, 160
    env = BatchedMiniWorld(rows, N, dynamic_levels=True, reset_draws=True, state_bank=4)
    seed_reset(env, 10 + np.arange(N))
    D = env.next_draws.shape[1]
    rs = np.random.default_rng(3)
    pend = np.zeros(N, np.uint8)
    nxt = np.full((N, D), np.nan)
    saved = {}                                            # slot -> episode_draws row of the saved env
    out = None
    took = loads = 0

    def check(reset, t, loaded):
        nonlocal took, loads
        got = host_array(env.episode_draws)
        lv = host_array(env.level_tensor)
        for i in np.nonzero(reset)[0]:
            if loaded[i] >= 0:
                assert np.array_equal(got[i], saved[loaded[i]], equal_nan=True), (t, i)
                loads += 1
                continue
            specs = env.draw_specs[lv[i]]
            assert np.isnan(got[i, len(specs):]).all(), (t, i)
            if pend[i]:
                for s in specs:
                    v = nxt[i, s["index"]]
                    if supports(s, v):
                        assert got[i, s["index"]] == v, (t, i)
                pend[i] = 0
                took += 1
        assert np.array_equal(host_array(env.draws_pending), pend), t
        assert np.array_equal(host_array(env.next_draws), nxt, equal_nan=True), t

    prev_done = np.zeros(N, bool)
    pending_load = np.full(N, -1)
    for t in range(T):
        ids = np.nonzero(rs.random(N) < 0.2)[0]
        if ids.size:
            k = int(rs.integers(0, D))
            v = rs.choice([0.0, 1.0, 2.0, 0.5, -0.3, np.nan], ids.size)
            env.set_env_draws(ids, k, v)
            nxt[ids, k] = v
            pend[ids] = 1
        if t % 23 == 7:                                   # save two envs, and load a saved slot at some envs' next resets
            src = rs.choice(N, 2, replace=False)
            slots = np.array([t % 4, (t + 1) % 4])
            env.save_states(src, slots)
            for s, i in zip(slots, src):
                saved[int(s)] = host_array(env.episode_draws)[i].copy()
        if t % 11 == 3 and saved:
            ids = rs.choice(N, 2, replace=False)
            slot = int(rs.choice(sorted(saved)))
            env.set_env_state(ids, slot)
            pending_load[ids] = slot
        if t % 37 == 5:                                   # a subset reset outside the step
            sub = np.array([1, 4], np.int32)
            env.engine.reset(sub)
            loaded = np.where(np.isin(np.arange(N), sub), pending_load, -1)
            pending_load[sub] = -1
            check(np.isin(np.arange(N), sub), t, loaded)
            prev_done[sub] = False
        env.set_env_level(np.nonzero(rs.random(N) < 0.2)[0], int(rs.integers(0, 3)))
        out = env.step_host(rs.integers(0, 3, N).astype(np.int32), out, render=False)
        loaded = np.where(prev_done, pending_load, -1)
        pending_load[prev_done] = -1
        check(prev_done, t, loaded)
        prev_done = (out["terminated"] | out["truncated"]).astype(bool)
    assert took > 20 and loads > 3
    env.close()


@pytest.mark.parametrize("level", ["MiniWorld-TMaze-v0", "MiniWorld-YMaze-v0"])
def test_a_designed_pose_wins_over_a_designed_side(hostsim_path, level):
    """A designed goal side together with a designed box pose puts the box at the pose; the side is still recorded and
    the stream advances as without either."""
    from miniworld_b200.batched import BatchedMiniWorld
    env = BatchedMiniWorld(level, 4, reset_draws=True, start_poses=True)
    env.set_env_draws(np.arange(4), 0, [0.0, 1.0, 0.0, 1.0])
    env.set_env_pose([0, 1], 0, [3.0, 4.0], [0.5, -0.5], 0.25)
    seed_reset(env, [5, 6, 7, 8])
    st = env.get_state()
    assert host_array(env.episode_draws)[:, 0].tolist() == [0.0, 1.0, 0.0, 1.0]
    for i, (x, z) in enumerate([(3.0, 0.5), (4.0, -0.5)]):
        assert st["ents"][i, 0]["pos"][0] == x and st["ents"][i, 0]["pos"][2] == z, i
    for i in range(4):
        opts = {"draws": {0: float(i % 2)}}
        if i < 2:
            opts["poses"] = {0: ((3.0, 0.5, 0.25), (4.0, -0.5, 0.25))[i]}
        assert_world_equals_host(env, i, host_env(level, {}, 5 + i, opts), i)
    env.close()


def test_snapshots_within_and_across_modes(hostsim_path):
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import EngineError
    make = lambda on: BatchedMiniWorld("MiniWorld-TMaze-v0", 4, reset_draws=on)
    a = make(True)
    seed_reset(a, [1, 2, 3, 4])
    a.set_env_draws([0, 2], 0, 1.0)
    blob = a.snapshot()
    assert blob[:4].tobytes() == b"MWB\xd3"
    st = full_state(a)
    arrays = [host_array(v).copy() for v in (a.next_draws, a.draws_pending, a.episode_draws)]
    acts = np.full(4, 2, np.int32)
    for _ in range(12):
        a.step_host(acts, render=False)
    a.restore(blob)
    for want, v in zip(arrays, (a.next_draws, a.draws_pending, a.episode_draws)):
        assert np.array_equal(host_array(v), want, equal_nan=True)
    for i in range(4):
        assert_env_equal(st, i, full_state(a), i, i)
    b = make(False)
    plain = b.snapshot()
    assert plain[:4].tobytes() == b"MWBS" and plain.size == blob.size - 4 * (2 * 8 * 2 + 1)
    seed_reset(b, [1, 2, 3, 4])
    same = make(False)
    seed_reset(same, [1, 2, 3, 4])
    assert np.array_equal(b.snapshot(), same.snapshot())
    with pytest.raises(EngineError, match="error -6"):
        b.restore(blob)
    with pytest.raises(EngineError, match="error -6"):
        a.restore(plain)
    for e in (a, b, same):
        e.close()


def test_a_bank_record_carries_episode_draws(hostsim_path):
    """With the bank on, a record holds episode_draws; the pending inputs stay out of it."""
    from miniworld_b200.batched import BatchedMiniWorld
    env = BatchedMiniWorld("MiniWorld-PickupObjects-v0", 3, reset_draws=True, state_bank=2)
    env.set_env_draws([0], 1, 4.0)
    seed_reset(env, [1, 2, 3])
    env.save_states([0], [1])
    want = host_array(env.episode_draws)[0].copy()
    env.set_env_draws([2], 0, 2.0)
    env.set_env_state([2], 1)
    env.engine.reset(np.array([2], np.int32))
    assert np.array_equal(host_array(env.episode_draws)[2], want) and want[1] == 4.0
    assert host_array(env.draws_pending).tolist() == [0, 0, 1]
    env.close()


def test_errors(hostsim_path):
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import EngineError
    from miniworld_b200.envs import LEVELS
    with pytest.raises(ValueError, match="reset draw"):
        BatchedMiniWorld("MiniWorld-OneRoom-v0", 2, reset_draws=True)
    with pytest.raises(ValueError, match="reset draw"):
        BatchedMiniWorld(["MiniWorld-OneRoom-v0", "MiniWorld-FourRooms-v0"], 2, reset_draws=True)
    host_only = type("HostOnlyTMaze", (LEVELS["MiniWorld-TMaze-v0"],), {"device_program": None})
    with pytest.raises(TypeError, match="host"):
        BatchedMiniWorld(host_only, 2, reset_draws=True)
    env = BatchedMiniWorld("MiniWorld-TMaze-v0", 4, reset_draws=True, state_bank=2)
    assert np.isnan(host_array(env.next_draws)).all() and np.isnan(host_array(env.episode_draws)).all()
    assert env.draw_specs[0][0] == dict(index=0, kind="choice", n=2, label=env.draw_specs[0][0]["label"])
    assert env.draw_specs[0][1]["kind"] == "uniform" and env.draw_specs[0][1]["hi"] == math.pi / 4
    with pytest.raises(EngineError, match="error -6"):
        env.engine.enable_reset_draws()                          # already on
    for args in [([4], 0, 1.0), ([-1], 0, 1.0), ([0], 2, 1.0), ([0], -1, 1.0), ([0], True, 1.0), ([0], "side", 1.0),
                 ([0], 0.0, 1.0), ([0, 1], 0, [1.0, 2.0, 3.0]), ([[0, 1]], 0, 1.0), ([0.5], 0, 1.0), ([0], 0, "a")]:
        with pytest.raises(ValueError):
            env.set_env_draws(*args)
    assert not host_array(env.draws_pending).any() and np.isnan(host_array(env.next_draws)).all()
    env.set_env_draws([1, 2, 1], 0, [1.0, 0.0, 0.0])
    assert host_array(env.next_draws)[:, 0].tolist()[1:3] == [0.0, 0.0]
    assert host_array(env.draws_pending).tolist() == [0, 1, 1, 0]
    env.close()
    banked = BatchedMiniWorld("MiniWorld-TMaze-v0", 2, state_bank=2)
    with pytest.raises(EngineError, match="error -6"):
        banked.engine.enable_reset_draws()                       # after the bank
    banked.close()
    off = BatchedMiniWorld("MiniWorld-TMaze-v0", 2)
    for name in ("next_draws", "draws_pending", "episode_draws"):
        with pytest.raises(EngineError, match="error -6"):
            off.engine.state_array(name)
        with pytest.raises(RuntimeError, match="reset_draws=True"):
            getattr(off, name)
    with pytest.raises(RuntimeError):
        off.set_env_draws([0], 0, 1.0)
    off.close()


def test_program_draw_indices_are_checked(hostsim_path):
    """A program whose CHOICE / UNIFORM ops do not number their draws 0, 1, ... in `room` is refused (MWB_EINVAL)."""
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import EngineError, OP_CHOICE
    env = BatchedMiniWorld("MiniWorld-TMaze-v0", 2)
    ops = env.program.op_array()
    ops["room"][ops["op"] == OP_CHOICE] = 1
    env.engine.set_program(ops)
    with pytest.raises(EngineError, match="error -1"):
        env.engine.enable_reset_draws()
    env.close()


def test_host_mirror_leaves_other_draws_alone():
    """reset(options={"draws": ...}) touches only _gen_world()'s own draws: placement, textures and Maze carves run
    as without the option, and without the option the reset is unchanged."""
    from miniworld_b200.envs import LEVELS
    for level in ("MiniWorld-MazeS3-v0", "MiniWorld-OneRoom-v0", "MiniWorld-FourRooms-v0"):
        a = host_env(level, {"domain_rand": True}, 9)
        b = host_env(level, {"domain_rand": True}, 9, {"draws": {0: 0.0, 1: 1.0, 2: 0.5}})
        assert b.episode_draws == [] and np.array_equal(a.agent.pos, b.agent.pos)
        assert a.np_random.bit_generator.state == b.np_random.bit_generator.state
    env = LEVELS["MiniWorld-TMaze-v0"](device=None)
    env.reset(seed=3, options={"draws": {0: 1}})
    assert env.box.pos[2] > 0 and env.episode_draws[0] == 1.0 and type(env.np_random).__name__ == "Generator"


def _shard_worker(rank, port, hostsim, q):
    import os
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=2)
    from miniworld_b200 import engine
    from miniworld_b200.dist import ShardedMiniWorld
    engine._override_library_for_tests(hostsim)
    env = ShardedMiniWorld(short_level("MiniWorld-TMaze-v0", 7), 7, dist=dist, reset_draws=True)
    seed_reset(env.local, [1000 + env.start + k for k in range(env.count)])
    outs = shard_run(env.local, env.start, 40, 7, rank, lambda a: env.scatter_actions(a, like=torch.zeros(1)),
                     env.gather_to_root)
    if rank == 0:
        q.put(outs)
    dist.barrier()
    dist.destroy_process_group()


def shard_run(env, start, steps, total, rank=0, scatter=None, gather=None):
    """Every step the done envs of a shard starting at global env `start` get a goal side keyed by their global index."""
    import torch
    acts_all = np.random.default_rng(5).integers(0, 3, size=(steps, total), dtype=np.int32)
    outs, out = [], None
    for t in range(steps):
        acts = acts_all[t] if scatter is None else scatter(torch.as_tensor(acts_all[t]) if rank == 0 else None).numpy()
        out = env.step_host(acts, out, render=t == steps - 1)
        done = np.nonzero((out["terminated"] | out["truncated"]).astype(bool))[0]
        gk = start + done
        if done.size:
            env.set_env_draws(done, 0, ((gk + t) % 2).astype(np.float64))
        got = [out["obs"], out["reward"], np.array(env.episode_draws), np.array(env.draws_pending)]
        if gather is not None:
            got = [gather(torch.as_tensor(x)).numpy() if rank == 0 else gather(torch.as_tensor(x)) for x in got]
        outs.append([np.array(x) for x in got] if rank == 0 else None)
    return outs


def test_sharded_draw_writes_equal_one_process(hostsim_path):
    """Two gloo ranks that write their envs' designs into their local batches equal one process."""
    import os
    import torch.multiprocessing as mp
    from miniworld_b200.batched import BatchedMiniWorld
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 41000 + os.getpid() % 2000
    procs = [ctx.Process(target=_shard_worker, args=(r, port, hostsim_path, q)) for r in range(2)]
    for p in procs:
        p.start()
    sharded = q.get(timeout=300)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    env = BatchedMiniWorld(short_level("MiniWorld-TMaze-v0", 7), 7, reset_draws=True)
    seed_reset(env, 1000 + np.arange(7))
    one = shard_run(env, 0, 40, 7)
    for t, (x, y) in enumerate(zip(one, sharded)):
        for k in (1, 2, 3):
            assert np.array_equal(x[k], y[k], equal_nan=True), (t, k)
    assert np.array_equal(one[-1][0], sharded[-1][0]) and 0 < one[-1][0].mean() < 255
    assert sum(int(x[3].sum()) for x in one) > 0
    env.close()


# ------------------------------------------------------------------ GPU (libmwb.so)
@pytest.mark.gpu
def test_gpu_balanced_sides_match_the_host_build(libmwb_path):
    """4096 TMaze envs, 300 steps in torch ops without a sync: every done env's next goal side is the side with fewer
    episodes so far, and per-side successes are counted from info["draws"].  A sample of envs replays on the host
    build with the recorded actions and designs: flags, rewards and info["draws"] every step, state at the end."""
    import subprocess
    import torch
    from conftest import ROOT
    from miniworld_b200 import engine
    from miniworld_b200.batched import BatchedMiniWorld
    level = short_level("MiniWorld-TMaze-v0", 15)
    N, T = 4096, 300
    env = BatchedMiniWorld(level, N, reset_draws=True)
    dev = torch.device("cuda")
    gen = torch.Generator(device="cuda")
    gen.manual_seed(3)
    env.reset(seed=500)
    acts = torch.randint(0, 3, (T, N), dtype=torch.int32, device=dev, generator=gen)
    turn = torch.arange(N, device=dev)                 # each env alternates sides, half of the envs starting at each
    episodes = torch.zeros(2, dtype=torch.float64, device=dev)
    wins = torch.zeros(2, dtype=torch.float64, device=dev)
    sample = np.sort(np.random.default_rng(4).choice(N, 64, replace=False))
    sample_t = torch.as_tensor(sample, device=dev)
    hist = {k: [] for k in ("draws", "rew", "te", "tr", "next", "pending")}
    for t in range(T):
        obs, rew, te, tr, info = env.step(acts[t])
        done = te | tr
        side = info["draws"][:, 0].long()
        episodes += torch.bincount(side[done], minlength=2).double()
        wins += torch.bincount(side[te], minlength=2).double()
        turn += done.long()
        env.next_draws[:, 0] = torch.where(done, (turn % 2).double(), env.next_draws[:, 0])
        env.draws_pending.copy_(torch.where(done, torch.ones_like(env.draws_pending), env.draws_pending))
        for k, v in (("draws", info["draws"]), ("rew", rew), ("te", te), ("tr", tr), ("next", env.next_draws),
                     ("pending", env.draws_pending)):
            hist[k].append(v[sample_t].clone())
    final = full_state(env)
    counts = episodes.cpu().numpy()
    hist = {k: torch.stack(v).cpu().numpy() for k, v in hist.items()}
    assert counts.sum() > 10000 and abs(counts[0] - counts[1]) <= 0.02 * counts.sum()
    assert (wins <= episodes).all()
    acts = acts.cpu().numpy()
    env.close()

    lib = subprocess.check_output([ROOT + "/tests/hostsim/build.sh"]).decode().strip().splitlines()[-1]
    engine._override_library_for_tests(lib)
    try:
        host = BatchedMiniWorld(level, len(sample), reset_draws=True)
        seed_reset(host, 500 + sample)
        out = None
        for t in range(T):
            out = host.step_host(acts[t, sample], out, render=False)
            assert np.array_equal(out["reward"], hist["rew"][t]), t
            assert np.array_equal(out["terminated"].astype(bool), hist["te"][t]), t
            assert np.array_equal(out["truncated"].astype(bool), hist["tr"][t]), t
            assert np.array_equal(host.episode_draws, hist["draws"][t], equal_nan=True), t
            host.next_draws[:] = hist["next"][t]
            host.draws_pending[:] = hist["pending"][t]
        st = full_state(host)
        for j, i in enumerate(sample):
            assert_env_equal(st, j, final, i, ("final", int(i)))
        host.close()
    finally:
        engine._override_library_for_tests(None)


@pytest.mark.gpu
@pytest.mark.parametrize("level", ["MiniWorld-PickupObjects-v0", "MiniWorld-PutNext-v0", "MiniWorld-YMaze-v0",
                                   "MiniWorld-RoomObjects-v0"])
def test_gpu_designed_frames_match_the_pixel_oracle(libmwb_path, softgl_lib, level):
    """Frames of designed resets (kinds, colours, sizes and sides in and out of support) against oracle/softgl.c
    rendering the host-built world of the same design, with no capacity fault."""
    from test_render_paths import assert_matches, oracle_frame
    from miniworld_b200.batched import BatchedMiniWorld
    rs = np.random.default_rng(6)
    probe = BatchedMiniWorld(level, 1, reset_draws=True)
    specs = probe.draw_specs[0]
    probe.close()
    ds = designs(specs, rs)[:16]
    N = len(ds)
    env = BatchedMiniWorld(level, N, reset_draws=True, want_depth=True)
    put(env, "next_draws", np.arange(N), draw_rows(ds, len(specs)))
    put(env, "draws_pending", np.arange(N), np.ones(N, np.uint8))
    obs, _ = env.reset(seed=60)
    obs = obs.cpu().numpy()
    depth = env._bufs["depth"].cpu().numpy()
    assert env.engine.overflow_count() == 0
    st = env.get_state(rng=True)
    for i, d in enumerate(ds):
        host = host_env(level, {}, 60 + i, {"draws": d})
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
    level = short_level("MiniWorld-PickupObjects-v0", 3)
    a, b = (BatchedMiniWorld(level, N, domain_rand=True, reset_draws=True) for _ in range(2))
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
            kinds = torch.tensor([2.0 - k, 4.0], dtype=torch.float64, device="cuda")
            b.next_draws[:, :2].copy_(kinds.expand(N, 2))
            b.draws_pending.fill_(1)
            torch.cuda.synchronize()
            torch.cuda._sleep(100_000_000)
            a.next_draws[:, :2].copy_(kinds.expand(N, 2))
            a.draws_pending.fill_(1)
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
            assert torch.equal(a.episode_draws, b.episode_draws), call
            assert bool((a.draws_pending[took] == 0).all()) and bool((a.draws_pending[~took] == 1).all()), call
            assert bool((a.episode_draws[took, :2] == kinds).all()), call
    a.close()
    b.close()


@pytest.mark.gpu
def test_gpu_reset_takes_pending_designs(libmwb_path):
    """reset() after set_env_draws (host values and a CUDA tensor) takes the designs, as the host's reset does."""
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    N = 16
    kw = {"domain_rand": True}
    env = BatchedMiniWorld("MiniWorld-RoomObjects-v0", N, level_kwargs=kw, reset_draws=True)
    rs = np.random.default_rng(2)
    cols = rs.integers(0, 6, (N, 3)).astype(np.float64)
    env.set_env_draws(np.arange(N), 0, cols[:, 0])
    env.set_env_draws(np.arange(N), 2, torch.as_tensor(cols[:, 2], device="cuda"))
    env.reset(seed=80)
    assert not host_array(env.draws_pending).any()
    for i in range(N):
        host = host_env("MiniWorld-RoomObjects-v0", kw, 80 + i, {"draws": {0: cols[i, 0], 2: cols[i, 2]}})
        assert_world_equals_host(env, i, host, i)
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(DRAW_CASES))
def test_gpu_designed_episodes_follow_the_reference(libmwb_path, case):
    """The reference goldens replayed on the device, designs written with torch ops."""
    replay_draw_golden(case)
