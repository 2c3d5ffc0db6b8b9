"""Domain randomisation per level (mwb_level.domain_rand): rows of a level table that share a level but differ in the
flag must each equal, bit for bit, a single-level batch built with that row's flag -- rewards, flags, state, RNG
streams, frames and depth -- also across level changes between flags, snapshots and sharding.  CPU cases run the
kernels' host build; `gpu` cases run libmwb.so on the device."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from level_parity import (ROOT, STATE_KEYS, Follower, Lockstep, assert_env_equal, full_state, gpu_curriculum,
                          replay_draws, run_sharded, seed_reset, short_level)

# short episodes (8 / 9 / 10 steps) so that truncations and auto-resets happen inside the mix
SHORT_FOURROOMS = short_level("MiniWorld-FourRooms-v0", 8)
SHORT_HALLWAY = short_level("MiniWorld-Hallway-v0", 9)
SHORT_PICKUP = short_level("MiniWorld-PickupObjects-v0", 10)
OFF, ON = {"domain_rand": False}, {"domain_rand": True}
MIXED_ROWS = [(SHORT_FOURROOMS, OFF), (SHORT_FOURROOMS, ON), (SHORT_PICKUP, OFF), (SHORT_PICKUP, ON),
              ("MiniWorld-PutNext-v0", ON), (SHORT_HALLWAY, OFF), ("MiniWorld-Sidewalk-v0", ON),
              ("MiniWorld-CollectHealth-v0", OFF)]


def narrowed_params(frac=0.25):
    """DEFAULT_PARAMS with every range shrunk to `frac` of its width around the default (a middle rung of a
    randomisation ladder)."""
    from miniworld_b200.params import DEFAULT_PARAMS
    p = DEFAULT_PARAMS.copy()
    for name, q in DEFAULT_PARAMS.params.items():
        if isinstance(q.default, np.ndarray):
            lo, hi = q.default - frac * (q.default - q.min), q.default + frac * (q.max - q.default)
        else:
            lo, hi = float(q.default - frac * (q.default - q.min)), float(q.default + frac * (q.max - q.default))
        p.set(name, q.default, lo, hi, q.type)
    return p


# ------------------------------------------------------------------ CPU (kernels' host build)
def test_mixed_flags_equal_single_level_batches(hostsim_path):
    ls = Lockstep(MIXED_ROWS, n_per=2)
    assert [bool(pe.domain_rand) for pe in ls.mix.proto_envs] == [k["domain_rand"] for _, k in MIXED_ROWS]
    rng = np.random.default_rng(7)
    ended = np.zeros(ls.N, np.int64)
    ls.check("reset", False)
    for t in range(70):
        render = t % 10 == 0 or t == 69
        ls.step(ls.actions(rng), render)
        ls.check(t, render)
        ended += ls.out_m["terminated"] | ls.out_m["truncated"]
        if render:
            assert 0 < ls.out_m["obs"].mean() < 255
    # every env of the short rows has truncated (and auto-reset) several times inside the mix
    short = np.isin(ls.el, [0, 1, 2, 3, 5])
    assert (ended[short] >= 5).all()
    assert ls.mix.engine.overflow_count() == 0
    # the flag changes what the envs see: the off and on rows of one level differ in their draws
    sm = full_state(ls.mix)
    assert not np.array_equal(sm["env_params"][ls.el == 0], sm["env_params"][ls.el == 1])
    ls.close()


def side_by_side(rows, per_env_worlds=False, steps=None, domain_rand=False):
    """Rows of one table, each (level, kwargs, golden name or None); envs interleaved over the rows.  A golden row's
    envs replay that golden trajectory (seeds 1000 + j, its actions) and must match it bit for bit every step; the other
    rows' envs take random actions from other seeds."""
    from conftest import golden
    from helpers import state_mismatches
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import RNG_DTYPE, rng_state_of
    gs = {k: golden(name) for k, (_, _, name) in enumerate(rows) if name}
    quota = [gs[k]["actions"].shape[1] if k in gs else 4 for k in range(len(rows))]
    el = []
    while len(el) < sum(quota):                     # round-robin until every row has its envs
        for k in range(len(rows)):
            if el.count(k) < quota[k]:
                el.append(k)
    el = np.array(el, np.int32)
    N = len(el)
    env = BatchedMiniWorld([lv for lv, _, _ in rows], N, env_level=el, level_kwargs=[kw for _, kw, _ in rows],
                           per_env_worlds=per_env_worlds, domain_rand=domain_rand)
    mine = {k: np.nonzero(el == k)[0] for k in range(len(rows))}
    seeds = np.zeros(N, np.int64)
    for k, ids in mine.items():
        seeds[ids] = (1000 if k in gs else 7000 + 100 * k) + np.arange(len(ids))
    env.engine.seed(np.arange(N), np.array([rng_state_of(int(s)) for s in seeds], RNG_DTYPE))
    env.engine.reset()

    class View:
        def __init__(self, ids):
            self.ids = ids

        def get_state(self, **kw):
            return {k: v[self.ids] if np.ndim(v) and len(v) == N else v for k, v in env.get_state(**kw).items()}

    T = min(g["actions"].shape[0] for g in gs.values())
    T = T if steps is None else min(T, steps)
    for k, g in gs.items():
        bad = state_mismatches(View(mine[k]), g, 0, len(mine[k]))
        assert not bad, "after reset: " + "; ".join(bad)
    rng = np.random.default_rng(1)
    acts = np.zeros(N, np.int32)
    out = None
    for t in range(T):
        acts[:] = rng.integers(0, 3, N)
        for k, g in gs.items():
            acts[mine[k]] = g["actions"][t]
        out = env.step_host(acts, out, render=False)
        for k, g in gs.items():
            sub = {key: out[key][mine[k]] for key in ("reward", "terminated", "truncated")}
            bad = state_mismatches(View(mine[k]), g, t + 1, len(mine[k]), sub)
            assert not bad, "%s step %d: %s" % (rows[k][2], t + 1, "; ".join(bad))
    assert env.engine.overflow_count() == 0
    env.close()


@pytest.mark.parametrize("case", ["fourrooms", "pickup", "putnext", "maze"])
def test_reference_trajectories_side_by_side(hostsim_path, case):
    if case == "fourrooms":        # the batch default is on; the off row says so in its kwargs
        side_by_side([("MiniWorld-FourRooms-v0", OFF, "fourrooms"), ("MiniWorld-FourRooms-v0", {}, "fourrooms_dr")],
                     domain_rand=True)
    elif case == "pickup":
        side_by_side([("MiniWorld-PickupObjects-v0", {}, "pickup"), ("MiniWorld-PickupObjects-v0", ON, "pickup_dr")])
    elif case == "putnext":
        side_by_side([("MiniWorld-PutNext-v0", ON, "putnext_dr"), ("MiniWorld-Hallway-v0", {}, None)])
    else:
        side_by_side([("MiniWorld-MazeS3-v0", {}, "mazes3"), ("MiniWorld-MazeS8-v0", ON, "maze_dr")],
                     per_env_worlds=True, steps=120)


SWITCH_ROWS = [(SHORT_FOURROOMS, OFF), (SHORT_FOURROOMS, ON), (SHORT_PICKUP, ON), (SHORT_PICKUP, OFF),
               ("MiniWorld-FourRooms-v0", dict(ON, params=narrowed_params()))]


def test_level_changes_across_the_flag(hostsim_path):
    """Off -> on and on -> off, by pending assignment (taken at K1's auto-reset) and by weight draws (at mwb_reset):
    after each switch the env equals a one-env batch of its new row, with that row's flag, seeded with the stream it
    carried; the weight draws follow batched.sample_level."""
    from miniworld_b200.batched import BatchedMiniWorld, sample_level
    L, N, seed = len(SWITCH_ROWS), 10, 5
    el = np.arange(N, dtype=np.int32) % L
    env = BatchedMiniWorld([lv for lv, _ in SWITCH_ROWS], N, env_level=el, level_kwargs=[k for _, k in SWITCH_ROWS],
                           want_depth=True, dynamic_levels=True, level_seed=seed)
    seed_reset(env, 60 + np.arange(N))
    rng = np.random.default_rng(2)
    out = None
    for t in range(3):                                   # mid-episode: the shortest episode is 8 steps
        out = env.step_host(rng.integers(0, 3, N).astype(np.int32), out, render=False)
    target = {0: 1, 1: 0, 2: 3, 3: 2, 5: 4, 6: 3}         # off->on, on->off, across levels, onto the narrowed row
    env.set_env_level(list(target), list(target.values()))
    followers, level = {}, el.copy()
    prev_done = np.zeros(N, bool)
    for t in range(40):
        carried = env.get_state(rng=True)["rng"].copy()
        acts = rng.integers(0, 3, N).astype(np.int32)
        render = t % 3 == 0
        out = env.step_host(acts, out, render=render)
        st = full_state(env)
        for f in followers.values():
            f.step_and_check(acts, out, st, render, t)
        for i in np.nonzero(prev_done)[0]:               # env i auto-reset in this step
            if int(i) in target and int(i) not in followers:
                level[i] = target[int(i)]
                followers[int(i)] = Follower(SWITCH_ROWS[level[i]], int(i), carried[i])
                followers[int(i)].check_state(st, ("switch", t))
        assert np.array_equal(env.env_level, level), t
        prev_done = (out["terminated"] | out["truncated"]).astype(bool)
    assert set(followers) == set(target)
    for f in followers.values():
        f.env.close()
    # weight draws at resets of every env: each env then equals a fresh env of its drawn row from its carried stream
    w = np.array([1.0, 2.0, 0.5, 1.0, 1.5], np.float32)
    draws = np.zeros(N, np.int64)
    moved = set()
    for r in range(3):
        env.set_level_weights(w)
        carried = env.get_state(rng=True)["rng"].copy()
        before = env.env_level.copy()
        env.engine.reset()
        want = [sample_level(seed, i, draws[i], w) for i in range(N)]
        draws += 1
        assert list(env.env_level) == want, r
        moved |= {(int(SWITCH_ROWS[a][1]["domain_rand"]), int(SWITCH_ROWS[b][1]["domain_rand"]))
                  for a, b in zip(before, want) if a != b}
        fol = [Follower(SWITCH_ROWS[want[i]], i, carried[i]) for i in range(N)]
        env.set_level_weights(np.zeros(L))              # an auto-reset below keeps its env's row, as the follower does
        st = full_state(env)
        for f in fol:
            f.check_state(st, ("draw", r))
        for t in range(3):
            acts = rng.integers(0, 3, N).astype(np.int32)
            out = env.step_host(acts, out, render=True)
            st = full_state(env)
            for f in fol:
                f.step_and_check(acts, out, st, True, ("draw", r, t))
        for f in fol:
            f.env.close()
    assert {(0, 1), (1, 0)} <= moved                     # the draws crossed the flag both ways
    assert env.engine.overflow_count() == 0
    env.close()


@pytest.mark.parametrize("batch_default", [False, True])
def test_row_kwargs_override_the_batch_default(hostsim_path, batch_default):
    """domain_rand=True with one row {"domain_rand": False}, and the reverse: the row's kwargs win, the batch argument
    is the default of the rows that do not set the flag (no duplicate keyword)."""
    rows = [("MiniWorld-FourRooms-v0", {}), ("MiniWorld-FourRooms-v0", {"domain_rand": not batch_default}),
            ("MiniWorld-PickupObjects-v0", {})]
    ls = Lockstep(rows, n_per=2, domain_rand=batch_default)
    assert [bool(pe.domain_rand) for pe in ls.mix.proto_envs] == [batch_default, not batch_default, batch_default]
    assert ls.mix.engine.cfg.domain_rand == int(batch_default)        # level 0's flag, as mwb_create fills it
    rng = np.random.default_rng(4)
    ls.check("reset", False)
    for t in range(20):
        render = t % 5 == 0
        ls.step((rng.random(ls.N) * ls.own_n).astype(np.int32), render)
        ls.check(t, render)
    ls.close()


@pytest.mark.parametrize("level", ["MiniWorld-FourRooms-v0", "MiniWorld-MazeS3-v0"])
@pytest.mark.parametrize("flag", [True, False])
def test_single_level_kwargs_flag_equals_batch_flag(hostsim_path, level, flag):
    """BatchedMiniWorld(level, level_kwargs={"domain_rand": flag}) equals BatchedMiniWorld(level, domain_rand=flag),
    whatever the batch argument says (before, a flag in level_kwargs was dropped, or raised a duplicate keyword)."""
    from miniworld_b200.batched import BatchedMiniWorld
    N = 4
    a = BatchedMiniWorld(level, N, level_kwargs={"domain_rand": flag}, domain_rand=not flag, want_depth=True)
    b = BatchedMiniWorld(level, N, domain_rand=flag, want_depth=True)
    assert a.domain_rand == b.domain_rand == flag and a.engine.cfg.domain_rand == int(flag)
    for e in (a, b):
        seed_reset(e, 30 + np.arange(N))
    rng = np.random.default_rng(6)
    oa = ob = None
    for t in range(25):
        acts = rng.integers(0, 3, N).astype(np.int32)
        render = t % 6 == 0
        oa = a.step_host(acts, oa, render=render)
        ob = b.step_host(acts, ob, render=render)
        for key in ("reward", "terminated", "truncated") + (("obs", "depth") if render else ()):
            assert np.array_equal(oa[key], ob[key]), (t, key)
        sa, sb = full_state(a), full_state(b)
        for i in range(N):
            assert_env_equal(sa, i, sb, i, t)
    a.close()
    b.close()


def test_c_abi_level_flag(hostsim_path):
    from miniworld_b200 import engine, pack
    from miniworld_b200.engine import Engine, EngineError, Level
    from miniworld_b200.envs import Hallway
    from miniworld_b200.program import ResetProgram
    with open(os.path.join(ROOT, "include", "mwb.h")) as f:
        assert re.search(r"#define MWB_ABI_VERSION 10\b", f.read())
    assert engine.ABI_VERSION == 10
    # the flag takes the place of the reserved field: mwb_level keeps its size and layout
    assert Level.domain_rand.offset == 20 and C.sizeof(Level) == 24 + C.sizeof(engine.Params)
    lib = engine.load_library()
    sizes = (C.c_int32 * 32)()
    n = lib.mwb_abi_sizes(sizes, 32)
    assert list(sizes[:n]) == engine._expected_sizes()
    pe = Hallway(device=None)
    prog = ResetProgram()
    pe.device_program(prog)
    geom = pack.pack_geometry(pe)
    eng = Engine(3, max_rooms=len(geom[0]), max_quads=len(geom[1]), max_segs=len(geom[2]), max_ents=2, rule=(1, 0))
    eng.sync_assets()
    eng.set_protos(prog.proto_array())
    lv = dict(rule=(1, 0), max_episode_steps=250, params=pe.params, geometry=geom, ops=prog.op_array())
    for bad in (2, -1):
        with pytest.raises(EngineError, match="error -1"):
            eng.set_levels([dict(lv, domain_rand=0), dict(lv, domain_rand=bad)], [0, 1, 1])
    # the handle is still usable: a valid table, a reset and a step
    eng.set_levels([dict(lv, domain_rand=0), dict(lv, domain_rand=1)], [0, 1, 1])
    eng.seed(np.arange(3), np.array([engine.rng_state_of(s) for s in (1, 2, 2)], engine.RNG_DTYPE))
    eng.reset()
    st = eng.get_state(rng=True)
    # envs 1 and 2 share a seed and the randomised row; env 1 drew its sky and camera, env 0 did not
    assert np.array_equal(st["env_params"][1], st["env_params"][2])
    assert np.array_equal(st["cam"][0], [pe.params.params[k].default for k in ("cam_height", "cam_fwd_disp",
                                                                                 "cam_pitch", "cam_fov_y")])
    assert not np.array_equal(st["cam"][1], st["cam"][0])
    reward = np.zeros(3)
    eng.step(np.zeros(3, np.int32), reward=reward)
    eng.close()


def test_snapshot_restore_of_a_dynamic_mixed_flag_handle(hostsim_path):
    from miniworld_b200.batched import BatchedMiniWorld
    N = 10
    make = lambda **kw: BatchedMiniWorld([lv for lv, _ in SWITCH_ROWS], N, level_kwargs=[k for _, k in SWITCH_ROWS],
                                         want_depth=True, dynamic_levels=True, **kw)
    env = make(level_seed=13)
    seed_reset(env, 200 + np.arange(N))
    env.set_level_weights([1, 1, 2, 1, 1])
    rng = np.random.default_rng(3)
    acts = rng.integers(0, 3, size=(70, N)).astype(np.int32)
    for t in range(20):
        env.step_host(acts[t], render=False)
    env.set_env_level([0, 3], [1, 4])
    blob = env.snapshot()

    def run(e):
        rec, o = [], None
        for t in range(20, 70):
            o = e.step_host(acts[t], o, render=t % 10 == 0)
            st = full_state(e)
            rec.append([np.array(o[k]) for k in ("reward", "terminated", "truncated", "obs", "depth")] +
                       [e.env_level.copy()] + [st[k].copy() for k in STATE_KEYS + ("cam", "env_params", "ents",
                                                                                        "room_tex")])
        return rec

    first = run(env)
    env.restore(blob)
    second = run(env)
    fresh = make(level_seed=0)                           # zero weights, another seed: the blob's are adopted
    fresh.restore(blob)
    third = run(fresh)
    for t, (a, b, c) in enumerate(zip(first, second, third)):
        for x, y, z in zip(a, b, c):
            assert np.array_equal(x, y) and np.array_equal(x, z), t
    assert len({int(v) for r in first for v in r[5]}) == len(SWITCH_ROWS)   # envs visited every row
    for e in (env, fresh):
        e.close()


# ------------------------------------------------------------------ multi-process sharding (gloo, host build)
SHARD_ROWS = [("MiniWorld-FourRooms-v0", OFF), ("MiniWorld-FourRooms-v0", dict(ON, params=narrowed_params())),
              ("MiniWorld-FourRooms-v0", ON), (("MiniWorld-Hallway-v0", 9), OFF), (("MiniWorld-Hallway-v0", 9), ON)]


def test_sharded_mixed_flag_curriculum_equals_single_process(hostsim_path):
    spec = dict(levels=[lv for lv, _ in SHARD_ROWS], level_kwargs=[k for _, k in SHARD_ROWS], level_seed=31,
                weights=[1, 1, 1, 2, 2])
    env, start = run_sharded(spec, total=10, steps=30, port_base=37500)
    assert not np.array_equal(env.env_level, start)
    env.close()


# ------------------------------------------------------------------ GPU (libmwb.so)
# a randomisation ladder of FourRooms (off / narrowed ranges / on) next to Hallway off and on
GPU_ROWS = [("MiniWorld-FourRooms-v0", OFF), ("MiniWorld-FourRooms-v0", dict(ON, params=narrowed_params())),
            ("MiniWorld-FourRooms-v0", ON), ("MiniWorld-Hallway-v0", OFF), ("MiniWorld-Hallway-v0", ON)]


def _gpu_run(N, steps, seed, level_seed, followers=None):
    """The ladder with weights rewritten by torch on the current stream every 50 steps (gpu_curriculum)."""
    import torch
    weights = lambda t, gen: torch.rand(len(GPU_ROWS), device="cuda", generator=gen) - 0.1
    return gpu_curriculum(GPU_ROWS, N, steps, seed, level_seed, weights, followers=followers)


@pytest.mark.gpu
def test_gpu_mixed_flag_ladder_at_scale(libmwb_path):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    N, steps, seed, level_seed = max(4096, 12 * sms), 300, 321, 77
    env, done_h, level_h, weight_h, _ = _gpu_run(N, steps, seed, level_seed)
    _, switches = replay_draws(env, level_seed, done_h, level_h, weight_h)
    env.close()
    flag = [k["domain_rand"] for _, k in GPU_ROWS]
    on_off = [sw for sw in switches if sw[1] < steps - 1 and flag[sw[2]] and not flag[sw[3]]]
    off_on = [sw for sw in switches if sw[1] < steps - 1 and not flag[sw[2]] and flag[sw[3]]]
    assert len(on_off) > 20 and len(off_on) > 20
    pick = np.random.default_rng(0)
    followers = {}
    for group in (on_off, off_on):
        for k in pick.choice(len(group), size=6, replace=False):
            followers.setdefault(group[k][0], group[k][1])
    env2, _, _, _, checked = _gpu_run(N, steps, seed, level_seed, followers=followers)
    assert set(checked) == set(followers) and min(checked.values()) >= 1 and sum(checked.values()) >= 2 * len(followers)
    env2.close()


@pytest.mark.gpu
def test_gpu_reference_frames_of_off_and_on_rows(libmwb_path):
    """FourRooms off and on in one table against the unmodified reference's frames (tests/golden/stream_fourrooms.npz,
    stream_fourrooms_dr.npz): RGB within 1 LSB with more than 99.5 % of channel values identical, depth identical."""
    from conftest import GOLDEN, golden
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import RNG_DTYPE, rng_state_of
    streams = []
    for name in ("fourrooms", "fourrooms_dr"):
        with np.load(os.path.join(GOLDEN, "stream_%s.npz" % name)) as z:
            streams.append({k: z[k] for k in z.files})
    gs = [golden(str(s["meta"][2])) for s in streams]
    H, W = streams[0]["rgb"].shape[1:3]
    n = max(int(s["sel"][:, 1].max()) + 1 for s in streams)
    N = 2 * n
    el = (np.arange(N) % 2).astype(np.int32)                  # off at the even slots, on at the odd ones
    env = BatchedMiniWorld(["MiniWorld-FourRooms-v0"] * 2, N, env_level=el, level_kwargs=[OFF, ON], want_depth=True,
                           obs_width=W, obs_height=H)
    mine = [np.nonzero(el == k)[0] for k in range(2)]
    env.engine.seed(np.arange(N), np.array([rng_state_of(1000 + int(i) // 2) for i in range(N)], RNG_DTYPE))
    env.engine.reset()
    rows = [{} for _ in streams]
    for r, s in zip(rows, streams):
        for k, (t, i) in enumerate(s["sel"]):
            r.setdefault(int(t), []).append((k, int(i)))
    out = dict(obs=np.zeros((N, H, W, 3), np.uint8), reward=np.zeros(N), terminated=np.zeros(N, np.uint8),
               truncated=np.zeros(N, np.uint8), depth=np.zeros((N, H, W, 1), np.float32))
    same, total, frames = [0, 0], [0, 0], [0, 0]

    def check(t):
        for b, (s, r) in enumerate(zip(streams, rows)):
            for k, i in r.get(t, []):
                d = np.abs(out["obs"][mine[b][i]].astype(int) - s["rgb"][k].astype(int))
                assert d.max() <= 1, (b, t, i)
                same[b], total[b], frames[b] = same[b] + int((d == 0).sum()), total[b] + d.size, frames[b] + 1
                if not s["event"][k]:
                    assert np.array_equal(out["depth"][mine[b][i]], s["depth"][k]), (b, t, i)

    env.engine.render(obs=out["obs"], depth=out["depth"])
    check(0)
    last = max(max(r) for r in rows)
    acts = np.zeros(N, np.int32)
    for t in range(1, last + 1):
        for b in range(2):
            acts[mine[b]] = gs[b]["actions"][t - 1, :n]
        render = any(t in r for r in rows)
        env.step_host(acts, out, render=render)
        if render:
            check(t)
    for b in range(2):
        assert frames[b] > 0 and same[b] > 0.995 * total[b], b
    assert env.engine.overflow_count() == 0
    env.close()
