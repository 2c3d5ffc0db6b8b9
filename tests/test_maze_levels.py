"""Maze-family levels in level tables (BatchedMiniWorld(levels, per_env_worlds=True), mwb_set_level_maze): every env of
a mix must equal, bit for bit, the same env in a batch of its own level -- rewards, flags, state, RNG streams, frames,
depth and static geometry -- also after level changes across template and per-env-world levels and across snapshots.
CPU cases run the kernels' host build; `gpu` cases run libmwb.so on the device."""
import os
import re

import numpy as np
import pytest

from level_parity import STATE_KEYS, Follower, Lockstep, full_state, geometry_equal, run_sharded, seed_reset

MAZE_KW = {"num_rows": 3, "num_cols": 5}        # non-square: a rows / cols mix-up changes the world
MIX = [("MiniWorld-MazeS2-v0", {}), ("MiniWorld-MazeS3-v0", {}), ("MiniWorld-MazeS3Fast-v0", {}),
       ("MiniWorld-Maze-v0", {}), ("MiniWorld-Maze-v0", MAZE_KW), ("MiniWorld-Hallway-v0", {}),
       ("MiniWorld-FourRooms-v0", {}), ("MiniWorld-PickupObjects-v0", {})]
LADDER = ["MiniWorld-OneRoom-v0", "MiniWorld-MazeS2-v0", "MiniWorld-MazeS3-v0", "MiniWorld-Maze-v0"]


def run_parity(levels, n_per, steps, domain_rand, render_every, geometry_every):
    ls = Lockstep(levels, n_per, domain_rand, per_env_worlds=True)
    rng = np.random.default_rng(3)
    ended = np.zeros(ls.N, np.int64)
    ls.check("reset", False, geometry=True)
    for t in range(steps):
        render = t % render_every == 0 or t == steps - 1
        ls.step((rng.random(ls.N) * ls.own_n).astype(np.int32), render)
        ls.check(t, render, geometry=t % geometry_every == 0 or t == steps - 1)
        ended += ls.out_m["terminated"] | ls.out_m["truncated"]
    assert ls.mix.engine.overflow_count() == 0
    return ls, ended


# ------------------------------------------------------------------ CPU (kernels' host build)
@pytest.mark.parametrize("domain_rand", [False, True])
def test_maze_mix_equals_single_level_batches(hostsim_path, domain_rand):
    ls, ended = run_parity(MIX, n_per=2, steps=110, domain_rand=domain_rand, render_every=22, geometry_every=10)
    # MazeS2 truncates at 96 steps: its envs regenerated their mazes through K1's auto-reset inside the mix
    assert ended[ls.el == 0].all()
    ls.close()


def mix_trajectory(name, g, lib_path=None, steps=None, check_every=1):
    """Replay golden trajectory `name` with its envs at the even slots of a batch whose odd slots run template levels."""
    from helpers import CASES, state_mismatches
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import RNG_DTYPE, rng_state_of
    level, dr = CASES[name]
    n = g["actions"].shape[1]
    N = 2 * n
    el = np.where(np.arange(N) % 2 == 0, 0, 1 + (np.arange(N) // 2) % 2).astype(np.int32)
    env = BatchedMiniWorld([level, "MiniWorld-FourRooms-v0", "MiniWorld-Hallway-v0"], N, env_level=el, domain_rand=dr,
                           per_env_worlds=True)
    seeds = np.where(el == 0, 1000 + np.arange(N) // 2, 7000 + np.arange(N))
    env.engine.seed(np.arange(N), np.array([rng_state_of(int(s)) for s in seeds], RNG_DTYPE))
    env.engine.reset()
    mine = np.nonzero(el == 0)[0]

    class View:
        def get_state(self, **kw):
            return {k: v[mine] if np.ndim(v) and len(v) == N else v for k, v in env.get_state(**kw).items()}

    T = g["actions"].shape[0] if steps is None else min(steps, g["actions"].shape[0])
    bad = state_mismatches(View(), g, 0, n)
    assert not bad, "after reset: " + "; ".join(bad)
    rng = np.random.default_rng(1)
    acts = np.zeros(N, np.int32)
    out = None
    for t in range(T):
        acts[:] = rng.integers(0, 3, N)
        acts[mine] = g["actions"][t, :n]
        out = env.step_host(acts, out, render=False)
        if (t + 1) % check_every == 0 or t == T - 1:
            sub = {k: out[k][mine] for k in ("reward", "terminated", "truncated")}
            bad = state_mismatches(View(), g, t + 1, n, sub)
            assert not bad, "step %d: %s" % (t + 1, "; ".join(bad))
    assert env.engine.overflow_count() == 0
    env.close()


@pytest.mark.parametrize("name", ["mazes3", "maze_dr"])
def test_reference_trajectories_inside_a_mix(hostsim_path, name):
    from conftest import golden
    mix_trajectory(name, golden(name), steps=200 if name == "maze_dr" else None)


def test_level_changes_across_world_kinds(hostsim_path):
    """OneRoom -> Maze, Maze -> OneRoom and Maze -> MazeS2 by pending assignment: after the switch the env equals a
    fresh env of its new level seeded with the stream it carried (state, frames, geometry); weight draws follow
    batched.sample_level."""
    from miniworld_b200.batched import BatchedMiniWorld, sample_level
    N = 6
    el = np.array([0, 3, 3, 1, 2, 0], np.int32)
    env = BatchedMiniWorld(LADDER, N, env_level=el, dynamic_levels=True, level_seed=9, per_env_worlds=True,
                           want_depth=True)
    seed_reset(env, 300 + np.arange(N))
    rng = np.random.default_rng(2)
    out = None
    for t in range(8):
        out = env.step_host(rng.integers(0, 3, N).astype(np.int32), out, render=False)
    moves = {0: 3, 1: 0, 2: 1}
    ids = np.array(sorted(moves), np.int32)
    carried = env.get_state(rng=True)["rng"][ids].copy()
    env.set_env_level(ids, [moves[i] for i in ids])
    env.engine.reset(ids)
    assert list(env.env_level[ids]) == [moves[i] for i in ids]
    followers = {int(i): Follower((LADDER[moves[int(i)]], {}), int(i), carried[k]) for k, i in enumerate(ids)}
    for t in range(12):
        acts = rng.integers(0, 3, N).astype(np.int32)
        render = t % 4 == 0
        out = env.step_host(acts, out, render=render)
        st = full_state(env)
        for i, f in followers.items():
            f.step_and_check(acts, out, st, render, t)
            assert geometry_equal(env, i, f.env, 0), (t, i)
    for f in followers.values():
        f.env.close()
    # weight-driven draws at resets of every env
    w = np.array([1.0, 0.5, 2.0, 1.5], np.float32)
    env.set_level_weights(w)
    draws = np.zeros(N, np.int64)
    for r in range(4):
        env.engine.reset()
        want = [sample_level(9, i, draws[i], w) for i in range(N)]
        draws += 1
        assert list(env.env_level) == want, r
        st = env.get_state(rng=True)
        for i in range(N):                                   # every env's geometry is its new level's
            lvl = int(env.env_level[i])
            if lvl == 0:
                assert len(env.engine.get_geometry(i)[0]) == 1
            else:
                assert len(env.engine.get_geometry(i)[0]) == {1: 2 * 4 - 1, 2: 2 * 9 - 1, 3: 2 * 64 - 1}[lvl]
        assert np.all(st["step_count"] == 0)
    assert env.engine.overflow_count() == 0
    env.close()


@pytest.mark.parametrize("dynamic", [False, True])
def test_snapshot_restore_with_per_env_worlds(hostsim_path, dynamic):
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import EngineError
    N = 6
    kw = dict(dynamic_levels=True, level_seed=4) if dynamic else {}
    env = BatchedMiniWorld(LADDER, N, domain_rand=True, per_env_worlds=True, want_depth=True, **kw)
    seed_reset(env, 40 + np.arange(N))
    rng = np.random.default_rng(8)
    acts = rng.integers(0, 3, (200, N)).astype(np.int32)
    out = None
    for t in range(15):
        out = env.step_host(acts[t], out, render=False)
    if dynamic:
        env.set_env_level([0, 2, 5], [3, 0, 1])
        env.engine.reset(np.array([0, 2, 5], np.int32))
        env.set_level_weights([1, 1, 1, 1])
    blob = env.snapshot()

    def run():
        o, rec = None, []
        for t in range(40):
            o = env.step_host(acts[20 + t], o, render=t % 10 == 0)
            st = env.get_state(rng=True)
            rec.append(({k: np.array(o[k]) for k in ("reward", "terminated", "truncated", "obs", "depth")},
                        {k: st[k].copy() for k in STATE_KEYS}, [env.engine.get_geometry(i) for i in range(N)],
                        env.env_level.copy()))
        return rec

    first = run()
    env.restore(blob)
    second = run()
    for t, (a, b) in enumerate(zip(first, second)):
        for k in a[0]:
            assert np.array_equal(a[0][k], b[0][k]), (t, k)
        for k in a[1]:
            assert np.array_equal(a[1][k], b[1][k]), (t, k)
        for ga, gb in zip(a[2], b[2]):
            for x, y in zip(ga, gb):
                assert all(np.array_equal(x[f], y[f]) for f in x.dtype.names if f != "reserved"), t
        assert np.array_equal(a[3], b[3])
    # a blob with per-env worlds does not restore into a handle without them, nor the other way round
    plain = BatchedMiniWorld(["MiniWorld-OneRoom-v0", "MiniWorld-Hallway-v0"], N, domain_rand=True, **kw)
    seed_reset(plain, np.arange(N))
    with pytest.raises(EngineError, match="error -6"):
        plain.restore(blob)
    with pytest.raises(EngineError, match="error -6"):
        env.restore(plain.snapshot())
    plain.close()
    env.close()


def _maze_desc(level="MiniWorld-MazeS2-v0"):
    from miniworld_b200 import pack
    from miniworld_b200.envs import LEVELS
    from miniworld_b200.maze_lowering import MazeTemplate
    cls = LEVELS[level]
    pe = cls(device=None)
    return MazeTemplate(cls), pack.room_cdf(pe.room_probs)


def test_c_abi_validates_set_level_maze(hostsim_path):
    from miniworld_b200 import pack
    from miniworld_b200.engine import Engine, EngineError
    from miniworld_b200.envs import Hallway
    from miniworld_b200.program import ResetProgram
    tmpl, cdf = _maze_desc()                 # MazeS2: 4 cells -> 7 rooms, 30 quads, 16 segments
    pe = Hallway(device=None)
    prog = ResetProgram()
    pe.device_program(prog)
    g = pack.pack_geometry(pe)
    lv = dict(rule=(1, 0), max_episode_steps=250, params=pe.params, geometry=g, ops=prog.op_array())
    ok = dict(max_rooms=7, max_quads=30, max_segs=16, max_ents=2)
    eng = Engine(3, **ok)
    eng.set_protos(prog.proto_array())
    with pytest.raises(EngineError, match="error -6"):
        eng.set_level_maze(0, tmpl, cdf)                    # before set_levels
    per_env = Engine(3, shared_geometry=False, **ok)
    with pytest.raises(EngineError, match="error -6"):
        per_env.set_level_maze(0, tmpl, cdf)                # shared_geometry = 0
    eng.set_levels([lv, lv], [0, 1, 1])
    for bad in (-1, 2):
        with pytest.raises(EngineError, match="error -1"):
            eng.set_level_maze(bad, tmpl, cdf)
    for field in ("max_rooms", "max_quads", "max_segs"):
        small = Engine(3, **dict(ok, **{field: ok[field] - 1}))
        small.set_protos(prog.proto_array())
        small.set_levels([lv], [0, 0, 0])
        with pytest.raises(EngineError, match="error -5"):
            small.set_level_maze(0, tmpl, cdf)
        small.close()
    big, big_cdf = _maze_desc()
    big.rows, big.cols = 16, 17                             # 272 cells > MWB_MAZE_MAX_CELLS
    with pytest.raises(EngineError, match="error -5"):
        eng.set_level_maze(1, big, np.zeros(2 * 272 - 1))
    eng.set_level_maze(1, tmpl, cdf)
    with pytest.raises(EngineError, match="error -6"):
        eng.set_levels([lv, lv], [0, 1, 1])                 # the table is fixed once it has Maze levels
    for e in (eng, per_env):
        e.close()


@pytest.mark.parametrize("levels,kw,match", [
    ("MiniWorld-MazeS3-v0", {}, "sequence of levels"),
    (["MiniWorld-Hallway-v0", "MiniWorld-MazeS3-v0"], {"per_env_worlds": False}, "per_env_worlds=True"),
])
def test_construction_errors(hostsim_path, levels, kw, match):
    from miniworld_b200.batched import BatchedMiniWorld
    with pytest.raises(ValueError, match=match):
        BatchedMiniWorld(levels, 4, **dict({"per_env_worlds": True}, **kw))


def test_flag_without_maze_levels_changes_nothing(hostsim_path):
    from miniworld_b200.batched import BatchedMiniWorld
    levels = ["MiniWorld-OneRoom-v0", "MiniWorld-FourRooms-v0"]
    a = BatchedMiniWorld(levels, 4, per_env_worlds=True)
    b = BatchedMiniWorld(levels, 4)
    for e in (a, b):
        seed_reset(e, np.arange(4))
    sa, sb = a.snapshot(), b.snapshot()
    assert len(sa) == len(sb) and bytes(sa[:4]) == bytes(sb[:4]) == b"MWBS"
    for i in range(4):
        assert geometry_equal(a, i, b, i)
    a.close()
    b.close()


def test_sharded_maze_curriculum_equals_single_process(hostsim_path):
    env, _ = run_sharded(dict(levels=LADDER, level_seed=12, per_env_worlds=True, weights=[1, 2, 2, 1]), total=8,
                         steps=30, port_base=35500)
    env.close()


# ------------------------------------------------------------------ GPU (libmwb.so)
GPU_MIX = [("MiniWorld-Maze-v0", {}), ("MiniWorld-MazeS3-v0", {}), ("MiniWorld-MazeS2-v0", {}),
           ("MiniWorld-FourRooms-v0", {}), ("MiniWorld-PickupObjects-v0", {}), ("MiniWorld-Hallway-v0", {})]


@pytest.mark.gpu
def test_gpu_maze_mix_at_scale(libmwb_path):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n_per = (12 * sms + len(GPU_MIX) - 1) // len(GPU_MIX)
    ls, ended = run_parity(GPU_MIX, n_per=n_per, steps=300, domain_rand=True, render_every=1, geometry_every=100)
    assert ended.sum() > 0
    ls.close()


@pytest.mark.gpu
def test_gpu_reference_trajectory_inside_a_mix(libmwb_path):
    from conftest import golden
    mix_trajectory("maze_long", golden("maze_long"), check_every=20)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["mazes3", "maze_dr"])
def test_gpu_reference_frames_inside_a_mix(libmwb_path, name):
    """Frames of the maze envs of a mix vs the unmodified reference's (tests/golden/stream_*.npz): RGB within 1 LSB
    with more than 99.5 % of channel values identical, depth identical."""
    from conftest import GOLDEN, golden
    from helpers import CASES
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import RNG_DTYPE, rng_state_of
    with np.load(os.path.join(GOLDEN, "stream_%s.npz" % name)) as z:
        s = {k: z[k] for k in z.files}
    g = golden(str(s["meta"][2]))
    level, dr = CASES[str(s["meta"][2])]
    H, W = s["rgb"].shape[1:3]
    n = int(s["sel"][:, 1].max()) + 1
    N = 2 * n
    el = np.where(np.arange(N) % 2 == 1, 0, 1).astype(np.int32)     # maze envs at the odd slots
    env = BatchedMiniWorld([level, "MiniWorld-FourRooms-v0"], N, env_level=el, domain_rand=dr, per_env_worlds=True,
                           want_depth=True, obs_width=W, obs_height=H)
    mine = np.nonzero(el == 0)[0]
    seeds = np.where(el == 0, 1000 + np.arange(N) // 2, 5000 + np.arange(N))
    env.engine.seed(np.arange(N), np.array([rng_state_of(int(x)) for x in seeds], RNG_DTYPE))
    env.engine.reset()
    rows = {}
    for k, (t, i) in enumerate(s["sel"]):
        rows.setdefault(int(t), []).append((k, int(i)))
    out = dict(obs=np.zeros((N, H, W, 3), np.uint8), reward=np.zeros(N), terminated=np.zeros(N, np.uint8),
               truncated=np.zeros(N, np.uint8), depth=np.zeros((N, H, W, 1), np.float32))
    same = total = frames = 0
    acts = np.zeros(N, np.int32)

    def check(t):
        nonlocal same, total, frames
        for k, i in rows[t]:
            d = np.abs(out["obs"][mine[i]].astype(int) - s["rgb"][k].astype(int))
            assert d.max() <= 1, (name, t, i)
            same, total, frames = same + int((d == 0).sum()), total + d.size, frames + 1
            if not s["event"][k]:
                assert np.array_equal(out["depth"][mine[i]], s["depth"][k]), (name, t, i)

    if 0 in rows:
        env.engine.render(obs=out["obs"], depth=out["depth"])
        check(0)
    for t in range(1, max(rows) + 1):
        acts[:] = 1
        acts[mine] = g["actions"][t - 1, :n]
        env.step_host(acts, out, render=t in rows)
        if t in rows:
            check(t)
    assert frames > 0 and same > 0.995 * total
    assert env.engine.overflow_count() == 0
    env.close()


@pytest.mark.gpu
def test_gpu_maze_curriculum_at_scale(libmwb_path):
    import torch
    from miniworld_b200.batched import BatchedMiniWorld, sample_level
    N, steps, seed = 4096, 200, 21
    env = BatchedMiniWorld(LADDER, N, dynamic_levels=True, level_seed=seed, per_env_worlds=True, domain_rand=True)
    env.reset(seed=0)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(3)
    acts = torch.randint(0, 3, (steps, N), dtype=torch.int32, device="cuda", generator=gen)
    dones, levels, weights = [], [], []
    for t in range(steps):
        if t % 50 == 0:
            env.level_weights.copy_(torch.rand(len(LADDER), device="cuda", generator=gen))
        weights.append(env.level_weights.clone())
        obs, rew, te, tr, info = env.step(acts[t])
        dones.append((te | tr).clone())
        levels.append(info["level"].clone())
    torch.cuda.synchronize()
    done = torch.stack(dones).cpu().numpy()
    lv = torch.stack(levels).cpu().numpy()
    w = torch.stack(weights).cpu().numpy()
    # the numpy restatement: an env that ended an episode at step t draws at step t + 1 (next-step auto-reset)
    draws = np.zeros(N, np.int64)
    cur = lv[0].copy()
    checked = 0
    for t in range(1, steps):
        for i in np.nonzero(done[t - 1])[0]:
            want = sample_level(seed, i, draws[i], w[t])
            draws[i] += 1
            cur[i] = want
            checked += 1
        assert np.array_equal(lv[t], cur), t
    assert checked > 0 and len(set(lv[-1])) == len(LADDER)
    # every env after the run equals a fresh env of its final level: a reset from one carried stream
    st = env.get_state(rng=True)
    sample = np.random.default_rng(0).choice(N, 16, replace=False)
    env.set_level_weights(np.zeros(len(LADDER)))
    env.engine.reset(sample.astype(np.int32))
    st2 = full_state(env)
    for i in sample:
        f = Follower((LADDER[int(lv[-1][i])], {}), int(i), st["rng"][i], batch_default=True)
        f.check_state(st2, i)
        assert geometry_equal(env, int(i), f.env, 0), i
        f.env.close()
    assert env.engine.overflow_count() == 0
    env.close()


def k2_report(monkeypatch, capfd, make):
    monkeypatch.setenv("MWB_DEBUG", "1")
    capfd.readouterr()
    obj = make()
    err = capfd.readouterr().err
    monkeypatch.delenv("MWB_DEBUG")
    lines = [ln for ln in err.splitlines() if ln.startswith("[mwb] K2 ")]
    assert lines, err
    return obj, lines[-1]


@pytest.mark.gpu
def test_gpu_k2_residence_per_level(libmwb_path, monkeypatch, capfd):
    from miniworld_b200.batched import BatchedMiniWorld
    env, line = k2_report(monkeypatch, capfd, lambda: BatchedMiniWorld(
        ["MiniWorld-FourRooms-v0", "MiniWorld-MazeS3-v0", "MiniWorld-Maze-v0"], 4096, per_env_worlds=True))
    m = re.search(r"dynamic smem (\d+) B .*shared-memory records (\d+), HBM lists: levels(( \d+)+| none)$", line)
    assert m, line
    assert m.group(3).split() == ["2"], line                    # only the 8 x 8 Maze
    E = env.engine.cfg.max_ents
    want = max(2 * (q + 6 * E) + 2 for q in (len(env.engine.get_geometry(0)[1]), 70))   # FourRooms, MazeS3
    assert int(m.group(2)) == want and int(m.group(1)) > 0, line
    env.close()
    # a mix without maze levels: exactly the launch of the parent commit (4096 envs, 80 x 60, 8x MSAA)
    env, line = k2_report(monkeypatch, capfd, lambda: BatchedMiniWorld(
        ["MiniWorld-OneRoom-v0", "MiniWorld-FourRooms-v0", "MiniWorld-Hallway-v0"], 4096, per_env_worlds=True))
    assert line == EXPECTED_PLAIN_MIX, line
    env.close()


EXPECTED_PLAIN_MIX = ("[mwb] K2 256 threads, 8x MSAA: dynamic smem 37504 B (local destination), parts 1, "
                      "resident blocks/SM 3")   # the parent commit's report for this mix on an H100
