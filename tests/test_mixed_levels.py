"""Several levels in one batch (mwb_set_levels): env i of a mixed batch must equal, bit for bit, env i of a batch of
its own level seeded the same way -- rewards, flags, poses, step counters, RNG streams, frames and depth maps.
CPU cases run the kernels' host build; `gpu` cases run libmwb.so on the device."""
import numpy as np
import pytest

from level_parity import STATE_KEYS, Lockstep, geometry_equal, run_sharded, seed_reset

# every rule kind but Sign; OneRoomS6Fast brings its own params and a 50-step truncation, ThreeRooms an ImageFrame
MIX = ["MiniWorld-Hallway-v0", "MiniWorld-FourRooms-v0", "MiniWorld-PickupObjects-v0", "MiniWorld-CollectHealth-v0",
       "MiniWorld-PutNext-v0", "MiniWorld-TMazeLeft-v0", "MiniWorld-Sidewalk-v0", "MiniWorld-OneRoomS6Fast-v0",
       "MiniWorld-ThreeRooms-v0"]


def rows(levels):
    return [(lv, {}) for lv in levels]


def run_parity(levels, n_per, steps, domain_rand, render_every, largest=False):
    ls = Lockstep(rows(levels), n_per, domain_rand)
    rng = np.random.default_rng(7)
    trunc = np.zeros(ls.N, np.int64)
    ended = np.zeros(ls.N, np.int64)
    for t in range(steps):
        render = t % render_every == 0 or t == steps - 1
        ls.step(ls.actions(rng, largest), render)
        ls.check(t, render)
        trunc += ls.out_m["truncated"]
        ended += ls.out_m["terminated"] | ls.out_m["truncated"]
        if render:
            assert 0 < ls.out_m["obs"].mean() < 255
    assert ls.mix.engine.overflow_count() == 0
    if "MiniWorld-OneRoomS6Fast-v0" in levels and steps > 50:
        # 50-step episodes: every env of that level has ended one (and auto-reset) within the rollout
        fast = ls.el == levels.index("MiniWorld-OneRoomS6Fast-v0")
        assert ended[fast].all()
        assert n_per < 32 or trunc[fast].any()
    assert ended.sum() > 0
    ls.close()


# ------------------------------------------------------------------ CPU (kernels' host build)
@pytest.mark.parametrize("domain_rand", [False, True])
def test_mixed_batch_equals_single_level_batches(hostsim_path, domain_rand):
    run_parity(MIX, n_per=2, steps=60, domain_rand=domain_rand, render_every=15)


def test_out_of_space_actions_match_single_level_batches(hostsim_path):
    """Actions are not masked: an action outside an env's own level space does what the single-level engine does."""
    run_parity(MIX, n_per=2, steps=40, domain_rand=True, render_every=20, largest=True)


def test_subset_reset_visible_ents_and_geometry(hostsim_path):
    ls = Lockstep(rows(MIX), n_per=2, domain_rand=True)
    rng = np.random.default_rng(11)
    for t in range(12):
        ls.step(ls.actions(rng), render=False)
    ids = np.array([1, 4, 9, 17], np.int32)
    seed_reset(ls.mix, 9000 + ids, ids)
    for k, s in enumerate(ls.singles):
        mine = np.nonzero(ls.el == k)[0]
        sub = [j for j, i in enumerate(mine) if i in ids]
        if sub:
            seed_reset(s, 9000 + mine[sub], sub)
    ls.check("reset", render=False)
    for t in range(12):
        ls.step(ls.actions(rng), render=t == 11)
        ls.check(t, render=t == 11)
    vis = np.zeros(ls.N, np.uint32)
    ls.mix.visible_ents(vis)
    for k, s in enumerate(ls.singles):
        v = np.zeros(s.num_envs, np.uint32)
        s.visible_ents(v)
        assert np.array_equal(vis[ls.el == k], v)
    for i in (0, 5, 16):           # mwb_get_geometry goes through the env's level
        assert geometry_equal(ls.singles[ls.el[i]], 0, ls.mix, i), i
    ls.close()


def test_snapshot_restore_and_assignment_check(hostsim_path):
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import EngineError
    levels = MIX[:5]
    ls = Lockstep(rows(levels), n_per=2, domain_rand=True)
    rng = np.random.default_rng(3)
    acts = [ls.actions(rng) for _ in range(40)]
    for t in range(15):
        ls.step(acts[t], render=False)
    blob = ls.mix.snapshot()

    def run(env):
        rec, out = [], None
        for t in range(15, 40):
            out = env.step_host(acts[t], out, render=False)
            st = env.get_state(rng=True)
            rec.append([out["reward"].copy(), out["terminated"].copy()] + [st[k].copy() for k in STATE_KEYS])
        return rec
    first = run(ls.mix)
    ls.mix.restore(blob)
    second = run(ls.mix)
    fresh = BatchedMiniWorld(levels, ls.N, env_level=ls.el, domain_rand=True)
    fresh.restore(blob)
    third = run(fresh)
    for a, b, c in zip(first, second, third):
        for x, y, z in zip(a, b, c):
            assert np.array_equal(x, y) and np.array_equal(x, z)
    # the single-level batches follow the same trajectory
    for t in range(15, 40):
        ls.outs = [s.step_host(acts[t][ls.el == k], render=False) for k, s in enumerate(ls.singles)]
        for k in range(ls.L):
            assert np.array_equal(first[t - 15][0][ls.el == k], ls.outs[k]["reward"])
    other = BatchedMiniWorld(levels, ls.N, env_level=ls.el[::-1].copy(), domain_rand=True)
    with pytest.raises(EngineError, match="error -6"):
        other.restore(blob)
    more = BatchedMiniWorld(levels + levels[:1], ls.N, env_level=ls.el, domain_rand=True)
    with pytest.raises(EngineError, match="error -6"):
        more.restore(blob)
    for e in (fresh, other, more):
        e.close()
    ls.close()


def test_one_level_list_and_kwargs_per_entry(hostsim_path):
    """The same id twice with different kwargs (OneRoom size 6 and 10), default contiguous assignment."""
    from miniworld_b200.batched import BatchedMiniWorld
    env = BatchedMiniWorld(["MiniWorld-OneRoom-v0", "MiniWorld-OneRoom-v0"], 5, level_kwargs=[{"size": 6}, {"size": 10}])
    assert env.env_level.tolist() == [0, 0, 0, 1, 1]
    assert [pe.size for pe in env.proto_envs] == [6, 10]
    assert env.level_ids == ["MiniWorld-OneRoom-v0"] * 2
    small = BatchedMiniWorld("MiniWorld-OneRoom-v0", 3, level_kwargs={"size": 6})
    big = BatchedMiniWorld("MiniWorld-OneRoom-v0", 2, level_kwargs={"size": 10})
    seed_reset(env, range(5))
    seed_reset(small, range(3))
    seed_reset(big, range(3, 5))
    a = np.random.default_rng(0).integers(0, 3, size=(30, 5), dtype=np.int32)
    for t in range(30):
        o = env.step_host(a[t], render=False)
        o1, o2 = small.step_host(a[t, :3], render=False), big.step_host(a[t, 3:], render=False)
        assert np.array_equal(o["reward"], np.concatenate([o1["reward"], o2["reward"]]))
    st, s1, s2 = env.get_state(), small.get_state(), big.get_state()
    assert np.array_equal(st["agent_pos"], np.concatenate([s1["agent_pos"], s2["agent_pos"]]))
    one = BatchedMiniWorld(["MiniWorld-Hallway-v0"], 2)
    assert one.env_level.tolist() == [0, 0] and one.single_action_space.n == 3
    for e in (env, small, big, one):
        e.close()


def test_top_view_needs_equal_extents(hostsim_path):
    from miniworld_b200.batched import BatchedMiniWorld
    env = BatchedMiniWorld(["MiniWorld-Hallway-v0", "MiniWorld-FourRooms-v0"], 2)
    with pytest.raises(ValueError, match="extents differ"):
        env.render_top_view(out=np.zeros((2, 60, 80, 3), np.uint8))
    env.close()
    env = BatchedMiniWorld(["MiniWorld-TMazeLeft-v0", "MiniWorld-TMazeRight-v0"], 2)
    seed_reset(env, [1, 2])
    out = np.zeros((2, 60, 80, 3), np.uint8)
    env.render_top_view(out=out)
    assert 0 < out.mean() < 255
    env.close()


@pytest.mark.parametrize("levels,kw,match", [
    (["MiniWorld-Hallway-v0", "MiniWorld-MazeS3-v0"], {}, "Maze family"),
    (["MiniWorld-Maze-v0"], {}, "Maze family"),
    (["MiniWorld-Hallway-v0", "MiniWorld-Sign-v0"], {}, "dict"),
    (["MiniWorld-Hallway-v0", "MiniWorld-OneRoom-v0"], {"env_level": [0, 1, 2, 0]}, r"\[0, 2\)"),
    (["MiniWorld-Hallway-v0", "MiniWorld-OneRoom-v0"], {"env_level": [0, 1]}, "shape"),
    (["MiniWorld-Hallway-v0", "MiniWorld-OneRoom-v0"], {"level_kwargs": [{}]}, "1 entries for 2 levels"),
    (["MiniWorld-Hallway-v0"] * 33, {}, "at most 32"),
    ("MiniWorld-Hallway-v0", {"env_level": [0, 0, 0, 0]}, "sequence of levels"),
])
def test_construction_errors(hostsim_path, levels, kw, match):
    from miniworld_b200.batched import BatchedMiniWorld
    with pytest.raises(ValueError, match=match):
        BatchedMiniWorld(levels, 4, **kw)


def test_c_abi_rejects_bad_level_tables(hostsim_path):
    """mwb_set_levels validates its input itself (callers other than BatchedMiniWorld)."""
    from miniworld_b200 import pack
    from miniworld_b200.engine import Engine, EngineError
    from miniworld_b200.envs import Hallway
    from miniworld_b200.program import ResetProgram
    pe = Hallway(device=None)
    prog = ResetProgram()
    pe.device_program(prog)
    geom = pack.pack_geometry(pe)
    lv = dict(rule=(1, 0), max_episode_steps=250, params=pe.params, geometry=geom, ops=prog.op_array())
    caps = dict(max_rooms=len(geom[0]), max_quads=len(geom[1]), max_segs=len(geom[2]), max_ents=2)
    eng = Engine(3, **caps)
    eng.set_protos(prog.proto_array())
    with pytest.raises(EngineError, match="error -1.*env_level"):
        eng.set_levels([lv, lv], [0, 2, 1])
    with pytest.raises(EngineError, match="error -5"):
        eng.set_levels([lv] * 33, [0, 0, 0])
    with pytest.raises(EngineError, match="error -5"):
        eng.set_levels([dict(lv, ops=np.concatenate([lv["ops"]] * 40))], [0, 0, 0])
    small = Engine(3, **dict(caps, max_quads=2))
    with pytest.raises(EngineError, match="error -5"):
        small.set_levels([lv], [0, 0, 0])
    maze = Engine(3, shared_geometry=False, **caps)
    with pytest.raises(EngineError, match="error -1.*shared_geometry"):
        maze.set_levels([lv], [0, 0, 0])
    eng.set_levels([lv, lv], [0, 1, 1])
    for e in (eng, small, maze):
        e.close()


# ------------------------------------------------------------------ multi-process sharding (gloo, host build)
def test_sharded_mixed_run_equals_single_process(hostsim_path):
    env, start = run_sharded(dict(levels=MIX[:4], domain_rand=True), total=10, steps=8, port_base=31500)
    assert start.tolist() == [0, 0, 0, 1, 1, 1, 2, 2, 3, 3]     # default assignment: blocks of 3, 3, 2, 2
    env.close()


# ------------------------------------------------------------------ GPU (libmwb.so)
@pytest.mark.gpu
@pytest.mark.parametrize("domain_rand", [False, True])
def test_gpu_mixed_batch_equals_single_level_batches(libmwb_path, domain_rand):
    run_parity(MIX, n_per=114, steps=300, domain_rand=domain_rand, render_every=25)     # 1026 envs


@pytest.mark.gpu
def test_gpu_out_of_space_actions(libmwb_path):
    run_parity(MIX, n_per=32, steps=120, domain_rand=True, render_every=30, largest=True)


@pytest.mark.gpu
def test_gpu_device_path_reset_subset_snapshot_and_info(libmwb_path):
    """The torch path: reset(seed, env_ids), step() on device tensors, visible_ents, snapshot / restore, info keys."""
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    levels = ["MiniWorld-TMazeLeft-v0", "MiniWorld-TMazeRight-v0", "MiniWorld-CollectHealth-v0"]
    N = 48
    el = (np.arange(N) % 3).astype(np.int32)
    mix = BatchedMiniWorld(levels, N, env_level=el, domain_rand=True, want_depth=True)
    singles = [BatchedMiniWorld(lv, N // 3, domain_rand=True, want_depth=True) for lv in levels]
    mix.reset(seed=list(range(N)))
    for k, s in enumerate(singles):
        s.reset(seed=list(np.nonzero(el == k)[0]))
    assert "goal_pos" not in mix._info and "health" not in mix._info    # only keys every level defines alike
    two = BatchedMiniWorld(levels[:2], 4)
    two.reset(seed=0)
    assert "goal_pos" in two.step(torch.zeros(4, dtype=torch.int32, device="cuda"))[4]
    two.close()
    rng = np.random.default_rng(1)
    blob = None
    for t in range(60):
        acts = torch.as_tensor(rng.integers(0, 3, size=N, dtype=np.int32), device="cuda")
        if t == 20:
            ids = np.array([0, 4, 8, 40], np.int32)
            mix.reset(seed=[77 + int(i) for i in ids], env_ids=ids)
            for k, s in enumerate(singles):
                mine = np.nonzero(el == k)[0]
                sub = [j for j, i in enumerate(mine) if i in ids]
                if sub:
                    s.reset(seed=[77 + int(mine[j]) for j in sub], env_ids=sub)
        if t == 30:
            blob = mix.snapshot()
            ref = [x.clone() for x in mix.step(acts)[:4]]
            mix.restore(blob)
        obs, rew, te, tr, info = mix.step(acts)
        for k, s in enumerate(singles):
            sel = torch.as_tensor(el == k, device="cuda")
            o, r, e, u, i = s.step(acts[sel])
            assert torch.equal(obs[sel], o) and torch.equal(rew[sel], r) and torch.equal(te[sel], e)
            assert torch.equal(tr[sel], u) and torch.equal(info["depth"][sel], i["depth"])
        if t == 30:
            assert torch.equal(ref[0], obs) and torch.equal(ref[1], rew)
    vis = mix.visible_ents().cpu().numpy()
    for k, s in enumerate(singles):
        assert np.array_equal(vis[el == k], s.visible_ents().cpu().numpy())
    assert mix.engine.overflow_count() == 0
    for e in [mix] + singles:
        e.close()
