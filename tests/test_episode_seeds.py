"""Episode seeds (mwb_enable_episode_seeds, BatchedMiniWorld(episode_seeds=True)): numpy's SeedSequence -> PCG64 inside
the device reset against numpy itself, a pending seed against today's host-seeded reset and the reference trajectories,
seed replay inside a rollout, together with level changes, snapshots, sharding and errors.  CPU cases run the kernels'
host build; `gpu` cases run libmwb.so on the device."""
import numpy as np
import pytest

from level_parity import (Follower, assert_env_equal, full_state, geometry_equal, seed_reset, short_level)

EDGE_SEEDS = [0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 1, 2 ** 63 - 1]
SHORT_FOURROOMS_ID, SHORT_PICKUP_ID, SHORT_MAZE_ID = (("MiniWorld-FourRooms-v0", 8), ("MiniWorld-PickupObjects-v0", 10),
                                                      ("MiniWorld-MazeS3-v0", 12))
SHORT_FOURROOMS, SHORT_PICKUP, SHORT_MAZE = (short_level(*lv) for lv in (SHORT_FOURROOMS_ID, SHORT_PICKUP_ID, SHORT_MAZE_ID))
POOL = np.array([11, 2 ** 32 + 5, 777, 2 ** 40 + 3, 5])


def many_seeds(n_each=2000):
    rs = np.random.default_rng(1)
    return np.array(EDGE_SEEDS + [int(x) for x in rs.integers(0, 2 ** 32, n_each)] +
                    [int(x) for x in rs.integers(0, 2 ** 63, n_each)], np.int64)


def queue_reset(env, seeds, ids=None):
    """reset(seed=...) of an episode_seeds batch without the render: queue the seeds, then mwb_reset."""
    ids = np.arange(env.num_envs) if ids is None else np.asarray(ids)
    env.set_env_seed(ids, seeds)
    env.engine.reset(None if len(ids) == env.num_envs else ids.astype(np.int32), stream=env._level_stream())
    env._seeded = True


def host_array(view):
    return np.array(view) if isinstance(view, np.ndarray) else view.cpu().numpy()


def streams_equal_numpy_twin(seeds, level="MiniWorld-Hallway-v0"):
    """A batch whose resets take `seeds` from next_seed against a twin whose streams numpy built (rng_state_of ->
    mwb_seed): the reset itself draws from the stream, so both are compared after it, every field of the stream."""
    from miniworld_b200.batched import BatchedMiniWorld
    N = len(seeds)
    env = BatchedMiniWorld(level, N, episode_seeds=True)
    twin = BatchedMiniWorld(level, N)
    queue_reset(env, seeds)
    seed_reset(twin, seeds)
    a, b = env.get_state(rng=True), twin.get_state(rng=True)
    for f in a["rng"].dtype.names:
        bad = np.nonzero(a["rng"][f] != b["rng"][f])[0]
        assert bad.size == 0, (f, [int(seeds[i]) for i in bad[:4]])
    for key in ("agent_pos", "agent_dir", "ents"):
        assert np.array_equal(a[key], b[key]), key
    assert np.array_equal(host_array(env.episode_seed), seeds) and (host_array(env.next_seed) == -1).all()
    assert env.engine.overflow_count() == 0
    env.close()
    twin.close()


def golden_replay(name, steps, n, check_every=10):
    """helpers.run_trajectory with the initial seeds installed by the device reset."""
    from conftest import golden
    from helpers import CASES, state_mismatches
    from miniworld_b200.batched import BatchedMiniWorld
    g = golden(name)
    level, dr = CASES[name]
    env = BatchedMiniWorld(level, n, domain_rand=dr, autoreset=True, episode_seeds=True)
    assert env.device_reset
    queue_reset(env, 1000 + np.arange(n))
    bad = state_mismatches(env, g, 0, n)
    assert not bad, "after reset: " + "; ".join(bad)
    out = None
    for t in range(min(steps, g["actions"].shape[0])):
        out = env.step_host(g["actions"][t, :n], out, render=False)
        if (t + 1) % check_every == 0:
            bad = state_mismatches(env, g, t + 1, n, out)
            assert not bad, "step %d: %s" % (t + 1, "; ".join(bad))
        else:
            assert np.array_equal(out["reward"], g["reward"][t + 1, :n]), t
    assert env.engine.overflow_count() == 0
    env.close()


# ------------------------------------------------------------------ CPU (kernels' host build)
def test_device_seeding_equals_numpy(hostsim_path):
    streams_equal_numpy_twin(many_seeds())


@pytest.mark.parametrize("level,kwargs", [(SHORT_FOURROOMS, {}), (SHORT_FOURROOMS, {"domain_rand": True}),
                                          (SHORT_PICKUP, {"domain_rand": True}), (short_level("MiniWorld-PutNext-v0", 9), {"domain_rand": True}),
                                          ("MiniWorld-CollectHealth-v0", {}), (SHORT_MAZE, {}), (SHORT_MAZE, {"domain_rand": True})],
                         ids=["fourrooms", "fourrooms_dr", "pickup_dr", "putnext_dr", "collecthealth", "mazes3", "mazes3_dr"])
def test_a_pending_seed_equals_the_host_seeded_reset(hostsim_path, level, kwargs):
    """next_seed + reset == mwb_seed + reset (today's reset(seed=[...])): state, stream and geometry, and the same over a
    rollout with auto-resets, during which both continue their streams."""
    from miniworld_b200.batched import BatchedMiniWorld
    N = 6
    seeds = np.array([3, 2 ** 32 + 9, 41, 2 ** 50, 6, 2 ** 63 - 1])
    a = BatchedMiniWorld(level, N, level_kwargs=kwargs, episode_seeds=True)
    b = BatchedMiniWorld(level, N, level_kwargs=kwargs)
    queue_reset(a, seeds)
    seed_reset(b, seeds)
    rng = np.random.default_rng(2)
    oa = ob = None
    resets = 0
    for t in range(90):
        if t % 6 == 0:
            sa, sb = full_state(a), full_state(b)
            for i in range(N):
                assert_env_equal(sa, i, sb, i, (t, i))
                assert geometry_equal(a, i, b, i), (t, i)
        acts = rng.integers(0, a.action_space.n, N).astype(np.int32)
        oa, ob = a.step_host(acts, oa, render=False), b.step_host(acts, ob, render=False)
        for key in ("reward", "terminated", "truncated"):
            assert np.array_equal(oa[key], ob[key]), (t, key)
        resets += int((oa["terminated"] | oa["truncated"]).sum())
    assert resets > 0
    assert a.engine.overflow_count() == 0
    a.close()
    b.close()


@pytest.mark.parametrize("name,steps,n", [("fourrooms", 80, 16), ("pickup_dr", 60, 8), ("mazes3", 120, 4), ("hallway", 60, 16)])
def test_reference_trajectories_from_device_installed_seeds(hostsim_path, name, steps, n):
    golden_replay(name, steps, n)


def test_seed_replay_inside_a_rollout(hostsim_path):
    """Done envs get a seed from a small pool (or none) every step.  After its auto-reset an env equals a one-env
    follower that was seeded on the host, and tracks it; envs that never got a seed equal a batch without the mode;
    episode_seed / next_seed follow a numpy model; one seed gives one episode, whichever env plays it and when."""
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import rng_state_of
    row = (SHORT_FOURROOMS, {"domain_rand": True})
    N, T, NEVER = 8, 300, 2                       # envs 0 and 1 are never given a seed
    a = BatchedMiniWorld(row[0], N, level_kwargs=row[1], episode_seeds=True)
    b = BatchedMiniWorld(row[0], N, level_kwargs=row[1])
    seed_reset(a, 900 + np.arange(N))
    seed_reset(b, 900 + np.arange(N))
    rng = np.random.default_rng(8)
    script = np.random.default_rng(9).integers(0, 3, size=(len(POOL), 16), dtype=np.int32)   # actions of a pool seed's episode
    ep, pend = np.full(N, -1, np.int64), np.full(N, -1, np.int64)
    prev_done, seeded_ever = np.zeros(N, bool), np.zeros(N, bool)
    live, episodes, made, compared = {}, {}, 0, 0
    oa = ob = None
    st = full_state(a)
    for t in range(T):
        acts = rng.integers(0, 3, N).astype(np.int32)
        for i in np.nonzero(ep >= 0)[0]:
            acts[i] = script[int(np.nonzero(POOL == ep[i])[0][0]), st["step_count"][i]]
        oa, ob = a.step_host(acts, oa, render=False), b.step_host(acts, ob, render=False)
        st, sb = full_state(a), full_state(b)
        just_reset = prev_done.copy()
        ep[just_reset] = np.where(pend[just_reset] >= 0, pend[just_reset], -1)
        pend[just_reset] = -1
        seeded_ever |= ep >= 0
        assert np.array_equal(a.episode_seed, ep) and np.array_equal(a.next_seed, pend), t
        for i in np.nonzero(~seeded_ever)[0]:
            assert_env_equal(st, i, sb, i, ("unseeded", t, i))
            assert oa["reward"][i] == ob["reward"][i]
        for i, f in list(live.items()):
            f.step_and_check(acts, oa, st, False, ("follow", t))
        for i in np.nonzero(just_reset & (ep >= 0))[0]:
            if made < 40:
                live[i] = Follower(row, i, rng_state_of(int(ep[i])))
                live[i].check_state(st, ("reset", t, i))
                made += 1
        for i in np.nonzero(ep >= 0)[0]:
            key = (int(ep[i]), int(st["step_count"][i]), bool(just_reset[i]))
            val = (st["agent_pos"][i].tobytes(), float(st["agent_dir"][i]), st["rng"][i].tobytes(), float(oa["reward"][i]))
            if key in episodes:
                assert episodes[key] == val, (t, i, key)
                compared += 1
            episodes[key] = val
        done = (oa["terminated"] | oa["truncated"]).astype(bool)
        for i in np.nonzero(done)[0]:
            if i in live:
                live.pop(i).env.close()
            if i >= NEVER and rng.random() < 0.7:
                pend[i] = POOL[rng.integers(len(POOL))]
        chosen = np.nonzero(done & (pend >= 0))[0]
        if t % 2:
            a.set_env_seed(chosen, pend[chosen])
        else:
            a.next_seed[chosen] = pend[chosen]
        prev_done = done
    assert made == 40 and compared > 200 and (~seeded_ever).sum() == NEVER
    assert a.engine.overflow_count() == 0
    a.close()
    b.close()


def test_a_reset_that_takes_a_level_and_a_seed(hostsim_path):
    """dynamic_levels and episode_seeds together, Maze row with per-env worlds included: a reset that takes a pending
    level and a pending seed equals a fresh env of the new level after reset(seed=s), geometry included."""
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import rng_state_of
    rows = [(SHORT_FOURROOMS, {}), (SHORT_PICKUP, {"domain_rand": True}), (SHORT_MAZE, {})]
    N, T = 6, 120
    env = BatchedMiniWorld([r[0] for r in rows], N, level_kwargs=[r[1] for r in rows], dynamic_levels=True,
                           per_env_worlds=True, episode_seeds=True, want_depth=True)
    seed_reset(env, 300 + np.arange(N))
    rng = np.random.default_rng(4)
    want_level, want_seed = env.env_level.copy(), np.full(N, -1, np.int64)
    level, ep = want_level.copy(), want_seed.copy()
    prev_done = np.zeros(N, bool)
    live, seen, out = {}, set(), None
    for t in range(T):
        acts = rng.integers(0, 3, N).astype(np.int32)
        out = env.step_host(acts, out, render=False)
        st = full_state(env)
        level[prev_done], ep[prev_done] = want_level[prev_done], want_seed[prev_done]
        assert np.array_equal(env.env_level, level) and np.array_equal(env.episode_seed, ep), t
        for i, f in list(live.items()):
            f.step_and_check(acts, out, st, False, ("follow", t))
        for i in np.nonzero(prev_done)[0]:
            live[i] = Follower(rows[want_level[i]], i, rng_state_of(int(want_seed[i])))
            live[i].check_state(st, ("reset", t, i))
            assert geometry_equal(env, i, live[i].env, 0), (t, i)
            seen.add(int(want_level[i]))
        done = (out["terminated"] | out["truncated"]).astype(bool)
        for i in np.nonzero(done)[0]:
            if i in live:
                live.pop(i).env.close()
            want_level[i], want_seed[i] = rng.integers(len(rows)), POOL[rng.integers(len(POOL))]
        env.set_env_level(np.nonzero(done)[0], want_level[done])
        env.set_env_seed(np.nonzero(done)[0], want_seed[done])
        prev_done = done
    assert seen == {0, 1, 2} and env.engine.overflow_count() == 0
    env.close()


@pytest.mark.parametrize("level,kwargs", [(SHORT_FOURROOMS, {"domain_rand": True}), (SHORT_MAZE, {})], ids=["fourrooms_dr", "mazes3"])
def test_an_idle_seed_batch_equals_a_batch_without_the_mode(hostsim_path, level, kwargs):
    from miniworld_b200.batched import BatchedMiniWorld
    N = 6
    a = BatchedMiniWorld(level, N, level_kwargs=kwargs, episode_seeds=True, want_depth=True)
    b = BatchedMiniWorld(level, N, level_kwargs=kwargs, want_depth=True)
    seed_reset(a, 40 + np.arange(N))
    seed_reset(b, 40 + np.arange(N))
    rng = np.random.default_rng(3)
    oa = ob = None
    for t in range(150):
        render = t % 50 == 49
        acts = rng.integers(0, 3, N).astype(np.int32)
        oa, ob = a.step_host(acts, oa, render=render), b.step_host(acts, ob, render=render)
        for key in ("reward", "terminated", "truncated") + (("obs", "depth") if render else ()):
            assert np.array_equal(oa[key], ob[key]), (t, key)
        if t % 10 == 9:
            sa, sb = full_state(a), full_state(b)
            for i in range(N):
                assert_env_equal(sa, i, sb, i, (t, i))
    assert (a.episode_seed == -1).all() and (a.next_seed == -1).all()
    a.close()
    b.close()


def test_snapshots_carry_pending_and_episode_seeds(hostsim_path):
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import EngineError
    N = 6
    make = lambda **kw: BatchedMiniWorld(SHORT_FOURROOMS, N, domain_rand=True, **kw)
    env = make(episode_seeds=True)
    queue_reset(env, 70 + np.arange(N))
    acts = np.random.default_rng(6).integers(0, 3, size=(60, N), dtype=np.int32)
    for t in range(20):
        env.step_host(acts[t], render=False)
    env.set_env_seed([0, 2, 5], [POOL[0], POOL[1], POOL[3]])          # pending when the snapshot is taken
    blob = env.snapshot()
    assert bytes(blob[:4]) == b"MWBs"

    def run(e):
        rec = []
        for t in range(20, 60):
            o = e.step_host(acts[t], render=False)
            st = full_state(e)
            rec.append([o["reward"].copy(), o["terminated"].copy()] + [st[k].copy() for k in ("agent_pos", "rng", "env_params")] +
                       [np.array(e.episode_seed), np.array(e.next_seed)])
        return rec
    first = run(env)
    assert {int(POOL[0]), int(POOL[1]), int(POOL[3])} <= {int(s) for r in first for s in r[5]}
    fresh = make(episode_seeds=True)
    fresh.restore(blob)
    assert np.array_equal(fresh.next_seed[[0, 2, 5]], [POOL[0], POOL[1], POOL[3]])
    for x, y in zip(first, run(fresh)):
        for u, v in zip(x, y):
            assert np.array_equal(u, v)
    # across the mode, either way
    off = make()
    seed_reset(off, 70 + np.arange(N))
    with pytest.raises(EngineError, match="error -6"):
        off.restore(blob)
    off_blob = off.snapshot()
    with pytest.raises(EngineError, match="error -6"):
        fresh.restore(off_blob)
    # a handle with the mode off writes the blob it always wrote: its magic, and no room for the two arrays
    assert bytes(off_blob[:4]) == b"MWBS" and len(off_blob) == len(blob) - 2 * 8 * N
    off.restore(off_blob)
    for e in (env, fresh, off):
        e.close()


def test_errors(hostsim_path):
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import EngineError
    from miniworld_b200.envs import LEVELS
    env = BatchedMiniWorld("MiniWorld-FourRooms-v0", 4, episode_seeds=True)
    seed_reset(env, [1, 2, 3, 4])
    with pytest.raises(EngineError, match="error -6"):
        env.engine.enable_episode_seeds()                        # already on
    for bad in (-1, 2 ** 63, [3, -2], np.array([1, 2 ** 63], np.uint64)):
        with pytest.raises(ValueError, match="2\\*\\*63"):
            env.set_env_seed([0, 1] if np.ndim(bad) else [0], bad)
    with pytest.raises(ValueError):
        env.set_env_seed([0, 1, 2], [1, 2])
    with pytest.raises(ValueError):
        env.set_env_seed([4], 1)
    assert (env.next_seed == -1).all()
    env.set_env_seed([1, 3, 1], [7, 8, 9])                       # an env listed twice takes its last entry
    assert env.next_seed.tolist() == [-1, 9, -1, 8]
    env.next_seed[2] = -5                                        # raw writes: any negative entry means none
    env.engine.reset()
    assert env.episode_seed.tolist() == [-1, 9, -1, 8] and (env.next_seed == -1).all()
    env.close()
    off = BatchedMiniWorld("MiniWorld-FourRooms-v0", 4)
    for name in ("next_seed", "episode_seed"):
        with pytest.raises(EngineError, match="error -6"):
            off.engine.state_array(name)
    with pytest.raises(RuntimeError):
        off.next_seed
    with pytest.raises(RuntimeError):
        off.set_env_seed([0], 1)
    off.close()
    base = LEVELS["MiniWorld-Hallway-v0"]
    host_only = type("HostOnly" + base.__name__, (base,), {"device_program": None})
    with pytest.raises(TypeError):
        BatchedMiniWorld(host_only, 2, episode_seeds=True)
    host = BatchedMiniWorld(host_only, 2)
    with pytest.raises(EngineError, match="error -6"):
        host.engine.enable_episode_seeds()                       # no device reset program
    host.close()


def shard_seeds(done, start, t):
    """Seeds the done envs of a shard starting at global env `start` get at step t (-1: none)."""
    g = start + np.arange(len(done))
    return np.where(done & ((g + t) % 3 != 0), 100 + (g * 31 + t) % 5, -1)


def shard_run(env, start, steps, total, rank=0, scatter=None, gather=None):
    import torch
    acts_all = np.random.default_rng(5).integers(0, 3, size=(steps, total), dtype=np.int32)
    outs, out = [], None
    for t in range(steps):
        acts = acts_all[t] if scatter is None else scatter(torch.as_tensor(acts_all[t]) if rank == 0 else None).numpy()
        out = env.step_host(acts, out, render=t == steps - 1)
        s = shard_seeds((out["terminated"] | out["truncated"]).astype(bool), start, t)
        env.set_env_seed(np.nonzero(s >= 0)[0], s[s >= 0])
        got = [out["obs"], out["reward"], np.array(env.episode_seed), env.get_state()["env_params"]]
        if gather is not None:
            got = [gather(torch.as_tensor(x)).numpy() if rank == 0 else gather(torch.as_tensor(x)) for x in got]
        outs.append([np.array(x) for x in got] if rank == 0 else None)
    return outs


def _shard_worker(rank, port, hostsim, q):
    import os
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=2)
    from miniworld_b200 import engine
    from miniworld_b200.dist import ShardedMiniWorld
    engine._override_library_for_tests(hostsim)
    env = ShardedMiniWorld(SHORT_FOURROOMS, 7, dist=dist, domain_rand=True, episode_seeds=True)
    seed_reset(env.local, [1000 + env.start + k for k in range(env.count)])
    outs = shard_run(env.local, env.start, 40, 7, rank, lambda a: env.scatter_actions(a, like=torch.zeros(1)), env.gather_to_root)
    if rank == 0:
        q.put(outs)
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_seed_writes_equal_one_process(hostsim_path):
    """Two gloo ranks that write their envs' seeds into their local batches equal one process: a seed belongs to an
    env, so no offset is involved."""
    import os
    import torch.multiprocessing as mp
    from miniworld_b200.batched import BatchedMiniWorld
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 35000 + os.getpid() % 2000
    procs = [ctx.Process(target=_shard_worker, args=(r, port, hostsim_path, q)) for r in range(2)]
    for p in procs:
        p.start()
    sharded = q.get(timeout=300)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    env = BatchedMiniWorld(SHORT_FOURROOMS, 7, domain_rand=True, episode_seeds=True)
    seed_reset(env, 1000 + np.arange(7))
    one = shard_run(env, 0, 40, 7)
    for t, (x, y) in enumerate(zip(one, sharded)):
        for k in (1, 2, 3):
            assert np.array_equal(x[k], y[k]), (t, k)
    assert np.array_equal(one[-1][0], sharded[-1][0]) and 0 < one[-1][0].mean() < 255
    assert any((x[2] >= 100).any() for x in one)
    env.close()


# ------------------------------------------------------------------ GPU (libmwb.so)
@pytest.mark.gpu
def test_gpu_device_seeding_equals_numpy(libmwb_path):
    streams_equal_numpy_twin(many_seeds())


@pytest.mark.gpu
def test_gpu_reset_takes_seeds_from_a_cuda_tensor_and_from_host_ints(libmwb_path):
    """reset(seed=<CUDA tensor>) and reset(seed=<ints>) of an episode_seeds batch == reset(seed=[...]) of a plain batch,
    observation included, and both record the seeds."""
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    N = 64
    seeds = many_seeds(29)[:N]
    a, b, c = (BatchedMiniWorld("MiniWorld-FourRooms-v0", N, domain_rand=True, episode_seeds=k < 2) for k in range(3))
    oa = a.reset(seed=torch.as_tensor(seeds, device="cuda"))[0].clone()
    ob = b.reset(seed=[int(s) for s in seeds])[0].clone()
    oc = c.reset(seed=[int(s) for s in seeds])[0].clone()
    assert torch.equal(oa, oc) and torch.equal(ob, oc) and 0 < oc.float().mean() < 255
    sa, sb, sc = full_state(a), full_state(b), full_state(c)
    for i in range(N):
        assert_env_equal(sa, i, sc, i, ("tensor", i))
        assert_env_equal(sb, i, sc, i, ("ints", i))
    assert np.array_equal(host_array(a.episode_seed), seeds) and np.array_equal(host_array(b.episode_seed), seeds)
    # the listed envs only, and a base seed
    a.reset(seed=torch.tensor([5, 6], device="cuda"), env_ids=[3, 9])
    b.reset(seed=1000)
    assert host_array(a.episode_seed)[[3, 9]].tolist() == [5, 6] and host_array(a.episode_seed)[4] == seeds[4]
    assert np.array_equal(host_array(b.episode_seed), 1000 + np.arange(N))
    for e in (a, b, c):
        e.close()


@pytest.mark.gpu
def test_gpu_level_replay_loop_matches_the_host_build(libmwb_path):
    """4096 envs, 300 steps of the level-replay loop in torch ops (scores per seed, multinomial picks, fresh seeds),
    never synchronising.  A sample of envs replays on the host build with the recorded actions and seed writes: flags
    and rewards and info["seed"] every step, state and streams at the end, frames at three steps."""
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    N, T, B = 4096, 300, 512
    frames_at = (60, 180, T - 1)
    env = BatchedMiniWorld(SHORT_FOURROOMS, N, domain_rand=True, episode_seeds=True)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(3)
    dev = torch.device("cuda")
    rand_seeds = lambda: torch.randint(0, 2 ** 62, (N,), device=dev, generator=gen)
    buf_seed = torch.arange(B, device=dev) * 3 + 1
    buf_score = torch.ones(B, device=dev)
    ret = torch.zeros(N, dtype=torch.float64, device=dev)
    first = rand_seeds()
    first[:B] = buf_seed
    env.reset(seed=first)
    acts = torch.randint(0, 3, (T, N), dtype=torch.int32, device=dev, generator=gen)
    sample = np.sort(np.random.default_rng(4).choice(N, 96, replace=False))
    sample_t = torch.as_tensor(sample, device=dev)
    hist = {k: [] for k in ("next", "seed", "rew", "te", "tr")}
    frames = {}
    for t in range(T):
        obs, rew, te, tr, info = env.step(acts[t])
        ret += rew
        done = te | tr
        slot = torch.searchsorted(buf_seed, info["seed"]).clamp(max=B - 1)
        hit = done & (buf_seed[slot] == info["seed"])
        buf_score[slot[hit]] = 0.9 * buf_score[slot[hit]] + 0.1 * (1.0 - ret[hit]).float()
        pick = buf_seed[torch.multinomial(buf_score, N, replacement=True, generator=gen)]
        nxt = torch.where(torch.rand(N, device=dev, generator=gen) < 0.5, pick, rand_seeds())
        nxt = torch.where(torch.rand(N, device=dev, generator=gen) < 0.1, torch.full_like(nxt, -1), nxt)   # some continue
        env.next_seed.copy_(torch.where(done, nxt, env.next_seed))
        ret[done] = 0
        for k, v in (("next", env.next_seed), ("seed", info["seed"]), ("rew", rew), ("te", te), ("tr", tr)):
            hist[k].append(v[sample_t].clone())
        if t in frames_at:
            frames[t] = obs[sample_t].clone()
    final = full_state(env)
    hist = {k: torch.stack(v).cpu().numpy() for k, v in hist.items()}
    frames = {t: f.cpu().numpy() for t, f in frames.items()}
    assert env.engine.overflow_count() == 0
    assert (hist["seed"] >= 0).mean() > 0.5 and (hist["seed"][-1] == -1).any() and hist["te"].sum() + hist["tr"].sum() > 1000
    first, acts = first.cpu().numpy(), acts.cpu().numpy()
    env.close()

    import subprocess
    from conftest import ROOT
    from miniworld_b200 import engine
    lib = subprocess.check_output([ROOT + "/tests/hostsim/build.sh"]).decode().strip().splitlines()[-1]
    engine._override_library_for_tests(lib)
    try:
        host = BatchedMiniWorld(SHORT_FOURROOMS, len(sample), domain_rand=True, episode_seeds=True)
        queue_reset(host, first[sample])
        out = None
        for t in range(T):
            out = host.step_host(acts[t, sample], out, render=t in frames_at)
            assert np.array_equal(out["reward"], hist["rew"][t]), t
            assert np.array_equal(out["terminated"].astype(bool), hist["te"][t]), t
            assert np.array_equal(out["truncated"].astype(bool), hist["tr"][t]), t
            assert np.array_equal(host.episode_seed, hist["seed"][t]), t
            if t in frames_at:
                d = np.abs(out["obs"].astype(int) - frames[t].astype(int))
                assert d.max() <= 1 and 0 < frames[t].mean() < 255, (t, int(d.max()))
            host.next_seed[:] = hist["next"][t]
        st = full_state(host)
        for j, i in enumerate(sample):
            assert_env_equal(st, j, final, i, ("final", int(i)))
        host.close()
    finally:
        engine._override_library_for_tests(None)


@pytest.mark.gpu
def test_gpu_seeds_written_on_a_side_stream_behind_a_busy_stream(libmwb_path):
    """Seeds written on a side stream behind a long-running kernel are seen by the step (auto-reset) and the reset that
    run behind them on that stream: `a` writes and goes on at once, `b` waits for the device after the same write."""
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    N = 64
    level = short_level("MiniWorld-FourRooms-v0", 3)
    a, b = (BatchedMiniWorld(level, N, domain_rand=True, episode_seeds=True) for _ in range(2))
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        acts = torch.randint(0, 3, (N,), dtype=torch.int32, device="cuda")
        for e in (a, b):
            e.reset(seed=5)
            for _ in range(3):
                _, _, te, tr, _ = e.step(acts)
            done = te | tr                                        # these envs reset in their next step
        assert int(done.sum()) > N // 2
        for k, call in enumerate(("step", "reset")):
            seeds = torch.arange(N, device="cuda") * 7 + 2 ** 33 * k
            b.next_seed.copy_(seeds)
            torch.cuda.synchronize()
            torch.cuda._sleep(100_000_000)
            a.next_seed.copy_(seeds)
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
            assert torch.equal(a.episode_seed[took], seeds[took]) and torch.equal(a.episode_seed, b.episode_seed), call
            assert bool((a.next_seed[took] == -1).all()) and torch.equal(a.next_seed[~took], seeds[~took])
    a.close()
    b.close()


@pytest.mark.gpu
def test_gpu_reference_trajectory_from_device_installed_seeds(libmwb_path):
    golden_replay("fourrooms", 120, 16)
    golden_replay("mazes3", 80, 4)
