"""Level params written while the batch runs (MWB_ARRAY_LEVEL_PARAMS, BatchedMiniWorld.set_level_param): the engine
must follow the reference's `env.params.set(...)` between steps bit for bit -- per-step draws from the next step,
reset draws and max_forward_step from each env's next reset -- and a batch whose params are never written must run
exactly as before.  CPU cases run the kernels' host build; `gpu` cases run libmwb.so on the device."""
import ctypes as C
import json

import numpy as np
import pytest

from level_parity import Follower, assert_env_equal, full_state, seed_reset, short_level, single_of

# golden case -> (level, kwargs of the level)
CASES = {"fourrooms_dr": ("MiniWorld-FourRooms-v0", {"domain_rand": True}),
         "oneroom": ("MiniWorld-OneRoom-v0", {}),
         "putnext_dr": ("MiniWorld-PutNext-v0", {"domain_rand": True}),
         "pickup_dr": ("MiniWorld-PickupObjects-v0", {"domain_rand": True})}
SHORT_FOURROOMS = short_level("MiniWorld-FourRooms-v0", 8)
SHORT_PICKUP = short_level("MiniWorld-PickupObjects-v0", 10)


def _host_only():
    from miniworld_b200.envs import LEVELS
    base = LEVELS["MiniWorld-Hallway-v0"]
    return type("HostOnly" + base.__name__, (base,), {"device_program": None})


HOST_ONLY = _host_only()          # a level without a device reset program: worlds come from the host


def schedule_of(g):
    """{step: [(name, default, min, max), ...]} of a traj_params_* golden."""
    return {int(t): calls for t, calls in zip(g["steps"], json.loads(str(g["schedule"])))}


def apply(env, level, calls):
    for name, default, *rest in calls:
        lo, hi = (list(rest) + [None, None])[:2]
        env.set_level_param(level, name, default, lo, hi)


def rng_of(g, t, n):
    return g["rng_state"][t, :n], g["rng_inc"][t, :n], g["rng_has32"][t, :n], g["rng_uint"][t, :n]


def golden_mismatches(st, ids, g, t, out=None):
    from helpers import state_mismatches

    class View:
        def get_state(self, **kw):
            return {k: v[ids] if np.ndim(v) and len(v) == len(st["agent_pos"]) else v for k, v in st.items()}
    bad = state_mismatches(View(), g, t, len(ids), out)
    rng = st["rng"][ids]
    want = rng_of(g, t, len(ids))
    got = (np.stack([rng["state_hi"], rng["state_lo"]], 1), np.stack([rng["inc_hi"], rng["inc_lo"]], 1),
           rng["has_uint32"], rng["uinteger"])
    for name, a, b in zip(("rng state", "rng inc", "has_uint32", "uinteger"), got, want):
        if not np.array_equal(a.astype(b.dtype), b):
            bad.append(name)
    if not np.array_equal(st["carrying"][ids], g["carrying"][t, :len(ids)]):
        bad.append("carrying")
    return bad


def replay(case, table):
    """Replay golden `case`: as a single-level batch, or as row 1 of a table whose rows 0 (another level) and 2 (the
    same level) are never written and must equal untouched single-level batches stepped with the same actions."""
    from conftest import golden
    from miniworld_b200.batched import BatchedMiniWorld
    g = golden("params_" + case)
    level, kw = CASES[case]
    sched = schedule_of(g)
    T, Ng = g["actions"].shape
    if not table:
        env = single_of(level, kw, Ng)
        ids, row, others = np.arange(Ng), 0, []
        seed_reset(env, 1000 + np.arange(Ng))
    else:
        rows = [("MiniWorld-Hallway-v0", {"domain_rand": True}), (level, kw), (level, kw)]
        el = np.array([1] * Ng + [0] * 3 + [2] * 3, np.int32)
        N = len(el)
        env = BatchedMiniWorld([r[0] for r in rows], N, env_level=el, level_kwargs=[r[1] for r in rows])
        seeds = np.where(el == 1, 1000 + np.arange(N), 7000 + np.arange(N))
        seed_reset(env, seeds)
        ids, row = np.nonzero(el == 1)[0], 1
        others = []
        for k in (0, 2):
            sel = np.nonzero(el == k)[0]
            s = single_of(rows[k][0], rows[k][1], len(sel))
            seed_reset(s, seeds[sel])
            others.append((sel, s, None))
    st = full_state(env)
    bad = golden_mismatches(st, ids, g, 0)
    assert not bad, "after reset: " + "; ".join(bad)
    rng = np.random.default_rng(3)
    out = None
    for t in range(T):
        if t in sched:
            apply(env, row, sched[t])
        acts = rng.integers(0, 3, env.num_envs).astype(np.int32)
        acts[ids] = g["actions"][t]
        out = env.step_host(acts, out, render=t == T - 1)
        st = full_state(env)
        sub = {key: out[key][ids] for key in ("reward", "terminated", "truncated")}
        bad = golden_mismatches(st, ids, g, t + 1, sub)
        assert not bad, "%s step %d: %s" % (case, t + 1, "; ".join(bad))
        for j, (sel, s, o) in enumerate(others):
            o = s.step_host(acts[sel], o, render=t == T - 1)
            others[j] = (sel, s, o)
            ss = full_state(s)
            for key in ("reward", "terminated", "truncated"):
                assert np.array_equal(out[key][sel], o[key]), (t, key)
            for a, i in enumerate(sel):
                assert_env_equal(st, i, ss, a, (case, t, int(i)))
    for sel, s, o in others:
        assert np.array_equal(out["obs"][sel], o["obs"])
        s.close()
    assert env.engine.overflow_count() == 0
    return env


# ------------------------------------------------------------------ CPU (kernels' host build)
@pytest.mark.parametrize("table", [False, True], ids=["single", "table"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_written_params_follow_the_reference(hostsim_path, case, table):
    env = replay(case, table)
    # what the schedule wrote is what the device holds now
    from conftest import golden
    from miniworld_b200.engine import PARAMS_COLUMN
    g = golden("params_" + case)
    last = schedule_of(g)[max(schedule_of(g))]
    got = env.get_level_params(1 if table else 0)
    for name, default, *rest in last:
        lo, hi = (list(rest) + [default, default])[:2]
        p = got.params[name]
        assert np.array_equal(p.default, default) and np.array_equal(p.min, lo), name
        assert np.allclose(p.max, hi, rtol=0, atol=1e-12), name
        if name == "forward_step":
            assert p.max == hi
    view = env.engine.state_array("level_params")
    assert view.shape[1] == PARAMS_COLUMN["max_forward_step"] + 1
    env.close()


def test_the_goldens_cover_a_captured_threshold(hostsim_path):
    """putnext_dr lowers forward_step's max at step 200 while its episodes run: until they reset, their carried boxes
    sit at the old max_forward_step (0.17), and the episodes after their resets take the new one (0.13).  The replay
    above matches those poses and thresholds."""
    from conftest import golden
    g = golden("params_putnext_dr")
    mfs, carrying = g["max_forward_step"], g["carrying"] >= 0
    assert (carrying[201:] & (mfs[201:] == 0.17)).any() and (mfs[201:] == 0.13).any()
    assert np.isfinite(golden("params_pickup_dr")["carry_pos"]).any()


def untouched_pair(rows, **kw):
    from miniworld_b200.batched import BatchedMiniWorld
    a, b = (BatchedMiniWorld([r[0] for r in rows], 8, level_kwargs=[r[1] for r in rows], want_depth=True, **kw)
            for _ in range(2))
    for e in (a, b):
        seed_reset(e, 50 + np.arange(8))
    return a, b


def test_no_op_writes_change_nothing(hostsim_path):
    rows = [(SHORT_FOURROOMS, {"domain_rand": True}), ("MiniWorld-OneRoom-v0", {}), (SHORT_PICKUP, {"domain_rand": True})]
    a, b = untouched_pair(rows)
    before = np.array(a.engine.state_array("level_params"))
    for lvl, pe in enumerate(b.proto_envs):
        b.set_level_params(lvl, pe.params)
    assert np.array_equal(np.array(b.engine.state_array("level_params")), before)
    rng = np.random.default_rng(0)
    oa = ob = None
    for t in range(40):
        acts = rng.integers(0, 5, 8).astype(np.int32)
        render = t % 13 == 0 or t == 39
        oa, ob = a.step_host(acts, oa, render=render), b.step_host(acts, ob, render=render)
        for key in ("reward", "terminated", "truncated") + (("obs", "depth") if render else ()):
            assert np.array_equal(oa[key], ob[key]), (t, key)
        sa, sb = full_state(a), full_state(b)
        for i in range(8):
            assert_env_equal(sa, i, sb, i, t)
    a.close()
    b.close()


def written_params(base, k):
    """A DomainParams `base` with wider step ranges and other reset ranges (k picks one of two variants)."""
    p = base.copy()
    p.set("forward_step", 0.2, 0.05 * (k + 1), 0.3 + 0.1 * k)
    p.set("turn_step", 20, 5, 35 + k)
    p.set("cam_fov_y", 50 + k, 30, 70)
    p.set("light_color", [0.6, 0.6, 0.6], [0.2, 0.3, 0.4], [0.9, 0.8, 0.7 + 0.1 * k])
    return p


def test_a_reset_after_a_write_equals_a_fresh_batch_with_the_written_params(hostsim_path):
    """After the writes, every env that resets (into its own level or, through set_env_level, into another one) equals
    a one-env batch built with the written params and seeded with the stream it carried into that reset."""
    from miniworld_b200.batched import BatchedMiniWorld
    rows = [(SHORT_FOURROOMS, {"domain_rand": True}), (SHORT_PICKUP, {"domain_rand": True})]
    N = 8
    env = BatchedMiniWorld([r[0] for r in rows], N, level_kwargs=[r[1] for r in rows], dynamic_levels=True,
                           want_depth=True)
    seed_reset(env, 300 + np.arange(N))
    written = [written_params(pe.params, k) for k, pe in enumerate(env.proto_envs)]
    rng = np.random.default_rng(1)
    out = None
    for t in range(3):
        out = env.step_host(rng.integers(0, 3, N).astype(np.int32), out, render=False)
    for lvl in range(2):
        env.set_level_params(lvl, written[lvl])
    env.set_env_level([0, 5], [1, 0])          # two envs also change level at their next reset
    followers, checked = {}, {}
    for t in range(40):
        carried = env.get_state(rng=True)["rng"]
        lv_before = env.env_level
        acts = rng.integers(0, 3, N).astype(np.int32)
        out = env.step_host(acts, out, render=t % 9 == 0)
        st = full_state(env)
        for i, f in list(followers.items()):
            f.step_and_check(acts, out, st, t % 9 == 0, t)
            checked[i] = f.steps
            if out["terminated"][i] or out["truncated"][i]:
                del followers[i]
        for i in np.nonzero(st["step_count"] == 0)[0]:     # reset in this step
            if i in followers or i in checked:
                continue
            lvl = int(env.env_level[i])
            kw = dict(rows[lvl][1], params=written[lvl])
            followers[i] = Follower((rows[lvl][0], kw), i, carried[i])
            followers[i].check_state(st, ("reset", t, int(i), int(lv_before[i]), lvl))
    assert len(checked) == N and min(checked.values()) >= 5
    assert env.env_level[0] == 1 and env.env_level[5] == 0
    env.close()


def test_a_snapshot_after_writes_restores_into_a_fresh_handle(hostsim_path):
    rows = [(SHORT_FOURROOMS, {"domain_rand": True}), (SHORT_PICKUP, {"domain_rand": True})]
    a, b = untouched_pair(rows)
    rng = np.random.default_rng(2)
    oa = ob = None
    for t in range(5):
        oa = a.step_host(rng.integers(0, 3, 8).astype(np.int32), oa, render=False)
    for lvl, pe in enumerate(a.proto_envs):
        a.set_level_params(lvl, written_params(pe.params, lvl))
    for t in range(5):
        oa = a.step_host(rng.integers(0, 3, 8).astype(np.int32), oa, render=False)
    a.set_level_param(0, "forward_step", 0.16, 0.15, 0.17)   # running episodes keep the max their reset took
    blob = a.snapshot()
    b.restore(blob)
    assert np.array_equal(np.array(b.engine.state_array("level_params")), np.array(a.engine.state_array("level_params")))
    for t in range(30):
        acts = rng.integers(0, 3, 8).astype(np.int32)
        render = t % 10 == 0
        oa, ob = a.step_host(acts, oa, render=render), b.step_host(acts, ob, render=render)
        for key in ("reward", "terminated", "truncated") + (("obs",) if render else ()):
            assert np.array_equal(oa[key], ob[key]), (t, key)
        sa, sb = full_state(a), full_state(b)
        for i in range(8):
            assert_env_equal(sa, i, sb, i, t)
    assert np.array_equal(a.snapshot(), b.snapshot())
    a.close()
    b.close()


def test_argument_errors(hostsim_path):
    from miniworld_b200.batched import BatchedMiniWorld
    env = BatchedMiniWorld(["MiniWorld-FourRooms-v0", "MiniWorld-OneRoom-v0"], 4)
    with pytest.raises(KeyError, match="forward_step"):
        env.set_level_param(0, "bot_radius", 0.4)
    with pytest.raises(ValueError, match="level"):
        env.set_level_param(2, "forward_step", 0.2)
    with pytest.raises(ValueError, match="level"):
        env.set_level_param(True, "forward_step", 0.2)
    with pytest.raises(ValueError, match="shape"):
        env.set_level_param(0, "sky_color", 0.5)
    with pytest.raises(ValueError, match="shape"):
        env.set_level_param(0, "forward_step", [0.1, 0.2, 0.3])
    with pytest.raises(ValueError, match="above"):
        env.set_level_param(0, "forward_step", 0.2, 0.1, 0.15)
    with pytest.raises(ValueError, match="above"):
        env.set_level_param(0, "turn_step", 10, 12, 20)
    with pytest.raises(ValueError, match="both"):
        env.set_level_param(0, "turn_step", None, 5)
    before = np.array(env.engine.state_array("level_params"))
    env.set_level_param(0, "turn_step")                        # nothing given: nothing written
    assert np.array_equal(np.array(env.engine.state_array("level_params")), before)
    env.set_level_param(1, "turn_step", None, 10, 50)          # the default stays
    p = env.get_level_params(1).params["turn_step"]
    assert (p.default, p.min, p.max) == (env.proto_envs[1].params.params["turn_step"].default, 10.0, 50.0)
    # an int-typed param cannot be set
    from miniworld_b200.params import DomainParams
    q = env.proto_envs[0].params.copy()
    q.params["turn_step"] = DomainParams.DomainParam(15, 10, 20, "int")
    env.proto_envs[0].params = q
    with pytest.raises(TypeError, match="int"):
        env.set_level_param(0, "turn_step", 15)
    env.close()
    # host-reset levels draw their params in Python
    host = BatchedMiniWorld(HOST_ONLY, 2)
    assert not host.device_reset
    with pytest.raises(TypeError):
        host.set_level_param(0, "forward_step", 0.2)
    with pytest.raises(TypeError):
        host.get_level_params(0)
    host.close()


def test_raw_state_array(hostsim_path):
    """mwb_state_array(MWB_ARRAY_LEVEL_PARAMS): n_levels records, valid with or without level changes, MWB_ESTATE on a
    handle without device resets, MWB_EINVAL for an unknown array."""
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import Params, lower_params
    for kw in ({}, {"dynamic_levels": True}):
        env = BatchedMiniWorld(["MiniWorld-FourRooms-v0", "MiniWorld-Hallway-v0", "MiniWorld-OneRoom-v0"], 3, **kw)
        ptr, count = C.c_void_p(), C.c_int64()
        assert env.engine.lib.mwb_state_array(env.engine.h, 9, C.byref(ptr), C.byref(count)) == 0
        assert count.value == 3
        rec = (Params * 3).from_address(ptr.value)
        for k, pe in enumerate(env.proto_envs):
            assert bytes(rec[k]) == bytes(lower_params(pe.params))
        assert env.engine.lib.mwb_state_array(env.engine.h, 10, C.byref(ptr), C.byref(count)) == -1
        env.close()
    host = BatchedMiniWorld(HOST_ONLY, 2)
    assert host.engine.lib.mwb_state_array(host.engine.h, 9, C.byref(ptr), C.byref(count)) == -6
    assert b"device resets" in host.engine.lib.mwb_last_error()
    host.close()


SHARD_ROWS = [(SHORT_FOURROOMS, {"domain_rand": True}), (SHORT_PICKUP, {"domain_rand": True})]
SHARD_WRITES = {3: [(0, "forward_step", 0.3, 0.1, 0.5), (1, "sky_color", [0.1, 0.2, 0.3])],
                7: [(1, "cam_fov_y", 70, 40, 90), (0, "turn_step", 30, 5, 60)]}


def shard_run(env, steps, rank=0, scatter=None, gather=None):
    """The schedule of SHARD_WRITES on `env` (a batch, or a rank's local batch); per step the (gathered) rewards and
    env params, and the observations of the last step."""
    import torch
    env.set_level_weights([1.0, 1.0])
    acts_all = np.random.default_rng(5).integers(0, 3, size=(steps, 8), dtype=np.int32)
    outs, out = [], None
    for t in range(steps):
        for lvl, name, *vals in SHARD_WRITES.get(t, []):
            env.set_level_param(lvl, name, *vals)
        acts = acts_all[t] if scatter is None else scatter(torch.as_tensor(acts_all[t]) if rank == 0 else None).numpy()
        out = env.step_host(acts, out, render=t == steps - 1)
        got = [out["obs"], out["reward"], env.get_state()["env_params"]]
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
    env = ShardedMiniWorld([r[0] for r in SHARD_ROWS], 8, dist=dist, level_kwargs=[r[1] for r in SHARD_ROWS],
                           dynamic_levels=True, level_seed=9)
    seed_reset(env.local, [1000 + env.start + k for k in range(env.count)])
    outs = shard_run(env.local, 14, rank, lambda a: env.scatter_actions(a, like=torch.zeros(1)), env.gather_to_root)
    if rank == 0:
        q.put(outs)
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_writes_equal_one_process(hostsim_path):
    """Two gloo ranks that write the same schedule into their local batches equal one process (ShardedMiniWorld needs
    no code of its own: each rank writes its `local` batch)."""
    import os
    import torch.multiprocessing as mp
    from miniworld_b200.batched import BatchedMiniWorld
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33000 + os.getpid() % 2000
    procs = [ctx.Process(target=_shard_worker, args=(r, port, hostsim_path, q)) for r in range(2)]
    for p in procs:
        p.start()
    sharded = q.get(timeout=300)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    env = BatchedMiniWorld([r[0] for r in SHARD_ROWS], 8, level_kwargs=[r[1] for r in SHARD_ROWS],
                           dynamic_levels=True, level_seed=9)
    seed_reset(env, 1000 + np.arange(8))
    one = shard_run(env, 14)
    for t, (a, b) in enumerate(zip(one, sharded)):
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]), t
    assert np.array_equal(one[-1][0], sharded[-1][0]) and 0 < one[-1][0].mean() < 255
    assert env.get_level_params(0).params["turn_step"].max == 60
    env.close()


# ------------------------------------------------------------------ GPU (libmwb.so)
@pytest.mark.gpu
def test_gpu_adr_loop_matches_the_host_build_and_the_reference(libmwb_path):
    """4096 FourRooms envs with domain_rand; every 50 steps torch widens or narrows each row's forward_step / turn_step
    ranges from the rewards.  A seeded sample of envs replays on the host build with the recorded schedule (state,
    streams, rewards, flags), and the golden envs follow the reference's fourrooms_dr schedule."""
    import torch
    from conftest import golden
    from miniworld_b200.batched import BatchedMiniWorld
    g = golden("params_fourrooms_dr")
    Ng = g["actions"].shape[1]
    N, T, L = 4096, 300, 2
    rows = ["MiniWorld-FourRooms-v0"] * L
    el = np.where(np.arange(N) < Ng, 0, 1 + np.arange(N) % (L - 1)).astype(np.int32)
    env = BatchedMiniWorld(rows, N, domain_rand=True, env_level=el)
    seeds = 1000 + np.arange(N)
    seed_reset(env, seeds)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(11)
    acts = torch.randint(0, 3, (T, N), dtype=torch.int32, device="cuda", generator=gen)
    acts[:, :Ng] = torch.as_tensor(g["actions"], device="cuda")
    sched = schedule_of(g)
    fs = torch.tensor([0.15, 0.12, 0.17], dtype=torch.float64, device="cuda")
    ts = torch.tensor([15.0, 10.0, 20.0], dtype=torch.float64, device="cuda")
    writes, rew_h, te_h, tr_h = [], [], [], []
    score = torch.zeros(N, dtype=torch.float64, device="cuda")
    for t in range(T):
        if t in sched:
            apply(env, 0, sched[t])
        if t and t % 50 == 0:
            # ADR: the row's success rate decides whether its ranges widen (success) or narrow
            rate = score[el == 1].mean()
            grow = torch.where(rate > 0.0, 1.25, 0.9).to(torch.float64)
            fs = torch.stack([fs[0], fs[0] - (fs[0] - fs[1]) * grow, fs[0] + (fs[2] - fs[0]) * grow])
            ts = torch.stack([ts[0], ts[0] - (ts[0] - ts[1]) * grow, ts[0] + (ts[2] - ts[0]) * grow])
            env.set_level_param(1, "forward_step", fs[0], fs[1], fs[2])
            env.set_level_param(1, "turn_step", ts[0], ts[1], ts[2])
            writes.append((t, fs.clone(), ts.clone()))
            score.zero_()
        obs, rew, te, tr, info = env.step(acts[t])
        score += rew
        rew_h.append(rew.clone())
        te_h.append(te.clone())
        tr_h.append(tr.clone())
    final = env.get_state(rng=True)
    rew_h, te_h, tr_h = (torch.stack(x).cpu().numpy() for x in (rew_h, te_h, tr_h))
    assert env.engine.overflow_count() == 0
    # the golden envs: the reference under the same schedule
    bad = golden_mismatches(full_state(env), np.arange(Ng), g, T, None)
    assert not bad, bad
    assert np.array_equal(rew_h[:, :Ng], g["reward"][1:]) and np.array_equal(te_h[:, :Ng], g["terminated"][1:])
    writes = [(t, a.cpu().numpy(), b.cpu().numpy()) for t, a, b in writes]
    acts = acts.cpu().numpy()
    env.close()
    # a seeded sample of the other envs, replayed on the host build with the recorded schedule
    sample = np.sort(np.random.default_rng(4).choice(np.arange(Ng, N), 64, replace=False))
    replay_sample(rows, el, seeds, acts, sched, writes, sample, final, rew_h, te_h, tr_h)


def replay_sample(rows, el, seeds, acts, sched, writes, sample, final, rew_h, te_h, tr_h):
    import subprocess
    from conftest import ROOT
    from miniworld_b200 import engine
    from miniworld_b200.batched import BatchedMiniWorld
    lib = subprocess.check_output([ROOT + "/tests/hostsim/build.sh"]).decode().strip().splitlines()[-1]
    engine._override_library_for_tests(lib)
    try:
        host = BatchedMiniWorld(rows, len(sample), domain_rand=True, env_level=el[sample])
        seed_reset(host, seeds[sample])
        w = {t: (a, b) for t, a, b in writes}
        out = None
        for t in range(acts.shape[0]):
            if t in w:
                host.set_level_param(1, "forward_step", *w[t][0])
                host.set_level_param(1, "turn_step", *w[t][1])
            out = host.step_host(acts[t, sample], out, render=False)
            assert np.array_equal(out["reward"], rew_h[t, sample]), t
            assert np.array_equal(out["terminated"].astype(bool), te_h[t, sample]), t
            assert np.array_equal(out["truncated"].astype(bool), tr_h[t, sample]), t
        st = host.get_state(rng=True)
        for key in ("agent_pos", "agent_dir", "step_count", "rng", "cam", "env_params", "ents"):
            assert np.array_equal(st[key], final[key][sample]), key
        host.close()
    finally:
        engine._override_library_for_tests(None)


@pytest.mark.gpu
def test_gpu_writes_enqueued_behind_a_busy_stream_reach_the_next_step_and_reset(libmwb_path):
    """A write enqueued on torch's stream behind a long-running kernel must be seen by the next step (step() and
    step_host()) and the next reset, which run behind it on that stream: `a` writes and goes on at once, `b` writes
    the same values and waits for the device first."""
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    N = 64
    a, b = (BatchedMiniWorld("MiniWorld-FourRooms-v0", N, domain_rand=True) for _ in range(2))
    a.reset(seed=5)
    b.reset(seed=5)
    acts = torch.randint(0, 3, (N,), dtype=torch.int32, device="cuda")
    for k, call in enumerate(("step", "step_host", "reset")):
        w = written_params(a.proto_envs[0].params, k % 2)
        w.set("forward_step", 0.2 + 0.05 * k, 0.05, 0.4 + 0.1 * k)
        b.set_level_params(0, w)
        torch.cuda.synchronize()
        torch.cuda._sleep(100_000_000)
        a.set_level_params(0, w)
        if call == "step":
            a.step(acts)
            b.step(acts)
        elif call == "step_host":
            ra = a.step_host(acts.cpu().numpy())
            rb = b.step_host(acts.cpu().numpy())
            assert np.array_equal(ra["obs"], rb["obs"]) and np.array_equal(ra["reward"], rb["reward"])
        else:
            a.reset(seed=9)
            b.reset(seed=9)
        torch.cuda.synchronize()
        sa, sb = full_state(a), full_state(b)
        for i in range(N):
            assert_env_equal(sa, i, sb, i, call)
    a.close()
    b.close()
