"""Level changes at episode boundaries (mwb_enable_level_changes, BatchedMiniWorld(dynamic_levels=True)): pending
assignments, the device-side level draw against its numpy restatement, snapshots, sharding and errors.  CPU cases
run the kernels' host build; `gpu` cases run libmwb.so on the device."""
import numpy as np
import pytest

from level_parity import (STATE_KEYS, Follower, full_state, gpu_curriculum, model_levels, replay_draws, run_sharded,
                          seed_reset, short_level)

MIX = ["MiniWorld-Hallway-v0", "MiniWorld-FourRooms-v0", "MiniWorld-PickupObjects-v0", "MiniWorld-CollectHealth-v0",
       "MiniWorld-PutNext-v0", "MiniWorld-TMazeLeft-v0", "MiniWorld-Sidewalk-v0", "MiniWorld-OneRoomS6Fast-v0",
       "MiniWorld-ThreeRooms-v0"]
SHORT_IDS = [("MiniWorld-OneRoomS6Fast-v0", 7), ("MiniWorld-Hallway-v0", 9), ("MiniWorld-FourRooms-v0", 8),
             ("MiniWorld-PickupObjects-v0", 10)]
SHORT = [short_level(*lv) for lv in SHORT_IDS]


def host_world_matches(env, i, cls, carried, domain_rand):
    """Env i right after a reset equals the level's host `_gen_world()` fed the stream env i carried into the reset:
    agent pose, entity list and the stream position afterwards."""
    from miniworld_b200.engine import generator_from_state, rng_state_of
    kw = {"domain_rand": True} if domain_rand else {}
    pe = cls(device=None, **kw)
    pe._np_random = generator_from_state(carried)
    pe.reset()
    st = env.get_state(rng=True)
    assert np.array_equal(st["agent_pos"][i], pe.agent.pos) and st["agent_dir"][i] == pe.agent.dir
    live = [e for e in range(st["ents"].shape[1]) if st["ents"][i, e]["proto"] >= 0]
    assert len(live) == len(pe.entities)
    for e, ent in zip(live, pe.entities):
        assert np.array_equal(st["ents"][i, e]["pos"], np.asarray(ent.pos, float)) and st["ents"][i, e]["dir"] == ent.dir
    want = rng_state_of(pe.np_random)
    for f in want.dtype.names:
        assert st["rng"][i][f] == want[f], f


# ------------------------------------------------------------------ CPU (kernels' host build)
@pytest.mark.parametrize("domain_rand", [False, True])
def test_idle_dynamic_batch_equals_static_batch(hostsim_path, domain_rand):
    """Zero weights and no pending assignment: level changes on change nothing."""
    from miniworld_b200.batched import BatchedMiniWorld
    L, N = len(MIX), 2 * len(MIX)
    el = np.arange(N, dtype=np.int32) % L
    static = BatchedMiniWorld(MIX, N, env_level=el, domain_rand=domain_rand, want_depth=True)
    dyn = BatchedMiniWorld(MIX, N, env_level=el, domain_rand=domain_rand, want_depth=True, dynamic_levels=True,
                           level_seed=3)
    seeds = 500 + np.arange(N)
    seed_reset(static, seeds)
    seed_reset(dyn, seeds)
    rng = np.random.default_rng(7)
    own_n = np.array([pe.action_space.n for pe in static.proto_envs])[el]
    o1 = o2 = None
    ended = 0
    for t in range(60):
        render = t % 15 == 0 or t == 59
        acts = (rng.random(N) * own_n).astype(np.int32)
        o1 = static.step_host(acts, o1, render=render)
        o2 = dyn.step_host(acts, o2, render=render)
        for key in ("reward", "terminated", "truncated") + (("obs", "depth") if render else ()):
            assert np.array_equal(o1[key], o2[key]), (t, key)
        s1, s2 = static.get_state(rng=True), dyn.get_state(rng=True)
        for key in STATE_KEYS:
            assert np.array_equal(s1[key], s2[key]), (t, key)
        ended += int((o1["terminated"] | o1["truncated"]).sum())
    assert ended > 0
    assert np.array_equal(dyn.env_level, el) and np.array_equal(dyn.level_tensor, el)
    assert (dyn._views()["next_level"] == -1).all()
    static.close()
    dyn.close()


def test_pending_assignment_takes_effect_at_the_next_reset(hostsim_path):
    from miniworld_b200.batched import BatchedMiniWorld
    L, N, dr = len(SHORT), 8, True
    el = np.arange(N, dtype=np.int32) % L
    env = BatchedMiniWorld(SHORT, N, env_level=el, domain_rand=dr, want_depth=True, dynamic_levels=True)
    seed_reset(env, 40 + np.arange(N))
    rng = np.random.default_rng(2)
    out = None
    for t in range(3):                                # mid-episode: the shortest episode is 7 steps
        out = env.step_host(rng.integers(0, 3, N).astype(np.int32), out, render=False)
    assert not (out["terminated"] | out["truncated"]).any()
    ids = np.array([0, 1, 2, 3, 5], np.int32)
    target = dict(zip(ids.tolist(), ((el[ids] + 1) % L).tolist()))
    env.set_env_level(ids, [target[i] for i in ids])
    assert np.array_equal(env.env_level, el)          # nothing moves before a reset
    followers, switched = {}, set()
    level = el.copy()
    prev_done = np.zeros(N, bool)
    for t in range(60):
        carried = env.get_state(rng=True)["rng"].copy()
        acts = rng.integers(0, 3, N).astype(np.int32)
        render = t % 5 == 0
        out = env.step_host(acts, out, render=render)
        st = full_state(env)
        for f in followers.values():
            if f.steps < 30:
                f.step_and_check(acts, out, st, render, t)
        for i in range(N):
            if prev_done[i] and i in target and i not in switched:     # env i reset in this step
                level[i] = target[i]
                switched.add(i)
                host_world_matches(env, i, SHORT[level[i]], carried[i], dr)
                followers[i] = Follower((SHORT[level[i]], {}), i, carried[i], dr)
        assert np.array_equal(env.env_level, level), t
        prev_done = (out["terminated"] | out["truncated"]).astype(bool)
    assert switched == set(target) and all(f.steps >= 30 for f in followers.values())
    assert (env._views()["next_level"] == -1).all()
    # an explicit reset applies a pending assignment at once
    carried = env.get_state(rng=True)["rng"].copy()
    env.set_env_level([6], [1])
    env.engine.reset([6])
    assert env.env_level[6] == 1 and env._views()["next_level"][6] == -1
    host_world_matches(env, 6, SHORT[1], carried[6], dr)
    for f in followers.values():
        f.env.close()
    env.close()


def test_level_draws_equal_numpy_restatement(hostsim_path):
    from miniworld_b200.batched import BatchedMiniWorld
    L, N, seed = len(SHORT), 8, 0xC0FFEE
    el = np.arange(N, dtype=np.int32) % L
    env = BatchedMiniWorld(SHORT, N, env_level=el, dynamic_levels=True, level_seed=seed)
    seed_reset(env, 7 + np.arange(N))
    schedule = {0: ("call", [1, 2, 3, 4]), 40: ("view", [0, -1, np.nan, 5]), 80: ("call", [0.5, 0, 0.25, 1e-3]),
                120: ("view", [0, 0, 0, 0]), 160: ("call", [-2, 1, 1, np.nan]), 200: ("view", [3, 0, 0, 1])}
    level, draws, pending = el.copy(), np.zeros(N, np.int64), np.full(N, -1)
    weights = np.zeros(L, np.float32)
    resets = np.zeros(N, np.int64)
    seen = [set() for _ in range(N)]
    rng = np.random.default_rng(9)
    prev_done = np.zeros(N, bool)
    out = None
    for t in range(240):
        if t in schedule:
            how, w = schedule[t]
            weights = np.asarray(w, np.float32)
            if how == "call":
                env.set_level_weights(w)
            else:
                env.level_weights[:] = weights
        if t == 100:                               # out-of-range pending entries written through the view: ignored
            env._views()["next_level"][2] = 7
            env._views()["next_level"][3] = -5
            pending[2], pending[3] = 7, -5
        out = env.step_host(rng.integers(0, 3, N).astype(np.int32), out, render=False)
        model_levels(seed, 0, level, draws, pending, weights, prev_done)
        resets += prev_done
        assert np.array_equal(env.env_level, level), t
        assert np.array_equal(env._views()["next_level"], np.where(pending == -1, -1, pending)), t
        for i in range(N):
            seen[i].add(int(level[i]))
        prev_done = (out["terminated"] | out["truncated"]).astype(bool)
    assert resets.min() >= 20
    assert draws.min() > 0 and max(len(s) for s in seen) == L      # the draws did move envs around
    env.close()


def test_snapshot_restore_continues_the_draws(hostsim_path):
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import EngineError
    L, N = len(SHORT), 8
    el = np.arange(N, dtype=np.int32) % L
    make = lambda **kw: BatchedMiniWorld(SHORT, N, env_level=el, domain_rand=True, **kw)
    env = make(dynamic_levels=True, level_seed=11)
    seed_reset(env, 100 + np.arange(N))
    env.set_level_weights([1, 1, 2, 0])
    rng = np.random.default_rng(4)
    acts = rng.integers(0, 3, size=(60, N)).astype(np.int32)
    for t in range(20):
        env.step_host(acts[t], render=False)
    env.set_env_level([4, 5], [3, 3])
    blob = env.snapshot()

    def run(e):
        rec = []
        for t in range(20, 60):
            o = e.step_host(acts[t], render=False)
            st = e.get_state(rng=True)
            rec.append([o["reward"].copy(), o["terminated"].copy(), e.env_level.copy()] + [st[k].copy() for k in STATE_KEYS])
        return rec
    first = run(env)
    env.restore(blob)
    second = run(env)
    fresh = make(dynamic_levels=True)              # another seed and zero weights: the blob's are adopted
    fresh.restore(blob)
    third = run(fresh)
    for a, b, c in zip(first, second, third):
        for x, y, z in zip(a, b, c):
            assert np.array_equal(x, y) and np.array_equal(x, z)
    assert any(not np.array_equal(r[2], el) for r in first)
    static = make()
    with pytest.raises(EngineError, match="error -6"):
        static.restore(blob)
    with pytest.raises(EngineError, match="error -6"):
        fresh.restore(static.snapshot())
    for e in (env, fresh, static):
        e.close()


def test_construction_and_argument_errors(hostsim_path):
    from miniworld_b200 import pack
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import Engine, EngineError
    from miniworld_b200.envs import Hallway
    from miniworld_b200.program import ResetProgram
    pe = Hallway(device=None)
    prog = ResetProgram()
    pe.device_program(prog)
    geom = pack.pack_geometry(pe)
    eng = Engine(3, max_rooms=len(geom[0]), max_quads=len(geom[1]), max_segs=len(geom[2]), max_ents=2)
    eng.set_protos(prog.proto_array())
    with pytest.raises(EngineError, match="error -6"):
        eng.enable_level_changes(1, 0)             # before mwb_set_levels
    with pytest.raises(EngineError, match="error -6"):
        eng.state_array("next_level")
    lv = dict(rule=(1, 0), max_episode_steps=250, params=pe.params, geometry=geom, ops=prog.op_array())
    eng.set_levels([lv, lv], [0, 1, 1])
    with pytest.raises(EngineError, match="error -1"):
        eng.enable_level_changes(1, -4)
    eng.enable_level_changes(1, 0)
    with pytest.raises(EngineError, match="error -6"):
        eng.enable_level_changes(1, 0)
    with pytest.raises(EngineError, match="error -6"):
        eng.set_levels([lv, lv], [0, 1, 1])        # the table is fixed once levels can change
    assert eng.state_array("level_weights").shape == (2,) and eng.state_array("env_level").tolist() == [0, 1, 1]
    eng.close()
    with pytest.raises(ValueError, match="sequence of levels"):
        BatchedMiniWorld("MiniWorld-Hallway-v0", 4, dynamic_levels=True)
    env = BatchedMiniWorld(["MiniWorld-Hallway-v0", "MiniWorld-OneRoom-v0"], 4, dynamic_levels=True)
    for ids, lvs, match in (([0], [2], r"\[0, 2\)"), ([4], [0], r"\[0, 4\)"), ([-1], [0], r"\[0, 4\)"),
                            ([0, 1], [1], "2 env ids but 1 levels"), ([0], [-1], r"\[0, 2\)")):
        with pytest.raises(ValueError, match=match):
            env.set_env_level(ids, lvs)
    with pytest.raises(ValueError, match="shape"):
        env.set_level_weights([1, 2, 3])
    assert (env._views()["next_level"] == -1).all()
    env.set_env_level([1, 3, 1], [1, 0, 0])                 # env 1 listed twice: its last entry wins
    assert env._views()["next_level"].tolist() == [-1, 0, -1, 0]
    static = BatchedMiniWorld(["MiniWorld-Hallway-v0", "MiniWorld-OneRoom-v0"], 4)
    with pytest.raises(RuntimeError, match="dynamic_levels"):
        static.set_env_level([0], [1])
    for e in (env, static):
        e.close()


# ------------------------------------------------------------------ multi-process sharding (gloo, host build)
def test_sharded_dynamic_run_equals_single_process(hostsim_path):
    env, start = run_sharded(dict(levels=SHORT_IDS, domain_rand=True, level_seed=77, weights=[1, 2, 0, 3]), total=10,
                             steps=30, port_base=33500)
    assert not np.array_equal(env.env_level, start)
    env.close()


# ------------------------------------------------------------------ GPU (libmwb.so)
GPU_LEVELS = ["MiniWorld-FourRooms-v0", "MiniWorld-Hallway-v0", "MiniWorld-OneRoomS6Fast-v0", "MiniWorld-PickupObjects-v0"]


def _gpu_run(N, steps, seed, level_seed, followers=None):
    """4 levels, weights replaced every 50 steps by torch ops on the current stream (gpu_curriculum)."""
    import torch

    def weights(t, gen):
        if t == 150:
            return torch.zeros(len(GPU_LEVELS), device="cuda")               # keep every level for a while
        return torch.rand(len(GPU_LEVELS), device="cuda", generator=gen) - 0.2
    return gpu_curriculum([(lv, {}) for lv in GPU_LEVELS], N, steps, seed, level_seed, weights, domain_rand=True,
                          followers=followers)


@pytest.mark.gpu
def test_gpu_device_curriculum_draws_equal_numpy_restatement(libmwb_path):
    N, steps, seed, level_seed = 4096, 300, 123, 99
    env, done_h, level_h, weight_h, _ = _gpu_run(N, steps, seed, level_seed)
    draws, switches = replay_draws(env, level_seed, done_h, level_h, weight_h)
    assert draws.sum() > N and len(switches) > 100
    env.close()
    # a seeded sample of switched envs: the episode after the switch equals a one-env batch from the carried stream
    early = [sw for sw in switches if sw[1] < steps - 1]           # switches with at least one step after them
    pick = np.random.default_rng(0).choice(len(early), size=8, replace=False)
    followers = {}
    for k in pick:
        i, t = early[k][:2]
        followers.setdefault(i, t)
    env2, _, _, _, checked = _gpu_run(N, steps, seed, level_seed, followers=followers)
    assert set(checked) == set(followers) and min(checked.values()) >= 1 and sum(checked.values()) >= 2 * len(followers)
    env2.close()


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["step", "step_host"])
def test_gpu_level_writes_just_before_step_reach_its_resets(libmwb_path, path):
    """Asynchronous torch kernels write the weights and a pending assignment right before step() / step_host(); the
    resets in that step see both."""
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    N = 256
    env = BatchedMiniWorld(["MiniWorld-OneRoomS6Fast-v0", "MiniWorld-Hallway-v0", "MiniWorld-OneRoomS6-v0"], N,
                           env_level=np.zeros(N, np.int32), dynamic_levels=True, level_seed=1)
    env.reset(seed=0)
    acts = np.zeros(N, np.int32)                                       # turn left: OneRoomS6Fast truncates at step 50
    acts_d = torch.as_tensor(acts, device="cuda")
    out = None
    for t in range(50):
        if path == "step":
            _, _, te, tr, _ = env.step(acts_d)
            done = (te | tr).cpu().numpy()
        else:
            out = env.step_host(acts, out, render=t == 49)
            done = (out["terminated"] | out["truncated"]).astype(bool)
    assert done.sum() > N // 2 and (env.env_level == 0).all()
    first = int(np.nonzero(done)[0][0])
    w_new = torch.tensor([0.0, 0.0, 1.0], device="cuda")               # on the device before the delay: no host copy below
    pending = torch.full((N,), -1, dtype=torch.int32, device="cuda")
    pending[first] = 1
    torch.cuda.synchronize()
    torch.cuda._sleep(200_000_000)                                     # the writes below run long after the call returned
    env.level_weights.copy_(w_new)
    env._views()["next_level"].copy_(pending)
    if path == "step":
        env.step(acts_d)
    else:
        env.step_host(acts, out, render=False)
    want = np.where(done, 2, 0)
    want[first] = 1                                                    # the pending assignment wins over the draw
    assert np.array_equal(env.env_level, want)
    env.close()
