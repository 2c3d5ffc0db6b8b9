"""Parity harness of the level-table tests (not collected by pytest, like helpers.py): a table of levels run side by
side with one single-level batch per row, one-env followers of envs that switched level, a gloo-sharded run against
one process, and a device-side curriculum loop.  A row is (level, kwargs); a row's single-level batch takes the row's
`domain_rand` (or the batch default) as its batch argument."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STATE_KEYS = ("agent_pos", "agent_dir", "step_count", "rng", "num_picked_up", "carrying")


def seed_reset(env, seeds, ids=None):
    """reset(seed=...) without the render: mwb_seed + mwb_reset of the listed envs."""
    from miniworld_b200.engine import RNG_DTYPE, rng_state_of
    ids = np.arange(env.num_envs, dtype=np.int32) if ids is None else np.asarray(ids, np.int32)
    env.engine.seed(ids, np.array([rng_state_of(int(s)) for s in seeds], RNG_DTYPE))
    env.engine.reset(None if len(ids) == env.num_envs else ids)


def short_level(name, steps):
    """The level `name` truncated after `steps` steps: many resets in a short rollout."""
    from miniworld_b200.envs import LEVELS
    base = LEVELS[name]

    def __init__(self, **kw):
        base.__init__(self, **kw)
        self.max_episode_steps = steps
    return type("Short" + base.__name__, (base,), {"__init__": __init__})


def model_levels(seed, offset, level, draws, pending, weights, resetting):
    """The numpy restatement of one step's level resolution for the envs in `resetting` (in place)."""
    from miniworld_b200.batched import sample_level
    L = len(weights)
    for i in np.nonzero(resetting)[0]:
        p = int(pending[i])
        if 0 <= p < L:
            level[i] = p
        else:
            d = sample_level(seed, offset + i, draws[i], weights)
            if d is not None:
                level[i] = d
                draws[i] += 1
        pending[i] = -1


def full_state(env):
    return env.get_state(rng=True, room_tex=True)


def assert_env_equal(sa, i, sb, j, where):
    """Env i of state `sa` equals env j of state `sb`: STATE_KEYS plus everything domain randomisation draws (camera,
    sky and light, entity colours, texture variants).  Capacities may differ: the smaller one is compared, and the
    larger one's extra entity slots must be empty.  (Proto indices are not compared: a table shifts each level's.)"""
    for key in STATE_KEYS + ("cam", "env_params"):
        assert np.array_equal(sa[key][i], sb[key][j]), (where, key)
    ea, eb = sa["ents"][i], sb["ents"][j]
    E = min(len(ea), len(eb))
    live = eb["proto"][:E] >= 0
    assert np.array_equal(ea["proto"][:E] >= 0, live), (where, "live slots")
    for f in ("pos", "dir", "color"):
        assert np.array_equal(ea[f][:E][live], eb[f][:E][live]), (where, f)
    assert (ea["proto"][E:] < 0).all() and (eb["proto"][E:] < 0).all(), where
    if "room_tex" in sa and "room_tex" in sb:
        R = min(sa["room_tex"].shape[1], sb["room_tex"].shape[1])
        assert np.array_equal(sa["room_tex"][i, :R], sb["room_tex"][j, :R]), (where, "room_tex")


def geometry_equal(a, i, b, j):
    """mwb_get_geometry of env i of batch `a` and env j of batch `b`, compared field by field (struct padding is not
    part of the geometry; a template's tex_id is its definition env's own draw, unused by device resets)."""
    for x, y in zip(a.engine.get_geometry(i), b.engine.get_geometry(j)):
        if len(x) != len(y):
            return False
        for f in x.dtype.names:
            if f not in ("reserved", "tex_id") and not np.array_equal(x[f], y[f]):
                return False
    return True


def single_of(level, kwargs, n, batch_default=False, **extra):
    """The single-level batch a row must equal: the row's flag (or the batch default) becomes its batch argument."""
    from miniworld_b200.batched import BatchedMiniWorld
    kw = dict(kwargs)
    flag = bool(kw.pop("domain_rand", batch_default))
    return BatchedMiniWorld(level, n, domain_rand=flag, level_kwargs=kw, want_depth=True, **extra)


class Lockstep:
    """A table (env i runs row i % L) and one single-level batch per row, stepped with the same per-env actions."""

    def __init__(self, rows, n_per, domain_rand=False, per_env_worlds=False, seed0=500, **kw):
        from miniworld_b200.batched import BatchedMiniWorld
        self.L, self.N = len(rows), n_per * len(rows)
        self.el = np.arange(self.N, dtype=np.int32) % self.L
        self.mix = BatchedMiniWorld([lv for lv, _ in rows], self.N, env_level=self.el, domain_rand=domain_rand,
                                    want_depth=True, level_kwargs=[k for _, k in rows], per_env_worlds=per_env_worlds,
                                    **kw)
        self.singles = [single_of(lv, k, n_per, domain_rand, **kw) for lv, k in rows]
        for k, s in enumerate(self.singles):
            assert s.device_reset
            assert bool(self.mix.proto_envs[k].domain_rand) == s.domain_rand == bool(s.engine.cfg.domain_rand)
        self.seeds = seed0 + np.arange(self.N)
        seed_reset(self.mix, self.seeds)
        for k, s in enumerate(self.singles):
            seed_reset(s, self.seeds[self.el == k])
        self.own_n = np.array([self.singles[k].action_space.n for k in self.el])
        self.out_m, self.outs = None, [None] * self.L

    def actions(self, rng, largest=False):
        high = np.full(self.N, self.mix.single_action_space.n) if largest else self.own_n
        return (rng.random(self.N) * high).astype(np.int32)

    def step(self, acts, render):
        self.out_m = self.mix.step_host(acts, self.out_m, render=render)
        for k, s in enumerate(self.singles):
            self.outs[k] = s.step_host(acts[self.el == k], self.outs[k], render=render)

    def check(self, t, render, geometry=False):
        """Outputs of the last step, the state of every env (assert_env_equal) and, with `geometry`, its geometry."""
        sm = full_state(self.mix)
        for k, s in enumerate(self.singles):
            sel, o, ss = np.nonzero(self.el == k)[0], self.outs[k], full_state(s)
            if o is not None:
                for key in ("reward", "terminated", "truncated") + (("obs", "depth") if render else ()):
                    assert np.array_equal(self.out_m[key][sel], o[key]), (t, self.mix.level_ids[k], key)
            for j, i in enumerate(sel):
                assert_env_equal(sm, i, ss, j, (t, k, int(i)))
                if geometry:
                    assert geometry_equal(self.mix, i, s, j), (t, k, int(i))

    def close(self):
        for e in [self.mix] + self.singles:
            e.close()


class Follower:
    """A one-env batch of `row`, seeded with the stream env i carried into its switch to that row and stepped with env
    i's actions: env i must equal it bit for bit."""

    def __init__(self, row, i, carried, batch_default=False):
        from miniworld_b200.engine import RNG_DTYPE
        self.i = i
        self.env = single_of(row[0], row[1], 1, batch_default)
        self.env.engine.seed([0], np.array([carried], RNG_DTYPE))
        self.env.engine.reset()
        self.out, self.steps = None, 0

    def check_state(self, st, where):
        assert_env_equal(st, self.i, full_state(self.env), 0, where)

    def step_and_check(self, acts, out, st, render, where):
        """`out` / `st`: the table's outputs and full_state after the step with `acts`."""
        i = self.i
        self.out = self.env.step_host(acts[i:i + 1], self.out, render=render)
        for key in ("reward", "terminated", "truncated") + (("obs", "depth") if render else ()):
            assert np.array_equal(out[key][i], self.out[key][0]), (where, i, key)
        self.check_state(st, where)
        self.steps += 1


# ------------------------------------------------------------------ multi-process sharding (gloo, host build)
def _spec_batch(spec):
    """spec -> (levels, BatchedMiniWorld keyword arguments).  A level given as (level id, steps) is short_level's
    truncation of it (classes made at run time do not pickle into a spawned worker)."""
    levels = [short_level(*lv) if isinstance(lv, tuple) else lv for lv in spec["levels"]]
    kw = dict(level_kwargs=spec.get("level_kwargs"), domain_rand=spec.get("domain_rand", False),
              per_env_worlds=spec.get("per_env_worlds", False))
    if spec.get("level_seed") is not None:
        kw.update(dynamic_levels=True, level_seed=spec["level_seed"])
    return levels, kw


def _sharded_worker(rank, world, port, hostsim, spec, total, steps, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from miniworld_b200 import engine
    from miniworld_b200.dist import ShardedMiniWorld
    engine._override_library_for_tests(hostsim)
    levels, kw = _spec_batch(spec)
    env = ShardedMiniWorld(levels, total, dist=dist, **kw)
    seed_reset(env.local, [1000 + env.start + k for k in range(env.count)])
    if spec.get("weights") is not None:
        env.local.set_level_weights(spec["weights"])
    acts_all = torch.as_tensor(np.random.default_rng(5).integers(0, 3, size=(steps, total), dtype=np.int32))
    outs, out = [], None
    for t in range(steps):
        mine = env.scatter_actions(acts_all[t] if rank == 0 else None, like=torch.zeros(1))
        out = env.local.step_host(mine.numpy(), out, render=t == steps - 1)
        got = [env.gather_to_root(torch.as_tensor(x)) for x in (out["obs"], out["reward"], env.local.env_level,
                                                                 env.local.get_state()["env_params"])]
        if rank == 0:
            outs.append([x.numpy().copy() for x in got])
    if rank == 0:
        q.put(outs)
    dist.barrier()
    dist.destroy_process_group()


def run_sharded(spec, total, steps, port_base):
    """`spec` (a picklable dict: levels, level_kwargs, weights, level_seed for level changes, per_env_worlds,
    domain_rand) run by two gloo ranks of the host build must equal one process step for step: rewards, levels and
    env_params every step, observations at the last.  Returns the one-process batch and its levels before the run."""
    import torch.multiprocessing as mp
    from miniworld_b200 import engine
    from miniworld_b200.batched import BatchedMiniWorld
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = port_base + os.getpid() % 2000
    procs = [ctx.Process(target=_sharded_worker, args=(r, 2, port, engine._test_library, spec, total, steps, q))
             for r in range(2)]
    for p in procs:
        p.start()
    sharded = q.get(timeout=300)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    levels, kw = _spec_batch(spec)
    env = BatchedMiniWorld(levels, total, **kw)
    seed_reset(env, 1000 + np.arange(total))
    if spec.get("weights") is not None:
        env.set_level_weights(spec["weights"])
    start = env.env_level.copy()
    acts_all = np.random.default_rng(5).integers(0, 3, size=(steps, total), dtype=np.int32)
    out = None
    for t in range(steps):
        out = env.step_host(acts_all[t], out, render=t == steps - 1)
        assert np.array_equal(out["reward"], sharded[t][1]) and np.array_equal(env.env_level, sharded[t][2]), t
        assert np.array_equal(env.get_state()["env_params"], sharded[t][3]), t
    assert np.array_equal(out["obs"], sharded[-1][0]) and 0 < out["obs"].mean() < 255
    return env, start


# ------------------------------------------------------------------ GPU curriculum (libmwb.so)
def gpu_curriculum(rows, N, steps, seed, level_seed, weights, domain_rand=False, followers=None):
    """A table of `rows` with level changes on; every 50 steps `weights(t, gen)` (a CUDA tensor drawn from the torch
    generator `gen`) replaces the level weights on the current stream.  Without `followers` the loop never
    synchronises: the flags, levels and weights of every step are cloned on the device and returned.  `followers`
    {env: switch step} replays the same run and compares those envs, frames included, every step against one-env
    batches of their new rows from the carried stream; `checked` then maps each of them to the number of steps
    compared after its switch."""
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    env = BatchedMiniWorld([lv for lv, _ in rows], N, level_kwargs=[k for _, k in rows], domain_rand=domain_rand,
                           want_depth=True, dynamic_levels=True, level_seed=level_seed)
    env.reset(seed=seed)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(5)
    acts_all = torch.randint(0, 3, (steps, N), dtype=torch.int32, device="cuda", generator=gen)
    done_h, level_h, weight_h = [], [], []
    live, checked = {}, {}
    for t in range(steps):
        if t % 50 == 0:
            env.level_weights.copy_(weights(t, gen))
        weight_h.append(env.level_weights.clone())
        if followers is not None:
            carried = None
            for i, ts in followers.items():
                if ts == t:
                    carried = carried if carried is not None else env.get_state(rng=True)["rng"]
                    live[i] = [None, carried[i].copy()]
        obs, rew, te, tr, info = env.step(acts_all[t])
        if followers is None:
            done_h.append((te | tr).clone())
            level_h.append(info["level"].clone())
            continue
        st = full_state(env) if live else None
        out = None
        for i, f in list(live.items()):
            if f[0] is None:                                             # the switch step: env i just reset
                f[0] = Follower(rows[int(env.level_tensor[i])], i, f[1], domain_rand)
                f[0].check_state(st, ("switch", t))
                continue
            if out is None:
                out = {"reward": rew.cpu().numpy(), "terminated": te.cpu().numpy(), "truncated": tr.cpu().numpy(),
                       "obs": obs.cpu().numpy(), "depth": info["depth"].cpu().numpy()}
            f[0].step_and_check(acts_all[t].cpu().numpy(), out, st, True, t)
            checked[i] = f[0].steps
            if out["terminated"][i] or out["truncated"][i] or f[0].steps >= 40:
                f[0].env.close()
                del live[i]
    assert env.engine.overflow_count() == 0
    return env, done_h, level_h, weight_h, checked


def replay_draws(env, level_seed, done_h, level_h, weight_h):
    """Check a gpu_curriculum run's levels step by step against model_levels; returns the draw counts and the switches
    (env, step, old level, new level)."""
    import torch
    done = torch.stack(done_h).cpu().numpy()
    levels = torch.stack(level_h).cpu().numpy()
    weights = torch.stack(weight_h).cpu().numpy()
    N = env.num_envs
    level = env._env_level.copy()                  # the initial assignment
    draws, pending = np.zeros(N, np.int64), np.full(N, -1)
    switches = []
    prev = np.zeros(N, bool)
    for t in range(len(done)):
        before = level.copy()
        model_levels(level_seed, 0, level, draws, pending, weights[t], prev)
        assert np.array_equal(levels[t], level), t
        switches += [(int(i), t, int(before[i]), int(level[i])) for i in np.nonzero(level != before)[0]]
        prev = done[t]
    return draws, switches
