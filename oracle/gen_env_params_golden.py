#!/usr/bin/env python
"""TEST INFRASTRUCTURE (oracle).  Golden trajectories of the UNMODIFIED reference whose episodes run on DomainParams
of their own -- what per-env ADR boundary sampling and robustness sweeps do with a private `env.params` per env.

Protocol of oracle/gen_params_golden.py (env i seeded 1000 + i, actions default_rng(12345) or a pickup / drop heavy
mix, "next-step" auto-reset, the stream, max_forward_step and the carry position recorded every row), with episodes
truncated after EPISODE_STEPS steps as in oracle/gen_pose_golden.py, and one addition: for each (env, episode) the file
holds a design, a pending flag and 22 element rows (default, min, max) in the order of mwb_enable_env_params
(sky_color, light_pos, light_color, light_ambient, obj_color_bias element by element, then forward_step,
forward_drift, turn_step, cam_pitch, cam_fov_y, cam_height, cam_fwd_disp), NaN where the element keeps the level's.
Before a reset whose design is pending (about 80 %) the env gets a private copy of its level's params overlaid by
name and element: a finite default replaces the param's default, a finite (min, max) pair its range.  Other resets run
on the level's params.  A design picks a random subset of elements; each one gets a range inside the level's, a range
beyond it, a boundary pin (v, v, v) or a default only.  min <= max always: the reference's Generator.uniform refuses
min > max.

    python oracle/gen_env_params_golden.py [case ...]     # writes tests/golden/traj_envparams_<case>.npz
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
from oracle.gen_golden import MAX_ENTS, snapshot  # noqa: E402
from oracle.gen_params_golden import record_rng  # noqa: E402
from oracle.ref_stub import make_reference_env  # noqa: E402

EPISODE_STEPS = 20
# the element rows of a design: (param name, element index or None for a scalar param)
VECTORS = ("sky_color", "light_pos", "light_color", "light_ambient", "obj_color_bias")
SCALARS = ("forward_step", "forward_drift", "turn_step", "cam_pitch", "cam_fov_y", "cam_height", "cam_fwd_disp")
ELEMENTS = [(n, k) for n in VECTORS for k in range(3)] + [(n, None) for n in SCALARS]

# name, env id, kwargs, N, T[, action probabilities]
CASES = [
    ("fourrooms_dr", "MiniWorld-FourRooms-v0", {"domain_rand": True}, 12, 300),
    ("oneroom", "MiniWorld-OneRoom-v0", {}, 12, 300),                   # randomisation off: only defaults count
    ("pickup_dr", "MiniWorld-PickupObjects-v0", {"domain_rand": True}, 12, 300, [0.2, 0.2, 0.35, 0.0, 0.25]),
    ("putnext_dr", "MiniWorld-PutNext-v0", {"domain_rand": True}, 8, 300, [0.2, 0.2, 0.3, 0.0, 0.15, 0.15, 0.0, 0.0]),
    ("mazes3_dr", "MiniWorld-MazeS3-v0", {"domain_rand": True}, 8, 300),
]


def element(params, name, k):
    p = params.params[name]
    pick = (lambda v: float(np.asarray(v, float)[k])) if k is not None else float
    return pick(p.default), pick(p.min), pick(p.max)


def draw_design(rs, base):
    """One [22, 3] design over the level's params `base`."""
    row = np.full((len(ELEMENTS), 3), np.nan)
    for e, (name, k) in enumerate(ELEMENTS):
        if rs.random() >= 0.35:
            continue
        d, lo, hi = element(base, name, k)
        span = hi - lo if hi > lo else max(abs(d), 1.0) * 0.2
        kind = rs.integers(0, 4)
        if kind == 0:                                     # a range inside the level's
            a, b = np.sort(lo + rs.random(2) * (hi - lo))
            row[e] = (a + rs.random() * (b - a), a, b)
        elif kind == 1:                                   # a range beyond it
            a, b = lo - rs.random() * 0.5 * span, hi + rs.random() * 0.5 * span
            row[e] = (a + rs.random() * (b - a), a, b)
        elif kind == 2:                                   # a boundary pin
            v = lo if rs.random() < 0.5 else hi
            row[e] = (v, v, v)
        else:                                             # a default only
            row[e, 0] = lo + rs.random() * (hi - lo) if hi > lo else d + (rs.random() - 0.5) * span
    return row


def overlay(base, row):
    """A private copy of `base` overlaid by design `row`, by param name and element."""
    out = base.copy()
    for name in VECTORS + SCALARS:
        p = out.params[name]
        vec = name in VECTORS
        d, lo, hi = (np.array(v, float).reshape(-1).copy() for v in (p.default, p.min, p.max))
        for e, (n, k) in enumerate(ELEMENTS):
            if n != name:
                continue
            j = k if vec else 0
            if np.isfinite(row[e, 0]):
                d[j] = row[e, 0]
            if np.isfinite(row[e, 1]) and np.isfinite(row[e, 2]):
                lo[j], hi[j] = row[e, 1], row[e, 2]
        vals = [v if vec else float(v[0]) for v in (d, lo, hi)]
        out.params[name] = type(p)(vals[0], vals[1], vals[2], p.type)
    return out


def run_case(name, env_id, kwargs, N, T, action_probs=None):
    env = make_reference_env(env_id, **kwargs)
    env = getattr(env, "unwrapped", env)
    env.max_episode_steps = EPISODE_STEPS
    base = env.params
    n_act = env.action_space.n
    if action_probs is None:
        actions = np.random.default_rng(12345).integers(0, n_act, size=(T, N), dtype=np.int32)
    else:
        actions = np.random.default_rng(12345).choice(n_act, size=(T, N), p=action_probs).astype(np.int32)
    K = T // 2 + 2
    rs = np.random.default_rng(len(name) + 7)
    pending = rs.random((N, K)) < 0.8
    design = np.stack([np.stack([draw_design(rs, base) for _ in range(K)]) for _ in range(N)])
    S = T + 1
    out = dict(
        pos=np.zeros((S, N, 3)), dir=np.zeros((S, N)), step_count=np.zeros((S, N), np.int32),
        reward=np.zeros((S, N)), terminated=np.zeros((S, N), bool), truncated=np.zeros((S, N), bool),
        was_reset=np.zeros((S, N), bool), n_ents=np.zeros((S, N), np.int32), carrying=np.zeros((S, N), np.int32),
        ent_pos=np.zeros((S, N, MAX_ENTS, 3)), ent_dir=np.zeros((S, N, MAX_ENTS)),
        ent_radius=np.zeros((S, N, MAX_ENTS)), ent_kind=np.zeros((S, N, MAX_ENTS), np.int8),
        ent_color=np.zeros((S, N, MAX_ENTS, 3)),
        sky_color=np.zeros((S, N, 3)), light_pos=np.zeros((S, N, 3)), light_color=np.zeros((S, N, 3)),
        light_ambient=np.zeros((S, N, 3)), cam=np.zeros((S, N, 4)), max_forward_step=np.zeros((S, N)),
        rng_state=np.zeros((S, N, 2), np.uint64), rng_inc=np.zeros((S, N, 2), np.uint64),
        rng_has32=np.zeros((S, N), np.int32), rng_uint=np.zeros((S, N), np.uint32),
        carry_pos=np.full((S, N, 3), np.nan), episode=np.zeros((S, N), np.int32),
    )
    carried = []
    orig = env._get_carry_pos

    def carry_pos(*a):
        carried.append(orig(*a))
        return carried[-1]
    env._get_carry_pos = carry_pos

    def reset(i, k, seed=None):
        env.params = overlay(base, design[i, k]) if pending[i, k] else base
        env.reset(seed=seed)

    def record(t, i):
        snapshot(env, out, t, i)
        c = env.agent.carrying
        out["carrying"][t, i] = env.entities.index(c) if c is not None else -1
        record_rng(env, out, t, i)
        out["max_forward_step"][t, i] = env.max_forward_step
        if carried:
            out["carry_pos"][t, i] = carried[-1]

    for i in range(N):
        k = 0
        carried.clear()
        reset(i, k, seed=1000 + i)
        record(0, i)
        out["was_reset"][0, i] = True
        done = False
        for t in range(T):
            carried.clear()
            if done:
                k += 1
                reset(i, k)
                r, te, tr = 0.0, False, False
                out["was_reset"][t + 1, i] = True
            else:
                _, r, te, tr, _ = env.step(int(actions[t, i]))
            done = bool(te or tr)
            out["reward"][t + 1, i] = r
            out["terminated"][t + 1, i] = te
            out["truncated"][t + 1, i] = tr
            record(t + 1, i)
            out["episode"][t + 1, i] = k
    env.params = base
    del env._get_carry_pos
    K = int(out["episode"][-1].max()) + 1
    out.update(actions=actions, design_pending=pending[:, :K], design=design[:, :K],
               episode_steps=np.array(EPISODE_STEPS, np.int32),
               meta=np.array([env_id, repr(sorted(kwargs.items())), str(N), str(T), str(n_act), np.__version__]))
    path = os.path.join(HERE, "..", "tests", "golden", "traj_envparams_%s.npz" % name)
    np.savez_compressed(path, **out)
    used = sum(int(pending[i, :out["episode"][-1, i] + 1].sum()) for i in range(N))
    print("%-13s N=%d T=%d  episodes=%d  designed resets=%d  terminated=%d  carrying steps=%d  -> %s (%d B)" % (
        name, N, T, int(out["episode"][-1].sum()) + N, used, int(out["terminated"].sum()),
        int((out["carrying"] >= 0).sum()), os.path.relpath(path), os.path.getsize(path)))


if __name__ == "__main__":
    only = set(sys.argv[1:])
    for case in CASES:
        if not only or case[0] in only:
            run_case(*case)
