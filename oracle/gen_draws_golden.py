#!/usr/bin/env python
"""TEST INFRASTRUCTURE (oracle).  Golden trajectories of the UNMODIFIED reference whose episodes take designed reset
draws -- what environment design over an episode's content (object kinds and colours, box sizes, goal sides, headings)
does.

Protocol of oracle/gen_pose_golden.py (env i seeded 1000 + i, actions default_rng(12345), "next-step" auto-reset,
episodes truncated after EPISODE_STEPS steps), with one addition: for each (env, episode) the stored schedule holds a
design -- a pending flag and one value per reset draw, NaN where there is none.  About 80 % of resets are designed, each
with a random subset of the draws, and some values lie outside the draw's support.  While a reset with a pending design
runs, and only then, the reference's `_gen_world()` runs with its np_random wrapped: the choice / integers / uniform
calls it makes itself (not those inside place_entity, which runs with the plain stream) are numbered 0, 1, ... in call
order, made as usual, and then replaced by the design's value when that lies in the draw's support (an integer in
[low, high); a finite value in [lo, hi]).

    python oracle/gen_draws_golden.py [case ...]     # writes tests/golden/traj_draws_<case>.npz
"""
import math
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
from oracle.gen_golden import snapshot  # noqa: E402
from oracle.gen_params_golden import record_rng  # noqa: E402
from oracle.gen_pose_golden import EPISODE_STEPS  # noqa: E402
from oracle.ref_stub import make_reference_env  # noqa: E402

# name, env id, kwargs, N, T
CASES = [
    ("tmaze", "MiniWorld-TMaze-v0", {}, 12, 300),
    ("ymaze_dr", "MiniWorld-YMaze-v0", {"domain_rand": True}, 12, 300),
    ("pickup", "MiniWorld-PickupObjects-v0", {}, 8, 300),
    ("roomobjects", "MiniWorld-RoomObjects-v0", {}, 8, 300),
    ("putnext_dr", "MiniWorld-PutNext-v0", {"domain_rand": True}, 8, 300),
    ("hallway", "MiniWorld-Hallway-v0", {}, 8, 300),
]


class Draws:
    """np_random of a designed `_gen_world()`: see the module docstring.  `specs` collects (kind, a, b) per draw: an
    integer draw over [a, b), a uniform over [a, b]."""

    def __init__(self, stream, design):
        self.stream, self.design, self.specs = stream, design, []

    def __getattr__(self, name):
        return getattr(self.stream, name)

    def _take(self, v, spec, ok):
        d = len(self.specs)
        self.specs.append(spec)
        x = float(self.design[d]) if d < len(self.design) else math.nan
        return type(v)(x) if ok(x) else v

    def _integer(self, v, lo, hi):
        return self._take(v, ("choice", lo, hi), lambda x: lo <= x < hi and x == math.floor(x))

    def choice(self, a, *args, **kw):
        v = self.stream.choice(a, *args, **kw)
        return self._integer(v, 0, int(a)) if isinstance(a, (int, np.integer)) and not args and not kw else v

    def integers(self, low, high=None, *args, **kw):
        v = self.stream.integers(low, high, *args, **kw)
        return self._integer(v, *((0, low) if high is None else (low, high))) if np.ndim(v) == 0 else v

    def uniform(self, low=0.0, high=1.0, *args, **kw):
        v = self.stream.uniform(low, high, *args, **kw)
        if np.ndim(v) or np.ndim(low) or np.ndim(high):
            return v
        return self._take(v, ("uniform", float(low), float(high)), lambda x: math.isfinite(x) and low <= x <= high)


def designed_reset(env, design, seed=None):
    """env.reset(seed) with `_gen_world()` drawing through Draws(design) (design None: a plain reset).  Returns the
    specs of the draws it made."""
    orig_gen, orig_place = env._gen_world, env.place_entity
    box = {}

    def gen_world():
        box["d"] = Draws(env.np_random, design)
        env.np_random = box["d"]
        try:
            orig_gen()
        finally:
            env.np_random = box["d"].stream

    def place_entity(*a, **kw):                # placement draws are not reset draws
        wrapped = env.np_random
        env.np_random = wrapped.stream if isinstance(wrapped, Draws) else wrapped
        try:
            return orig_place(*a, **kw)
        finally:
            env.np_random = wrapped

    if design is not None:
        env._gen_world, env.place_entity = gen_world, place_entity
    try:
        env.reset(seed=seed)
    finally:
        for name in ("_gen_world", "place_entity"):
            env.__dict__.pop(name, None)
    return box["d"].specs if "d" in box else None


def draw_designs(rs, N, K, specs):
    """pending [N, K] and values [N, K, D] of every (env, episode): a random subset of the draws per design, one in
    five values outside its draw's support."""
    D = len(specs)
    pending = rs.random((N, K)) < 0.8
    vals = np.full((N, K, D), np.nan)
    for i in range(N):
        for k in range(K):
            for d, (kind, lo, hi) in enumerate(specs):
                if rs.random() >= 0.6:
                    continue
                if rs.random() < 0.8:
                    vals[i, k, d] = rs.integers(lo, hi) if kind == "choice" else rs.uniform(lo, hi)
                elif kind == "choice":
                    vals[i, k, d] = rs.choice([hi, lo - 1, lo + 0.5])
                else:
                    vals[i, k, d] = rs.choice([lo - 0.05, hi + 0.05, math.inf, -math.inf])
    return pending, vals


def run_case(name, env_id, kwargs, N, T):
    env = make_reference_env(env_id, **kwargs)
    env = getattr(env, "unwrapped", env)
    env.max_episode_steps = EPISODE_STEPS
    specs = designed_reset(env, [], seed=0)
    K = T // 2 + 2                                   # an episode takes at least two rows (its reset and a step)
    rs = np.random.default_rng(len(name))
    pending, vals = draw_designs(rs, N, K, specs)
    n_act = env.action_space.n
    actions = np.random.default_rng(12345).integers(0, n_act, size=(T, N), dtype=np.int32)
    from oracle.gen_golden import MAX_ENTS
    S = T + 1
    out = dict(
        pos=np.zeros((S, N, 3)), dir=np.zeros((S, N)), step_count=np.zeros((S, N), np.int32),
        reward=np.zeros((S, N)), terminated=np.zeros((S, N), bool), truncated=np.zeros((S, N), bool),
        was_reset=np.zeros((S, N), bool), n_ents=np.zeros((S, N), np.int32), carrying=np.zeros((S, N), np.int32),
        ent_pos=np.zeros((S, N, MAX_ENTS, 3)), ent_dir=np.zeros((S, N, MAX_ENTS)),
        ent_radius=np.zeros((S, N, MAX_ENTS)), ent_kind=np.zeros((S, N, MAX_ENTS), np.int8),
        ent_color=np.zeros((S, N, MAX_ENTS, 3)),
        sky_color=np.zeros((S, N, 3)), light_pos=np.zeros((S, N, 3)), light_color=np.zeros((S, N, 3)),
        light_ambient=np.zeros((S, N, 3)), cam=np.zeros((S, N, 4)),
        rng_state=np.zeros((S, N, 2), np.uint64), rng_inc=np.zeros((S, N, 2), np.uint64),
        rng_has32=np.zeros((S, N), np.int32), rng_uint=np.zeros((S, N), np.uint32),
        episode=np.zeros((S, N), np.int32),
    )

    def reset(i, k, seed=None):
        designed_reset(env, list(vals[i, k]) if pending[i, k] else None, seed)

    for i in range(N):
        k = 0
        reset(i, k, seed=1000 + i)
        snapshot(env, out, 0, i)
        record_rng(env, out, 0, i)
        out["was_reset"][0, i] = True
        done = False
        for t in range(T):
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
            snapshot(env, out, t + 1, i)
            c = env.agent.carrying
            out["carrying"][t + 1, i] = env.entities.index(c) if c is not None else -1
            record_rng(env, out, t + 1, i)
            out["episode"][t + 1, i] = k
    K = int(out["episode"][-1].max()) + 1                 # the episodes that ran
    out.update(actions=actions, design_pending=pending[:, :K], design_draws=vals[:, :K],
               episode_steps=np.array(EPISODE_STEPS, np.int32),
               meta=np.array([env_id, repr(sorted(kwargs.items())), str(N), str(T), str(n_act), np.__version__]))
    path = os.path.join(HERE, "..", "tests", "golden", "traj_draws_%s.npz" % name)
    np.savez_compressed(path, **out)
    used = sum(int(pending[i, :out["episode"][-1, i] + 1].sum()) for i in range(N))
    print("%-12s N=%d T=%d D=%d  episodes=%d  designed resets=%d  terminated=%d  -> %s (%d B)" % (
        name, N, T, len(specs), int(out["episode"][-1].sum()) + N, used, int(out["terminated"].sum()),
        os.path.relpath(path), os.path.getsize(path)))


if __name__ == "__main__":
    only = set(sys.argv[1:])
    for case in CASES:
        if not only or case[0] in only:
            run_case(*case)
