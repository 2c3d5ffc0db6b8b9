#!/usr/bin/env python
"""TEST INFRASTRUCTURE (oracle).  Golden trajectories of the UNMODIFIED reference whose episodes start from designed
poses -- what start-state and goal-placement curricula do with `place_entity(pos=..., dir=...)`.

Protocol of oracle/gen_golden.py (env i seeded 1000 + i, actions default_rng(12345), "next-step" auto-reset), with
episodes truncated after EPISODE_STEPS steps so that every env plays many episodes, and one addition: for each
(env, episode) the stored schedule holds a design -- a pending flag, an (x, z, dir) row per entity-list slot and one for
the agent, NaN where there is none.  While a reset with a pending design runs, and only then, the reference's own
place_entity is wrapped: the call that fills slot e = len(self.entities) (the agent's call: the agent row first) gets
pos = [x, y, z] (y of the pos the level passed, else 0) and dir = the designed dir when finite, else the level's, and
then runs unchanged -- the reference's `pos=` branch.  Slots whose entity has a radius of 3 or more (Sidewalk's
building) are never designed: a design there could leave a later searched placement no free spot.

    python oracle/gen_pose_golden.py [case ...]     # writes tests/golden/traj_poses_<case>.npz
"""
import math
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
from oracle.gen_golden import MAX_ENTS, snapshot  # noqa: E402
from oracle.gen_params_golden import record_rng  # noqa: E402
from oracle.ref_stub import make_reference_env  # noqa: E402

EPISODE_STEPS = 20

# name, env id, kwargs, N, T
CASES = [
    ("oneroom", "MiniWorld-OneRoom-v0", {}, 12, 300),
    ("fourrooms_dr", "MiniWorld-FourRooms-v0", {"domain_rand": True}, 12, 300),
    ("tmaze", "MiniWorld-TMaze-v0", {}, 12, 300),
    ("pickup", "MiniWorld-PickupObjects-v0", {}, 8, 300),
    ("putnext_dr", "MiniWorld-PutNext-v0", {"domain_rand": True}, 8, 300),
    ("sidewalk", "MiniWorld-Sidewalk-v0", {}, 8, 300),
]


def placed_slots(env):
    """Slots filled by place_entity in one reset (append-only entities are not), with the agent's slot and the radii."""
    calls = []
    orig = env.place_entity

    def spy(ent, *a, **kw):
        calls.append((len(env.entities), ent is env.agent))
        return orig(ent, *a, **kw)
    env.place_entity = spy
    env.reset(seed=0)
    del env.place_entity
    radius = [float(e.radius) for e in env.entities]
    return [(e, agent, radius[e]) for e, agent in calls]


def draw_designs(rs, N, K, slots, lo, hi):
    """pending [N, K], slot rows [N, K, MAX_ENTS, 3] and agent rows [N, K, 3] of every (env, episode)."""
    pending = rs.random((N, K)) < 0.8
    pose = np.full((N, K, MAX_ENTS, 3), np.nan)
    agent = np.full((N, K, 3), np.nan)
    for i in range(N):
        for k in range(K):
            xz = lambda: lo + rs.random(2) * (hi - lo)
            d = lambda: rs.uniform(-math.pi, math.pi) if rs.random() < 0.5 else math.nan
            for e, is_agent, radius in slots:
                if radius < 3 and rs.random() < 0.5:
                    pose[i, k, e] = (*xz(), d())
            if rs.random() < 0.6:
                agent[i, k] = (*xz(), d())
    return pending, pose, agent


def run_case(name, env_id, kwargs, N, T):
    env = make_reference_env(env_id, **kwargs)
    env = getattr(env, "unwrapped", env)
    env.max_episode_steps = EPISODE_STEPS
    slots = placed_slots(env)
    lo = np.array([min(r.min_x for r in env.rooms), min(r.min_z for r in env.rooms)]) + 0.5
    hi = np.array([max(r.max_x for r in env.rooms), max(r.max_z for r in env.rooms)]) - 0.5
    K = T // 2 + 2                                   # an episode takes at least two rows (its reset and a step)
    rs = np.random.default_rng(len(name))
    pending, pose, agent = draw_designs(rs, N, K, slots, lo, hi)
    n_act = env.action_space.n
    actions = np.random.default_rng(12345).integers(0, n_act, size=(T, N), dtype=np.int32)
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
    orig = env.place_entity
    active = [None]

    def place_entity(ent, room=None, pos=None, dir=None, **kw):
        if active[0] is not None:
            rows, agent_row = active[0]
            e = len(env.entities)
            cands = ([agent_row] if ent is env.agent else []) + ([rows[e]] if e < MAX_ENTS else [])
            for row in cands:
                if math.isfinite(row[0]) and math.isfinite(row[1]):
                    pos = np.array([row[0], 0.0 if pos is None else float(pos[1]), row[1]])
                    dir = float(row[2]) if math.isfinite(row[2]) else dir
                    break
        return orig(ent, room=room, pos=pos, dir=dir, **kw)

    def reset(i, k, seed=None):
        active[0] = (pose[i, k], agent[i, k]) if pending[i, k] else None
        env.place_entity = place_entity
        env.reset(seed=seed)
        del env.place_entity
        active[0] = None

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
    out.update(actions=actions, design_pending=pending[:, :K], design_pose=pose[:, :K], design_agent=agent[:, :K],
               episode_steps=np.array(EPISODE_STEPS, np.int32),
               meta=np.array([env_id, repr(sorted(kwargs.items())), str(N), str(T), str(n_act), np.__version__]))
    path = os.path.join(HERE, "..", "tests", "golden", "traj_poses_%s.npz" % name)
    np.savez_compressed(path, **out)
    used = sum(int(pending[i, :out["episode"][-1, i] + 1].sum()) for i in range(N))
    print("%-13s N=%d T=%d  episodes=%d  designed resets=%d  terminated=%d  -> %s (%d B)" % (
        name, N, T, int(out["episode"][-1].sum()) + N, used, int(out["terminated"].sum()), os.path.relpath(path),
        os.path.getsize(path)))


if __name__ == "__main__":
    only = set(sys.argv[1:])
    for case in CASES:
        if not only or case[0] in only:
            run_case(*case)
