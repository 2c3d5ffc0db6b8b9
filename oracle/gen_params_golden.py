#!/usr/bin/env python
"""TEST INFRASTRUCTURE (oracle).  Golden trajectories of the UNMODIFIED reference whose DomainParams change while
the episodes run -- what automatic domain randomisation does with `env.params.set(...)` between steps.

Protocol of oracle/gen_golden.py (env i seeded 1000 + i, actions default_rng(12345), "next-step" auto-reset), with
two additions:
  * every env runs on a private copy of its level's params (the reference's DEFAULT_PARAMS is one module-global
    object), and before step STEPS[k] of every env -- the step itself, or the reset that takes its place -- the
    calls of schedule k are applied to that copy with DomainParams.set;
  * the env's numpy stream state is recorded after every step (rng_state / rng_inc / rng_has32 / rng_uint), and so
    are self.max_forward_step and the carry position the step computed (carry_pos, NaN when it computed none).
The schedule is stored in the file (JSON), so that a test can replay it without this module.

    python oracle/gen_params_golden.py [case ...]     # writes tests/golden/traj_params_<case>.npz
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
from oracle.gen_golden import MAX_ENTS, snapshot  # noqa: E402
from oracle.ref_stub import make_reference_env  # noqa: E402

STEPS = (100, 200)

# name, env id, kwargs, N, T, [calls before step 100, calls before step 200][, action probabilities]; a call is
# (name, default, min, max)
CASES = [
    # wider step and camera ranges and a wider sky, then a forward_step max below the first one (a smaller near()
    # threshold for episodes that reset after step 200, the old one for those still running)
    ("fourrooms_dr", "MiniWorld-FourRooms-v0", {"domain_rand": True}, 32, 300, [
        [("forward_step", 0.2, 0.1, 0.35), ("turn_step", 15, 5, 30), ("cam_fov_y", 60, 40, 80),
         ("sky_color", [0.25, 0.82, 1.0], [0.0, 0.0, 0.0], [1.0, 1.0, 1.0])],
        [("forward_step", 0.13, 0.11, 0.14), ("forward_drift", 0.0, -0.1, 0.1)],
    ]),
    # randomisation off: only the defaults count
    ("oneroom", "MiniWorld-OneRoom-v0", {}, 16, 300, [
        [("forward_step", 0.45), ("turn_step", 30), ("sky_color", [0.5, 0.5, 0.5]), ("cam_height", 1.2)],
        [("forward_step", 0.95), ("turn_step", 60), ("light_ambient", [0.6, 0.6, 0.6])],
    ]),
    # near() between two entities
    ("putnext_dr", "MiniWorld-PutNext-v0", {"domain_rand": True}, 8, 300, [
        [("forward_step", 0.15, 0.12, 0.9)],
        [("forward_step", 0.125, 0.12, 0.13)],
    ], [0.2, 0.2, 0.3, 0.0, 0.15, 0.15, 0.0, 0.0]),
    # the carry position
    ("pickup_dr", "MiniWorld-PickupObjects-v0", {"domain_rand": True}, 16, 300, [
        [("forward_step", 0.15, 0.12, 0.6)],
        [("forward_step", 0.125, 0.12, 0.13), ("obj_color_bias", [0.0, 0.0, 0.0], [-0.5, -0.5, -0.5], [0.5, 0.5, 0.5])],
    ], [0.2, 0.2, 0.35, 0.0, 0.25]),
]


def apply_calls(params, calls):
    for name, default, *rest in calls:
        lo, hi = (rest + [None, None])[:2]
        params.set(name, default, lo, hi)


def record_rng(env, out, t, i):
    st = env.np_random.bit_generator.state
    s, inc = st["state"]["state"], st["state"]["inc"]
    m = (1 << 64) - 1
    out["rng_state"][t, i] = (s >> 64, s & m)
    out["rng_inc"][t, i] = (inc >> 64, inc & m)
    out["rng_has32"][t, i] = st["has_uint32"]
    out["rng_uint"][t, i] = st["uinteger"]


def run_case(name, env_id, kwargs, N, T, schedule, action_probs=None):
    env = make_reference_env(env_id, **kwargs)
    base = env.params
    n_act = env.action_space.n
    if action_probs is None:
        actions = np.random.default_rng(12345).integers(0, n_act, size=(T, N), dtype=np.int32)
    else:       # a pickup / drop heavy mix, so that carrying and putting next happen
        actions = np.random.default_rng(12345).choice(n_act, size=(T, N), p=action_probs).astype(np.int32)
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
        carry_pos=np.full((S, N, 3), np.nan),
    )
    # the carry position of each step (PickupObjects removes a picked-up object in the same step, so only this shows
    # where _get_carry_pos put it): recorded from the reference's own call, which is left to run unchanged
    carried = []
    orig = env._get_carry_pos

    def carry_pos(*a):
        carried.append(orig(*a))
        return carried[-1]
    env._get_carry_pos = carry_pos
    for i in range(N):
        env.params = base.copy()
        env.reset(seed=1000 + i)
        snapshot(env, out, 0, i)
        record_rng(env, out, 0, i)
        out["max_forward_step"][0, i] = env.max_forward_step
        out["was_reset"][0, i] = True
        done = False
        for t in range(T):
            if t in STEPS:
                apply_calls(env.params, schedule[STEPS.index(t)])
            carried.clear()
            if done:
                env.reset()
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
            if carried:
                out["carry_pos"][t + 1, i] = carried[-1]
            out["max_forward_step"][t + 1, i] = env.max_forward_step
    env.params = base
    del env._get_carry_pos
    out["actions"] = actions
    out["steps"] = np.array(STEPS, np.int32)
    out["schedule"] = np.array(json.dumps(schedule))
    out["meta"] = np.array([env_id, repr(sorted(kwargs.items())), str(N), str(T), str(n_act),
                            str(env.max_episode_steps), np.__version__])
    path = os.path.join(HERE, "..", "tests", "golden", "traj_params_%s.npz" % name)
    np.savez_compressed(path, **out)
    print("%-14s N=%d T=%d  episodes ended=%d  reward sum=%.3f  carrying steps=%d  -> %s (%d B)" % (
        name, N, T, int((out["terminated"] | out["truncated"]).sum()), out["reward"].sum(),
        int((out["carrying"] >= 0).sum()), os.path.relpath(path), os.path.getsize(path)))


if __name__ == "__main__":
    only = set(sys.argv[1:])
    for case in CASES:
        if not only or case[0] in only:
            run_case(*case)
