"""K1 at its decision boundaries: one step from constructed pre-states against the reference's own step.

tests/golden/contact_cases.npz (oracle/gen_contact_golden.py) holds states a few ulps either side of wall and
entity contact, carry blocking, pickup reach, goal and box-pair thresholds, the Sidewalk street edge, Sign's
object rule, CollectHealth's kit respawn, PickupObjects' last object and truncation, each with the post-state the
unmodified reference produced.  Every case of a level runs in one batch, one case per env, on the host-reset path
(the level's Python world, pre-state uploaded with mwb_set_world, stream with mwb_seed), and the post-state must
match bit for bit: poses, entity order, carrying, reward, flags, the level counter and the RNG state."""
import os

import numpy as np
import pytest

from conftest import GOLDEN

_CASES = None


def cases():
    global _CASES
    if _CASES is None:
        with np.load(os.path.join(GOLDEN, "contact_cases.npz")) as z:
            _CASES = {k: z[k] for k in z.files}
    return _CASES


# golden level key -> (level id, domain_rand)
LEVELS = {"fourrooms": ("MiniWorld-FourRooms-v0", False), "fourrooms_dr": ("MiniWorld-FourRooms-v0", True),
          "wallgap": ("MiniWorld-WallGap-v0", False), "hallway": ("MiniWorld-Hallway-v0", False),
          "oneroom": ("MiniWorld-OneRoom-v0", False), "sidewalk": ("MiniWorld-Sidewalk-v0", False),
          "pickup": ("MiniWorld-PickupObjects-v0", False), "collecthealth": ("MiniWorld-CollectHealth-v0", False),
          "putnext": ("MiniWorld-PutNext-v0", False), "sign": ("MiniWorld-Sign-v0", False)}
SEED = 7


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def level_batch(key, n, case_env):
    """Host-reset batch of n envs of the level; env case_env[c] starts from case c's pre-state, every other env from
    the level's reset.  Returns (env, indices of the level's cases)."""
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.envs import LEVELS as PY_LEVELS
    from miniworld_b200.engine import RNG_DTYPE, rng_state_of
    g = cases()
    level, dr = LEVELS[key]
    idx = np.nonzero(g["level"] == key)[0]
    host_only = type("HostOnly" + PY_LEVELS[level].__name__, (PY_LEVELS[level],), {"device_program": None})
    env = BatchedMiniWorld(host_only, n, domain_rand=dr, autoreset=False)
    assert not env.device_reset
    env._host_reset(np.zeros(1, np.int32), [SEED])
    w0 = env._workers[0]
    from miniworld_b200 import pack
    base = pack.pack_world(w0)
    # the level's Python world is the reference's: walls and entity radii as the generator recorded them
    assert np.array_equal(base["segs"]["ax"], g["segs_" + key][:, 0, 0])
    assert np.array_equal(base["segs"]["bz"], g["segs_" + key][:, 1, 2])
    assert np.array_equal(base["protos"]["radius"], g["radius_" + key])
    worlds = [base] * n
    rngs = np.array([rng_state_of(w0.np_random)] * n, RNG_DTYPE)
    for c, i in zip(idx, case_env):
        order = g["pre_order"][c]
        order = order[order >= 0]
        ents = base["ents"][order].copy()
        ents["pos"] = g["pre_pos"][c, :len(order)]
        ents["dir"] = g["pre_dir"][c, :len(order)]
        w = dict(base, ents=ents, agent_slot=int(np.nonzero(order == base["agent_slot"])[0][0]),
                 carrying=int(g["pre_carrying"][c]), step_count=int(g["pre_step_count"][c]),
                 num_picked_up=int(g["pre_counter"][c]))
        worlds[i] = w
        rngs[i] = g["pre_rng"][c]
    env.engine.set_world(np.arange(n, dtype=np.int32), worlds)
    env.engine.seed(np.arange(n, dtype=np.int32), rngs)
    return env, idx


def check_cases(env, idx, case_env, out):
    """Mismatches between the post-states of the listed envs and the reference's."""
    g = cases()
    st = env.get_state(rng=True)
    bad = []
    for c, i in zip(idx, case_env):
        what = []
        order = g["post_order"][c]
        order = order[order >= 0]
        ents = st["ents"][i]
        live = np.nonzero(ents["proto"] >= 0)[0]
        if not np.array_equal(ents["proto"][live], order):
            what.append("entity order %s, want %s" % (ents["proto"][live].tolist(), order.tolist()))
        else:
            if not np.array_equal(bits(ents["pos"][live]), bits(g["post_pos"][c, :len(order)])):
                what.append("entity positions")
            if not np.array_equal(bits(ents["dir"][live]), bits(g["post_dir"][c, :len(order)])):
                what.append("entity headings")
            car = int(st["carrying"][i])
            want = int(g["post_carrying"][c])
            got = -1 if car < 0 else int(np.nonzero(live == car)[0][0])
            if got != want:
                what.append("carrying slot %d, want %d" % (got, want))
        if not (bits(out["reward"][i]) == bits(g["reward"][c])):
            what.append("reward %r, want %r" % (out["reward"][i], g["reward"][c]))
        if bool(out["terminated"][i]) != bool(g["terminated"][c]) or bool(out["truncated"][i]) != bool(g["truncated"][c]):
            what.append("flags (%d, %d), want (%d, %d)" % (out["terminated"][i], out["truncated"][i],
                                                           g["terminated"][c], g["truncated"][c]))
        if int(st["step_count"][i]) != int(g["post_step_count"][c]):
            what.append("step_count")
        if int(st["num_picked_up"][i]) != int(g["post_counter"][c]):
            what.append("counter %d, want %d" % (st["num_picked_up"][i], g["post_counter"][c]))
        if st["rng"][i].tobytes() != g["post_rng"][c].tobytes():
            what.append("rng state")
        if what:
            bad.append("%s (%s): %s" % (g["name"][c], g["branch"][c], ", ".join(what)))
    return bad


def run_level(key, n=None, seed=0):
    """Every case of the level through one batch and one step; with n, the cases sit at random envs of a batch of n
    whose other envs take random actions from the level's reset."""
    g = cases()
    m = int((g["level"] == key).sum())
    if n is None:
        n, case_env = m, np.arange(m)
    else:
        case_env = np.random.default_rng(seed).choice(n, m, replace=False)
    env, idx = level_batch(key, n, case_env)
    actions = np.random.default_rng(seed + 1).integers(0, 3, n).astype(np.int32)
    actions[case_env] = g["action"][idx]
    out = env.step_host(actions, render=False)
    bad = check_cases(env, idx, case_env, out)
    env.close()
    assert not bad, "%d of %d cases differ from the reference:\n  %s" % (len(bad), m, "\n  ".join(bad))


BRANCHES = ["circle_hits_walls", "world_intersect", "move with carry", "turn with carry", "pickup reach", "near_point",
            "near_pair", "room_contains", "Sign", "CollectHealth", "PickupObjects", "truncation", "drift"]


def outcome(c):
    """What a boundary decides, as the reference recorded it: did the agent move or turn, reward, flags, counter,
    carrying and the entity list."""
    g = cases()
    order = g["pre_order"][c]
    slot = int(np.nonzero(order == g["agent_" + str(g["level"][c])])[0][0])
    post_slot = int(np.nonzero(g["post_order"][c] == order[slot])[0][0])
    return (not np.array_equal(g["pre_pos"][c, slot], g["post_pos"][c, post_slot]),
            g["pre_dir"][c, slot] != g["post_dir"][c, post_slot], float(g["reward"][c]), bool(g["terminated"][c]),
            bool(g["truncated"][c]), int(g["post_counter"][c]), int(g["post_carrying"][c]),
            g["post_order"][c].tobytes())


@pytest.mark.parametrize("branch", BRANCHES)
def test_golden_has_both_sides_of_each_boundary(branch):
    """Each branch has boundary cases, and the two adjacent doubles of every boundary led the reference to different
    outcomes (so the recorded states sit on the boundary)."""
    g = cases()
    names = [str(s) for s in g["name"]]
    sel = [k for k, s in enumerate(names) if str(g["branch"][k]) == branch and s.endswith("[a]")]
    assert sel, "no boundary case for " + branch
    for a in sel:
        b = names.index(names[a][:-3] + "[b]")
        assert outcome(a) != outcome(b), names[a]


def level_id(key):
    g = cases()
    return "%s:%s" % (key, "+".join(sorted(set(g["branch"][g["level"] == key].tolist()))).replace(" ", "_"))


@pytest.mark.parametrize("key", sorted(LEVELS), ids=level_id)
def test_contact_cases_host_build(hostsim_path, key):
    run_level(key)


@pytest.mark.gpu
@pytest.mark.parametrize("key", sorted(LEVELS), ids=level_id)
def test_contact_cases_gpu(libmwb_path, key):
    run_level(key)


@pytest.mark.gpu
@pytest.mark.parametrize("key", sorted(LEVELS), ids=level_id)
def test_contact_cases_gpu_large_batch(libmwb_path, key):
    """The same cases scattered among 4096 envs that step from the level's reset: K1's warp-per-env wall loop at
    full occupancy."""
    run_level(key, n=4096, seed=11)
