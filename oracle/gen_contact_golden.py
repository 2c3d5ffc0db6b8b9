#!/usr/bin/env python
"""TEST INFRASTRUCTURE (oracle).  One-step cases at K1's decision boundaries, recorded from the UNMODIFIED reference.

Random-action trajectories (gen_golden.py) almost never end a step within a few ulps of a wall, an entity, a reach
or goal threshold or a room edge, and those are the states where a restatement of the reference's arithmetic goes
wrong.  This script builds such states on purpose.  For each case it resets a reference env of the level with a
fixed seed, overwrites the state the case needs (agent and entity poses, the entity list's order, what the agent
carries, step_count, the level counter and the RNG state), records that pre-state, calls the reference's step()
once and records the post-state.

Boundary cases are found, not written down: one coordinate of the pre-state is scanned coarsely until the
reference's outcome (moved or not, picked up or not, reward, ...) flips, and then bisected to two adjacent doubles.
Those two, and their neighbours 1 and 3 ulps further out, are recorded with the outcome the reference produced; a
boundary is kept only if its two sides differ.  A few positions are chosen for the arithmetic they exercise: the
distance to a wall exactly equal to the radius (strict `<`), and an entity distance whose fused and unfused
evaluations fall on different sides of the threshold (np.linalg.norm goes through BLAS ddot, which fuses).

    python oracle/gen_contact_golden.py       # writes tests/golden/contact_cases.npz

tests/test_physics_contact.py replays every case through K1 (host build and libmwb.so) and compares bit for bit.
"""
import math
import os
import sys
from fractions import Fraction

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
from oracle.ref_stub import make_reference_env  # noqa: E402
from miniworld_b200.engine import RNG_DTYPE, rng_state_of  # noqa: E402

MAX_ENTS = 20
SEED = 7
OUT = os.path.join(HERE, "..", "tests", "golden", "contact_cases.npz")

# level key -> (gym id, kwargs, counter attribute)
LEVELS = {
    "fourrooms": ("MiniWorld-FourRooms-v0", {}, None),
    "fourrooms_dr": ("MiniWorld-FourRooms-v0", {"domain_rand": True}, None),
    "wallgap": ("MiniWorld-WallGap-v0", {}, None),
    "hallway": ("MiniWorld-Hallway-v0", {}, None),
    "oneroom": ("MiniWorld-OneRoom-v0", {}, None),
    "sidewalk": ("MiniWorld-Sidewalk-v0", {}, None),
    "pickup": ("MiniWorld-PickupObjects-v0", {}, "num_picked_up"),
    "collecthealth": ("MiniWorld-CollectHealth-v0", {}, "health"),
    "putnext": ("MiniWorld-PutNext-v0", {}, None),
    "sign": ("MiniWorld-Sign-v0", {}, None),
}


def ulps(x, k):
    """x moved by k ulps (k may be negative)."""
    for _ in range(abs(k)):
        x = np.nextafter(x, np.inf if k > 0 else -np.inf)
    return float(x)


def fma(a, b, c):
    return float(Fraction(a) * Fraction(b) + Fraction(c))


class Level:
    """A reference env reset with SEED, and the means to put it into any pre-state and step it once."""

    def __init__(self, key):
        self.key = key
        env_id, kwargs, self.counter_attr = LEVELS[key]
        self.env = env = make_reference_env(env_id, **kwargs)
        env.reset(seed=SEED)
        self.base = list(env.entities)
        self.agent = self.base.index(env.agent)
        self.base_pos = [np.array(e.pos, dtype=float) for e in self.base]
        self.base_dir = [float(e.dir) for e in self.base]
        self.base_rng = env.np_random.bit_generator.state
        self.base_counter = getattr(env, self.counter_attr) if self.counter_attr else 0
        self.segs = np.array(env.wall_segs, dtype=float)

    def state(self, **kw):
        """Pre-state: the reset's state with the listed fields replaced.  `order` lists base entity indices;
        `pos` / `dir` map base index -> value; `carrying` is a base index (its pose is set to the carry pose)."""
        st = dict(order=list(range(len(self.base))), pos={}, dir={}, carrying=-1, step_count=0,
                  counter=self.base_counter, rng=self.base_rng)
        for k, v in kw.items():
            if k in ("pos", "dir"):
                st[k] = dict(v)
            else:
                st[k] = v
        return st

    def apply(self, st):
        env = self.env
        env.entities = [self.base[j] for j in st["order"]]
        for j in st["order"]:
            e = self.base[j]
            p = st["pos"].get(j, self.base_pos[j])
            e.pos = np.array([float(p[0]), float(p[1]), float(p[2])]) if len(p) == 3 else \
                np.array([float(p[0]), 0.0, float(p[1])])
            e.dir = float(st["dir"].get(j, self.base_dir[j]))
        env.agent.carrying = None
        if st["carrying"] >= 0:
            c = self.base[st["carrying"]]
            env.agent.carrying = c
            c.pos = env._get_carry_pos(env.agent.pos, c)
            c.dir = env.agent.dir
        env.step_count = int(st["step_count"])
        if self.counter_attr:
            setattr(env, self.counter_attr, int(st["counter"]))
        env.np_random.bit_generator.state = st["rng"]

    def record(self, st):
        """The applied pre-state in packed form (per slot: base index, pose)."""
        env = self.env
        order = [self.base.index(e) for e in env.entities]
        pos = np.zeros((MAX_ENTS, 3))
        dr = np.zeros(MAX_ENTS)
        for k, e in enumerate(env.entities):
            pos[k] = np.asarray(e.pos, dtype=float)
            dr[k] = float(e.dir)
        car = env.agent.carrying
        return dict(order=order, pos=pos, dir=dr, carrying=env.entities.index(car) if car is not None else -1,
                    step_count=env.step_count, counter=getattr(env, self.counter_attr) if self.counter_attr else 0,
                    rng=rng_state_of(env.np_random))

    def run(self, st, action):
        """(pre record, post record) of one reference step from pre-state `st`."""
        env = self.env
        self.apply(st)
        pre = self.record(st)
        pos0, dir0 = np.array(env.agent.pos, dtype=float), float(env.agent.dir)
        _, r, te, tr, _ = env.step(int(action))
        post = self.record(st)
        post.update(reward=float(r), terminated=bool(te), truncated=bool(tr))
        car = env.agent.carrying
        post["carried"] = self.base.index(car) if car is not None else -1
        post["agent_pos"] = np.array(env.agent.pos, dtype=float)
        post["agent_dir"] = float(env.agent.dir)
        post["moved"] = not np.array_equal(post["agent_pos"], pos0)
        post["turned"] = post["agent_dir"] != dir0
        return pre, post


CASES = []      # (level, name, branch, action, pre, post)


def emit(L, name, branch, action, st):
    pre, post = L.run(st, action)
    CASES.append((L.key, name, branch, int(action), pre, post))
    return post


def boundary(L, name, branch, action, make, outcome, lo, hi, n=80, extra=()):
    """Scan make(x) for x in [lo, hi] until outcome(post) flips, bisect to adjacent doubles a, b and record a, b and
    1 and 3 ulps beyond each (plus `extra` coordinates).  Returns (a, b)."""
    f = lambda x: outcome(L.run(make(x), action)[1])
    xs = np.linspace(lo, hi, n)
    f0 = f(xs[0])
    k = next((k for k in range(1, n) if f(xs[k]) != f0), None)
    assert k is not None, "%s: outcome does not change over [%r, %r]" % (name, lo, hi)
    a, b = float(xs[k - 1]), float(xs[k])
    while True:
        m = (a + b) / 2
        if m == a or m == b:
            break
        if f(m) == f0:
            a = m
        else:
            b = m
    assert f(a) != f(b) and np.nextafter(a, b) == b, name
    step = 1 if b > a else -1
    for tag, x in (("a-3", ulps(a, -3 * step)), ("a-1", ulps(a, -step)), ("a", a), ("b", b), ("b+1", ulps(b, step)),
                   ("b+3", ulps(b, 3 * step))) + tuple(("x%d" % i, x) for i, x in enumerate(extra)):
        emit(L, "%s[%s]" % (name, tag), branch, action, make(x))
    return a, b


def gen_walls():
    # --- FourRooms: wall interior at a non-axis heading, forward and back; door corner (3, 1) forward and back
    L = Level("fourrooms")
    A = L.agent
    for name, act, d in (("fwd", 2, 0.3), ("back", 3, 0.3 + math.pi)):
        mk = lambda x, d=d: L.state(pos={A: (x, 4.0)}, dir={A: d})
        boundary(L, "walls_interior_" + name, "circle_hits_walls", act, mk,
                 lambda p: p["moved"], 6.30, 6.60)
    for name, act, d in (("fwd", 2, 2.3), ("back", 3, 2.3 + math.pi)):
        mk = lambda x, d=d: L.state(pos={A: (x, 1.5)}, dir={A: d})
        boundary(L, "walls_endpoint_" + name, "circle_hits_walls", act, mk,
                 lambda p: p["moved"], 3.30, 3.10)
    # --- WallGap: the gap's corner (1.5, 0.5) at a non-axis heading
    L = Level("wallgap")
    A = L.agent
    mk = lambda x: L.state(pos={A: (x, 1.0)}, dir={A: 0.8})
    boundary(L, "walls_endpoint_gap", "circle_hits_walls", 2, mk, lambda p: p["moved"], 1.20, 1.40)
    # distance to the wall z = 0.5 exactly equal to the agent's radius: strict `<` lets the move through
    from miniworld.math import intersect_circle_segs
    d = 0.2
    mk = lambda z: L.state(pos={A: (4.0, z)}, dir={A: d})
    a, b = boundary(L, "walls_interior_gap", "circle_hits_walls", 2, mk, lambda p: p["moved"], 0.98, 0.90)
    ties = []
    z = ulps(a, 40)
    for _ in range(120):
        L.apply(mk(z))
        ag = L.env.agent
        nxt = ag.pos + ag.dir_vec * 0.15 + ag.right_vec * 0.0
        r = ag.radius
        if not intersect_circle_segs(nxt, r, L.env.wall_segs) and \
                intersect_circle_segs(nxt, float(np.nextafter(r, np.inf)), L.env.wall_segs):
            ties.append(z)
        z = ulps(z, -1)
    assert ties, "no exact wall tie found"
    for k, z in enumerate(ties[:2]):
        emit(L, "walls_tie[%d]" % k, "circle_hits_walls", 2, mk(z))
    # --- drift: FourRooms with domain randomisation (fwd_drift drawn from the stream)
    L = Level("fourrooms_dr")
    A = L.agent
    mk = lambda x: L.state(pos={A: (x, 4.0)}, dir={A: 0.3})
    boundary(L, "drift_wall_fwd", "drift", 2, mk, lambda p: p["moved"], 6.20, 6.70)
    mk = lambda x: L.state(pos={A: (x, 1.5)}, dir={A: 2.3})
    boundary(L, "drift_wall_endpoint", "drift", 2, mk, lambda p: p["moved"], 3.40, 3.00)


def fused_split(L, target, R, mk, xs):
    """Coordinates x (of xs) whose final agent position is at an entity distance where the fused (BLAS ddot) and the
    unfused sum of squares fall on different sides of R."""
    out = []
    for x in xs:
        L.apply(mk(x))
        ag = L.env.agent
        p = ag.pos + ag.dir_vec * 0.15 + ag.right_vec * 0
        t = np.asarray(L.base[target].pos, dtype=float)
        dx, dz = t[0] - p[0], t[2] - p[2]
        df = math.sqrt(fma(dz, dz, dx * dx))
        du = math.sqrt(dz * dz + dx * dx)
        if (df < R) != (du < R):
            out.append(x)
    return out


def gen_entities():
    # --- Box (float64 radius): OneRoom's goal box; scan headings for a fused / unfused split at the threshold
    L = Level("oneroom")
    A, B = L.agent, 0
    bx, bz = L.base_pos[B][0], L.base_pos[B][2]
    R = 0.4 + L.base[B].radius
    got = 0
    for k in range(60):
        d = 0.1 + 0.013 * k
        dz0 = 0.35
        mk = lambda x, d=d: L.state(pos={A: (x, bz + dz0)}, dir={A: d})
        lo, hi = bx - 2.0, bx - 0.3
        f = lambda x: L.run(mk(x), 2)[1]["moved"]
        xs = np.linspace(lo, hi, 60)
        i = next(i for i in range(1, 60) if f(xs[i]) != f(xs[0]))
        a, b = xs[i - 1], xs[i]
        while True:
            m = (a + b) / 2
            if m == a or m == b:
                break
            a, b = (m, b) if f(m) == f(xs[0]) else (a, m)
        split = fused_split(L, B, R, mk, [ulps(a, j) for j in range(-4, 5)])
        if split:
            boundary(L, "entity_box_f64_fma%d" % got, "world_intersect", 2, mk,
                     lambda p: p["moved"], lo, hi, extra=split)
            got += 1
            if got == 2:
                break
    assert got, "no fused / unfused split found for the box"
    mk = lambda x: L.state(pos={A: (x, bz - 0.2)}, dir={A: -0.15})
    boundary(L, "entity_box_f64", "world_intersect", 2, mk, lambda p: p["moved"], bx - 2.0, bx - 0.3)
    # --- MeshEnt (float32 radius): PickupObjects' keys, CollectHealth's med-kits
    L = Level("pickup")
    A = L.agent
    park = {0: (9.5, 3.4), 1: (1.0, 1.0), 2: (11.0, 11.0), 3: (1.0, 11.0), 4: (11.0, 1.0)}
    R = np.float32(np.float32(0.4) + L.base[0].radius)
    got = 0
    for k in range(60):
        d = 0.05 + 0.011 * k
        mk = lambda x, d=d: L.state(pos={**park, A: (x, 3.7)}, dir={A: d})
        split = []
        f = lambda x: L.run(mk(x), 2)[1]["moved"]
        xs = np.linspace(7.0, 9.0, 60)
        i = next(i for i in range(1, 60) if f(xs[i]) != f(xs[0]))
        a, b = xs[i - 1], xs[i]
        while True:
            m = (a + b) / 2
            if m == a or m == b:
                break
            a, b = (m, b) if f(m) == f(xs[0]) else (a, m)
        split = fused_split(L, 0, float(R), mk, [ulps(a, j) for j in range(-4, 5)])
        if split:
            boundary(L, "entity_mesh_f32_fma%d" % got, "world_intersect", 2, mk,
                     lambda p: p["moved"], 7.0, 9.0, extra=split)
            got += 1
            if got == 2:
                break
    mk = lambda x: L.state(pos={**park, A: (x, 3.2)}, dir={A: 0.12})
    boundary(L, "entity_mesh_f32", "world_intersect", 2, mk, lambda p: p["moved"], 7.0, 9.0)
    L = Level("collecthealth")
    A = L.agent
    kx, kz = L.base_pos[0][0], L.base_pos[0][2]
    mk = lambda x: L.state(pos={A: (x, kz + 0.3)}, dir={A: 0.25}, counter=60)
    boundary(L, "entity_mesh_medkit", "world_intersect", 2, mk, lambda p: p["moved"], kx - 1.5, kx - 0.2)


def gen_carry():
    L = Level("putnext")
    A, RED, YEL = L.agent, 4, 5      # boxes in COLOR_NAMES order: blue, green, grey, purple, red, yellow
    park = {0: (1.0, 1.0), 1: (1.0, 11.0), 2: (11.0, 1.0), 3: (6.0, 1.0), YEL: (1.0, 6.0)}
    # the agent is free, the carried box hits the east wall
    mk = lambda x: L.state(pos={**park, A: (x, 6.0)}, dir={A: 0.3}, carrying=RED)
    boundary(L, "carry_move_wall", "move with carry", 2, mk, lambda p: p["moved"], 9.8, 10.8)
    # the carried box hits the yellow box
    mk = lambda x: L.state(pos={**park, YEL: (7.0, 5.5), A: (x, 6.0)}, dir={A: 0.3}, carrying=RED)
    boundary(L, "carry_move_entity", "move with carry", 2, mk, lambda p: p["moved"], 3.5, 5.5)
    # moving back: the carried box (ahead of the agent, moving with it) grazes the green box beside its path
    mk = lambda z: L.state(pos={**park, 1: (7.28, z), A: (8.0, 6.0)}, dir={A: math.pi + 0.2}, carrying=RED)
    boundary(L, "carry_move_back_entity", "move with carry", 3, mk, lambda p: p["moved"], 7.4, 6.8)
    # turn with carry: the carried box would hit the east wall at the new heading -> heading and box unchanged
    mk = lambda x: L.state(pos={**park, A: (x, 6.0)}, dir={A: math.pi / 2}, carrying=RED)
    boundary(L, "carry_turn_wall", "turn with carry", 1, mk, lambda p: p["turned"], 10.9, 11.5)
    mk = lambda x: L.state(pos={**park, YEL: (x, 5.2), A: (5.0, 6.0)}, dir={A: math.pi / 2 + 0.1}, carrying=RED)
    boundary(L, "carry_turn_entity", "turn with carry", 0, mk, lambda p: p["turned"], 3.0, 4.6)
    # pickup while carrying: refused, another box in reach before the carried one in the list
    emit(L, "pickup_while_carrying", "pickup reach", 4,
         L.state(pos={**park, 1: (5.8, 6.0), A: (5.0, 6.0)}, dir={A: 0.0}, carrying=RED))
    # near_pair while carrying: the boxes are near, no reward
    emit(L, "near_pair_carrying", "near_pair", 6,
         L.state(pos={**park, YEL: (6.5, 6.8), A: (5.0, 6.0)}, dir={A: 0.0}, carrying=RED))
    # after a drop: the red box lands at its carry position, yellow box either side of the threshold
    mk = lambda x: L.state(pos={**park, YEL: (x, 6.3), A: (5.0, 6.0)}, dir={A: 0.1}, carrying=RED)
    boundary(L, "near_pair_drop", "near_pair", 5, mk, lambda p: p["reward"], 7.0, 8.2)
    # no carry: a noop step with the boxes at the threshold
    mk = lambda x: L.state(pos={**park, RED: (5.0, 5.0), YEL: (x, 5.4), A: (9.0, 9.0)})
    boundary(L, "near_pair_still", "near_pair", 6, mk, lambda p: p["reward"], 5.5, 7.0)


def gen_pickup():
    L = Level("pickup")
    A = L.agent
    park = {0: (1.0, 1.0), 1: (1.0, 11.0), 2: (11.0, 11.0), 3: (11.0, 1.0), 4: (6.0, 1.0)}
    for name, j in (("box", 2), ("key", 0)):
        mk = lambda x, j=j: L.state(pos={**park, j: (8.0, 6.0), A: (x, 6.2)}, dir={A: -0.1})
        boundary(L, "pickup_reach_" + name, "pickup reach", 4, mk, lambda p: p["reward"], 5.8, 7.5)
    # the last object: num_picked_up reaches num_objs
    mk = lambda x: L.state(order=[1, A], pos={1: (8.0, 6.0), A: (x, 6.2)}, dir={A: -0.1}, counter=4)
    boundary(L, "pickup_last_object", "PickupObjects", 4, mk, lambda p: p["terminated"], 5.8, 7.5)
    # a static entity in reach: refused
    L = Level("sidewalk")
    A = L.agent
    emit(L, "pickup_static", "pickup reach", 4, L.state(pos={A: (-0.2, 2.0)}, dir={A: 0.05}))


def gen_goals():
    L = Level("hallway")
    A, B = L.agent, 0
    bx, bz = L.base_pos[B][0], L.base_pos[B][2]
    mk = lambda x: L.state(pos={A: (x, bz + 0.25)}, dir={A: 0.05})
    boundary(L, "near_goal_box_hallway", "near_point", 2, mk, lambda p: p["terminated"], bx - 2.0, bx - 0.9)
    mk = lambda x: L.state(pos={A: (x, bz + 0.25)}, dir={A: 0.05}, step_count=249)
    boundary(L, "truncation_goal", "truncation", 2, mk, lambda p: p["reward"], bx - 2.0, bx - 0.9)
    L = Level("oneroom")
    A, B = L.agent, 0
    bx, bz = L.base_pos[B][0], L.base_pos[B][2]
    mk = lambda x: L.state(pos={A: (x, bz - 0.4)}, dir={A: 0.4})
    boundary(L, "near_goal_box_oneroom", "near_point", 2, mk, lambda p: p["terminated"], bx - 2.0, bx - 0.9)
    # Sign: a BigKey (MeshEnt, float32 radius) reached; blue box is slot 0, blue key slot 3
    L = Level("sign")
    A = L.agent
    mk = lambda z: L.state(pos={A: (5.05, z)}, dir={A: math.pi / 2 - 0.1})
    boundary(L, "near_goal_bigkey", "near_point", 2, mk, lambda p: p["reward"], 3.3, 4.2)
    # two objects near at once: the box (reward +1) and the key, later in the loop (-1) -- the last hit wins
    mk = lambda x: L.state(pos={0: (4.0, 4.0), 3: (x, 5.0), A: (5.0, 5.0)}, dir={A: 0.3})
    boundary(L, "sign_two_near", "Sign", 0, mk, lambda p: p["reward"], 6.0, 7.2)
    # action 3 (end the episode; it also moves back) with an object at the threshold
    mk = lambda x: L.state(pos={3: (x, 3.0), A: (5.0, 4.0)}, dir={A: math.pi / 2})
    boundary(L, "sign_action3_near", "Sign", 3, mk, lambda p: p["reward"], 5.2, 6.6)
    emit(L, "sign_action3_nothing_near", "Sign", 3, L.state(pos={A: (5.0, 4.0)}, dir={A: math.pi / 2}))


def gen_street():
    L = Level("sidewalk")
    A, BOX = L.agent, 6
    mk = lambda x: L.state(pos={A: (x, 3.0)}, dir={A: 0.2})
    boundary(L, "street_edge", "room_contains", 2, mk, lambda p: p["terminated"], -0.3, 0.1)
    # the street rule and the goal on the same step, the goal either side of its threshold
    mk = lambda x: L.state(pos={A: (-0.05, 3.0), BOX: (x, 2.97)}, dir={A: 0.2})
    boundary(L, "street_and_goal", "room_contains", 2, mk, lambda p: p["reward"], 1.0, 1.4)


def gen_health():
    L = Level("collecthealth")
    A = L.agent

    def draws(st):
        """How many doubles the kit's respawn took from the stream."""
        pre, post = L.run(st, 4)
        g = np.random.Generator(np.random.PCG64())
        g.bit_generator.state = st["rng"]
        for n in range(200):
            if rng_state_of(g) == post["rng"]:
                return n
            g.random()
        return -1

    kx, kz = L.base_pos[0][0], L.base_pos[0][2]
    base = L.state(pos={A: (kx - 0.9, kz)}, dir={A: 0.0}, counter=40)
    # a stream position at which place_entity rejects several draws (4 per try, then the heading)
    g = np.random.Generator(np.random.PCG64())
    g.bit_generator.state = L.base_rng
    rng = None
    for _ in range(400):
        st = dict(base, rng=g.bit_generator.state)
        if draws(st) >= 13:
            rng = st["rng"]
            break
        g.random()
    assert rng is not None
    for name, order in (("kit_before_agent", list(range(19))), ("kit_after_agent", list(range(1, 19)) + [0])):
        mk = lambda x, order=order: L.state(order=order, pos={A: (x, kz)}, dir={A: 0.0}, counter=40, rng=rng)
        boundary(L, "health_" + name, "CollectHealth", 4, mk, lambda p: p["counter"], kx - 2.0, kx - 0.5)


def main():
    gen_walls()
    gen_entities()
    gen_carry()
    gen_pickup()
    gen_goals()
    gen_street()
    gen_health()
    n = len(CASES)
    out = dict(level=np.array([c[0] for c in CASES]), name=np.array([c[1] for c in CASES]),
               branch=np.array([c[2] for c in CASES]), action=np.array([c[3] for c in CASES], np.int32))
    for side in ("pre", "post"):
        recs = [c[4] if side == "pre" else c[5] for c in CASES]
        order = np.full((n, MAX_ENTS), -1, np.int32)
        for i, r in enumerate(recs):
            order[i, :len(r["order"])] = r["order"]
        out[side + "_order"] = order
        out[side + "_pos"] = np.stack([r["pos"] for r in recs])
        out[side + "_dir"] = np.stack([r["dir"] for r in recs])
        out[side + "_carrying"] = np.array([r["carrying"] for r in recs], np.int32)
        out[side + "_step_count"] = np.array([r["step_count"] for r in recs], np.int32)
        out[side + "_counter"] = np.array([r["counter"] for r in recs], np.int32)
        out[side + "_rng"] = np.array([r["rng"][()] for r in recs], RNG_DTYPE)
    post = [c[5] for c in CASES]
    out["reward"] = np.array([p["reward"] for p in post])
    out["terminated"] = np.array([p["terminated"] for p in post])
    out["truncated"] = np.array([p["truncated"] for p in post])
    levels = sorted(set(out["level"]))
    for key in levels:
        L = Level(key)
        out["segs_" + key] = L.segs
        out["radius_" + key] = np.array([float(e.radius) for e in L.base])
        out["agent_" + key] = np.int32(L.agent)
    out["meta"] = np.array([str(SEED), np.__version__])
    np.savez_compressed(OUT, **out)
    for key in levels:
        sel = out["level"] == key
        print("%-14s %3d cases" % (key, sel.sum()))
    print("%d cases -> %s (%d B)" % (n, os.path.relpath(OUT), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
