"""Goal distance in numpy: the definitions the batched engine's goal distance kernel computes (csrc/navigation.cuh,
include/mwb.h mwb_enable_goal_distance), restated operation for operation so that both agree bit for bit.

A goal level gets a grid of step H over the bounding box of its rooms' outlines.  For a world at a reset, a node is a
source when an agent standing there is near(goal), and free when no wall lies within r + H/2 and no entity other than
the agent and the goal within r + H/2 + its radius (r: the agent's radius).  Edges join free-or-source 8-neighbours,
5 units orthogonally and 7 diagonally (a diagonal needs both orthogonal nodes it passes free-or-source); one unit is
H / 5 = 0.05 m.  The field is the integer distance from the nearest source (Dijkstra), capped at 0xFFFE, with 0xFFFF
for every other node.  `query` reads the agent's geodesic distance and an expert action from it.

The world comes as the engine stores it: mwb_room records (ROOM_DTYPE), mwb_seg records (SEG_DTYPE) and an entity list
of (x, y, z, radius, radius_is_float32) tuples, None for an empty slot.  `world_of` builds that from a MiniWorldEnv.
"""
import heapq
import math
from fractions import Fraction

import numpy as np

from .engine import GOAL_GRID_CAP, GOAL_GRID_STEP

H = GOAL_GRID_STEP
NONE = 0xFFFF
MAX = 0xFFFE
PASS, FREE, SOURCE = 1, 2, 4            # node class bits, as in navigation.cuh
TURN_LEFT, TURN_RIGHT, MOVE_FORWARD = 0, 1, 2
_DEG = 0.017453292519943295              # math.pi / 180


def level_grid(env):
    """(min_x, min_z, nx, nz) of a level's definition instance: its rooms' bounding box, ceil(extent / H) nodes per
    axis.  ValueError beyond GOAL_GRID_CAP nodes."""
    min_x = min(float(r.min_x) for r in env.rooms)
    max_x = max(float(r.max_x) for r in env.rooms)
    min_z = min(float(r.min_z) for r in env.rooms)
    max_z = max(float(r.max_z) for r in env.rooms)
    nx, nz = max(1, math.ceil((max_x - min_x) / H)), max(1, math.ceil((max_z - min_z) / H))
    if nx * nz > GOAL_GRID_CAP:
        raise ValueError("%s: a goal grid of %d x %d nodes at %g m is more than %d nodes"
                         % (type(env).__name__, nx, nz, H, GOAL_GRID_CAP))
    return min_x, min_z, nx, nz


def world_of(env):
    """(rooms, segs, ents, agent slot) of a MiniWorldEnv as the engine would hold them."""
    from .pack import pack_geometry
    rooms, _, segs = pack_geometry(env)
    ents = [(float(e.pos[0]), float(e.pos[1]), float(e.pos[2]), float(e.radius), isinstance(e.radius, np.float32))
            for e in env.entities]
    return rooms, segs, ents, env.entities.index(env.agent)


def _fma(a, b, c):
    """a * b + c rounded once (the device's d_fma; Fraction arithmetic is exact, int / int rounds correctly)."""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def _norm3(dx, dy, dz):
    """np.linalg.norm of (dx, dy, dz) as BLAS ddot evaluates it: sqrt(fma(dz, dz, fma(dy, dy, dx * dx)))."""
    return math.sqrt(_fma(dz, dz, _fma(dy, dy, dx * dx)))


def _near_threshold(r0, r0_f32, r1, r1_f32, extra):
    if r0_f32 or r1_f32:
        return float(np.float32(np.float32(np.float32(r0) + np.float32(r1)) + np.float32(extra)))
    return (r0 + r1) + extra


def near(goal, x, y, z, agent_radius, mfs):
    """MiniWorldEnv.near(goal) for an agent of radius `agent_radius` at (x, y, z)."""
    gx, gy, gz, gr, gf = goal
    return _norm3(gx - x, gy - y, gz - z) < _near_threshold(gr, gf, agent_radius, False, 1.1 * mfs)


def _nodes(grid):
    min_x, min_z, nx, nz = grid
    k, l = np.meshgrid(np.arange(nx), np.arange(nz))
    return min_x + (k.ravel() + 0.5) * H, min_z + (l.ravel() + 0.5) * H


def node_classes(grid, rooms, segs, ents, agent, goal, mfs):
    """uint8 [nz * nx] class bits (PASS, FREE, SOURCE) of every node, flat index l * nx + k."""
    x, z = _nodes(grid)
    inside = np.zeros(x.shape, bool)
    for r in rooms:
        ok = np.ones(x.shape, bool)
        for e in range(int(r["num_edges"])):
            ok &= r["edge_nx"][e] * (x - r["edge_px"][e]) + r["edge_nz"][e] * (z - r["edge_pz"][e]) > 0
        inside |= ok
    ax, ay, az, ar, _ = ents[agent]
    cls = np.zeros(x.shape, np.uint8)
    # near(goal): evaluated exactly wherever a plain-arithmetic estimate cannot settle the comparison
    gx, gy, gz, gr, gf = ents[goal]
    thr = _near_threshold(gr, gf, ar, False, 1.1 * mfs)
    est = np.sqrt((gx - x) ** 2 + (gy - ay) ** 2 + (gz - z) ** 2)
    src = inside & (est < thr)
    for n in np.nonzero(inside & (np.abs(est - thr) <= 1e-9 * (1.0 + thr)))[0]:
        src[n] = near(ents[goal], x[n], ay, z[n], ar, mfs)
    cls[src] |= PASS | SOURCE
    rad = ar + 0.5 * H
    free = inside.copy()
    for s in segs:      # circle_hits_walls, one segment at a time over every node
        abx, abz = s["bx"] - s["ax"], s["bz"] - s["az"]
        apx, apz = x - s["ax"], z - s["az"]
        t = (apx * abx + apz * abz) / (abx * abx + abz * abz)
        t = np.where(t < 0.0, 0.0, np.where(t > 1.0, 1.0, t))
        dx, dz = (s["ax"] + t * abx) - x, (s["az"] + t * abz) - z
        free &= ~(np.sqrt(dx * dx + dz * dz) < rad)
    for e, ent in enumerate(ents):
        if ent is None or e in (agent, goal):
            continue
        ex, _, ez, er, ef = ent
        lim = float(np.float32(np.float32(rad) + np.float32(er))) if ef else rad + er
        for n in np.nonzero(free)[0]:
            dx, dz = ex - x[n], ez - z[n]
            if math.sqrt(_fma(dz, dz, dx * dx)) < lim:
                free[n] = False
    cls[free] |= PASS | FREE
    return cls


def _edges(cls, nx, nz, n):
    """(neighbour, cost) of every edge of node n, in increasing neighbour index."""
    k, l = n % nx, n // nx
    passable = lambda kk, ll: 0 <= kk < nx and 0 <= ll < nz and cls[ll * nx + kk] & PASS
    for dl in (-1, 0, 1):
        for dk in (-1, 0, 1):
            if (dk or dl) and passable(k + dk, l + dl):
                if dk and dl and not (passable(k + dk, l) and passable(k, l + dl)):
                    continue
                yield (l + dl) * nx + k + dk, 7 if dk and dl else 5


def distance_field(cls, nx, nz):
    """uint16 [nz * nx]: Dijkstra from every SOURCE node over the edges between PASS nodes, capped at MAX."""
    dist = np.full(nx * nz, NONE, np.int64)
    heap = [(0, int(n)) for n in np.nonzero(cls & SOURCE)[0]]
    for _, n in heap:
        dist[n] = 0
    heapq.heapify(heap)
    while heap:
        d, n = heapq.heappop(heap)
        if d > dist[n]:
            continue
        for m, w in _edges(cls, nx, nz, n):
            v = min(d + w, MAX)
            if v < dist[m]:
                dist[m] = v
                heapq.heappush(heap, (v, m))
    return dist.astype(np.uint16)


def query(grid, field, cls, ents, agent, goal, mfs, agent_dir, turn_step):
    """(goal_dist, expert_action) of an agent in slot `agent` facing `agent_dir`; `turn_step` is the level's default
    turn step in degrees."""
    min_x, min_z, nx, nz = grid
    ax, ay, az, ar, _ = ents[agent]
    is_near = near(ents[goal], ax, ay, az, ar, mfs)
    best, dist = -1, 0.0 if is_near else math.inf
    if not is_near:
        k0 = math.floor((ax - min_x) / H - 0.5)
        l0 = math.floor((az - min_z) / H - 0.5)
        for l in range(l0 - 1, l0 + 3):
            for k in range(k0 - 1, k0 + 3):
                if not (0 <= k < nx and 0 <= l < nz):
                    continue
                n = l * nx + k
                if not cls[n] & FREE or field[n] == NONE:
                    continue
                dx, dz = (min_x + (k + 0.5) * H) - ax, (min_z + (l + 0.5) * H) - az
                v = float(field[n]) * 0.05 + math.sqrt(dx * dx + dz * dz)
                if v < dist:
                    dist, best = v, n
    if not is_near and best < 0:
        return math.inf, -1
    wx, wz = ents[goal][0], ents[goal][2]
    if not is_near and field[best] != 0:
        m = min(_edges(cls, nx, nz, best), key=lambda e: (int(field[e[0]]) + e[1] if field[e[0]] != NONE else 1 << 20,
                                                           e[0]))[0]
        wx, wz = min_x + (m % nx + 0.5) * H, min_z + (m // nx + 0.5) * H
    co, si = math.cos(agent_dir), math.sin(agent_dir)
    vx, vz = wx - ax, wz - az
    vf = vx * co + vz * -si
    vv = vx * vx + vz * vz
    ch = math.cos(0.5 * turn_step * _DEG)
    if vf > 0.0 and vf * vf >= vv * (ch * ch):
        return dist, MOVE_FORWARD
    return dist, TURN_LEFT if vx * -si + vz * -co > 0.0 else TURN_RIGHT
