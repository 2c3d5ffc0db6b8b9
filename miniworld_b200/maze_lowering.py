"""Lowering of the Maze level's per-episode topology (reference envs/maze.py:73-153) for the
device-side reset kernel.

Maze worlds differ per episode only in WHICH neighbouring cells are connected; every piece of
geometry is a translate of a few templates: one grid cell (floor, ceiling, four walls) and one
connector room per direction.  The templates are not re-derived by hand: they are cut out of
worlds built by the host-side `connect_rooms` / `_gen_static_data` code (which is
bit-identical to the reference), and `verify()` checks that translating them reproduces a
full host-generated maze exactly.  With the default sizes (3 m cells, 0.25 m gaps) every
coordinate is a multiple of 0.25, so translation is exact in float64 and float32.
"""
import numpy as np

from . import pack
from .engine import QUAD_DTYPE, ROOM_DTYPE, SEG_DTYPE

# neighbour order of envs/maze.py: orders = [(0, 1), (0, -1), (-1, 0), (1, 0)] as (dj, di)
DIRS = [(0, 1), (0, -1), (-1, 0), (1, 0)]


def _shift_room(rec, dx, dz):
    r = rec.copy()
    for k in ("min_x", "max_x"):
        r[k] += dx
    for k in ("min_z", "max_z"):
        r[k] += dz
    n = int(r["num_edges"])
    r["edge_px"][:n] += dx
    r["edge_pz"][:n] += dz
    return r


def _shift_quad(q, dx, dz, floor_like):
    o = q.copy()
    nv = int(o["num_verts"])
    o["pos"][:nv, 0] += np.float32(dx)
    o["pos"][:nv, 2] += np.float32(dz)
    if floor_like:                       # floor / ceiling texcoords are world (x, z)
        o["uvm"][:nv, 0] += dx
        o["uvm"][:nv, 1] += dz
    return o


def _shift_seg(s, dx, dz):
    o = s.copy()
    o["ax"] += dx
    o["bx"] += dx
    o["az"] += dz
    o["bz"] += dz
    return o


class MazeTemplate:
    def __init__(self, level_cls, **kwargs):
        probe = level_cls(device=None, **kwargs)
        self.rows, self.cols = probe.num_rows, probe.num_cols
        self.pitch = float(probe.room_size + probe.gap_size)
        self.level_cls, self.kwargs = level_cls, kwargs
        mk = lambda: level_cls.__new__(level_cls)

        def blank():
            e = mk()
            e.__dict__.update(probe.__dict__)
            e.rooms, e.entities, e.wall_segs = [], [], []
            return e

        def cell(env, i, j):
            x, z = i * self.pitch, j * self.pitch
            return env.add_rect_room(min_x=x, max_x=x + probe.room_size, min_z=z, max_z=z + probe.room_size,
                                     wall_tex="brick_wall")

        # an isolated cell: floor, ceiling, 4 walls
        env = blank()
        cell(env, 0, 0)
        env._gen_static_data()
        rooms, quads, segs = pack.pack_geometry(env)
        assert len(quads) == 6 and len(segs) == 4
        self.cell_room, self.cell_quads, self.cell_segs = rooms[0], quads, segs
        # one connection per direction: which walls open, and the connector room
        self.open_a, self.open_b, self.conn = [], [], []
        for dj, di in DIRS:
            env = blank()
            a = cell(env, 0, 0)
            b = cell(env, di, dj)
            if di == 0:
                env.connect_rooms(a, b, min_x=a.min_x, max_x=a.max_x)
            else:
                env.connect_rooms(a, b, min_z=a.min_z, max_z=a.max_z)
            assert len(env.rooms) == 3
            env._gen_static_data()
            rooms, quads, segs = pack.pack_geometry(env)
            open_a = [e for e in range(4) if len(env.rooms[0].portals[e])]
            open_b = [e for e in range(4) if len(env.rooms[1].portals[e])]
            assert len(open_a) == 1 and len(open_b) == 1
            self.open_a.append(open_a[0])
            self.open_b.append(open_b[0])
            cq = quads[quads["room"] == 2]
            assert len(cq) == 4 and len(segs) == 3 + 3 + 2
            self.conn.append((rooms[2], cq, segs[6:]))
        self.num_rooms = 2 * self.rows * self.cols - 1
        # pick probabilities: grid rooms first, then the rows*cols - 1 connectors (list order is fixed)
        areas = np.array([float(self.cell_room["max_x"] - self.cell_room["min_x"]) *
                          float(self.cell_room["max_z"] - self.cell_room["min_z"])] * (self.rows * self.cols) +
                         [None] * (self.rows * self.cols - 1), dtype=object)
        self._cell_area = areas[0]

    # ---- reference construction on the host (for verify()): rebuild a world from its topology
    def assemble(self, connections):
        """connections: list of (i, j, dir_index) in creation order -> (rooms, quads, segs)."""
        R, C, p = self.rows, self.cols, self.pitch
        opened = np.zeros((R, C, 4), bool)
        for i, j, d in connections:
            dj, di = DIRS[d]
            opened[j, i, self.open_a[d]] = True
            opened[j + dj, i + di, self.open_b[d]] = True
        rooms, quads, segs = [], [], []
        for j in range(R):
            for i in range(C):
                dx, dz = i * p, j * p
                ri = len(rooms)
                rooms.append(_shift_room(self.cell_room, dx, dz))
                for q in self.cell_quads[:2]:
                    qq = _shift_quad(q, dx, dz, True)
                    qq["room"] = ri
                    quads.append(qq)
                for e in range(4):
                    if not opened[j, i, e]:
                        qq = _shift_quad(self.cell_quads[2 + e], dx, dz, False)
                        qq["room"] = ri
                        quads.append(qq)
                        segs.append(_shift_seg(self.cell_segs[e], dx, dz))
        for i, j, d in connections:
            dx, dz = i * p, j * p
            room, cq, cs = self.conn[d]
            ri = len(rooms)
            rooms.append(_shift_room(room, dx, dz))
            for k, q in enumerate(cq):
                qq = _shift_quad(q, dx, dz, k < 2)
                qq["room"] = ri
                quads.append(qq)
            segs.extend(_shift_seg(s, dx, dz) for s in cs)
        return np.array(rooms, ROOM_DTYPE), np.array(quads, QUAD_DTYPE), np.array(segs, SEG_DTYPE)

    def topology_of(self, env):
        """Connections (i, j, dir) in creation order, read back from a host-generated maze."""
        R, C, p = self.rows, self.cols, self.pitch
        out = []
        for room in env.rooms[R * C:]:
            cx, cz = float(room.mid_x), float(room.mid_z)
            best = None
            for d, (dj, di) in enumerate(DIRS):
                tr = self.conn[d][0]
                tx = (float(tr["min_x"]) + float(tr["max_x"])) / 2
                tz = (float(tr["min_z"]) + float(tr["max_z"])) / 2
                i, j = (cx - tx) / p, (cz - tz) / p
                if abs(i - round(i)) < 1e-9 and abs(j - round(j)) < 1e-9:
                    # the connector's first outline vertex tells a (cell, +1) from the neighbour's (cell, -1)
                    sh = _shift_room(tr, round(i) * p, round(j) * p)
                    if np.array_equal(sh["edge_px"][:4], room.outline[:, 0]) and np.array_equal(sh["edge_pz"][:4], room.outline[:, 2]):
                        best = (int(round(i)), int(round(j)), d)
            assert best is not None, "connector does not match any template"
            out.append(best)
        return out

    def layout_of(self, connections):
        """uint8 [rows, cols] layout (bit 0: wall to (j, i + 1) open, bit 1: wall to (j + 1, i) open) of connections
        (i, j, dir): a connector in direction d opens the +x or +z bit of the cell on its -x / -z side."""
        out = np.zeros((self.rows, self.cols), np.uint8)
        for i, j, d in connections:
            dj, di = DIRS[d]
            if dj == 0:
                out[j, min(i, i + di)] |= 1
            else:
                out[min(j, j + dj), i] |= 2
        return out

    def layout_connections(self, layout):
        """The connections a designed reset creates from `layout`, in its order: per cell in row-major order, +x
        (template direction 0), then +z (direction 3); bits that point outside the grid are ignored."""
        out = []
        for j in range(self.rows):
            for i in range(self.cols):
                bits = int(layout[j, i])
                if bits & 1 and i + 1 < self.cols:
                    out.append((i, j, 0))
                if bits & 2 and j + 1 < self.rows:
                    out.append((i, j, 3))
        return out

    def verify_layouts(self, layouts):
        """Assembling the canonical connections of each layout reproduces the world the host builds from it
        (Maze.reset(options={"maze": layout})) field for field."""
        for layout in layouts:
            env = self.level_cls(device=None, **self.kwargs)
            env.reset(seed=0, options={"maze": layout})
            want = pack.pack_geometry(env)
            got = self.assemble(self.layout_connections(layout))
            for w, g, name in zip(want, got, ("rooms", "quads", "segs")):
                assert len(w) == len(g), (name, len(w), len(g))
                for field in w.dtype.names:
                    if field in ("cdf", "reserved"):
                        continue
                    assert np.array_equal(w[field], g[field]), (name, field)
        return True

    def verify(self, seeds=(0, 1, 2)):
        """Translating the templates reproduces host-generated mazes field for field."""
        for seed in seeds:
            env = self.level_cls(device=None, **self.kwargs)
            env.reset(seed=seed)
            want = pack.pack_geometry(env)
            got = self.assemble(self.topology_of(env))
            for w, g, name in zip(want, got, ("rooms", "quads", "segs")):
                assert len(w) == len(g), (name, len(w), len(g))
                for field in w.dtype.names:
                    if field in ("cdf", "reserved"):
                        continue
                    assert np.array_equal(w[field], g[field]), (name, field, seed)
        return True
