"""Builder for the device-side reset program (include/mwb.h: mwb_op).

A level's `device_program(prog)` re-states its `_gen_world()` placement calls against this
builder; the result is the short CHOICE / UNIFORM / PLACE program csrc/reset.cuh interprets
per environment on the GPU, drawing from that env's numpy-exact PCG64 stream in the same
order as the Python `_gen_world()` does (reference miniworld.py:839-909).
`tests/test_hostsim_kernels.py` (CPU) and `tests/test_gpu_physics.py` (GPU) check every level's program against its `_gen_world()`.
"""
import math

import numpy as np

from .engine import OP_CHOICE, OP_DTYPE, OP_IFEQ, OP_MAZE, OP_PLACE, OP_PUT, OP_UNIFORM, PROTO_DTYPE
from .entity import Agent
from .pack import proto_record


class _Reg:
    def __init__(self, index):
        self.index = index


class ProtoTable:
    def __init__(self, base, strides, size):
        self.base, self.strides, self.size = base, strides, size


class ResetProgram:
    def __init__(self):
        self.ops = []
        self.protos = []
        self.proto_kinds = []          # class name of each prototype's entity
        self.slots = []                # (kind, is_agent, takes a designed pose) of each entity-list slot the reset fills
        self.draws = []                # spec of each reset draw (CHOICE / UNIFORM op), in program order
        self._ireg = 0
        self._freg = 0
        self.agent_proto = self.proto(Agent())
        self.num_placed = 0
        self.uses_maze = False

    # ---- prototypes
    def proto(self, ent):
        self.protos.append(proto_record(ent))
        self.proto_kinds.append(type(ent).__name__)
        return len(self.protos) - 1

    def _fill_slot(self, proto, agent, designable):
        """Record the slot the next placement fills (the branches of one `if` fill one slot: recorded once)."""
        if self.num_placed < len(self.slots):
            return
        if isinstance(proto, ProtoTable):
            kind = "/".join(sorted(set(self.proto_kinds[proto.base:proto.base + proto.size])))
        else:
            kind = self.proto_kinds[int(proto)]
        self.slots.append((kind, bool(agent), bool(designable)))

    def set_agent(self, agent):
        """The level changes the agent's physical constants (RoomObjects: `self.agent.radius = 1.5`)."""
        self.protos[self.agent_proto] = proto_record(agent)

    def proto_row(self, ents):
        """1-D table of entities indexed by one CHOICE result."""
        base = len(self.protos)
        for ent in ents:
            self.proto(ent)
        return ProtoTable(base, (1, 0), len(ents))

    def proto_table(self, nested):
        """2-D table of entities indexed by two CHOICE results."""
        base = len(self.protos)
        rows, cols = len(nested), len(nested[0])
        for row in nested:
            assert len(row) == cols
            for ent in row:
                self.proto(ent)
        return ProtoTable(base, (cols, 1), rows * cols)

    # ---- per-episode topology
    def maze(self):
        """Maze._gen_world()'s room carving runs on the device (csrc/maze.cuh)."""
        op = np.zeros((), OP_DTYPE)
        op["op"] = OP_MAZE
        self.ops.append(op)
        self.uses_maze = True

    # ---- random draws
    def _draw(self, op, spec, label):
        """Number reset draw `op` (its index in `room`, mwb_enable_reset_draws) and keep its spec."""
        op["room"] = len(self.draws)
        self.draws.append(dict(index=len(self.draws), **spec, label=label))
        self.ops.append(op)

    def choice(self, n, label=None):
        op = np.zeros((), OP_DTYPE)
        op["op"], op["a"], op["b"] = OP_CHOICE, self._ireg, int(n)
        self._draw(op, dict(kind="choice", n=int(n)), label)
        self._ireg += 1
        assert self._ireg <= 8
        return _Reg(self._ireg - 1)

    def uniform(self, lo, hi, label=None):
        op = np.zeros((), OP_DTYPE)
        op["op"], op["a"] = OP_UNIFORM, self._freg
        op["f"][:2] = (float(lo), float(hi))
        self._draw(op, dict(kind="uniform", lo=float(lo), hi=float(hi)), label)
        self._freg += 1
        assert self._freg <= 8
        return _Reg(self._freg - 1)

    # ---- placement
    def put(self, proto, pos, dir=None, append_only=False):
        """place_entity(ent, pos=pos, dir=dir): no search; dir=None draws uniform(-pi, pi).  append_only: a bare
        `self.entities.append(ent)` (does not trigger the static-data texture draws)."""
        op = np.zeros((), OP_DTYPE)
        op["op"], op["a"], op["b"] = OP_PUT, int(proto), int(append_only)
        op["f"] = [float(pos[0]), float(pos[1]), float(pos[2]), math.nan if dir is None else float(dir)]
        self.ops.append(op)
        self._fill_slot(proto, False, not append_only)
        self.num_placed += 1
        return self.num_placed - 1

    def place(self, proto, index=None, room=None, dir=None, min_x=None, max_x=None, min_z=None, max_z=None,
              when=None, same_slot=False, size=None, _agent=False):
        """place_entity(...).  when=(reg, value): the call sits in an `if reg == value:` branch of _gen_world();
        the other branches are stated with further place(..., when=..., same_slot=True) calls -- exactly one of
        them runs per reset and fills the one entity slot."""
        if when is not None:
            cond = np.zeros((), OP_DTYPE)
            cond["op"], cond["a"], cond["b"] = OP_IFEQ, when[0].index, int(when[1])
            self.ops.append(cond)
        if same_slot:
            self.num_placed -= 1
        self._fill_slot(proto, _agent, True)
        op = np.zeros((), OP_DTYPE)
        op["op"] = OP_PLACE
        op["ireg_a"] = op["ireg_b"] = -1
        if isinstance(proto, ProtoTable):
            op["a"] = proto.base
            ia, ib = index if isinstance(index, (tuple, list)) else (index, None)
            op["ireg_a"], op["stride_a"] = ia.index, proto.strides[0]
            if ib is not None:
                op["ireg_b"], op["stride_b"] = ib.index, proto.strides[1]
        else:
            op["a"] = int(proto)
        if size is not None:           # Box(size=<a value drawn for this episode>): overrides the prototype's size
            op["b"] = 1 + size.index
        op["room"] = -1 if room is None else int(room)
        op["dir_freg"] = -1 if dir is None else dir.index
        op["is_agent"] = int(_agent)
        op["f"] = [math.nan if v is None else float(v) for v in (min_x, max_x, min_z, max_z)]
        self.ops.append(op)
        # reset registers are per-program-run, but CHOICE results feeding a PLACE are dead after it
        if isinstance(proto, ProtoTable):
            self._ireg = 0
        self.num_placed += 1
        return self.num_placed - 1

    def place_agent(self, **kw):
        return self.place(self.agent_proto, _agent=True, **kw)

    # ---- output
    def op_array(self):
        return np.array(self.ops, OP_DTYPE)

    def proto_array(self):
        return np.array(self.protos, PROTO_DTYPE)
