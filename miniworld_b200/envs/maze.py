"""MiniWorld-Maze-v0 family: recursive-backtracker maze of 3x3 m cells (reference envs/maze.py)."""
import numpy as np

from .._gym import spaces, utils
from ..entity import Box
from ..params import DEFAULT_PARAMS
from ..world import MiniWorldEnv
from ._goal import GoalBoxRule


class Maze(GoalBoxRule, MiniWorldEnv, utils.EzPickle):
    def __init__(self, num_rows=8, num_cols=8, room_size=3, max_episode_steps=None, **kwargs):
        self.num_rows, self.num_cols = num_rows, num_cols
        self.room_size = room_size
        self.gap_size = 0.25
        MiniWorldEnv.__init__(self, max_episode_steps=max_episode_steps or num_rows * num_cols * 24, **kwargs)
        utils.EzPickle.__init__(self, num_rows=num_rows, num_cols=num_cols, room_size=room_size,
                                max_episode_steps=max_episode_steps, **kwargs)
        self.action_space = spaces.Discrete(self.actions.move_forward + 1)

    def _gen_world(self):
        """The recursive-backtracker carve, or with reset(options={"maze": ...}) a designed layout (_build_layout)."""
        pitch = self.room_size + self.gap_size
        grid = []
        for j in range(self.num_rows):
            row = []
            for i in range(self.num_cols):
                min_x, min_z = i * pitch, j * pitch
                row.append(self.add_rect_room(min_x=min_x, max_x=min_x + self.room_size,
                                              min_z=min_z, max_z=min_z + self.room_size,
                                              wall_tex="brick_wall"))
            grid.append(row)
        options = getattr(self, "reset_options", None) or {}
        if "maze" in options:
            self._build_layout(grid, options)
            return
        seen = set()

        def carve(i, j):
            cell = grid[j][i]
            seen.add(cell)
            remaining = [(0, 1), (0, -1), (-1, 0), (1, 0)]
            order = []
            while len(order) < 4:                      # shuffle by repeated choice (4 draws)
                pick = remaining[self._stream().choice(len(remaining))]   # a carve draw, not a reset draw
                remaining.remove(pick)
                order.append(pick)
            for dj, di in order:
                ni, nj = i + di, j + dj
                if not (0 <= nj < self.num_rows and 0 <= ni < self.num_cols):
                    continue
                other = grid[nj][ni]
                if other in seen:
                    continue
                if di == 0:
                    self.connect_rooms(cell, other, min_x=cell.min_x, max_x=cell.max_x)
                elif dj == 0:
                    self.connect_rooms(cell, other, min_z=cell.min_z, max_z=cell.max_z)
                carve(ni, nj)

        carve(0, 0)
        self.box = self.place_entity(Box(color="red"))
        self.place_agent()

    def _build_layout(self, grid, options):
        """The maze of a designed layout (options "maze": uint8 [rows, cols] or larger, bit 0 of cell (j, i) opening the
        wall to (j, i + 1), bit 1 the wall to (j + 1, i); cells and bits outside the grid are ignored) with the goal box
        in cell "goal_cell" and the agent in cell "agent_cell" (flat j * layout_cols + i; -1, absent or outside the grid:
        anywhere).  No carve draws; loops, isolated cells and unreachable goals are allowed."""
        layout = np.asarray(options["maze"])
        R, C = self.num_rows, self.num_cols
        for j in range(R):
            for i in range(C):
                cell, bits = grid[j][i], int(layout[j, i]) if j < layout.shape[0] and i < layout.shape[1] else 0
                if bits & 1 and i + 1 < C:
                    self.connect_rooms(cell, grid[j][i + 1], min_z=cell.min_z, max_z=cell.max_z)
                if bits & 2 and j + 1 < R:
                    self.connect_rooms(cell, grid[j + 1][i], min_x=cell.min_x, max_x=cell.max_x)

        def room_of(key):
            f = int(options.get(key, -1))
            j, i = divmod(f, layout.shape[1])
            return grid[j][i] if f >= 0 and j < R and i < C else None
        self.box = self.place_entity(Box(color="red"), room=room_of("goal_cell"))
        self.place_agent(room=room_of("agent_cell"))

    def device_program(self, prog):
        """Topology is random per episode: the carving itself is lowered (csrc/maze.cuh), using
        geometry templates that maze_lowering.MazeTemplate cuts out of host-built worlds."""
        prog.maze()
        prog.place(prog.proto(Box(color="red")))
        prog.place_agent()


class MazeS2(Maze):
    def __init__(self, num_rows=2, num_cols=2, **kwargs):
        Maze.__init__(self, num_rows=num_rows, num_cols=num_cols, **kwargs)


class MazeS3(Maze):
    def __init__(self, num_rows=3, num_cols=3, **kwargs):
        Maze.__init__(self, num_rows=num_rows, num_cols=num_cols, **kwargs)


fast_params = DEFAULT_PARAMS.no_random()
fast_params.set("forward_step", 0.7)
fast_params.set("turn_step", 45)


class MazeS3Fast(Maze):
    def __init__(self, num_rows=3, num_cols=3, max_episode_steps=300, params=fast_params,
                 domain_rand=False, **kwargs):
        Maze.__init__(self, num_rows=num_rows, num_cols=num_cols, max_episode_steps=max_episode_steps,
                      params=params, domain_rand=domain_rand, **kwargs)
