"""MiniWorld-TMaze-v0 / -TMazeLeft-v0 / -TMazeRight-v0: corridor into a cross arm, red box at
one end (reference envs/tmaze.py)."""
import math

from .._gym import spaces, utils
from ..entity import Box
from ..world import MiniWorldEnv


class TMaze(MiniWorldEnv, utils.EzPickle):
    def __init__(self, goal_pos=None, **kwargs):
        self.goal_pos = goal_pos
        MiniWorldEnv.__init__(self, max_episode_steps=280, **kwargs)
        utils.EzPickle.__init__(self, goal_pos, **kwargs)
        self.action_space = spaces.Discrete(self.actions.move_forward + 1)

    def _gen_world(self):
        stem = self.add_rect_room(min_x=-1, max_x=8, min_z=-2, max_z=2)
        bar = self.add_rect_room(min_x=8, max_x=12, min_z=-8, max_z=8)
        self.connect_rooms(stem, bar, min_z=-2, max_z=2)
        self.box = Box(color="red")
        if self.goal_pos is not None:
            gx, _, gz = self.goal_pos
            self.place_entity(self.box, min_x=gx, max_x=gx, min_z=gz, max_z=gz)
        elif self.np_random.integers(0, 2) == 0:
            self.place_entity(self.box, room=bar, max_z=bar.min_z + 2)
        else:
            self.place_entity(self.box, room=bar, min_z=bar.max_z - 2)
        heading = self.np_random.uniform(-math.pi / 4, math.pi / 4)
        self.place_agent(dir=heading, room=stem)

    device_rule = ("goal", 0)
    device_info = {"goal_pos": ("entity_pos", 0)}      # info["goal_pos"] = self.box.pos: the box is entity 0

    def device_program(self, prog):
        stem, bar = self.rooms[0], self.rooms[1]
        box = prog.proto(Box(color="red"))
        if self.goal_pos is not None:
            gx, _, gz = self.goal_pos
            prog.place(box, min_x=gx, max_x=gx, min_z=gz, max_z=gz)
        else:
            side = prog.choice(2, label="goal side (0: -z arm, 1: +z arm)")
            prog.place(box, room=1, max_z=bar.min_z + 2, when=(side, 0))
            prog.place(box, room=1, min_z=bar.max_z - 2, when=(side, 1), same_slot=True)
        heading = prog.uniform(-math.pi / 4, math.pi / 4, label="agent heading")
        prog.place_agent(dir=heading, room=0)

    def step(self, action):
        obs, reward, termination, truncation, info = super().step(action)
        if self.near(self.box):
            reward += self._reward()
            termination = True
        info["goal_pos"] = self.box.pos
        return obs, reward, termination, truncation, info


class TMazeLeft(TMaze):
    def __init__(self, goal_pos=[10, 0, -6], **kwargs):
        super().__init__(goal_pos=goal_pos, **kwargs)


class TMazeRight(TMaze):
    def __init__(self, goal_pos=[10, 0, 6], **kwargs):
        super().__init__(goal_pos=goal_pos, **kwargs)
