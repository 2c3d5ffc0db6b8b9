"""MiniWorld-YMaze-v0 / -YMazeLeft-v0 / -YMazeRight-v0: three arms around a triangular hub
(non-rectangular rooms; reference envs/ymaze.py)."""
import math

import numpy as np

from .._gym import spaces, utils
from ..entity import Box
from ..math import gen_rot_matrix
from ..world import MiniWorldEnv


class YMaze(MiniWorldEnv, utils.EzPickle):
    def __init__(self, goal_pos=None, **kwargs):
        self.goal_pos = goal_pos
        MiniWorldEnv.__init__(self, max_episode_steps=280, **kwargs)
        utils.EzPickle.__init__(self, goal_pos, **kwargs)
        self.action_space = spaces.Discrete(self.actions.move_forward + 1)

    def _gen_world(self):
        arm = np.array([[-9.15, 0, -2], [-9.15, 0, +2], [-1.15, 0, +2], [-1.15, 0, -2]])
        xz = lambda pts: np.delete(pts, 1, 1)
        main_arm = self.add_room(outline=xz(arm))
        hub = self.add_room(outline=np.array([[-1.15, -2], [-1.15, +2], [2.31, 0]]))
        turn = lambda deg: np.dot(arm, gen_rot_matrix(np.array([0, 1, 0]), deg * (math.pi / 180)))
        left_arm = self.add_room(outline=xz(turn(-120)))
        right_arm = self.add_room(outline=xz(turn(+120)))
        self.connect_rooms(main_arm, hub, min_z=-2, max_z=2)
        self.connect_rooms(left_arm, hub, min_z=-1.995, max_z=0)
        self.connect_rooms(right_arm, hub, min_z=0, max_z=1.995)
        self.box = Box(color="red")
        if self.goal_pos is not None:
            gx, _, gz = self.goal_pos
            self.place_entity(self.box, min_x=gx, max_x=gx, min_z=gz, max_z=gz)
        elif self.np_random.integers(0, 2) == 0:
            self.place_entity(self.box, room=left_arm, max_z=left_arm.min_z + 2.5)
        else:
            self.place_entity(self.box, room=right_arm, min_z=right_arm.max_z - 2.5)
        heading = self.np_random.uniform(-math.pi / 4, math.pi / 4)
        self.place_agent(dir=heading, room=main_arm)

    device_rule = ("goal", 0)

    def device_program(self, prog):
        left_arm, right_arm = self.rooms[2], self.rooms[3]     # add_room order: main arm, hub, left, right
        box = prog.proto(Box(color="red"))
        if self.goal_pos is not None:
            gx, _, gz = self.goal_pos
            prog.place(box, min_x=gx, max_x=gx, min_z=gz, max_z=gz)
        else:
            side = prog.choice(2, label="goal side (0: left arm, 1: right arm)")
            prog.place(box, room=2, max_z=left_arm.min_z + 2.5, when=(side, 0))
            prog.place(box, room=3, min_z=right_arm.max_z - 2.5, when=(side, 1), same_slot=True)
        heading = prog.uniform(-math.pi / 4, math.pi / 4, label="agent heading")
        prog.place_agent(dir=heading, room=0)

    def step(self, action):
        obs, reward, termination, truncation, info = super().step(action)
        if self.near(self.box):
            reward += self._reward()
            termination = True
        info["goal_pos"] = self.box.pos
        return obs, reward, termination, truncation, info


class YMazeLeft(YMaze):
    def __init__(self, goal_pos=[3.9, 0, -7.0], **kwargs):
        super().__init__(goal_pos=goal_pos, **kwargs)


class YMazeRight(YMaze):
    def __init__(self, goal_pos=[3.9, 0, 7.0], **kwargs):
        super().__init__(goal_pos=goal_pos, **kwargs)
