"""MiniWorld-Hallway-v0: red box at the far end of a corridor (reference envs/hallway.py)."""
import math

from .._gym import spaces, utils
from ..entity import Box
from ..world import MiniWorldEnv
from ._goal import GoalBoxRule


class Hallway(GoalBoxRule, MiniWorldEnv, utils.EzPickle):
    def __init__(self, length=12, **kwargs):
        assert length >= 2
        self.length = length
        MiniWorldEnv.__init__(self, max_episode_steps=250, **kwargs)
        utils.EzPickle.__init__(self, length, **kwargs)
        self.action_space = spaces.Discrete(self.actions.move_forward + 1)

    def _layout(self):
        return self.add_rect_room(min_x=-1, max_x=-1 + self.length, min_z=-2, max_z=2)

    def _gen_world(self):
        room = self._layout()
        self.box = self.place_entity(Box(color="red"), min_x=room.max_x - 2)
        heading = self.np_random.uniform(-math.pi / 4, math.pi / 4)
        self.place_agent(dir=heading, max_x=room.max_x - 2)

    def device_program(self, prog):
        room = self.rooms[0]
        prog.place(prog.proto(Box(color="red")), min_x=room.max_x - 2)
        heading = prog.uniform(-math.pi / 4, math.pi / 4, label="agent heading")
        prog.place_agent(dir=heading, max_x=room.max_x - 2)
