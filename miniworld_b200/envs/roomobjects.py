"""MiniWorld-RoomObjects-v0: one room with a box, a ball and a key to look at and carry; no
reward, no time limit (reference envs/roomobjects.py)."""
import math

from .._gym import utils
from ..entity import COLOR_NAMES, Ball, Box, Key
from ..world import MiniWorldEnv


class RoomObjects(MiniWorldEnv, utils.EzPickle):
    def __init__(self, size=10, **kwargs):
        assert size >= 2
        self.size = size
        MiniWorldEnv.__init__(self, max_episode_steps=math.inf, **kwargs)
        utils.EzPickle.__init__(self, size, **kwargs)

    def _gen_world(self):
        self.add_rect_room(min_x=0, max_x=self.size, min_z=0, max_z=self.size, wall_tex="brick_wall",
                           floor_tex="asphalt", no_ceiling=True)
        self.agent.radius = 1.5          # keeps spawned objects far enough away to be seen
        pick = lambda: COLOR_NAMES[self.np_random.choice(len(COLOR_NAMES))]
        self.place_entity(Box(color=pick(), size=0.9))
        self.place_entity(Ball(color=pick(), size=0.9))
        self.place_entity(Key(color=pick()))
        self.place_agent()

    device_rule = ("none", 0)

    def device_program(self, prog):
        prog.set_agent(self.agent)                           # radius 1.5
        for name, make in (("Box", lambda c: Box(color=c, size=0.9)), ("Ball", lambda c: Ball(color=c, size=0.9)),
                           ("Key", lambda c: Key(color=c))):
            # drawn while the entity is constructed, before place_entity
            colour = prog.choice(len(COLOR_NAMES), label="colour of the %s (index into COLOR_NAMES)" % name)
            prog.place(prog.proto_row([make(c) for c in COLOR_NAMES]), index=colour)
        prog.place_agent()

    def step(self, action):
        return super().step(action)
