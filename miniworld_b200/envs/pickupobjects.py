"""MiniWorld-PickupObjects-v0: +1 per collected ball / box / key (reference envs/pickupobjects.py)."""
from .._gym import spaces, utils
from ..entity import COLOR_NAMES, Ball, Box, Key
from ..world import MiniWorldEnv


class PickupObjects(MiniWorldEnv, utils.EzPickle):
    def __init__(self, size=12, num_objs=5, **kwargs):
        assert size >= 2
        self.size = size
        self.num_objs = num_objs
        MiniWorldEnv.__init__(self, max_episode_steps=400, **kwargs)
        utils.EzPickle.__init__(self, size, num_objs, **kwargs)
        self.action_space = spaces.Discrete(self.actions.pickup + 1)

    @property
    def device_rule(self):
        return ("pickup", self.num_objs)

    @staticmethod
    def _make(kind, color):
        return (Ball(color=color, size=0.9), Box(color=color, size=0.9), Key(color=color))[kind]

    def _layout(self):
        return self.add_rect_room(min_x=0, max_x=self.size, min_z=0, max_z=self.size,
                                  wall_tex="brick_wall", floor_tex="asphalt", no_ceiling=True)

    def _gen_world(self):
        self._layout()
        for _ in range(self.num_objs):
            kind = self.np_random.choice(3)                 # Ball, Box, Key
            color = COLOR_NAMES[self.np_random.choice(len(COLOR_NAMES))]
            self.place_entity(self._make(kind, color))
        self.place_agent()
        self.num_picked_up = 0

    def device_program(self, prog):
        ncol = len(COLOR_NAMES)
        table = prog.proto_table([[self._make(k, c) for c in COLOR_NAMES] for k in range(3)])
        for k in range(self.num_objs):
            kind = prog.choice(3, label="kind of object %d (0 Ball, 1 Box, 2 Key)" % k)
            color = prog.choice(ncol, label="colour of object %d (index into COLOR_NAMES)" % k)
            prog.place(table, index=(kind, color))
        prog.place_agent()

    def step(self, action):
        obs, reward, termination, truncation, info = super().step(action)
        if self.agent.carrying:
            self.entities.remove(self.agent.carrying)
            self.agent.carrying = None
            self.num_picked_up += 1
            reward = 1
            if self.num_picked_up == self.num_objs:
                termination = True
        return obs, reward, termination, truncation, info
