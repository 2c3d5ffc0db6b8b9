"""MiniWorld-PutNext-v0: carry the red box next to the yellow one (reference envs/putnext.py)."""
from .._gym import utils
from ..entity import COLOR_NAMES, Box
from ..world import MiniWorldEnv


class PutNext(MiniWorldEnv, utils.EzPickle):
    def __init__(self, size=12, **kwargs):
        assert size >= 2
        self.size = size
        MiniWorldEnv.__init__(self, max_episode_steps=250, **kwargs)
        utils.EzPickle.__init__(self, size, **kwargs)

    def _gen_world(self):
        self.add_rect_room(min_x=0, max_x=self.size, min_z=0, max_z=self.size)
        for color in COLOR_NAMES:
            box = self.place_entity(Box(color=color, size=self.np_random.uniform(0.6, 0.85)))
            if color == "red":
                self.red_box = box
            elif color == "yellow":
                self.yellow_box = box
        self.place_agent()

    @property
    def device_rule(self):
        return ("putnext", COLOR_NAMES.index("red") | (COLOR_NAMES.index("yellow") << 8))

    def device_program(self, prog):
        for color in COLOR_NAMES:
            size = prog.uniform(0.6, 0.85, label="size of the %s box" % color)   # drawn while the Box is constructed
            prog.place(prog.proto(Box(color=color, size=0.8)), size=size)
        prog.place_agent()

    def step(self, action):
        obs, reward, termination, truncation, info = super().step(action)
        if not self.agent.carrying and self.near(self.red_box, self.yellow_box):
            reward += self._reward()
            termination = True
        return obs, reward, termination, truncation, info
