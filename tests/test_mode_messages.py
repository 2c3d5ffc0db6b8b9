"""The exact refusals of every run-time mode, on the host build of the kernels: the libmwb error code and text of each
enable call (already on, after the state bank, on a host-reset handle, without what the mode needs), the "X is off"
text of every mode array, the mode names of a cross-mode restore, and the Python exceptions of BatchedMiniWorld's
accessors and constructor.  Other tests match these refusals by error code only."""
import numpy as np


def _refusal(call):
    try:
        call()
    except Exception as err:                      # noqa: BLE001 -- the type is part of what is pinned
        return "%s: %s" % (type(err).__name__, err)
    raise AssertionError("no refusal")


def _collect():
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import GOAL_GRID_DTYPE, Engine
    from miniworld_b200.envs import LEVELS
    got = {}
    host_only = type("HostOnlyRoom", (LEVELS["MiniWorld-OneRoom-v0"],), {"device_program": None})
    room, maze, pickup = "MiniWorld-OneRoom-v0", "MiniWorld-MazeS3-v0", "MiniWorld-PickupObjects-v0"
    table = ["MiniWorld-OneRoom-v0", "MiniWorld-FourRooms-v0"]
    worlds = ["MiniWorld-MazeS2-v0", "MiniWorld-OneRoom-v0"]

    def enables(env):
        e = env.engine
        grids = getattr(env, "goal_grids", None)
        if grids is None:
            grids = np.zeros(len(env.level_ids), GOAL_GRID_DTYPE)
            grids["goal_slot"] = -1
        return dict(level_changes=lambda: e.enable_level_changes(0, 0), episode_seeds=e.enable_episode_seeds,
                    maze_layouts=e.enable_maze_layouts, start_poses=e.enable_start_poses,
                    reset_draws=e.enable_reset_draws, goal_distance=lambda: e.enable_goal_distance(grids),
                    state_bank=lambda: e.enable_state_bank(2))

    # every enable call on a handle without the engine, a second time, after the state bank and on host resets
    env = BatchedMiniWorld(room, 2)
    lib = env.engine.lib
    for name, call in (("level_changes", lambda: lib.mwb_enable_level_changes(None, 0, 0)),
                       ("episode_seeds", lambda: lib.mwb_enable_episode_seeds(None)),
                       ("maze_layouts", lambda: lib.mwb_enable_maze_layouts(None)),
                       ("start_poses", lambda: lib.mwb_enable_start_poses(None)),
                       ("reset_draws", lambda: lib.mwb_enable_reset_draws(None)),
                       ("goal_distance", lambda: lib.mwb_enable_goal_distance(None, None)),
                       ("state_bank", lambda: lib.mwb_enable_state_bank(None, 2))):
        got["null handle: " + name] = "%d %s" % (call(), lib.mwb_last_error().decode())
    env.close()
    on = dict(level_changes=(table, dict(dynamic_levels=True)), episode_seeds=(room, dict(episode_seeds=True)),
              maze_layouts=(maze, dict(maze_layouts=True)), start_poses=(room, dict(start_poses=True)),
              reset_draws=(pickup, dict(reset_draws=True)), goal_distance=(room, dict(goal_distance=True)),
              state_bank=(room, dict(state_bank=2)))
    for name, (level, kw) in on.items():
        env = BatchedMiniWorld(level, 2, **kw)
        got["already on: " + name] = _refusal(enables(env)[name])
        env.close()
    for level in (room, maze, pickup):
        env = BatchedMiniWorld(level, 2, state_bank=2)
        for name, call in enables(env).items():
            if name not in ("goal_distance", "state_bank"):
                got["after the bank: %s: %s" % (level, name)] = _refusal(call)
        env.close()
    env = BatchedMiniWorld(host_only, 2)
    for name, call in enables(env).items():
        got["host resets: " + name] = _refusal(call)
    env.close()
    env = BatchedMiniWorld(room, 2)
    got["no Maze level"] = _refusal(env.engine.enable_maze_layouts)
    got["no draw"] = _refusal(env.engine.enable_reset_draws)
    got["no goal slot"] = _refusal(enables(env)["goal_distance"])
    got["no slots"] = _refusal(lambda: env.engine.enable_state_bank(0))

    # the arrays of every mode on a handle without it
    for name in Engine.ARRAYS:
        if Engine.ARRAYS[name][0] >= 6 and name != "level_params":
            got["array off: " + name] = _refusal(lambda: env.engine.state_array(name))
    host = BatchedMiniWorld(host_only, 2)
    got["array off: level_params"] = _refusal(lambda: host.engine.state_array("level_params"))

    # BatchedMiniWorld's accessors on a batch without the mode
    for name in ("level_tensor", "level_weights", "next_seed", "episode_seed", "next_maze", "next_maze_cells",
                 "maze_pending", "episode_maze", "next_pose", "next_agent_pose", "pose_pending", "episode_start",
                 "next_draws", "draws_pending", "episode_draws", "next_state", "episode_state", "bank_level",
                 "goal_dist", "expert_action", "episode_shortest", "goal_field", "grid_shape"):
        got["accessor: " + name] = _refusal(lambda: getattr(env, name))
    for name, call in (("set_level_weights", lambda: env.set_level_weights([1.0])),
                       ("set_env_level", lambda: env.set_env_level([0], 0)),
                       ("set_env_seed", lambda: env.set_env_seed([0], 1)),
                       ("set_env_maze", lambda: env.set_env_maze([0], np.zeros((3, 3), np.uint8))),
                       ("set_env_pose", lambda: env.set_env_pose([0], "agent", 1.0, 1.0)),
                       ("set_env_draws", lambda: env.set_env_draws([0], 0, 0.0)),
                       ("save_states", lambda: env.save_states([0], [0])),
                       ("set_env_state", lambda: env.set_env_state([0], 0)),
                       ("get_level_params", lambda: host.get_level_params(0)),
                       ("set_level_param", lambda: host.set_level_param(0, "forward_step", 0.1))):
        got["accessor: " + name] = _refusal(call)
    env.close()
    host.close()

    # the constructor's refusals
    for name, kw in (("episode_seeds", dict(episode_seeds=True)), ("maze_layouts", dict(maze_layouts=True)),
                     ("start_poses", dict(start_poses=True)), ("reset_draws", dict(reset_draws=True)),
                     ("goal_distance", dict(goal_distance=True)), ("state_bank", dict(state_bank=2)),
                     ("seeds and poses", dict(episode_seeds=True, start_poses=True))):
        got["host-reset batch: " + name] = _refusal(lambda: BatchedMiniWorld(host_only, 2, **kw))
    for name, level, kw in (("maze_layouts", room, dict(maze_layouts=True)), ("reset_draws", room, dict(reset_draws=True)),
                            ("goal_distance", pickup, dict(goal_distance=True)), ("state_bank", room, dict(state_bank=0)),
                            ("dynamic_levels", room, dict(dynamic_levels=True))):
        got["constructor: " + name] = _refusal(lambda: BatchedMiniWorld(level, 2, **kw))

    # the modes a snapshot names when it is restored into a handle with other modes
    pew = dict(per_env_worlds=True)
    for name, (level, kw) in list(on.items()) + [("worlds", (worlds, dict(pew, episode_seeds=True))),
                                                 ("worlds+levels", (worlds, dict(pew, dynamic_levels=True)))]:
        a, b = BatchedMiniWorld(level, 2, **kw), BatchedMiniWorld(level, 2, **(pew if level is worlds else {}))
        got["restore: " + name] = _refusal(lambda: b.restore(a.snapshot()))
        a.close()
        b.close()
    both = BatchedMiniWorld(room, 2, episode_seeds=True, start_poses=True, goal_distance=True, state_bank=2)
    plain = BatchedMiniWorld(room, 2)
    got["restore: several"] = _refusal(lambda: plain.restore(both.snapshot()))
    both.close()
    plain.close()
    return got


EXPECTED = {
    'null handle: level_changes': '-1 null handle',
    'null handle: episode_seeds': '-1 null handle',
    'null handle: maze_layouts': '-1 null handle',
    'null handle: start_poses': '-1 null handle',
    'null handle: reset_draws': '-1 null handle',
    'null handle: goal_distance': '-1 null handle',
    'null handle: state_bank': '-1 null handle',
    'already on: level_changes': 'EngineError: libmwb error -6: level changes are already on',
    'already on: episode_seeds': 'EngineError: libmwb error -6: episode seeds are already on',
    'already on: maze_layouts': 'EngineError: libmwb error -6: maze layouts are already on',
    'already on: start_poses': 'EngineError: libmwb error -6: start poses are already on',
    'already on: reset_draws': 'EngineError: libmwb error -6: reset draws are already on',
    'already on: goal_distance': 'EngineError: libmwb error -6: goal distance is already on',
    'already on: state_bank': 'EngineError: libmwb error -6: the state bank is already on',
    'after the bank: MiniWorld-OneRoom-v0: level_changes': 'EngineError: libmwb error -6: level changes cannot be '
                                                           'turned on once the state bank is on (its record layout '
                                                           'depends on it)',
    'after the bank: MiniWorld-OneRoom-v0: episode_seeds': 'EngineError: libmwb error -6: episode seeds cannot be '
                                                           'turned on once the state bank is on (its record layout '
                                                           'depends on it)',
    'after the bank: MiniWorld-OneRoom-v0: maze_layouts': 'EngineError: libmwb error -6: maze layouts cannot be '
                                                          'turned on once the state bank is on (its record layout '
                                                          'depends on it)',
    'after the bank: MiniWorld-OneRoom-v0: start_poses': 'EngineError: libmwb error -6: start poses cannot be turned '
                                                         'on once the state bank is on (its record layout depends on '
                                                         'it)',
    'after the bank: MiniWorld-OneRoom-v0: reset_draws': 'EngineError: libmwb error -6: reset draws cannot be turned '
                                                         'on once the state bank is on (its record layout depends on '
                                                         'it)',
    'after the bank: MiniWorld-MazeS3-v0: level_changes': 'EngineError: libmwb error -6: level changes need a level '
                                                          'table (mwb_set_levels first)',
    'after the bank: MiniWorld-MazeS3-v0: episode_seeds': 'EngineError: libmwb error -6: episode seeds cannot be '
                                                          'turned on once the state bank is on (its record layout '
                                                          'depends on it)',
    'after the bank: MiniWorld-MazeS3-v0: maze_layouts': 'EngineError: libmwb error -6: maze layouts cannot be turned '
                                                         'on once the state bank is on (its record layout depends on '
                                                         'it)',
    'after the bank: MiniWorld-MazeS3-v0: start_poses': 'EngineError: libmwb error -6: start poses cannot be turned '
                                                        'on once the state bank is on (its record layout depends on '
                                                        'it)',
    'after the bank: MiniWorld-MazeS3-v0: reset_draws': 'EngineError: libmwb error -6: reset draws cannot be turned '
                                                        'on once the state bank is on (its record layout depends on '
                                                        'it)',
    'after the bank: MiniWorld-PickupObjects-v0: level_changes': 'EngineError: libmwb error -6: level changes cannot '
                                                                 'be turned on once the state bank is on (its record '
                                                                 'layout depends on it)',
    'after the bank: MiniWorld-PickupObjects-v0: episode_seeds': 'EngineError: libmwb error -6: episode seeds cannot '
                                                                 'be turned on once the state bank is on (its record '
                                                                 'layout depends on it)',
    'after the bank: MiniWorld-PickupObjects-v0: maze_layouts': 'EngineError: libmwb error -6: maze layouts cannot be '
                                                                'turned on once the state bank is on (its record '
                                                                'layout depends on it)',
    'after the bank: MiniWorld-PickupObjects-v0: start_poses': 'EngineError: libmwb error -6: start poses cannot be '
                                                               'turned on once the state bank is on (its record '
                                                               'layout depends on it)',
    'after the bank: MiniWorld-PickupObjects-v0: reset_draws': 'EngineError: libmwb error -6: reset draws cannot be '
                                                               'turned on once the state bank is on (its record '
                                                               'layout depends on it)',
    'host resets: level_changes': 'EngineError: libmwb error -6: level changes need a level table (mwb_set_levels '
                                  'first)',
    'host resets: episode_seeds': 'EngineError: libmwb error -6: episode seeds need device resets (params and a reset '
                                  'program: mwb_set_levels, or mwb_set_params and mwb_set_program); host-generated '
                                  'worlds keep their streams on the host',
    'host resets: maze_layouts': 'EngineError: libmwb error -6: maze layouts need device resets (mwb_set_maze or '
                                 'mwb_set_level_maze on a handle with a reset program); host-generated worlds are '
                                 'built on the host',
    'host resets: start_poses': 'EngineError: libmwb error -6: start poses need device resets (params and a reset '
                                'program: mwb_set_levels, or mwb_set_params and mwb_set_program); host-generated '
                                'worlds are placed on the host',
    'host resets: reset_draws': 'EngineError: libmwb error -6: reset draws need device resets (params and a reset '
                                'program: mwb_set_levels, or mwb_set_params and mwb_set_program); host-generated '
                                'worlds draw on the host',
    'host resets: goal_distance': 'EngineError: libmwb error -6: goal distance needs device resets (params and a '
                                  'reset program: mwb_set_levels, or mwb_set_params and mwb_set_program); '
                                  'host-generated worlds arrive without a reset kernel',
    'host resets: state_bank': 'EngineError: libmwb error -6: the state bank needs device resets (params and a reset '
                               'program: mwb_set_levels, or mwb_set_params and mwb_set_program); host-generated '
                               'worlds are reset on the host',
    'no Maze level': 'EngineError: libmwb error -6: maze layouts need a Maze level (mwb_set_maze or '
                     'mwb_set_level_maze)',
    'no draw': 'EngineError: libmwb error -1: no level of this handle makes a reset draw (CHOICE / UNIFORM op)',
    'no goal slot': 'EngineError: libmwb error -1: no level of this handle has a goal slot',
    'no slots': 'EngineError: libmwb error -1: slots must be at least 1',
    'array off: env_level': 'EngineError: libmwb error -6: level changes are off (mwb_enable_level_changes)',
    'array off: next_level': 'EngineError: libmwb error -6: level changes are off (mwb_enable_level_changes)',
    'array off: level_weights': 'EngineError: libmwb error -6: level changes are off (mwb_enable_level_changes)',
    'array off: next_seed': 'EngineError: libmwb error -6: episode seeds are off (mwb_enable_episode_seeds)',
    'array off: episode_seed': 'EngineError: libmwb error -6: episode seeds are off (mwb_enable_episode_seeds)',
    'array off: next_maze': 'EngineError: libmwb error -6: maze layouts are off (mwb_enable_maze_layouts)',
    'array off: next_maze_cells': 'EngineError: libmwb error -6: maze layouts are off (mwb_enable_maze_layouts)',
    'array off: maze_pending': 'EngineError: libmwb error -6: maze layouts are off (mwb_enable_maze_layouts)',
    'array off: episode_maze': 'EngineError: libmwb error -6: maze layouts are off (mwb_enable_maze_layouts)',
    'array off: next_pose': 'EngineError: libmwb error -6: start poses are off (mwb_enable_start_poses)',
    'array off: next_agent_pose': 'EngineError: libmwb error -6: start poses are off (mwb_enable_start_poses)',
    'array off: pose_pending': 'EngineError: libmwb error -6: start poses are off (mwb_enable_start_poses)',
    'array off: episode_start': 'EngineError: libmwb error -6: start poses are off (mwb_enable_start_poses)',
    'array off: next_state': 'EngineError: libmwb error -6: the state bank is off (mwb_enable_state_bank)',
    'array off: episode_state': 'EngineError: libmwb error -6: the state bank is off (mwb_enable_state_bank)',
    'array off: bank_level': 'EngineError: libmwb error -6: the state bank is off (mwb_enable_state_bank)',
    'array off: next_draws': 'EngineError: libmwb error -6: reset draws are off (mwb_enable_reset_draws)',
    'array off: draws_pending': 'EngineError: libmwb error -6: reset draws are off (mwb_enable_reset_draws)',
    'array off: episode_draws': 'EngineError: libmwb error -6: reset draws are off (mwb_enable_reset_draws)',
    'array off: goal_dist': 'EngineError: libmwb error -6: goal distance is off (mwb_enable_goal_distance)',
    'array off: expert_action': 'EngineError: libmwb error -6: goal distance is off (mwb_enable_goal_distance)',
    'array off: episode_shortest': 'EngineError: libmwb error -6: goal distance is off (mwb_enable_goal_distance)',
    'array off: goal_field': 'EngineError: libmwb error -6: goal distance is off (mwb_enable_goal_distance)',
    'array off: level_params': 'EngineError: libmwb error -6: the handle has no device resets (params and a reset '
                               'program: mwb_set_levels, or mwb_set_params and mwb_set_program); host-generated '
                               'worlds carry their own draws',
    'accessor: level_tensor': 'RuntimeError: levels are fixed in this batch: construct it with dynamic_levels=True',
    'accessor: level_weights': 'RuntimeError: levels are fixed in this batch: construct it with dynamic_levels=True',
    'accessor: next_seed': 'RuntimeError: this batch has no episode seeds: construct it with episode_seeds=True',
    'accessor: episode_seed': 'RuntimeError: this batch has no episode seeds: construct it with episode_seeds=True',
    'accessor: next_maze': 'RuntimeError: this batch has no maze layouts: construct it with maze_layouts=True',
    'accessor: next_maze_cells': 'RuntimeError: this batch has no maze layouts: construct it with maze_layouts=True',
    'accessor: maze_pending': 'RuntimeError: this batch has no maze layouts: construct it with maze_layouts=True',
    'accessor: episode_maze': 'RuntimeError: this batch has no maze layouts: construct it with maze_layouts=True',
    'accessor: next_pose': 'RuntimeError: this batch has no start poses: construct it with start_poses=True',
    'accessor: next_agent_pose': 'RuntimeError: this batch has no start poses: construct it with start_poses=True',
    'accessor: pose_pending': 'RuntimeError: this batch has no start poses: construct it with start_poses=True',
    'accessor: episode_start': 'RuntimeError: this batch has no start poses: construct it with start_poses=True',
    'accessor: next_draws': 'RuntimeError: this batch has no reset draws: construct it with reset_draws=True',
    'accessor: draws_pending': 'RuntimeError: this batch has no reset draws: construct it with reset_draws=True',
    'accessor: episode_draws': 'RuntimeError: this batch has no reset draws: construct it with reset_draws=True',
    'accessor: next_state': 'RuntimeError: this batch has no state bank: construct it with state_bank=K',
    'accessor: episode_state': 'RuntimeError: this batch has no state bank: construct it with state_bank=K',
    'accessor: bank_level': 'RuntimeError: this batch has no state bank: construct it with state_bank=K',
    'accessor: goal_dist': 'RuntimeError: this batch has no goal distance: construct it with goal_distance=True',
    'accessor: expert_action': 'RuntimeError: this batch has no goal distance: construct it with goal_distance=True',
    'accessor: episode_shortest': 'RuntimeError: this batch has no goal distance: construct it with '
                                  'goal_distance=True',
    'accessor: goal_field': 'RuntimeError: this batch has no goal distance: construct it with goal_distance=True',
    'accessor: grid_shape': 'RuntimeError: this batch has no goal distance: construct it with goal_distance=True',
    'accessor: set_level_weights': 'RuntimeError: levels are fixed in this batch: construct it with '
                                   'dynamic_levels=True',
    'accessor: set_env_level': 'RuntimeError: levels are fixed in this batch: construct it with dynamic_levels=True',
    'accessor: set_env_seed': 'RuntimeError: this batch has no episode seeds: construct it with episode_seeds=True',
    'accessor: set_env_maze': 'RuntimeError: this batch has no maze layouts: construct it with maze_layouts=True',
    'accessor: set_env_pose': 'RuntimeError: this batch has no start poses: construct it with start_poses=True',
    'accessor: set_env_draws': 'RuntimeError: this batch has no reset draws: construct it with reset_draws=True',
    'accessor: save_states': 'RuntimeError: this batch has no state bank: construct it with state_bank=K',
    'accessor: set_env_state': 'RuntimeError: this batch has no state bank: construct it with state_bank=K',
    'accessor: get_level_params': 'TypeError: level params change at device resets; host-reset levels draw theirs in '
                                  "Python (set them on the level's own DomainParams)",
    'accessor: set_level_param': 'TypeError: level params change at device resets; host-reset levels draw theirs in '
                                 "Python (set them on the level's own DomainParams)",
    'host-reset batch: episode_seeds': 'TypeError: episode seeds are taken by device resets; host-reset levels keep '
                                       'RNG streams in Python',
    'host-reset batch: maze_layouts': 'ValueError: maze_layouts needs a Maze-family level in the batch',
    'host-reset batch: start_poses': 'TypeError: start poses are taken by device resets; host-reset levels place '
                                     'entities in Python (reset(options={"poses": ...}) of the level itself)',
    'host-reset batch: reset_draws': 'TypeError: reset draws are taken by device resets; host-reset levels draw in '
                                     'Python (reset(options={"draws": ...}) of the level itself)',
    'host-reset batch: goal_distance': 'TypeError: goal distance is built by device resets; host-reset levels build '
                                       'their worlds in Python (MiniWorldEnv.goal_distance() of the level itself)',
    'host-reset batch: state_bank': 'TypeError: the state bank loads states at device resets; host-reset levels keep '
                                    'their worlds and RNG streams in Python',
    'host-reset batch: seeds and poses': 'TypeError: episode seeds are taken by device resets; host-reset levels keep '
                                         'RNG streams in Python',
    'constructor: maze_layouts': 'ValueError: maze_layouts needs a Maze-family level in the batch',
    'constructor: reset_draws': 'ValueError: reset_draws needs a level with a reset draw; MiniWorld-OneRoom-v0 make '
                                'none',
    'constructor: goal_distance': 'ValueError: goal_distance needs a level with a goal rule; '
                                  'MiniWorld-PickupObjects-v0 have none',
    'constructor: state_bank': 'ValueError: state_bank is a number of slots >= 1, got 0',
    'constructor: dynamic_levels': 'ValueError: dynamic_levels moves envs between levels: pass `level` as a sequence '
                                   'of levels',
    'restore: level_changes': 'EngineError: libmwb error -6: snapshot of a handle with level changes on, no per-env '
                              'worlds, episode seeds off, maze layouts off, start poses off, state bank off, reset '
                              'draws off, goal distance off (this one has level changes off, no per-env worlds, '
                              'episode seeds off, maze layouts off, start poses off, state bank off, reset draws off, '
                              'goal distance off)',
    'restore: episode_seeds': 'EngineError: libmwb error -6: snapshot of a handle with level changes off, no per-env '
                              'worlds, episode seeds on, maze layouts off, start poses off, state bank off, reset '
                              'draws off, goal distance off (this one has level changes off, no per-env worlds, '
                              'episode seeds off, maze layouts off, start poses off, state bank off, reset draws off, '
                              'goal distance off)',
    'restore: maze_layouts': 'EngineError: libmwb error -6: snapshot of a handle with level changes off, no per-env '
                             'worlds, episode seeds off, maze layouts on, start poses off, state bank off, reset '
                             'draws off, goal distance off (this one has level changes off, no per-env worlds, '
                             'episode seeds off, maze layouts off, start poses off, state bank off, reset draws off, '
                             'goal distance off)',
    'restore: start_poses': 'EngineError: libmwb error -6: snapshot of a handle with level changes off, no per-env '
                            'worlds, episode seeds off, maze layouts off, start poses on, state bank off, reset draws '
                            'off, goal distance off (this one has level changes off, no per-env worlds, episode seeds '
                            'off, maze layouts off, start poses off, state bank off, reset draws off, goal distance '
                            'off)',
    'restore: reset_draws': 'EngineError: libmwb error -6: snapshot of a handle with level changes off, no per-env '
                            'worlds, episode seeds off, maze layouts off, start poses off, state bank off, reset '
                            'draws on, goal distance off (this one has level changes off, no per-env worlds, episode '
                            'seeds off, maze layouts off, start poses off, state bank off, reset draws off, goal '
                            'distance off)',
    'restore: goal_distance': 'EngineError: libmwb error -6: snapshot of a handle with level changes off, no per-env '
                              'worlds, episode seeds off, maze layouts off, start poses off, state bank off, reset '
                              'draws off, goal distance on (this one has level changes off, no per-env worlds, '
                              'episode seeds off, maze layouts off, start poses off, state bank off, reset draws off, '
                              'goal distance off)',
    'restore: state_bank': 'EngineError: libmwb error -6: snapshot of a handle with level changes off, no per-env '
                           'worlds, episode seeds off, maze layouts off, start poses off, state bank on, reset draws '
                           'off, goal distance off (this one has level changes off, no per-env worlds, episode seeds '
                           'off, maze layouts off, start poses off, state bank off, reset draws off, goal distance '
                           'off)',
    'restore: worlds': 'EngineError: libmwb error -6: snapshot of a handle with level changes off, per-env worlds, '
                       'episode seeds on, maze layouts off, start poses off, state bank off, reset draws off, goal '
                       'distance off (this one has level changes off, per-env worlds, episode seeds off, maze layouts '
                       'off, start poses off, state bank off, reset draws off, goal distance off)',
    'restore: worlds+levels': 'EngineError: libmwb error -6: snapshot of a handle with level changes on, per-env '
                              'worlds, episode seeds off, maze layouts off, start poses off, state bank off, reset '
                              'draws off, goal distance off (this one has level changes off, per-env worlds, episode '
                              'seeds off, maze layouts off, start poses off, state bank off, reset draws off, goal '
                              'distance off)',
    'restore: several': 'EngineError: libmwb error -6: snapshot of a handle with level changes off, no per-env '
                        'worlds, episode seeds on, maze layouts off, start poses on, state bank on, reset draws off, '
                        'goal distance on (this one has level changes off, no per-env worlds, episode seeds off, maze '
                        'layouts off, start poses off, state bank off, reset draws off, goal distance off)',
}


def test_mode_messages(hostsim_path):
    got = _collect()
    assert sorted(got) == sorted(EXPECTED)
    for key in EXPECTED:
        assert got[key] == EXPECTED[key], key
