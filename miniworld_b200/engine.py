"""ctypes binding of libmwb.so (include/mwb.h) -- the only way into the CUDA kernels.

There is no fallback: if the shared library is missing, or CUDA is unavailable when a
handle is created, construction raises.  The package only ever loads `libmwb.so` from its
own directory and no product class takes a library argument (tests reach the g++ build of
the kernels' inner functions through the private `_override_library_for_tests` seam).
"""
import ctypes as C
import os

import numpy as np

ABI_VERSION = 10
RULE_NONE, RULE_GOAL, RULE_PICKUP, RULE_SIDEWALK, RULE_SIGN, RULE_HEALTH, RULE_PUTNEXT = 0, 1, 2, 3, 4, 5, 6
SURF_WALL, SURF_FLOOR, SURF_CEIL = 0, 1, 2
OP_END, OP_CHOICE, OP_UNIFORM, OP_PLACE, OP_MAZE, OP_IFEQ, OP_PUT = 0, 1, 2, 3, 4, 5, 6
MAX_EDGES = 8
MAX_ENTS_CAP = 32
LEVEL_CAP = 32
MAX_OPS = 64

_HERE = os.path.dirname(os.path.abspath(__file__))
DEFAULT_LIB = os.path.join(_HERE, "libmwb.so")


class EngineError(RuntimeError):
    pass


# --------------------------------------------------------------------- struct mirrors

class Config(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "abi_version", "device", "num_envs", "obs_width", "obs_height", "msaa_samples",
        "shared_geometry", "max_rooms", "max_quads", "max_segs", "max_ents", "rule_kind",
        "rule_arg", "domain_rand", "max_episode_steps", "autoreset")] + [("reserved", C.c_int32 * 4)]


_VEC_PARAMS = ("sky_color", "light_pos", "light_color", "light_ambient", "obj_color_bias")
_SCALAR_PARAMS = ("forward_step", "forward_drift", "turn_step", "cam_pitch", "cam_fov_y",
                  "cam_height", "cam_fwd_disp")


class Params(C.Structure):
    _fields_ = ([(n + s, C.c_double * 3) for n in _VEC_PARAMS for s in ("", "_lo", "_rng")] +
                [(n + s, C.c_double) for n in _SCALAR_PARAMS for s in ("", "_lo", "_rng")] +
                [("max_forward_step", C.c_double)])


LOWERED_PARAMS = _VEC_PARAMS + _SCALAR_PARAMS     # the DomainParams entries the engine reads
# element rows of an env params row (mwb_enable_env_params): param name -> its row index, or a slice of three rows
ENV_PARAM_ROWS = dict([(n, slice(3 * k, 3 * k + 3)) for k, n in enumerate(_VEC_PARAMS)] +
                      [(n, 15 + k) for k, n in enumerate(_SCALAR_PARAMS)])
ENV_PARAM_ELEMS = 22
PARAMS_DOUBLES = C.sizeof(Params) // 8
# field of mwb_params -> its column in a float64 view of the params table
PARAMS_COLUMN = {name: getattr(Params, name).offset // 8 for name, _ in Params._fields_}


class TexDesc(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("offset", C.c_int64)]


class MeshDesc(C.Structure):
    _fields_ = [("num_tris", C.c_int32), ("reserved", C.c_int32), ("offset", C.c_int64)]


ROOM_DTYPE = np.dtype([
    ("min_x", "f8"), ("max_x", "f8"), ("min_z", "f8"), ("max_z", "f8"), ("cdf", "f8"),
    ("edge_px", "f8", MAX_EDGES), ("edge_pz", "f8", MAX_EDGES),
    ("edge_nx", "f8", MAX_EDGES), ("edge_nz", "f8", MAX_EDGES),
    ("num_edges", "i4"), ("tex_first", "i4", 3), ("tex_count", "i4", 3), ("tex_id", "i4", 3),
    ("reserved", "i4")], align=True)
QUAD_DTYPE = np.dtype([
    ("pos", "f4", (4, 3)), ("nrm", "f4", 3), ("room", "i4"), ("surf", "i4"), ("num_verts", "i4"),
    ("uvm", "f8", (4, 2))], align=True)
SEG_DTYPE = np.dtype([("ax", "f8"), ("az", "f8"), ("bx", "f8"), ("bz", "f8")], align=True)
PROTO_DTYPE = np.dtype([
    ("kind", "i4"), ("is_static", "i4"), ("mesh_id", "i4"), ("radius_is_f32", "i4"),
    ("radius", "f8"), ("height", "f8"), ("size", "f8", 3), ("color", "f8", 3),
    ("scale", "f4"), ("deg_form", "i4")], align=True)
ENTITY_DTYPE = np.dtype([
    ("proto", "i4"), ("reserved", "i4"), ("pos", "f8", 3), ("dir", "f8"), ("color", "f8", 3)], align=True)
OP_DTYPE = np.dtype([
    ("op", "i4"), ("a", "i4"), ("b", "i4"), ("ireg_a", "i4"), ("stride_a", "i4"), ("ireg_b", "i4"),
    ("stride_b", "i4"), ("room", "i4"), ("dir_freg", "i4"), ("is_agent", "i4"), ("f", "f8", 4)], align=True)
# mwb_goal_grid (mwb_enable_goal_distance): one level's grid and goal slot (-1 = no goal rule)
GOAL_GRID_DTYPE = np.dtype([("min_x", "<f8"), ("min_z", "<f8"), ("nx", "<i4"), ("nz", "<i4"), ("goal_slot", "<i4"),
                            ("reserved", "<i4")])
GOAL_GRID_STEP = 0.25
GOAL_GRID_CAP = 65536
RNG_DTYPE = np.dtype([
    ("state_hi", "u8"), ("state_lo", "u8"), ("inc_hi", "u8"), ("inc_lo", "u8"),
    ("has_uint32", "i4"), ("uinteger", "u4")], align=True)


class Geometry(C.Structure):
    _fields_ = [("num_rooms", C.c_int32), ("num_quads", C.c_int32), ("num_segs", C.c_int32),
                ("reserved", C.c_int32), ("rooms", C.c_void_p), ("quads", C.c_void_p), ("segs", C.c_void_p)]


class World(C.Structure):
    _fields_ = [("geom", Geometry), ("num_slots", C.c_int32), ("agent_slot", C.c_int32),
                ("carrying", C.c_int32), ("step_count", C.c_int32), ("num_picked_up", C.c_int32),
                ("hold", C.c_int32), ("ents", C.c_void_p),
                ("cam_height", C.c_double), ("cam_fwd_disp", C.c_double), ("cam_pitch", C.c_double),
                ("cam_fov_y", C.c_double), ("sky_color", C.c_double * 3), ("light_pos", C.c_double * 3),
                ("light_color", C.c_double * 3), ("light_ambient", C.c_double * 3)]


class MazeDesc(C.Structure):
    _fields_ = [("rows", C.c_int32), ("cols", C.c_int32), ("pitch", C.c_double),
                ("cell_room", C.c_byte * ROOM_DTYPE.itemsize), ("cell_quads", C.c_byte * (6 * QUAD_DTYPE.itemsize)),
                ("cell_segs", C.c_byte * (4 * SEG_DTYPE.itemsize)), ("open_a", C.c_int32 * 4), ("open_b", C.c_int32 * 4),
                ("conn_room", C.c_byte * (4 * ROOM_DTYPE.itemsize)), ("conn_quads", C.c_byte * (16 * QUAD_DTYPE.itemsize)),
                ("conn_segs", C.c_byte * (8 * SEG_DTYPE.itemsize)), ("cdf", C.c_void_p)]


class StateView(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "agent_pos", "agent_dir", "step_count", "carrying", "num_slots", "agent_slot", "ents",
        "cam", "env_params", "rng", "room_tex", "num_picked_up", "episodes_done")]


class Level(C.Structure):
    _fields_ = [("rule_kind", C.c_int32), ("rule_arg", C.c_int32), ("max_episode_steps", C.c_int32),
                ("op_first", C.c_int32), ("num_ops", C.c_int32), ("domain_rand", C.c_int32), ("params", Params)]


def _expected_sizes():
    return [C.sizeof(Config), C.sizeof(Params), C.sizeof(TexDesc), C.sizeof(MeshDesc),
            ROOM_DTYPE.itemsize, QUAD_DTYPE.itemsize, SEG_DTYPE.itemsize, PROTO_DTYPE.itemsize,
            ENTITY_DTYPE.itemsize, OP_DTYPE.itemsize, C.sizeof(Geometry), C.sizeof(World),
            RNG_DTYPE.itemsize, C.sizeof(StateView), C.sizeof(MazeDesc), C.sizeof(Level), GOAL_GRID_DTYPE.itemsize]


EXPORTS = (
    "mwb_create", "mwb_destroy", "mwb_last_error", "mwb_upload_textures", "mwb_upload_meshes",
    "mwb_set_params", "mwb_set_protos", "mwb_set_template", "mwb_set_program", "mwb_seed",
    "mwb_reset", "mwb_set_world", "mwb_step", "mwb_render_obs", "mwb_get_state",
    "mwb_launch_count", "mwb_abi_sizes", "mwb_profile", "mwb_profile_read", "mwb_set_maze", "mwb_get_geometry",
    "mwb_overflow_count", "mwb_shared_alloc", "mwb_shared_open", "mwb_shared_close",
    "mwb_render_top_view", "mwb_visible_ents", "mwb_set_action_noise",
    "mwb_snapshot_size", "mwb_snapshot", "mwb_restore", "mwb_set_obs_format",
    "mwb_flag_write", "mwb_flag_wait_geq", "mwb_flag_mode", "mwb_state_array", "mwb_debug_camera", "mwb_set_obs_peer",
    "mwb_set_levels", "mwb_enable_level_changes", "mwb_state_in_host_memory", "mwb_set_level_maze",
    "mwb_enable_episode_seeds", "mwb_enable_maze_layouts", "mwb_enable_start_poses", "mwb_enable_state_bank",
    "mwb_save_states", "mwb_enable_reset_draws", "mwb_enable_goal_distance", "mwb_render_views", "mwb_visible_ents_from",
    "mwb_render_views_at", "mwb_visible_ents_from_at",
    "mwb_enable_env_params",
)
OBS_FORMATS = {"hwc": 0, "cwh": 1, "grey": 2}

_libs = {}


_test_library = None


def _override_library_for_tests(path):
    """TEST SEAM, not product API: tests/ point the binding at the g++ build of the kernels' inner functions
    (tests/hostsim) to debug kernel logic on a GPU-less box.  No product class takes a library argument; the
    override only works inside a pytest / tools process that imports this private name on purpose."""
    global _test_library
    _test_library = os.path.abspath(path) if path else None


def load_library():
    """dlopen the in-tree libmwb.so, declare prototypes, verify the struct mirrors.  No compute happens."""
    path = _test_library or os.path.abspath(DEFAULT_LIB)
    if path in _libs:
        return _libs[path]
    if not os.path.exists(path):
        raise EngineError("%s not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(there is no CPU fallback)" % path)
    lib = C.CDLL(path)
    vp, i32p = C.c_void_p, C.POINTER(C.c_int32)
    lib.mwb_last_error.restype = C.c_char_p
    lib.mwb_create.argtypes = [C.POINTER(Config), C.POINTER(vp)]
    lib.mwb_destroy.argtypes = [vp]
    lib.mwb_upload_textures.argtypes = [vp, vp, C.c_int, vp]
    lib.mwb_upload_meshes.argtypes = [vp, vp, C.c_int, vp, vp, vp, vp, vp]
    lib.mwb_set_params.argtypes = [vp, C.POINTER(Params)]
    lib.mwb_set_protos.argtypes = [vp, vp, C.c_int]
    lib.mwb_set_template.argtypes = [vp, C.POINTER(Geometry)]
    lib.mwb_set_program.argtypes = [vp, vp, C.c_int]
    lib.mwb_set_levels.argtypes = [vp, C.c_int, vp, vp, vp, C.c_int, vp]
    lib.mwb_enable_level_changes.argtypes = [vp, C.c_uint64, C.c_int32]
    lib.mwb_enable_episode_seeds.argtypes = [vp]
    lib.mwb_enable_maze_layouts.argtypes = [vp]
    lib.mwb_enable_start_poses.argtypes = [vp]
    lib.mwb_enable_state_bank.argtypes = [vp, C.c_int32]
    lib.mwb_enable_reset_draws.argtypes = [vp]
    lib.mwb_enable_goal_distance.argtypes = [vp, vp]
    lib.mwb_enable_env_params.argtypes = [vp]
    lib.mwb_save_states.argtypes = [vp, vp, vp, C.c_int, vp]
    lib.mwb_state_in_host_memory.argtypes = []
    lib.mwb_seed.argtypes = [vp, vp, C.c_int, vp]
    lib.mwb_reset.argtypes = [vp, vp, C.c_int, vp]
    lib.mwb_set_world.argtypes = [vp, vp, C.c_int, vp]
    lib.mwb_step.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.mwb_render_obs.argtypes = [vp, vp, vp, vp]
    lib.mwb_render_top_view.argtypes = [vp, C.POINTER(C.c_double), C.c_int, vp, vp]
    lib.mwb_visible_ents.argtypes = [vp, vp, vp]
    lib.mwb_render_views.argtypes = [vp, vp, C.c_int, C.c_int, vp, vp, vp]
    lib.mwb_visible_ents_from.argtypes = [vp, vp, vp, vp]
    lib.mwb_render_views_at.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp]
    lib.mwb_visible_ents_from_at.argtypes = [vp, vp, C.c_int, vp, vp]
    lib.mwb_set_action_noise.argtypes = [vp, C.c_int, C.c_double, C.c_int]
    lib.mwb_set_obs_format.argtypes = [vp, C.c_int]
    lib.mwb_snapshot_size.argtypes = [vp, C.POINTER(C.c_size_t)]
    lib.mwb_snapshot.argtypes = [vp, vp, C.c_size_t]
    lib.mwb_restore.argtypes = [vp, vp, C.c_size_t]
    lib.mwb_get_state.argtypes = [vp, C.POINTER(StateView)]
    lib.mwb_launch_count.argtypes = [vp]
    lib.mwb_launch_count.restype = C.c_int64
    lib.mwb_abi_sizes.argtypes = [i32p, C.c_int]
    lib.mwb_set_maze.argtypes = [vp, C.POINTER(MazeDesc)]
    lib.mwb_set_level_maze.argtypes = [vp, C.c_int, C.POINTER(MazeDesc)]
    lib.mwb_get_geometry.argtypes = [vp, C.c_int, i32p, vp, vp, vp]
    lib.mwb_shared_alloc.argtypes = [C.c_int, C.c_size_t, C.POINTER(vp), C.c_char_p]
    lib.mwb_shared_open.argtypes = [C.c_int, C.c_char_p, C.POINTER(vp)]
    lib.mwb_shared_close.argtypes = [vp, C.c_int]
    lib.mwb_flag_write.argtypes = [vp, vp, C.c_uint32]
    lib.mwb_flag_wait_geq.argtypes = [vp, vp, C.c_uint32]
    lib.mwb_flag_mode.argtypes = []
    lib.mwb_debug_camera.argtypes = [vp, vp]
    lib.mwb_set_obs_peer.argtypes = [vp, C.c_int]
    lib.mwb_state_array.argtypes = [vp, C.c_int, C.POINTER(vp), C.POINTER(C.c_int64)]
    lib.mwb_overflow_count.argtypes = [vp]
    lib.mwb_overflow_count.restype = C.c_int64
    lib.mwb_profile.argtypes = [vp, C.c_int]
    lib.mwb_profile_read.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int64),
                                     C.POINTER(C.c_int64)]
    for name in EXPORTS:
        if name not in ("mwb_last_error", "mwb_launch_count", "mwb_overflow_count"):
            getattr(lib, name).restype = C.c_int
    sizes = (C.c_int32 * 32)()
    n = lib.mwb_abi_sizes(sizes, 32)
    got, want = list(sizes[:n]), _expected_sizes()
    if got != want:
        raise EngineError("ABI struct size mismatch: library %r vs binding %r" % (got, want))
    _libs[path] = lib
    return lib


class SharedDeviceBuffer:
    """Device memory that other processes on the box can map (CUDA IPC), exposed to torch
    through __cuda_array_interface__ (zero copy)."""

    def __init__(self, device, shape, handle=None):
        self.lib = load_library()
        self.shape = tuple(int(v) for v in shape)
        self.nbytes = int(np.prod(self.shape))
        self.device = int(device)
        self.ptr = C.c_void_p()
        self.opened = handle is not None
        if handle is None:
            buf = C.create_string_buffer(64)
            rc = self.lib.mwb_shared_alloc(self.device, self.nbytes, C.byref(self.ptr), buf)
            self.handle = buf.raw
        else:
            self.handle = bytes(handle)
            rc = self.lib.mwb_shared_open(self.device, self.handle, C.byref(self.ptr))
        if rc != 0:
            raise EngineError("peer buffer: %s" % (self.lib.mwb_last_error() or b"").decode())

    @property
    def __cuda_array_interface__(self):
        return {"shape": self.shape, "typestr": "|u1", "data": (self.ptr.value, False), "version": 3, "strides": None}

    def tensor(self):
        import torch
        return torch.as_tensor(self, device=torch.device("cuda", self.device))

    def close(self):
        if self.ptr:
            self.lib.mwb_shared_close(self.ptr, int(self.opened))
            self.ptr = C.c_void_p()


def rng_state_of(seed_or_generator):
    """numpy PCG64 state -> mwb_rng_state record (what gym.Env.reset(seed=...) installs)."""
    if isinstance(seed_or_generator, np.random.Generator):
        st = seed_or_generator.bit_generator.state
    else:
        st = np.random.PCG64(np.random.SeedSequence(int(seed_or_generator))).state
    rec = np.zeros((), RNG_DTYPE)
    s, inc = st["state"]["state"], st["state"]["inc"]
    mask = (1 << 64) - 1
    rec["state_hi"], rec["state_lo"] = s >> 64, s & mask
    rec["inc_hi"], rec["inc_lo"] = inc >> 64, inc & mask
    rec["has_uint32"], rec["uinteger"] = st["has_uint32"], st["uinteger"]
    return rec


def generator_from_state(rec):
    """mwb_rng_state record -> numpy Generator positioned at the same point of the stream."""
    bg = np.random.PCG64()
    st = bg.state
    st["state"]["state"] = (int(rec["state_hi"]) << 64) | int(rec["state_lo"])
    st["state"]["inc"] = (int(rec["inc_hi"]) << 64) | int(rec["inc_lo"])
    st["has_uint32"], st["uinteger"] = int(rec["has_uint32"]), int(rec["uinteger"])
    bg.state = st
    return np.random.Generator(bg)


def lower_params(params):
    """DomainParams table -> mwb_params (defaults, lows and numpy's `high - low`)."""
    out = Params()
    for name in _VEC_PARAMS:
        p = params.params[name]
        for k in range(3):
            getattr(out, name)[k] = float(p.default[k])
            getattr(out, name + "_lo")[k] = float(p.min[k])
        rng = np.subtract(np.asarray(p.max, float), np.asarray(p.min, float))
        for k in range(3):
            getattr(out, name + "_rng")[k] = float(rng[k])
    for name in _SCALAR_PARAMS:
        p = params.params[name]
        setattr(out, name, float(p.default))
        setattr(out, name + "_lo", float(p.min))
        setattr(out, name + "_rng", float(p.max) - float(p.min))
    out.max_forward_step = float(params.get_max("forward_step"))
    return out


def _ptr(arr):
    return None if arr is None else C.c_void_p(arr.ctypes.data)


def _dev_or_host_ptr(x):
    """numpy array, torch tensor (cpu or cuda) or raw int address -> c_void_p."""
    if x is None:
        return None
    if isinstance(x, np.ndarray):
        return C.c_void_p(x.ctypes.data)
    if isinstance(x, int):
        return C.c_void_p(x)
    return C.c_void_p(x.data_ptr())


class Engine:
    """One mwb_handle: N environments resident on one GPU."""

    def __init__(self, num_envs, obs_width=80, obs_height=60, msaa_samples=8, shared_geometry=True,
                 max_rooms=8, max_quads=64, max_segs=64, max_ents=8, rule=(RULE_NONE, 0), domain_rand=False,
                 max_episode_steps=1500, autoreset=False, device=0):
        self.lib = load_library()
        cfg = Config(ABI_VERSION, int(device), int(num_envs), int(obs_width), int(obs_height), int(msaa_samples),
                     int(bool(shared_geometry)), int(max_rooms), int(max_quads), int(max_segs), int(max_ents),
                     int(rule[0]), int(rule[1]), int(bool(domain_rand)), int(max_episode_steps), int(bool(autoreset)))
        self.cfg = cfg
        self.h = C.c_void_p()
        self._check(self.lib.mwb_create(C.byref(cfg), C.byref(self.h)))
        self.N, self.W, self.H = int(num_envs), int(obs_width), int(obs_height)
        self.max_ents, self.max_rooms = int(max_ents), int(max_rooms)
        self._tex_uploaded = 0
        self._mesh_uploaded = 0
        self.num_levels = 1
        # the CPU build of the kernels (tests) keeps its "device" arrays in host memory
        self.host_memory = bool(self.lib.mwb_state_in_host_memory())

    def _check(self, rc):
        if rc != 0:
            raise EngineError("libmwb error %d: %s" % (rc, (self.lib.mwb_last_error() or b"").decode()))

    def close(self):
        if getattr(self, "h", None) is not None and self.h:
            self.lib.mwb_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- assets
    def sync_assets(self):
        """Upload textures / meshes registered since the last call."""
        from .assets import ObjMesh, Texture
        if len(Texture.registry) != self._tex_uploaded:
            descs = (TexDesc * len(Texture.registry))()
            blobs, off = [], 0
            for k, t in enumerate(Texture.registry):
                descs[k] = TexDesc(t.width, t.height, off)
                blobs.append(t.texels.reshape(-1))
                off += t.texels.size
            blob = np.concatenate(blobs)
            self._check(self.lib.mwb_upload_textures(self.h, C.cast(descs, C.c_void_p), len(descs), _ptr(blob)))
            self._tex_uploaded = len(Texture.registry)
        if len(ObjMesh.registry) != self._mesh_uploaded and ObjMesh.registry:
            descs = (MeshDesc * len(ObjMesh.registry))()
            off = 0
            for k, m in enumerate(ObjMesh.registry):
                descs[k] = MeshDesc(m.num_tris, 0, off)
                off += m.num_tris
            cat = lambda name: np.ascontiguousarray(np.concatenate([getattr(m, name) for m in ObjMesh.registry]), np.float32)
            pos, nrm, uv, rgb = cat("verts"), cat("norms"), cat("texcs"), cat("colors")
            tri_tex = np.ascontiguousarray(np.concatenate([m.tri_tex for m in ObjMesh.registry]), np.int32)
            self._check(self.lib.mwb_upload_meshes(self.h, C.cast(descs, C.c_void_p), len(descs),
                                                   _ptr(pos), _ptr(nrm), _ptr(uv), _ptr(rgb), _ptr(tri_tex)))
            self._mesh_uploaded = len(ObjMesh.registry)

    # ---- level definition
    def set_params(self, params):
        p = lower_params(params)
        self._check(self.lib.mwb_set_params(self.h, C.byref(p)))

    def set_protos(self, protos):
        protos = np.ascontiguousarray(protos, PROTO_DTYPE)
        self._check(self.lib.mwb_set_protos(self.h, _ptr(protos), len(protos)))

    @staticmethod
    def _geometry(rooms, quads, segs):
        g = Geometry(len(rooms), len(quads), len(segs), 0,
                     rooms.ctypes.data if len(rooms) else None, quads.ctypes.data if len(quads) else None,
                     segs.ctypes.data if len(segs) else None)
        return g

    def set_template(self, rooms, quads, segs):
        self._keep = (rooms, quads, segs)
        g = self._geometry(rooms, quads, segs)
        self._check(self.lib.mwb_set_template(self.h, C.byref(g)))

    def set_maze(self, tmpl, cdf):
        """tmpl: maze_lowering.MazeTemplate; cdf: float64[2 rows cols - 1]."""
        d = self._maze_desc(tmpl, cdf)
        self._check(self.lib.mwb_set_maze(self.h, C.byref(d)))

    def set_level_maze(self, level, tmpl, cdf):
        """Level `level` of the table (set_levels) becomes a Maze level with per-env worlds (mwb_set_level_maze)."""
        d = self._maze_desc(tmpl, cdf)
        self._check(self.lib.mwb_set_level_maze(self.h, int(level), C.byref(d)))

    def _maze_desc(self, tmpl, cdf):
        d = MazeDesc()
        d.rows, d.cols, d.pitch = tmpl.rows, tmpl.cols, tmpl.pitch

        def put(field, arr):
            raw = np.ascontiguousarray(arr).tobytes()
            assert len(raw) == C.sizeof(field), (len(raw), C.sizeof(field))
            C.memmove(field, raw, len(raw))

        put(d.cell_room, np.array(tmpl.cell_room, ROOM_DTYPE))
        put(d.cell_quads, np.array(tmpl.cell_quads, QUAD_DTYPE))
        put(d.cell_segs, np.array(tmpl.cell_segs, SEG_DTYPE))
        for k in range(4):
            d.open_a[k], d.open_b[k] = tmpl.open_a[k], tmpl.open_b[k]
        put(d.conn_room, np.array([c[0] for c in tmpl.conn], ROOM_DTYPE))
        put(d.conn_quads, np.array([c[1] for c in tmpl.conn], QUAD_DTYPE))
        put(d.conn_segs, np.array([c[2] for c in tmpl.conn], SEG_DTYPE))
        self._maze_cdf = np.ascontiguousarray(cdf, np.float64)
        d.cdf = self._maze_cdf.ctypes.data
        return d

    def get_geometry(self, env):
        counts = (C.c_int32 * 3)()
        rooms = np.zeros(self.cfg.max_rooms, ROOM_DTYPE)
        quads = np.zeros(self.cfg.max_quads, QUAD_DTYPE)
        segs = np.zeros(self.cfg.max_segs, SEG_DTYPE)
        self._check(self.lib.mwb_get_geometry(self.h, int(env), counts, _ptr(rooms), _ptr(quads), _ptr(segs)))
        return rooms[:counts[0]], quads[:counts[1]], segs[:counts[2]]

    def overflow_count(self):
        return int(self.lib.mwb_overflow_count(self.h))

    def set_program(self, ops):
        ops = np.ascontiguousarray(ops, OP_DTYPE)
        self._check(self.lib.mwb_set_program(self.h, _ptr(ops), len(ops)))

    def set_levels(self, levels, env_level):
        """Several levels in one handle (mwb_set_levels).  levels: list of dicts with "rule" (kind, arg),
        "max_episode_steps", "params" (DomainParams), "geometry" (rooms, quads, segs), "ops" (this level's
        program, proto indices already absolute) and optionally "domain_rand" (0 or 1; default: the handle's
        construction flag); env_level: int [num_envs] level of each env."""
        n = len(levels)
        table = (Level * n)()
        geoms = (Geometry * n)()
        first = 0
        for k, lv in enumerate(levels):
            rec = table[k]
            rec.rule_kind, rec.rule_arg = int(lv["rule"][0]), int(lv["rule"][1])
            rec.max_episode_steps = int(lv["max_episode_steps"])
            rec.op_first, rec.num_ops = first, len(lv["ops"])
            rec.domain_rand = int(lv.get("domain_rand", self.cfg.domain_rand))
            rec.params = lower_params(lv["params"])
            geoms[k] = self._geometry(*lv["geometry"])
            first += len(lv["ops"])
        ops = np.ascontiguousarray(np.concatenate([lv["ops"] for lv in levels]), OP_DTYPE)
        env_level = np.ascontiguousarray(env_level, np.int32)
        self._keep = [lv["geometry"] for lv in levels]
        self._check(self.lib.mwb_set_levels(self.h, n, C.cast(table, C.c_void_p), C.cast(geoms, C.c_void_p),
                                            _ptr(ops), len(ops), _ptr(env_level)))
        self.num_levels = n

    def enable_level_changes(self, seed=0, env_offset=0):
        """Levels change at resets from now on (mwb_enable_level_changes): pending assignments ("next_level") and
        draws from "level_weights", keyed by `seed` and the env's global index env_offset + i."""
        self._check(self.lib.mwb_enable_level_changes(self.h, int(seed) & (2 ** 64 - 1), int(env_offset)))

    def enable_episode_seeds(self):
        """Resets take a pending seed from "next_seed" and record it in "episode_seed" from now on
        (mwb_enable_episode_seeds); needs device resets."""
        self._check(self.lib.mwb_enable_episode_seeds(self.h))

    def enable_maze_layouts(self):
        """Resets at Maze levels build a pending layout from "next_maze" / "next_maze_cells" / "maze_pending" and record
        every episode's layout in "episode_maze" from now on (mwb_enable_maze_layouts); needs device resets, a Maze
        level and capacities that fit its all-open maze."""
        self._check(self.lib.mwb_enable_maze_layouts(self.h))

    def enable_start_poses(self):
        """Resets with "pose_pending" set place the agent and the entities at the designed poses of "next_pose" /
        "next_agent_pose", and every reset records the agent's start pose in "episode_start" from now on
        (mwb_enable_start_poses); needs device resets."""
        self._check(self.lib.mwb_enable_start_poses(self.h))

    def enable_reset_draws(self):
        """Resets with "draws_pending" set replace the outcomes of their level's reset draws with the in-support values
        of "next_draws", and every reset records its outcomes in "episode_draws" from now on (mwb_enable_reset_draws);
        needs device resets and a level with a draw, before the state bank."""
        self._check(self.lib.mwb_enable_reset_draws(self.h))

    def enable_env_params(self):
        """Resets with "params_pending" set run on their level's params merged with the (default, min, max) rows of
        "next_params", and every reset records its rows in "episode_params" from now on (mwb_enable_env_params); needs
        device resets, before the state bank."""
        self._check(self.lib.mwb_enable_env_params(self.h))

    def enable_goal_distance(self, grids):
        """`grids` (GOAL_GRID_DTYPE [n_levels]): the goal distance kernel follows every step and reset from now on and
        fills "goal_dist", "expert_action", "episode_shortest" and "goal_field" (mwb_enable_goal_distance); needs
        device resets, a level with a goal slot and grids of at most GOAL_GRID_CAP nodes."""
        grids = np.ascontiguousarray(grids, GOAL_GRID_DTYPE)
        self._check(self.lib.mwb_enable_goal_distance(self.h, _ptr(grids)))

    def enable_state_bank(self, slots):
        """`slots` state records; resets with "next_state" set load a filled one, and every reset records the loaded
        slot in "episode_state" from now on (mwb_enable_state_bank); needs device resets, after every other mode."""
        self._check(self.lib.mwb_enable_state_bank(self.h, int(slots)))

    def save_states(self, env_ids, slots, stream=None):
        """Env env_ids[t] into slot slots[t] (mwb_save_states): int32 numpy arrays (checked) or int32 CUDA tensors
        (enqueued on `stream`, out-of-range entries skipped on the device)."""
        if isinstance(env_ids, np.ndarray):
            env_ids, slots = np.ascontiguousarray(env_ids, np.int32), np.ascontiguousarray(slots, np.int32)
        self._check(self.lib.mwb_save_states(self.h, _dev_or_host_ptr(env_ids), _dev_or_host_ptr(slots), len(env_ids),
                                             stream))

    # ---- reset
    def seed(self, env_ids, states):
        ids = np.ascontiguousarray(env_ids, np.int32)
        states = np.ascontiguousarray(states, RNG_DTYPE)
        self._check(self.lib.mwb_seed(self.h, _ptr(ids), len(ids), _ptr(states)))

    def reset(self, env_ids=None, stream=None):
        if env_ids is None:
            self._check(self.lib.mwb_reset(self.h, None, self.N, stream))
        else:
            ids = np.ascontiguousarray(env_ids, np.int32)
            self._check(self.lib.mwb_reset(self.h, _ptr(ids), len(ids), stream))

    def set_world(self, env_ids, worlds):
        """worlds: list of dicts from pack.pack_world()."""
        ids = np.ascontiguousarray(env_ids, np.int32)
        arr = (World * len(worlds))()
        keep = []
        for k, w in enumerate(worlds):
            ws = arr[k]
            rooms, quads, segs = w["rooms"], w["quads"], w["segs"]
            ws.geom = self._geometry(rooms, quads, segs)
            ents = np.ascontiguousarray(w["ents"], ENTITY_DTYPE)
            keep.append((rooms, quads, segs, ents))
            ws.num_slots, ws.agent_slot, ws.carrying = len(ents), int(w["agent_slot"]), int(w["carrying"])
            ws.step_count, ws.num_picked_up = int(w["step_count"]), int(w.get("num_picked_up", 0))
            ws.hold = int(w.get("hold", 0))
            ws.ents = ents.ctypes.data if len(ents) else None
            ws.cam_height, ws.cam_fwd_disp, ws.cam_pitch, ws.cam_fov_y = (float(v) for v in w["cam"])
            for name in ("sky_color", "light_pos", "light_color", "light_ambient"):
                for c in range(3):
                    getattr(ws, name)[c] = float(w[name][c])
        self._check(self.lib.mwb_set_world(self.h, _ptr(ids), len(ids), C.cast(arr, C.c_void_p)))

    # ---- hot path
    def step(self, actions, obs=None, depth=None, reward=None, terminated=None, truncated=None,
             step_params=None, stream=None):
        self._check(self.lib.mwb_step(self.h, _dev_or_host_ptr(actions), _dev_or_host_ptr(step_params),
                                      _dev_or_host_ptr(obs), _dev_or_host_ptr(depth), _dev_or_host_ptr(reward),
                                      _dev_or_host_ptr(terminated), _dev_or_host_ptr(truncated), stream))

    def render(self, obs=None, depth=None, stream=None):
        self._check(self.lib.mwb_render_obs(self.h, _dev_or_host_ptr(obs), _dev_or_host_ptr(depth), stream))

    def set_obs_format(self, fmt):
        """"hwc": uint8 [N,H,W,3]; "cwh": uint8 [N,3,W,H] (PyTorchObsWrapper); "grey": float64 [N,H,W,1]
        (GreyscaleWrapper) -- written in that layout by the render kernel itself."""
        self._check(self.lib.mwb_set_obs_format(self.h, OBS_FORMATS[fmt]))

    def snapshot(self):
        """uint8 array holding the restorable state of every env (mwb_snapshot)."""
        n = C.c_size_t()
        self._check(self.lib.mwb_snapshot_size(self.h, C.byref(n)))
        blob = np.zeros(n.value, np.uint8)
        self._check(self.lib.mwb_snapshot(self.h, C.c_void_p(blob.ctypes.data), n.value))
        return blob

    def restore(self, blob):
        blob = np.ascontiguousarray(blob, np.uint8)
        self._check(self.lib.mwb_restore(self.h, C.c_void_p(blob.ctypes.data), blob.size))

    def set_action_noise(self, prob=None, random_action=None):
        """StochasticActionWrapper inside the step kernel; prob=None switches it off."""
        self._check(self.lib.mwb_set_action_noise(self.h, int(prob is not None), float(prob or 0.0),
                                                  -1 if random_action is None else int(random_action)))

    def render_top_view(self, extents, obs, render_agent=True, stream=None):
        """Map view of every env (reference render_top_view); extents = (min_x, max_x, min_z, max_z)."""
        ext = (C.c_double * 4)(*[float(v) for v in extents])
        self._check(self.lib.mwb_render_top_view(self.h, ext, int(bool(render_agent)), _dev_or_host_ptr(obs), stream))

    def visible_ents(self, mask, stream=None, poses=None, row_width=3):
        """uint32[N] (numpy or CUDA tensor): bit e = entity slot e passes the reference's occlusion query -- from the
        agent's camera, or with `poses` (float64 [N, row_width] rows (x, z, dir[, cam_height, cam_fwd_disp, cam_pitch,
        cam_fov_y]), row_width 3 or 7) from each env's designed camera (mwb_visible_ents_from_at; a skipped row leaves
        its entry as it is)."""
        if poses is None:
            self._check(self.lib.mwb_visible_ents(self.h, _dev_or_host_ptr(mask), stream))
        else:
            self._check(self.lib.mwb_visible_ents_from_at(self.h, _dev_or_host_ptr(poses), int(row_width),
                                                          _dev_or_host_ptr(mask), stream))

    def render_views(self, poses, views, obs=None, depth=None, render_agent=False, stream=None, row_width=3, size=None,
                     samples=None):
        """Views of every env from designed cameras (mwb_render_views_at): poses float64 [views, N, row_width] rows
        (x, z, dir[, cam_height, cam_fwd_disp, cam_pitch, cam_fov_y]), obs [views, N, frame] in the observation format
        and / or depth float32 [views, N, H, W, 1] (numpy or CUDA tensors, contiguous) at size (W, H) (default: the
        observation size) with `samples` samples per pixel (default: the handle's); frames of skipped rows are left as
        they are."""
        W, H = (self.W, self.H) if size is None else (int(size[0]), int(size[1]))
        S = self.cfg.msaa_samples if samples is None else int(samples)
        self._check(self.lib.mwb_render_views_at(self.h, _dev_or_host_ptr(poses), int(row_width), int(views), W, H, S,
                                                 int(bool(render_agent)), _dev_or_host_ptr(obs), _dev_or_host_ptr(depth),
                                                 stream))

    # name -> (mwb_state_array id, element type, shape): "env" = [N], "ents" = [max_ents, N], "level" = [count]
    # ([n_levels], or [slots] for bank_level),
    # "params" = [n_levels, PARAMS_DOUBLES] (mwb_params records as float64 words), "env_rows" = [N, count / N],
    # "env_slots" = [N, count / (3 N), 3] ([N, max_ents, 3], or [N, 22, 3] for the env params rows)
    ARRAYS = {"counter": (0, "<i4", "env"), "step_count": (1, "<i4", "env"), "ent_x": (2, "<f8", "ents"),
              "ent_y": (3, "<f8", "ents"), "ent_z": (4, "<f8", "ents"), "ent_dir": (5, "<f8", "ents"),
              "env_level": (6, "<i4", "env"), "next_level": (7, "<i4", "env"), "level_weights": (8, "<f4", "level"),
              "level_params": (9, "<f8", "params"), "next_seed": (16, "<i8", "env"), "episode_seed": (17, "<i8", "env"),
              "next_maze": (18, "|u1", "env_rows"), "next_maze_cells": (19, "<i4", "env_rows"),
              "maze_pending": (20, "|u1", "env"), "episode_maze": (21, "|u1", "env_rows"),
              "next_pose": (22, "<f8", "env_slots"), "next_agent_pose": (23, "<f8", "env_rows"),
              "pose_pending": (24, "|u1", "env"), "episode_start": (25, "<f8", "env_rows"),
              "next_state": (26, "<i4", "env"), "episode_state": (27, "<i4", "env"), "bank_level": (28, "<i4", "level"),
              "next_draws": (29, "<f8", "env_rows"), "draws_pending": (30, "|u1", "env"),
              "episode_draws": (31, "<f8", "env_rows"), "goal_dist": (32, "<f8", "env"),
              "expert_action": (33, "<i4", "env"), "episode_shortest": (34, "<f8", "env"),
              "goal_field": (35, "<u2", "env_rows")}
    # ARRAYS holds the arrays of the modes up to goal distance; its key set is what pinned refusal texts walk, so
    # later modes list theirs in a table of their own (state_array reads ARRAYS, then those tables).  A later mode adds
    # a table here, or the tables are merged together with those texts.
    ENV_PARAM_ARRAYS = {"next_params": (36, "<f8", "env_slots"), "params_pending": (37, "|u1", "env"),
                        "episode_params": (38, "<f8", "env_slots")}

    def state_array(self, name, shape=None):
        """Zero-copy view of a state array (mwb_state_array) as an object with __cuda_array_interface__:
        "counter" / "step_count" int32 [N]; "ent_x|y|z|dir" float64 [max_ents, N]; with level changes on,
        "env_level" / "next_level" int32 [N] and "level_weights" float32 [n_levels]; with device resets,
        "level_params" float64 [n_levels, PARAMS_DOUBLES] (column of a field: PARAMS_COLUMN); with episode seeds on,
        "next_seed" / "episode_seed" int64 [N]; with maze layouts on, "next_maze" / "episode_maze" uint8
        [N, rows * cols], "next_maze_cells" int32 [N, 2] and "maze_pending" uint8 [N]; with start poses on,
        "next_pose" float64 [N, max_ents, 3], "next_agent_pose" / "episode_start" float64 [N, 3] and "pose_pending"
        uint8 [N]; with the state bank on, "next_state" / "episode_state" int32 [N] and "bank_level" int32 [slots];
        with reset draws on, "next_draws" / "episode_draws" float64 [N, D] and "draws_pending" uint8 [N]; with goal
        distance on, "goal_dist" / "episode_shortest" float64 [N], "expert_action" int32 [N] and "goal_field" uint16
        [N, G]; with env params on, "next_params" / "episode_params" float64 [N, 22, 3] and "params_pending" uint8 [N].
        `shape` gives the view
        another shape of the same size (the maze layouts as [N, rows, cols]).  On the host build of the kernels the
        arrays live in host memory, and the view is a numpy array over the same memory instead."""
        which, typestr, axis = self.ARRAYS[name] if name in self.ARRAYS else self.ENV_PARAM_ARRAYS[name]
        ptr, count = C.c_void_p(), C.c_int64()
        self._check(self.lib.mwb_state_array(self.h, which, C.byref(ptr), C.byref(count)))
        n = count.value
        shape = tuple(shape or {"env": (self.N,), "ents": (n // self.N, self.N), "level": (n,),
                                "params": (n, PARAMS_DOUBLES), "env_rows": (self.N, n // self.N),
                                "env_slots": (self.N, n // (3 * self.N), 3)}[axis])
        if int(np.prod(shape)) != (n * PARAMS_DOUBLES if axis == "params" else n):
            raise ValueError("%s has %d entries, not shape %s" % (name, n, shape))
        if self.host_memory:
            dt = np.dtype(typestr)
            buf = (C.c_char * (int(np.prod(shape)) * dt.itemsize)).from_address(ptr.value)
            return np.frombuffer(buf, dt).reshape(shape)

        class _View:
            __cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr.value, False), "version": 3, "strides": None}
        return _View()

    def set_obs_peer(self, peer):
        """peer: True / False = observations go to another GPU's / this GPU's memory; None = look it up per pointer."""
        self._check(self.lib.mwb_set_obs_peer(self.h, -1 if peer is None else int(bool(peer))))

    def debug_camera(self):
        """float32 [N, 16]: eye, right, up, forward, (cot / aspect, cot), (za, zb) of every env's camera as K2 derives it."""
        out = np.zeros((self.N, 16), np.float32)
        self._check(self.lib.mwb_debug_camera(self.h, _ptr(out)))
        return out

    def launch_count(self):
        return int(self.lib.mwb_launch_count(self.h))

    def profile(self, enable=True):
        self._check(self.lib.mwb_profile(self.h, int(enable)))

    def profile_read(self):
        """(k1_ms, k2_ms, k1_launches, k2_launches) since the last read, CUDA-event timed."""
        a, b, na, nb = C.c_double(), C.c_double(), C.c_int64(), C.c_int64()
        self._check(self.lib.mwb_profile_read(self.h, C.byref(a), C.byref(b), C.byref(na), C.byref(nb)))
        return a.value, b.value, na.value, nb.value

    # ---- state
    def get_state(self, rng=False, room_tex=False):
        N, E = self.N, self.max_ents
        out = dict(agent_pos=np.zeros((N, 3)), agent_dir=np.zeros(N), step_count=np.zeros(N, np.int32),
                   carrying=np.zeros(N, np.int32), num_slots=np.zeros(N, np.int32),
                   agent_slot=np.zeros(N, np.int32), ents=np.zeros((N, E), ENTITY_DTYPE),
                   cam=np.zeros((N, 4)), env_params=np.zeros((N, 12)), num_picked_up=np.zeros(N, np.int32),
                   episodes_done=np.zeros(1, np.int64))
        if rng:
            out["rng"] = np.zeros(N, RNG_DTYPE)
        if room_tex:
            out["room_tex"] = np.zeros((N, self.max_rooms, 3), np.int32)
        view = StateView()
        for k, v in out.items():
            setattr(view, k, v.ctypes.data)
        self._check(self.lib.mwb_get_state(self.h, C.byref(view)))
        return out


class SingleEnvEngine:
    """N = 1 engine behind `world.MiniWorldEnv`: the env's Python objects stay authoritative;
    before each GPU call the (possibly user-modified) state is pushed, afterwards pulled."""

    def __init__(self, obs_width, obs_height, msaa_samples, device):
        self.args = (obs_width, obs_height, msaa_samples)
        self.device = 0 if device in ("cuda", None) else int(str(device).split(":")[-1])
        self.engine = None
        self.caps = None
        self.W, self.H = obs_width, obs_height

    def close(self):
        if self.engine is not None:
            self.engine.close()
            self.engine = None

    def push(self, env, full):
        from . import pack
        world = pack.pack_world(env)
        need = (max(8, len(world["rooms"])), max(64, len(world["quads"])), max(64, len(world["segs"])),
                max(8, len(world["ents"])))
        max_steps = int(min(env.max_episode_steps, 2 ** 31 - 1))     # math.inf -> never truncates
        if self.engine is None or any(n > c for n, c in zip(need, self.caps)) or \
                self.engine.cfg.max_episode_steps != max_steps:
            if self.engine is not None:
                self.engine.close()
            caps = tuple(int(2 ** np.ceil(np.log2(n))) for n in need)
            W, H, msaa = self.args
            self.engine = Engine(1, W, H, msaa, shared_geometry=False, max_rooms=caps[0], max_quads=caps[1],
                                 max_segs=caps[2], max_ents=min(caps[3], MAX_ENTS_CAP), rule=(RULE_NONE, 0),
                                 domain_rand=False, max_episode_steps=max_steps, autoreset=False,
                                 device=self.device)
            self.caps = caps
            self.engine.set_params(env.params)
        self.engine.sync_assets()
        self.engine.set_protos(world["protos"])
        self.engine.set_world([0], [world])
        self._slots = world["slot_entities"]

    def pull(self, env):
        st = self.engine.get_state()
        env.step_count = int(st["step_count"][0])
        ents = st["ents"][0]
        for slot, ent in enumerate(self._slots):
            rec = ents[slot]
            ent.pos = np.array(rec["pos"])
            ent.dir = float(rec["dir"])
        c = int(st["carrying"][0])
        env.agent.carrying = self._slots[c] if c >= 0 else None

    def step_single(self, action, fwd_step, fwd_drift, turn_step):
        obs = np.zeros((self.H, self.W, 3), np.uint8)
        acts = np.array([action], np.int32)
        sp = np.array([[fwd_step, fwd_drift, turn_step]], np.float64)
        self.engine.step(acts, obs=obs, step_params=sp)
        return obs

    def render(self, want_depth):
        obs = np.zeros((self.H, self.W, 3), np.uint8)
        depth = np.zeros((self.H, self.W, 1), np.float32) if want_depth else None
        self.engine.render(obs=obs, depth=depth)
        return obs, depth

    def render_top_view(self, extents, render_agent):
        obs = np.zeros((self.H, self.W, 3), np.uint8)
        self.engine.render_top_view(extents, obs, render_agent)
        return obs

    def visible_ents(self):
        mask = np.zeros(1, np.uint32)
        self.engine.visible_ents(mask)
        return {ent for slot, ent in enumerate(self._slots) if (int(mask[0]) >> slot) & 1}

    def render_view(self, pose, render_agent):
        """pose: a 3- or 7-column row, rendered at this engine's own frame size and sample count"""
        pose = np.asarray(pose, np.float64).reshape(1, 1, -1)
        obs = np.zeros((self.H, self.W, 3), np.uint8)
        depth = np.zeros((self.H, self.W, 1), np.float32)
        self.engine.render_views(pose, 1, obs=obs, depth=depth, render_agent=render_agent, row_width=pose.shape[-1])
        return obs, depth
