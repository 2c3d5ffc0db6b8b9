/*
 * mwb.h -- C ABI of libmwb.so, the H100-native batched MiniWorld step engine.
 *
 * The reference (Farama-Foundation/Miniworld) has no plugin / FFI layer of its own: its
 * only foreign-function crossing is pyglet's per-GL-call ctypes binding, hit thousands of
 * times per frame from MiniWorldEnv.step / render_obs.  This header replaces that
 * crossing with ONE batched call per step over N independent environments.  Every entry
 * point below names the reference code it stands in for (paths relative to the reference
 * root, pinned at c660156 / v2.1.0).
 *
 * Conventions
 *   - plain C, no C++ / torch types; loaded with ctypes.CDLL (miniworld_b200/engine.py).
 *   - every function returns 0 on success, a negative MWB_E* code otherwise;
 *     mwb_last_error() returns a thread-local, library-owned message.
 *   - every buffer is caller-owned.  Output / action pointers may be host or device
 *     memory (detected with cudaPointerGetAttributes); host pointers make the call
 *     synchronous, device pointers enqueue on `stream` and return.
 *   - a handle is bound to one CUDA device and is not thread-safe; that device must be the calling
 *     thread's current device for every call on the handle (one process per GPU is the intended use).
 *   - there is no CPU execution path: mwb_create fails with MWB_ENOCUDA without a GPU.
 */
#ifndef MWB_H_
#define MWB_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MWB_ABI_VERSION 10

/* error codes */
#define MWB_OK 0
#define MWB_EINVAL (-1)
#define MWB_ENOCUDA (-2)
#define MWB_ECUDA (-3)
#define MWB_EABI (-4)
#define MWB_ECAPACITY (-5)
#define MWB_ESTATE (-6)

/* fixed capacities of the flat records */
#define MWB_MAX_EDGES 8   /* outline vertices per room (rect rooms and connectors: 4) */
#define MWB_MAX_OPS 64    /* reset-program length */
#define MWB_LEVEL_CAP 32  /* levels one handle can run side by side (mwb_set_levels) */

/* entity kinds (reference miniworld/entity.py: Box :386, MeshEnt :124, Agent :455) */
#define MWB_KIND_NONE 0
#define MWB_KIND_BOX 1
#define MWB_KIND_MESH 2
#define MWB_KIND_AGENT 3

/* level rule evaluated after the base step (reference envs/<level>.py step()) */
#define MWB_RULE_NONE 0   /* base MiniWorldEnv.step only (miniworld.py:670-730)               */
#define MWB_RULE_GOAL 1   /* near(box) -> +_reward(), terminated (hallway.py:67-74, oneroom.py */
                          /* :64-71, fourrooms.py:66-73, maze.py:155-162)                      */
#define MWB_RULE_PICKUP 2 /* carrying -> remove, reward = 1 (pickupobjects.py:83-95)          */
#define MWB_RULE_SIDEWALK 3 /* agent inside the street room -> terminated (reward 0), then the  */
                          /* GOAL rule (sidewalk.py:93-104); rule_arg = box slot | room << 8   */

#define MWB_RULE_SIGN 4   /* action 3 ends the episode; touching one of the six objects (slots 0..5:   */
                          /* kind = slot / 3, colour = slot % 3) ends it with reward +1 / -1            */
                          /* (sign.py:158-173); rule_arg = colour index | goal << 8                     */

#define MWB_RULE_HEALTH 5 /* health -= 2 per step; pickup while carrying: the kit is removed from the list, */
                          /* placed again (place_entity on the env's stream) and health = 100; reward 2, or  */
                          /* -100 and terminated once health <= 0 (collecthealth.py:62-86).  The per-env     */
                          /* level counter (num_picked_up in mwb_state_view) holds the health.               */

#define MWB_RULE_PUTNEXT 6 /* near(ent a, ent b) and not carrying -> +_reward(), terminated (putnext.py:61-66);  */
                          /* rule_arg = slot a | slot b << 8                                                  */

/* surfaces of a room */
#define MWB_SURF_WALL 0
#define MWB_SURF_FLOOR 1
#define MWB_SURF_CEIL 2

/* reset-program opcodes: a lowered _gen_world() (reference miniworld.py:544-604, 839-909) */
#define MWB_OP_END 0
#define MWB_OP_CHOICE 1   /* ireg[a] = np_random.choice(b)            (== integers(0, b))      */
#define MWB_OP_UNIFORM 2  /* freg[a] = np_random.uniform(f[0], f[1])                           */
#define MWB_OP_PLACE 3    /* place_entity(); see mwb_op                                         */
#define MWB_OP_IFEQ 5     /* run the next op only if ireg[a] == b (a level's `if rng.integers(0, 2) == 0:`)   */
#define MWB_OP_PUT 6      /* place_entity(ent, pos=f[0..2], dir=f[3]) (miniworld.py:862-869): no search, no    */
                          /* draw unless f[3] is NaN (then dir = uniform(-pi, pi)); b = 1: a bare               */
                          /* entities.append(ent), which does not trigger _gen_static_data                      */
#define MWB_OP_MAZE 4     /* Maze._gen_world() room topology (reference envs/maze.py:73-153): recursive  */
                          /* backtracker on the env's RNG stream, geometry from mwb_set_maze templates   */

typedef struct mwb_handle mwb_handle;

typedef struct mwb_config {
  int32_t abi_version;       /* must be MWB_ABI_VERSION                                          */
  int32_t device;            /* CUDA ordinal                                                     */
  int32_t num_envs;          /* N                                                                */
  int32_t obs_width;         /* MiniWorldEnv(obs_width=80)  (miniworld.py:473)                   */
  int32_t obs_height;        /* MiniWorldEnv(obs_height=60) (miniworld.py:474)                   */
  int32_t msaa_samples;      /* 1, 4 or 8; FrameBuffer(obs_w, obs_h, 8) (miniworld.py:515)       */
  int32_t shared_geometry;   /* 1: all envs share one static room template; 0: per-env geometry  */
  int32_t max_rooms, max_quads, max_segs, max_ents;   /* per-env capacities                      */
  int32_t rule_kind;         /* MWB_RULE_*                                                       */
  int32_t rule_arg;          /* GOAL: entity slot of the box; PICKUP: num_objs                   */
  int32_t domain_rand;       /* MiniWorldEnv(domain_rand=...) (miniworld.py:478) of level 0      */
  int32_t max_episode_steps; /* (miniworld.py:472)                                               */
  int32_t autoreset;         /* 1: the step after terminated|truncated resets on the device      */
  int32_t reserved[4];
} mwb_config;

/* DomainParams table (reference params.py:115-130), lowered: lo and (hi - lo) per element,
 * as numpy's Generator.uniform consumes them (low + (high - low) * random()). */
typedef struct mwb_params {
  double sky_color[3], sky_color_lo[3], sky_color_rng[3];
  double light_pos[3], light_pos_lo[3], light_pos_rng[3];
  double light_color[3], light_color_lo[3], light_color_rng[3];
  double light_ambient[3], light_ambient_lo[3], light_ambient_rng[3];
  double obj_color_bias[3], obj_color_bias_lo[3], obj_color_bias_rng[3];
  double forward_step, forward_step_lo, forward_step_rng;
  double forward_drift, forward_drift_lo, forward_drift_rng;
  double turn_step, turn_step_lo, turn_step_rng;
  double cam_pitch, cam_pitch_lo, cam_pitch_rng;
  double cam_fov_y, cam_fov_y_lo, cam_fov_y_rng;
  double cam_height, cam_height_lo, cam_height_rng;
  double cam_fwd_disp, cam_fwd_disp_lo, cam_fwd_disp_rng;
  double max_forward_step;   /* params.get_max("forward_step") (miniworld.py:581)                */
} mwb_params;

/* one mip-mapped texture (reference opengl.py:147-184: GL_RGB, rows bottom-up, REPEAT,
 * LINEAR / LINEAR_MIPMAP_LINEAR); texels passed top row first, RGB8, engine builds mips. */
typedef struct mwb_tex_desc {
  int32_t width, height;
  int64_t offset;            /* byte offset of this texture's level 0 in the texel blob          */
} mwb_tex_desc;

/* one triangle mesh (reference objmesh.py:36-216): per face-vertex arrays; each triangle names
 * the texture of its material chunk (map_Kd) or -1.  ImageFrame / TextFrame (entity.py:168-383)
 * are lowered to small meshes of this form too. */
typedef struct mwb_mesh_desc {
  int32_t num_tris;
  int32_t reserved;
  int64_t offset;            /* index of the first triangle in the vertex arrays                 */
} mwb_mesh_desc;

/* Room (reference miniworld.py:122-194): extents, outline + inward edge normals for
 * point_inside (:272-284), pick probability for place_entity (:873-880), textures. */
typedef struct mwb_room {
  double min_x, max_x, min_z, max_z;
  double cdf;                               /* cumulative room_probs, as Generator.choice(p=) */
  double edge_px[MWB_MAX_EDGES], edge_pz[MWB_MAX_EDGES];   /* outline                          */
  double edge_nx[MWB_MAX_EDGES], edge_nz[MWB_MAX_EDGES];   /* edge_norms                       */
  int32_t num_edges;
  int32_t tex_first[3];                     /* first texture id of the wall/floor/ceil family */
  int32_t tex_count[3];                     /* number of variants (Texture.get, opengl.py:113) */
  int32_t tex_id[3];                        /* variant in use (host-generated worlds)          */
  int32_t reserved;
} mwb_room;

/* One static quad of Room._render (miniworld.py:401-434): floor / ceiling polygon or a wall
 * piece from _gen_static_data (:313-344).  uvm = texcoords in metres; the engine applies
 * TEX_DENSITY / tex size (gen_texcs_wall :82-103, gen_texcs_floor :106-119). */
typedef struct mwb_quad {
  float pos[4][3];
  float nrm[3];
  int32_t room;
  int32_t surf;              /* MWB_SURF_*                                                       */
  int32_t num_verts;         /* 4 (3 for a triangular floor fan piece)                          */
  double uvm[4][2];
} mwb_quad;

/* collision segment, stored as the reference stores it: [s_p1, s_p0] (miniworld.py:325) */
typedef struct mwb_seg {
  double ax, az, bx, bz;
} mwb_seg;

/* Entity prototype: everything about an entity that does not change during an episode. */
typedef struct mwb_proto {
  int32_t kind;              /* MWB_KIND_*                                                       */
  int32_t is_static;         /* Entity.is_static (entity.py:115-121, :163-165)                   */
  int32_t mesh_id;           /* MeshEnt: index into the uploaded meshes, else -1                 */
  int32_t radius_is_f32;     /* MeshEnt radii are np.float32 under numpy >= 2 (SURVEY R2)        */
  double radius, height;
  double size[3];            /* Box size                                                         */
  double color[3];           /* COLORS[color] (entity.py:30-40)                                  */
  float scale;               /* MeshEnt.scale (entity.py:144)                                    */
  int32_t deg_form;          /* how render() forms glRotatef's angle: 1 = dir * 180 / pi (MeshEnt, entity.py:158), */
                             /* 0 = dir * (180 / pi) (Box, ImageFrame, TextFrame: entity.py:206, 316, 421)          */
} mwb_proto;

/* Per-env entity instance (host-generated worlds / state exchange). */
typedef struct mwb_entity {
  int32_t proto;             /* index into the handle's proto table, -1 = empty slot             */
  int32_t reserved;
  double pos[3];
  double dir;
  double color[3];           /* Box.color_vec after randomize (entity.py:405-407)                */
} mwb_entity;

typedef struct mwb_op {
  int32_t op;                /* MWB_OP_*                                                         */
  int32_t a, b;              /* CHOICE: dst ireg, n.  UNIFORM: dst freg.  PLACE: proto base, 1 + freg holding   */
                             /* this episode's Box edge length (0: the prototype's).  IFEQ: ireg, value.        */
                             /* PUT: proto, append-only flag                                                    */
  int32_t ireg_a, stride_a;  /* PLACE: proto = a + ireg[ireg_a]*stride_a + ireg[ireg_b]*stride_b */
  int32_t ireg_b, stride_b;  /*        (ireg_* = -1: unused)                                     */
  int32_t room;              /* PLACE: fixed room index or -1 (sample by area).  CHOICE / UNIFORM: the draw's    */
                             /* index d, 0, 1, ... in program order (mwb_enable_reset_draws)                    */
  int32_t dir_freg;          /* PLACE: freg holding dir, or -1 (draw uniform(-pi, pi))           */
  int32_t is_agent;          /* PLACE: this is place_agent()                                     */
  double f[4];               /* UNIFORM: lo, hi.  PLACE: min_x, max_x, min_z, max_z (NaN = room) */
} mwb_op;

/* Static template + reset program shared by all envs (shared_geometry = 1), or the
 * geometry of one env (shared_geometry = 0, via mwb_set_world). */
typedef struct mwb_geometry {
  int32_t num_rooms, num_quads, num_segs, reserved;
  const mwb_room* rooms;
  const mwb_quad* quads;
  const mwb_seg* segs;
} mwb_geometry;

/* Complete per-env world, produced by host-side world generation (reset()). */
typedef struct mwb_world {
  mwb_geometry geom;         /* ignored when shared_geometry = 1                                 */
  int32_t num_slots;         /* length of the entity list (miniworld.py:560)                     */
  int32_t agent_slot;        /* index of the agent in it                                         */
  int32_t carrying;          /* slot being carried or -1                                         */
  int32_t step_count;
  int32_t num_picked_up;
  int32_t hold;              /* 1: the next mwb_step reports this env as just reset (reward 0, flags
                              * 0) instead of stepping it -- host-side "next-step" auto-reset       */
  const mwb_entity* ents;    /* num_slots entries                                                */
  double cam_height, cam_fwd_disp, cam_pitch, cam_fov_y;   /* Agent (entity.py:455-516)        */
  double sky_color[3], light_pos[3], light_color[3], light_ambient[3];
} mwb_world;

/* numpy Generator(PCG64) state as exposed by bit_generator.state */
typedef struct mwb_rng_state {
  uint64_t state_hi, state_lo, inc_hi, inc_lo;
  int32_t has_uint32;
  uint32_t uinteger;
} mwb_rng_state;

/* Readback of the dynamic state (all host pointers, any may be NULL). */
typedef struct mwb_state_view {
  double* agent_pos;         /* [N][3]                                                           */
  double* agent_dir;         /* [N]                                                              */
  int32_t* step_count;       /* [N]                                                              */
  int32_t* carrying;         /* [N]                                                              */
  int32_t* num_slots;        /* [N]                                                              */
  int32_t* agent_slot;       /* [N]                                                              */
  mwb_entity* ents;          /* [N][max_ents]                                                    */
  double* cam;               /* [N][4] height, fwd_disp, pitch, fov_y                            */
  double* env_params;        /* [N][12] sky, light_pos, light_color, light_ambient               */
  mwb_rng_state* rng;        /* [N]                                                              */
  int32_t* room_tex;         /* [N][max_rooms][3] texture id in use per room surface             */
  int32_t* num_picked_up;    /* [N]                                                              */
  int64_t* episodes_done;    /* [1] steps that ended an episode (terminated|truncated) so far    */
} mwb_state_view;

/* ---- lifetime ------------------------------------------------------------------------
 * replaces MiniWorldEnv.__init__ GL context + FrameBuffer creation (miniworld.py:508-518,
 * opengl.py:202-327) */
int mwb_create(const mwb_config* cfg, mwb_handle** out);
int mwb_destroy(mwb_handle* h);
const char* mwb_last_error(void);

/* ---- assets: Texture.load (opengl.py:147-184), ObjMesh.__init__ (objmesh.py:36-216) ---- */
int mwb_upload_textures(mwb_handle* h, const mwb_tex_desc* descs, int n, const uint8_t* texels_rgb8);
int mwb_upload_meshes(mwb_handle* h, const mwb_mesh_desc* descs, int n, const float* pos /*[T][3][3]*/,
                      const float* nrm /*[T][3][3]*/, const float* uv /*[T][3][2]*/,
                      const float* rgb /*[T][3][3]*/, const int32_t* tri_tex /*[T] texture id or -1*/);

/* ---- level definition ------------------------------------------------------------------ */
int mwb_set_params(mwb_handle* h, const mwb_params* p);                    /* params.py:115-130  */
int mwb_set_protos(mwb_handle* h, const mwb_proto* protos, int n);         /* entity.py ctor data */
int mwb_set_template(mwb_handle* h, const mwb_geometry* g);                /* shared static rooms */
int mwb_set_program(mwb_handle* h, const mwb_op* ops, int n);              /* lowered _gen_world  */

/* Several levels in one batch (the reference's vector env built from a list of env constructors, each with its own
 * level id and kwargs).  A handle holds a table of levels; mwb_create's rule fields and domain_rand, mwb_set_params,
 * mwb_set_template and mwb_set_program fill level 0 of it, so a handle that never calls mwb_set_levels runs one level.
 * mwb_set_levels replaces the whole table: level l gets templates[l] as its static rooms and the reset program
 * ops[op_first, op_first + num_ops).  env_level[i] names the level of env i; the proto table (mwb_set_protos) is
 * shared, so each level's ops address it with absolute indices.  Only for shared_geometry = 1 handles (MWB_EINVAL
 * otherwise); MWB_ECAPACITY for more than MWB_LEVEL_CAP levels, a program longer than MWB_MAX_OPS or a template
 * above the handle's max_rooms / max_quads / max_segs; MWB_EINVAL for an env_level entry outside [0, n_levels) or a
 * domain_rand other than 0 or 1.
 * Each level has its own domain_rand: an env's reset draws (texture variants, sky and light, entity colours, agent
 * camera) follow the flag of the level it resets into, and its per-step draws the flag of its episode's level, so rows
 * that share a level definition but differ in the flag (and in their params' ranges) make a randomisation curriculum.
 * The flag is table data, not env state: snapshots do not carry it.  The rows' params are the initial content of the
 * params table, which the caller may rewrite while the batch runs (MWB_ARRAY_LEVEL_PARAMS).
 * Per-handle settings (observation size, MSAA, autoreset, action noise) apply to every level. */
typedef struct mwb_level {
  int32_t rule_kind;         /* MWB_RULE_*                                                       */
  int32_t rule_arg;
  int32_t max_episode_steps;
  int32_t op_first, num_ops; /* this level's slice of the shared op array                        */
  int32_t domain_rand;       /* 0 or 1: MiniWorldEnv(domain_rand=...) of this level              */
  mwb_params params;
} mwb_level;
int mwb_set_levels(mwb_handle* h, int n_levels, const mwb_level* levels, const mwb_geometry* templates /*[n_levels]*/,
                   const mwb_op* ops, int n_ops, const int32_t* env_level /*[num_envs]*/);

/* Level changes at episode boundaries (curricula: promote an env once it succeeds, re-weight levels by success rate).
 * Valid after mwb_set_levels (MWB_ESTATE before it, or when already on; the level table is fixed from then on).  It
 * allocates next_level [N] (all -1), level_draws [N] (all 0) and level_weights [L] (all 0: no draws), and makes the
 * device's env_level authoritative: the resets rewrite it, and the caller reads and writes these arrays in place
 * through mwb_state_array (MWB_ARRAY_ENV_LEVEL / NEXT_LEVEL / LEVEL_WEIGHTS), stream-ordered, without a sync.
 *
 * A level changes only at a reset: mwb_reset, and the next-step auto-reset inside mwb_step.  An env never changes
 * level mid-episode.  At every reset of env i, before the level is read:
 *   1. if next_level[i] is in [0, L): the env takes that level, and next_level[i] is cleared to -1;
 *   2. otherwise, if the level weights sum to more than 0: the next level is drawn from them;
 *   3. otherwise the env keeps its level.
 * A next_level entry outside [-1, L) counts as -1 and is cleared.
 * The draw does not touch the env's numpy stream, so after a switch env i equals, bit for bit, a fresh env of the new
 * level whose stream was set to the state env i carried into that reset.  It is defined exactly:
 *   k      = (uint64)(env_offset + i) << 32 | level_draws[i]     (the env's global index; sharded = single process)
 *   h      = splitmix64 output at position k for `seed`:
 *            z = seed + (k + 1) * 0x9E3779B97F4A7C15;  z = (z ^ z >> 30) * 0xBF58476D1CE4E5B9;
 *            z = (z ^ z >> 27) * 0x94D049BB133111EB;  h = z ^ z >> 31              (all mod 2^64)
 *   w_l    = level_weights[l] if it is > 0, else 0 (NaN and negative weights count as 0)
 *   total  = w_0 + w_1 + ... in level order, float32;  target = float32(h >> 40) * 2^-24 * total, float32
 *   level  = the first l with w_l > 0 whose running float32 sum w_0 + ... + w_l exceeds target (the last such l
 *            if none does, which only an infinite weight can cause); level_draws[i] += 1.
 * Handles that never call this behave exactly as before it existed.  Snapshots of a handle with level changes on
 * carry env_level, next_level, level_draws, level_weights, seed and env_offset; restoring one needs a handle with
 * the same level count and level changes on, and adopts all of them.  Restoring a blob into a handle whose level
 * changes are on / off while the blob's were off / on fails with MWB_ESTATE. */
int mwb_enable_level_changes(mwb_handle* h, uint64_t seed, int32_t env_offset /* global index of env 0, >= 0 */);

/* Episode seeds (level replay: restart an env on a chosen seed when its episode ends, and know which seed every
 * finished episode ran).  Stands in for env.reset(seed=s) of the reference (gymnasium seeds self.np_random with
 * Generator(PCG64(SeedSequence(s))), miniworld.py:551), decided per env on the device instead of by a host call.
 * Valid on a handle with device resets (params and a reset program set: mwb_set_levels, or mwb_set_params and
 * mwb_set_program; MWB_ESTATE otherwise, since host-generated worlds keep their streams on the host, and when already
 * on).  It needs neither a level table nor level changes.  It allocates next_seed int64 [N] and episode_seed int64 [N],
 * both all -1, which the caller reads and writes in place through mwb_state_array (MWB_ARRAY_NEXT_SEED /
 * MWB_ARRAY_EPISODE_SEED), stream-ordered, without a sync.
 *
 * A seed is taken only at a reset: mwb_reset, and the next-step auto-reset inside mwb_step.  At every reset of env i,
 * before anything is drawn:
 *   1. if next_seed[i] >= 0: the env's numpy stream is replaced by the one SeedSequence(next_seed[i]) starts,
 *      episode_seed[i] = next_seed[i], and next_seed[i] is cleared to -1;
 *   2. otherwise the env continues its stream and episode_seed[i] = -1 (any negative next_seed counts as -1 and is
 *      cleared).
 * So env i then equals, bit for bit, a fresh env of its level after reset(seed=s): what mwb_seed with
 * bit_generator.state of Generator(PCG64(SeedSequence(s))) followed by mwb_reset gives.  With level changes on, the
 * level is resolved as before (the level draw never touches the env's stream): a reset that takes a pending level and
 * a pending seed equals a fresh env of the new level after reset(seed=s).  episode_seed names the running episode; after
 * a terminating step it still names the episode that ended, because the reset happens inside the next step.
 * The stream of seed s, 0 <= s < 2^63, all 32-bit values mod 2^32:
 *   entropy  = (s & 0xFFFFFFFF, s >> 32, 0, 0)       (SeedSequence pads the pool's input with zeros, so [s] for
 *                                                     s < 2^32 and [low, high] otherwise are both this)
 *   hashmix(v):  v ^= hc;  hc *= 0x931e8875;  v *= hc;  v ^= v >> 16      (hc starts at 0x43b0d7e5 and carries on
 *                                                                          through every call below)
 *   mix(x, y):   r = 0xca01f9dd * x - 0x4973f715 * y;  r ^= r >> 16
 *   pool[k]  = hashmix(entropy[k])                    for k = 0..3
 *   for src = 0..3, for dst = 0..3, src != dst:  pool[dst] = mix(pool[dst], hashmix(pool[src]))
 *   w[k]     = pool[k % 4] ^ hc';  hc' *= 0x58f38ded;  w[k] *= hc';  w[k] ^= w[k] >> 16      for k = 0..7,
 *              hc' starting at 0x8b51f9dd
 *   q[k]     = w[2k] | w[2k + 1] << 32                for k = 0..3 (uint64)
 *   inc      = (q[2] << 64 | q[3]) << 1 | 1           (mod 2^128)
 *   state    = 0;  state = state * M + inc;  state += q[0] << 64 | q[1];  state = state * M + inc
 *              (M = 0x2360ED051FC65DA44385DF649FCCF645);  has_uint32 = 0, uinteger = 0
 * Handles that never call this behave exactly as before it existed, and the addition changes no struct and no existing
 * entry point, so MWB_ABI_VERSION stays as it is and blobs of such handles restore as before.  Snapshots of a handle with episode seeds on carry
 * both arrays, are marked as such in the header, and a restore adopts them; restoring a blob into a handle whose
 * episode seeds are on / off while the blob's were off / on fails with MWB_ESTATE before anything else is compared. */
int mwb_enable_episode_seeds(mwb_handle* h);

/* Maze level (reference envs/maze.py): every episode's world is a translate-and-select of these
 * templates -- one grid cell and one connector room per neighbour direction, in the order of
 * maze.py:110 `orders = [(0, 1), (0, -1), (-1, 0), (1, 0)]` as (dj, di).  All records are for
 * cell (0, 0); the kernel adds (i, j) * pitch. */
typedef struct mwb_maze_desc {
  int32_t rows, cols;
  double pitch;                      /* room_size + gap_size                                       */
  mwb_room cell_room;
  mwb_quad cell_quads[6];            /* floor, ceiling, walls of edges 0..3                        */
  mwb_seg cell_segs[4];
  int32_t open_a[4], open_b[4];      /* edge opened in the current cell / in the neighbour          */
  mwb_room conn_room[4];             /* connector created by connect_rooms (miniworld.py:768-837)  */
  mwb_quad conn_quads[4][4];         /* floor, ceiling, two side walls                             */
  mwb_seg conn_segs[4][2];
  const double* cdf;                 /* [2 rows cols - 1] cumulative room_probs (list order fixed) */
} mwb_maze_desc;
int mwb_set_maze(mwb_handle* h, const mwb_maze_desc* maze);

/* Maze layouts (environment design: PAIRED's adversary writes the maze, ACCEL edits the walls of past levels and
 * replays them).  Valid after mwb_set_maze / mwb_set_level_maze on a handle with device resets; MWB_ESTATE when the
 * handle has no Maze level, resets on the host, or has the mode on already; MWB_ECAPACITY when some Maze level's
 * all-open maze does not fit the handle: for c = R C cells and E = R (C - 1) + (R - 1) C inner edges, max_rooms
 * c + E, max_quads 6c + 2E and max_segs 4c (a tree needs 2c - 1, 8c - 2 and 4c).  K2's per-level triangle capacity and
 * the HBM triangle lists are sized from the all-open bound from then on.
 *
 * A layout is uint8 [maze_rows][maze_cols], the maxima of mwb_maze_desc rows / cols over the handle's Maze levels.  Bit 0 of cell (j, i) opens the
 * wall to (j, i + 1), bit 1 the wall to (j + 1, i); cells outside a level's grid, bits that point outside it and the
 * other six bits are ignored.  Loops, isolated cells and unreachable goals are allowed.  Four arrays, all zero (and
 * the cells -1) at the call, read and written in place through mwb_state_array, stream-ordered, without a sync:
 *   next_maze uint8 [N][rows][cols]    layout of the env's next reset at a Maze level;
 *   next_maze_cells int32 [N][2]       (goal cell, agent cell) of that layout, each j * maze_cols + i, or -1 (an index
 *                                      outside the level's grid counts as -1): where the goal box / agent are placed;
 *   maze_pending uint8 [N]             nonzero: next_maze waits for the env's next reset at a Maze level;
 *   episode_maze uint8 [N][rows][cols] layout of each env's running episode, masked to its grid.
 * At every reset of env i (mwb_reset, and the next-step auto-reset inside mwb_step), after the level is resolved:
 *   1. at a Maze level with maze_pending[i] set: episode_maze[i] = next_maze[i] masked, maze_pending[i] = 0, and the
 *      world is built as this host code builds it (Maze._gen_world with options={"maze": ...}): the grid rooms row by
 *      row; for each cell in row-major order, connect_rooms(cell, cell + x, min_z, max_z) if bit 0 is set, then
 *      connect_rooms(cell, cell + z, min_x, max_x) if bit 1 is set; place_entity(Box(color="red"), room=goal cell's
 *      room or none); place_agent(room=agent cell's room or none).  No carve draws are made; textures, sky and light
 *      and the camera draws follow as at every reset.  The room pick probabilities are the env's own:
 *      p = areas / np.sum(areas) (numpy's pairwise summation), cdf = p.cumsum() / p.cumsum()[-1];
 *   2. at a Maze level without a pending layout: the random carve, as before, and episode_maze[i] records its topology
 *      (a connector from a cell in direction d sets the +x or +z bit of the cell on its -x / -z side).  Replaying such
 *      a layout builds the same walls but creates the connectors in another order, so the placement draws differ;
 *   3. at any other level: episode_maze[i] = 0, and a pending layout stays pending.
 * After a terminating step episode_maze still names the episode that ended, because the reset happens inside the next
 * step.  With episode seeds on, a layout, its two cells and a seed reproduce an episode exactly.  Handles that never
 * call this behave exactly as before it existed, and the addition changes no struct, so MWB_ABI_VERSION stays as it
 * is.  Snapshots of a handle with the mode on carry the four arrays and are marked as such in the header; restoring a
 * blob into a handle whose layouts are on / off while the blob's were off / on fails with MWB_ESTATE before anything
 * else is compared. */
int mwb_enable_maze_layouts(mwb_handle* h);

/* Start poses (reverse curricula, start-state curricula, goal-placement environment design).  Valid on a handle with
 * device resets (params and a reset program); MWB_ESTATE when the handle resets on the host or has the mode on already.
 * A pose is (x, z, dir) in float64.  Four arrays, read and written in place through mwb_state_array, stream-ordered,
 * without a sync; the designed rows are all NaN and the rest zero at the call:
 *   next_pose float64 [N][max_ents][3]   designed pose of each entity-list slot at the env's next reset;
 *   next_agent_pose float64 [N][3]       designed pose of the agent at the env's next reset;
 *   pose_pending uint8 [N]               nonzero: the rows wait for the env's next reset;
 *   episode_start float64 [N][3]         the agent's (x, z, dir) at the start of the env's running episode.
 * At every reset of env i (mwb_reset, and the next-step auto-reset inside mwb_step) with pose_pending[i] set, at any
 * level, pose_pending[i] = 0 and the level's program runs with these placements replaced (the rows stay as written):
 *   - the place_entity call that fills entity-list slot e (a PLACE op, or a PUT op that is not append-only) takes
 *     next_pose[i][e] when its x and z are finite; the agent's call (place_agent) takes next_agent_pose[i] when its x
 *     and z are finite, and otherwise its slot's row as any other call.  In a level table a slot is a slot of the
 *     level the reset runs; next_agent_pose is the agent at every level;
 *   - a designed call runs the reference's place_entity(pos=[x, y, z], dir=...) branch: y is the y of the pos the
 *     level passed (0 for a searched placement), dir is the designed dir when finite, else the dir the level passed,
 *     else uniform(-pi, pi) drawn from the env's stream.  No room is picked, no position searched and no collision
 *     checked, as in the reference; a pose outside the floor plan is kept as written.  A design that leaves a later
 *     searched placement of the same reset no free spot makes that search run forever, as it would in the reference;
 *   - every other draw (choices, sizes, other slots' searches, textures, sky and light, colours, camera) happens as
 *     before and in order, so with episode seeds on a seed and a design reproduce an episode;
 *   - a designed pose wins over the goal or agent cell of a designed maze (mwb_enable_maze_layouts) for that call.
 * Every reset writes the agent's pose into episode_start[i], designed or drawn; after a terminating step it still names
 * the episode that ended, because the reset happens inside the next step.  Handles that never call this behave
 * exactly as before it existed, and the addition changes no struct, so MWB_ABI_VERSION stays as it is.  Snapshots of
 * a handle with the mode on carry the four arrays and are marked as such in the header; restoring a blob into a handle
 * whose start poses are on / off while the blob's were off / on fails with MWB_ESTATE before anything else is
 * compared. */
int mwb_enable_start_poses(mwb_handle* h);

/* Reset draws (environment design over what an episode contains: object kinds and colours, box sizes, goal sides,
 * headings).  Valid on a handle with device resets (params and a reset program), before the state bank: MWB_ESTATE
 * when the handle resets on the host, has the mode on already or has the bank on.  A level's reset draws are the CHOICE
 * and UNIFORM ops of its program; op.room of each must hold its index d = 0, 1, ... in program order (MWB_EINVAL
 * otherwise), and D is the largest draw count over the handle's levels at the call (MWB_EINVAL when it is 0).  Three
 * arrays, read and written in place through mwb_state_array, stream-ordered, without a sync:
 *   next_draws float64 [N][D]      designed outcome of draw d at the env's next reset (all NaN at the call);
 *   draws_pending uint8 [N]        nonzero: the rows wait for the env's next reset (all 0 at the call);
 *   episode_draws float64 [N][D]   outcome of each draw of the env's running episode (all NaN at the call).
 * At every reset of env i (mwb_reset, and the next-step auto-reset inside mwb_step) that runs a program, at any level,
 * draws_pending[i] = 0 when it was set, and the rows stay as written.  With it set, each draw d of the level the reset
 * resolves to (after the level, seed and bank rules) is made from the env's stream as usual, and its result is then
 * replaced by next_draws[i][d] when that value lies in the draw's support: for a choice over n an integer in [0, n),
 * for a uniform over [lo, hi] a finite value with lo <= v <= hi.  Otherwise (NaN included) the drawn value stays.  So
 * the stream advances as without a design, a seed plus a design reproduces an episode, and a design only selects an
 * outcome the level can produce itself.  Rows beyond the level's draw count are ignored.  Every such reset writes the
 * outcome of each draw, designed or drawn, into episode_draws[i][d] (choices as exact integers) and NaN beyond the
 * level's count; after a terminating step it still names the episode that ended.  A designed start pose
 * (mwb_enable_start_poses) still wins for the position and dir of its placement.  A state-bank load consumes only
 * next_state: pending draws wait for the next reset that runs a program, and episode_draws is part of the record.
 * Handles that never call this behave exactly as before it existed, and the addition changes no struct, so
 * MWB_ABI_VERSION stays as it is.  Snapshots of a handle with the mode on carry the three arrays and are marked as such
 * in the header; restoring across the mode fails with MWB_ESTATE before anything else is compared. */
int mwb_enable_reset_draws(mwb_handle* h);

/* Env params (automatic domain randomisation with per-env boundary sampling, robustness sweeps over camera, lighting
 * and dynamics): give an env's next episode DomainParams of its own.  Valid on a handle with device resets (params and
 * a reset program), before the state bank: MWB_ESTATE when the handle resets on the host, has the mode on already or
 * has the bank on.  A params row is MWB_ENV_PARAM_ELEMS element rows in the order of mwb_params with each vector param
 * expanded element by element (sky_color[0..2] 0-2, light_pos 3-5, light_color 6-8, light_ambient 9-11,
 * obj_color_bias 12-14, forward_step 15, forward_drift 16, turn_step 17, cam_pitch 18, cam_fov_y 19, cam_height 20,
 * cam_fwd_disp 21); an element row is float64 (default, min, max).  Three arrays, read and written in place through
 * mwb_state_array, stream-ordered, without a sync:
 *   next_params float64 [N][22][3]     the row env i's next episode runs (all NaN at the call);
 *   params_pending uint8 [N]           nonzero: the row waits for the env's next reset (all 0 at the call);
 *   episode_params float64 [N][22][3]  the row of the env's running episode, all NaN when it runs its level's params.
 * At every reset of env i (mwb_reset, and the next-step auto-reset inside mwb_step) that runs a program, at any level,
 * after the level, seed and bank rules: with params_pending[i] set, params_pending[i] = 0 and next_params[i] is copied
 * into episode_params[i], the rows staying as written; otherwise episode_params[i] is set to all NaN.  The episode then
 * runs on its level's params merged with episode_params[i], element by element:
 *   - the range is the env's (min, max) when both are finite, else the level's; the default is the env's when finite,
 *     else the level's.  A range is lowered as lo = min and rng = max - min in float64 (numpy's uniform());
 *   - "the level's" means the level row as it stands at the reset for the params read at resets (sky, light,
 *     obj_color_bias, the camera params), and at every step for forward_step, forward_drift and turn_step, so that
 *     writes to MWB_ARRAY_LEVEL_PARAMS keep reaching every entry an episode did not design, mid-episode included;
 *   - max_forward_step (the near() threshold and the carry distance) is the env's forward_step max when that element's
 *     range applies, else the level's at the reset; the episode keeps it.
 * A design changes no draw count: under the level's domain_rand flag every element is still one uniform(), without it
 * only defaults are read, so the stream advances as without a design and a seed plus a design reproduces an episode.
 * (v, v, v) pins an element either way.  A range with min > max runs on the device only (lo + (max - min) * u with
 * a negative span); the reference and the drop-in class draw with numpy's Generator.uniform, which refuses it.  The goal distance
 * mode uses the merged max_forward_step for its near-goal nodes and the merged turn_step default for its expert.  A
 * state-bank load consumes only next_state: a pending row waits for the next reset that runs a program, and
 * episode_params is part of the record (528 B more per record).  Handles that never call this behave exactly as
 * before it existed, and the addition changes no struct, so MWB_ABI_VERSION stays as it is.  Snapshots of a handle
 * with the mode on carry the three arrays and are marked as such in the header; restoring across the mode fails with
 * MWB_ESTATE before anything else is compared.  Memory: 2 x 528 + 1 B per env for the arrays, plus a 536 B per-env
 * scratch for the merged row. */
#define MWB_ENV_PARAM_ELEMS 22
int mwb_enable_env_params(mwb_handle* h);

/* State bank (Go-Explore, backplay and demonstration-start curricula, branching rollouts): save env states into device
 * records and start an env's next episode from one.  Valid on a handle with device resets, after the level table, any
 * Maze levels and the other modes are set up: MWB_ESTATE when the handle resets on the host or has the bank on already,
 * and every later mwb_enable_* / mwb_set_levels / mwb_set_maze / mwb_set_level_maze call fails with MWB_ESTATE, because
 * the record layout depends on them.  MWB_EINVAL for slots < 1.  Allocates `slots` records and three int32 arrays,
 * read and written in place through mwb_state_array, stream-ordered, without a sync:
 *   next_state [N]         slot env i's next reset loads, -1 = none (all -1 at the call);
 *   episode_state [N]      slot the running episode was loaded from, -1 = it ran the level's program; after a
 *                          terminating step it still names the episode that ended;
 *   bank_level [slots]     level of the state each slot holds, -1 = empty (all -1 at the call; treat as read-only).
 * A record is everything a running episode is: the entity list (proto, pose, colour, size), num_slots, agent_slot,
 * carrying, step_count, the counter (CollectHealth's health), the camera, sky and light parameters, max_forward_step,
 * the ghost entity, the RNG stream, the env's room texture variants, env_level, the episode_seed / episode_maze /
 * episode_start / episode_draws records of the modes that are on and, when the saved env's level has per-env worlds, its world block
 * (the rooms, quads and segments in use).  Not in a record: needs_reset, the pending inputs (next_level, level_draws,
 * next_seed, the pending layout, cells, poses and draws), next_state, episode_state, episodes_done, the level table and its
 * params.
 * At every reset of env i (mwb_reset, and the next-step auto-reset inside mwb_step) with next_state[i] = s >= 0, before
 * anything else, next_state[i] = -1; then, when slot s exists and is filled and its level is the env's level or level
 * changes are on, env i becomes the record bit for bit (env_level included), episode_state[i] = s, and no program runs
 * and nothing is drawn: every other pending input stays pending for the next reset that runs a program.  Otherwise the
 * entry is dropped, the reset runs as it would have, and episode_state[i] = -1.  So a loaded env's future under the
 * same actions is the saved env's, its auto-resets included; the level's current params apply to its per-step draws,
 * and its step_count is the saved one.  Handles that never call this behave exactly as before it existed, and the
 * addition changes no struct, so MWB_ABI_VERSION stays as it is.  Snapshots of a handle with the bank carry the
 * records and the three arrays and are marked as such in the header; restoring across the mode fails with MWB_ESTATE,
 * and into a bank of another size with MWB_EINVAL. */
int mwb_enable_state_bank(mwb_handle* h, int32_t slots);
/* Copy env env_ids[t] into slot slots[t] for t in [0, n) and set bank_level[slots[t]] to the env's level.  A slot
 * named more than once takes its last entry.  Both arrays are host memory, checked here (MWB_EINVAL for an env or slot
 * out of range), or both device memory: then the call enqueues on `stream` (null: the handle's stream, and the call
 * returns finished) without a check on the host, and entries with an env or slot out of range are skipped on the
 * device.  MWB_ESTATE without the bank. */
int mwb_save_states(mwb_handle* h, const int32_t* env_ids, const int32_t* slots, int n, void* stream);

/* Goal distance (SPL, shortest-path filters of environment design, distance-shaped rewards, imitation): the geodesic
 * distance from every env's agent to its goal, the running episode's shortest path and an expert action, on the
 * device.  One grid per level, grids[l] for level l: node (k, l') of nx x nz sits at (min_x + (k + 0.5) h,
 * min_z + (l' + 0.5) h), h = MWB_GOAL_GRID_STEP, flat index l' * nx + k; goal_slot is the entity-list slot of the
 * goal of a level whose rule is near(goal) (MWB_RULE_GOAL), -1 for a level without one. */
#define MWB_GOAL_GRID_STEP 0.25
#define MWB_GOAL_GRID_CAP 65536        /* nodes of one grid */
typedef struct mwb_goal_grid {
  double min_x, min_z;
  int32_t nx, nz;
  int32_t goal_slot;         /* -1 = no goal rule: the level's envs report NaN / -1                */
  int32_t reserved;          /* 0                                                                  */
} mwb_goal_grid;
/* Valid on a handle with device resets and a level table or Maze level set up (MWB_ESTATE when it resets on the host
 * or has the mode on already; mwb_set_levels, mwb_set_maze and mwb_set_level_maze fail with MWB_ESTATE afterwards,
 * since the grids cover the levels' rooms).  MWB_EINVAL for a null array, a nonzero reserved field, no level with a
 * goal slot, a goal slot outside [0, max_ents) or a grid with nx or nz < 1; MWB_ECAPACITY for a grid of more than
 * MWB_GOAL_GRID_CAP nodes.  G is the largest grid (nx * nz) over the levels with a goal.  Arrays, read in place through
 * mwb_state_array, stream-ordered, all read-only:
 *   goal_dist float64 [N]        metres from the agent's pose after the last mwb_step / mwb_reset (NaN before the
 *                                first, and at levels without a goal);
 *   expert_action int32 [N]      0 turn_left, 1 turn_right, 2 move_forward, -1 = none;
 *   episode_shortest float64 [N] goal_dist right after the reset that started the running episode (a program reset
 *                                or a state-bank load); after a terminating step it still names the episode that ended;
 *   goal_field uint16 [N][G]     the env's distance field, in units of h / 5, 0xFFFF = unreachable or blocked.
 * A reset of env i (program or bank load) builds env i's field from its world as the reset left it, in a kernel that
 * follows the reset in mwb_reset and K1 in mwb_step; that kernel then writes goal_dist and expert_action of every env,
 * and episode_shortest of the envs it reset.  With r the agent prototype's radius, a node inside some room is a source
 * when an agent standing there is near(goal) (the rule's own threshold, walls ignored), and free when no wall lies
 * within r + h/2 and no entity other than the agent and the goal within r + h/2 + its radius.  Edges join free-or-source
 * 8-neighbours; orthogonal ones cost 5, diagonal ones 7 and need both orthogonal neighbours they pass free-or-source;
 * the field is the shortest-path distance from the nearest source, capped at 0xFFFE.  goal_dist is 0 when the agent is
 * near(goal), else the minimum over the free nodes with a finite field of the 4 x 4 block k0 - 1 .. k0 + 2 (k0 =
 * floor((x - min_x) / h - 0.5), same for z) of field * 0.05 + the straight distance, +inf when there is none.  The
 * expert heads for the goal when that node's field is 0 or the agent is near, else for the node's neighbour with the
 * least field + edge cost (ties: lowest flat index), moving forward when within half the level's default turn_step of
 * the heading to it and turning towards it otherwise.  mwb_restore rebuilds every field and keeps episode_shortest
 * from the blob.  Handles that never call this behave exactly as before it existed, and the addition changes no
 * existing struct, so MWB_ABI_VERSION stays as it is.  Snapshots of a handle with the mode on carry episode_shortest
 * and are marked as such in the header; restoring across the mode fails with MWB_ESTATE. */
int mwb_enable_goal_distance(mwb_handle* h, const mwb_goal_grid* grids /* [n_levels] */);

/* Maze levels in a level table (curricula over maze sizes: MazeS2 -> MazeS3 -> Maze, next to fixed-layout levels).
 * Valid on a shared_geometry = 1 handle after mwb_set_levels (MWB_ESTATE otherwise).  Level `level` (MWB_EINVAL
 * outside [0, L)) becomes a per-env-world level: every reset of an env at that level carves a fresh maze from these
 * templates into the env's own world, as mwb_set_maze does for a one-level handle.  MWB_ECAPACITY when the maze has more
 * than MWB_MAZE_MAX_CELLS (256) cells or does not fit max_rooms (2c - 1 for c cells), max_quads (8c - 2) or max_segs
 * (4c).  The first call adds one world block per env after the L templates (every env, since level changes can move
 * any env into a maze level) and fixes the level table (mwb_set_levels returns MWB_ESTATE from then on).  An env's
 * world holds its last maze until its next reset; envs at template levels read their level's template.
 * K2 then keeps each level's triangle lists in shared memory or HBM by the level's own size (levels above 512 triangle
 * records: HBM), and snapshots carry the per-env worlds, marked as such in the header (a restore into a handle without
 * per-env worlds, or the other way round, fails with MWB_ESTATE before anything else is compared). */
int mwb_set_level_maze(mwb_handle* h, int level, const mwb_maze_desc* maze);

/* static geometry of one env as currently on the device (tests, debugging); arrays sized by the
 * handle's max_rooms / max_quads / max_segs */
int mwb_get_geometry(mwb_handle* h, int env, int32_t counts[3], mwb_room* rooms, mwb_quad* quads, mwb_seg* segs);

/* ---- reset: MiniWorldEnv.reset (miniworld.py:544-604) ----------------------------------
 * mwb_seed      = gym.Env.reset(seed=...): installs Generator(PCG64(SeedSequence(seed))) state
 * mwb_reset     = device-side reset of the listed envs with the lowered program (RNG on device)
 * mwb_set_world = host-generated world for the listed envs (any level, any _gen_world)       */
int mwb_seed(mwb_handle* h, const int32_t* env_ids, int n, const mwb_rng_state* states);
int mwb_reset(mwb_handle* h, const int32_t* env_ids /*NULL = all*/, int n, void* stream);
int mwb_set_world(mwb_handle* h, const int32_t* env_ids, int n, const mwb_world* worlds);

/* ---- the hot path: MiniWorldEnv.step (miniworld.py:670-730) + level rule + render_obs
 * (:1177-1221) [+ render_depth (:1223-1236)] for all N envs.
 *   actions      int32[N]          (host or device)
 *   step_params  double[N][3] or NULL: forward_step, forward_drift, turn_step drawn by the
 *                caller (single-env host-RNG path); NULL = defaults / device RNG (:677-680)
 *   obs          uint8[N][H][W][3] or NULL (skip rendering)
 *   depth        float[N][H][W]    or NULL
 *   reward       double[N], terminated / truncated uint8[N]  (may be NULL)                    */
int mwb_step(mwb_handle* h, const int32_t* actions, const double* step_params, uint8_t* obs,
             float* depth, double* reward, uint8_t* terminated, uint8_t* truncated, void* stream);

/* Observation layout written by the render kernel's epilogue (all `obs` arguments of this header):
 *   MWB_OBS_HWC_U8    uint8 [N][H][W][3]  MiniWorldEnv.render_obs (default)
 *   MWB_OBS_CWH_U8    uint8 [N][3][W][H]  PyTorchObsWrapper.observation: transpose(2, 1, 0) (wrappers.py:24-25)
 *   MWB_OBS_GREY_F64  double [N][H][W][1] GreyscaleWrapper.observation: 0.30 R + 0.59 G + 0.11 B in float64,
 *                                         as numpy evaluates it on the uint8 frame (wrappers.py:43-46)      */
#define MWB_OBS_HWC_U8 0
#define MWB_OBS_CWH_U8 1
#define MWB_OBS_GREY_F64 2
int mwb_set_obs_format(mwb_handle* h, int format);

/* StochasticActionWrapper (reference wrappers.py:49-71) applied inside mwb_step: before an env steps, one
 * np_random.uniform() is drawn from ITS stream; if it is not below `prob` the action is replaced by
 * `random_action`, or, when that is negative, by np_random.integers(0, 6).  Envs that reset in this
 * step draw nothing.  enabled = 0 turns it off (the default). */
int mwb_set_action_noise(mwb_handle* h, int enabled, double prob, int random_action);

/* render_obs / render_depth without stepping (observation returned by reset()) */
int mwb_render_obs(mwb_handle* h, uint8_t* obs, float* depth, void* stream);

/* render_top_view (miniworld.py:1088-1175): orthographic map of every env, rendered at the handle's
 * observation size with its MSAA setting.  extents = {min_x, max_x, min_z, max_z} as the reference
 * has them after the aspect-ratio adjustment (:1109-1133), i.e. glOrtho(min_x, max_x, -max_z, -min_z,
 * -100, 100); render_agent != 0 also draws Agent.render()'s marker triangle (entity.py:518-539).
 *   obs          uint8[N][H][W][3] (host or device)                                             */
int mwb_render_top_view(mwb_handle* h, const double extents[4], int render_agent, uint8_t* obs, void* stream);

/* get_visible_ents (miniworld.py:1238-1333): occlusion queries of a 0.2 m box at every entity
 * against the rooms, at the observation frame buffer's resolution and sample count.
 *   mask         uint32[N] (host or device): bit e = entity-list slot e passed its query          */
int mwb_visible_ents(mwb_handle* h, uint32_t* mask, void* stream);

/* ---- designed cameras: views of every env from poses the caller writes ------------------------------
 * A pose row is (x, z, dir), float64, with the level's heading convention dir_vec = (cos dir, 0, -sin dir).
 * The view of env i from row (x, z, dir) is exactly what the reference's render_obs() / render_depth() return
 * after agent.pos = (x, agent.pos[1], z) and agent.dir = dir with nothing else changed: the same entity list (a
 * carried object at its own pose), textures, sky, light and the running episode's cam_height, cam_fwd_disp,
 * cam_pitch and cam_fov_y.  The agent's body is not drawn (render_obs's render_agent=False); render_agent != 0
 * additionally draws Agent.render()'s marker triangle (entity.py:518-539) at the agent's REAL pose in the state,
 * as the top view does: a third-person view.  Frame size, MSAA and observation format are the handle's own.
 * A row with any non-finite entry, or with |dir| >= 105414350 (the range in which the glibc-exact sin / cos are
 * validated; reduce headings modulo 2 pi first), is skipped: that env's frame and depth in that view are left
 * untouched and no camera is computed for it.
 * Neither call changes any env state.
 *   poses        float64[views][N][3] (host or device)
 *   obs          frames [views][N] in the observation format (host or device), or NULL for depth only
 *   depth        float32[views][N][H][W] (host or device) or NULL
 * Host destinations go through the handle's staging one view at a time; device ones are written in place on
 * `stream` without a host sync. */
int mwb_render_views(mwb_handle* h, const double* poses, int views, int render_agent, uint8_t* obs, float* depth,
                     void* stream);

/* get_visible_ents (as mwb_visible_ents) with the agent moved to env i's row of poses float64[N][3] (host or
 * device) as mwb_render_views defines it; a skipped row leaves mask[i] as it is. */
int mwb_visible_ents_from(mwb_handle* h, const double* poses, uint32_t* mask, void* stream);

/* ---- designed cameras with their own intrinsics, frame size and sample count --------------------------
 * mwb_render_views with rows of row_width 3 or 7 columns, rendered at width x height with `samples` samples per
 * pixel (1, 4, 8 or 16).  A 7-column row is (x, z, dir, cam_height, cam_fwd_disp, cam_pitch, cam_fov_y): the view
 * of env i is what the reference's render_obs(FrameBuffer(width, height, samples)) / render_depth(...) return after
 * agent.pos = (x, agent.pos[1], z), agent.dir = dir and each camera attribute set to the row's value, nothing else
 * changed.  NaN in columns 3-6 means the running episode's value (the one its reset drew, or the merged env params
 * value): an all-NaN 7-column row renders the same bytes as its 3-column row.  Besides the 3-column skip rule, a
 * 7-column row is skipped when an intrinsic column is +-inf, a given cam_fov_y lies outside (0, 180) or a given
 * |cam_pitch| >= 90 (gluLookAt's basis is undefined at 90).  Frames come back in the observation format at
 * width x height: obs [views][N] frames of that size, depth float32[views][N][height][width].  Host destinations
 * use the handle's staging, which grows on the first call at a larger size and is never shrunk.
 * mwb_render_views(h, poses, views, ...) is mwb_render_views_at(h, poses, 3, views, obs_width, obs_height,
 * msaa_samples, ...). */
int mwb_render_views_at(mwb_handle* h, const double* rows, int row_width, int views, int width, int height, int samples,
                        int render_agent, uint8_t* obs, float* depth, void* stream);

/* mwb_visible_ents_from with rows float64[N][row_width], row_width 3 or 7, as mwb_render_views_at defines them.  The
 * reference's get_visible_ents always renders into obs_fb, so the query uses the row's camera attributes but the
 * handle's own frame size and sample count. */
int mwb_visible_ents_from_at(mwb_handle* h, const double* rows, int row_width, uint32_t* mask, void* stream);

/* ---- state exchange (env.agent.pos, env.entities[i].pos ... views; checkpointing) ------ */
int mwb_get_state(mwb_handle* h, const mwb_state_view* out);

/* ---- checkpointing: the complete restorable state of all N envs (entity lists, counters, camera and
 * lighting parameters, numpy streams, pending auto-resets, geometry on the device, the level params table and each
 * env's max_forward_step) as one host blob.
 * Restoring into a handle created with the same configuration and level definition resumes every env
 * bit for bit.  (The reference has no equivalent: its state lives in Python objects.)  The blob of a handle with
 * several levels also carries env_level; restoring it into a handle with another level count or assignment fails
 * with MWB_ESTATE (handles with level changes on: see mwb_enable_level_changes; their blobs are marked as such in the
 * header, and a blob whose mark differs from the handle's mode is refused with MWB_ESTATE before anything else is
 * compared; the same holds for episode seeds, mwb_enable_episode_seeds). */
int mwb_snapshot_size(mwb_handle* h, size_t* bytes);
int mwb_snapshot(mwb_handle* h, void* blob, size_t bytes);
int mwb_restore(mwb_handle* h, const void* blob, size_t bytes);

/* number of kernels this handle has launched so far (bench.py's gpu_launches) */
int64_t mwb_launch_count(mwb_handle* h);

/* capacity faults (must stay 0): frames whose culled triangle list did not fit the kernel's budget, frames that keep
 * more than 65 535 triangles after culling (triangle ids are 16-bit and 0xFFFF is the sky: about 26 full Balls in
 * view; such a frame renders wrong), device-side maze generation that ran out of room / quad / segment capacity (the
 * env is left empty instead of searching forever) */
int64_t mwb_overflow_count(mwb_handle* h);

/* Device-side timing of the two kernels: when enabled, every K1 / K2 launch is bracketed by
 * CUDA events on the launching stream; mwb_profile_read synchronises, returns the summed
 * milliseconds and launch counts since the last read, and clears them (bench.py roofline). */
int mwb_profile(mwb_handle* h, int enable);
int mwb_profile_read(mwb_handle* h, double* k1_ms, double* k2_ms, int64_t* k1_launches, int64_t* k2_launches);

/* ---- peer-memory observation buffer (multi-GPU, SURVEY 8e "fused option") ---------------
 * One process per GPU: rank 0 allocates the global observation buffer with mwb_shared_alloc and
 * publishes its 64-byte CUDA IPC handle; the other ranks map it with mwb_shared_open and pass
 * `mapped + start_env * H * W * 3` as the `obs` argument of mwb_step, so K2's row-segment stores
 * land directly in rank 0's HBM over NVLink -- the gather collective disappears.  */
int mwb_shared_alloc(int device, size_t bytes, void** dev_ptr, unsigned char handle[64]);
int mwb_shared_open(int device, const unsigned char handle[64], void** dev_ptr);
int mwb_shared_close(void* dev_ptr, int opened /* 1: from mwb_shared_open, 0: from mwb_shared_alloc */);
/* Tell the handle whether the `obs` pointer of the following mwb_step / mwb_render_obs calls is another GPU's memory
 * (1), local memory (0), or to look it up per pointer (-1, the default).  For a peer destination K2 stages each
 * frame (or band of a frame) in shared memory and writes it out as address-ordered 16-byte stores, which is what NVLink
 * needs; for local HBM it stores row segments directly. */
int mwb_set_obs_peer(mwb_handle* h, int peer);

/* The camera K2 derives for every env, read back for parity tests against the reference's Agent.cam_pos / cam_dir /
 * cam_fov_y (entity.py:476-503) and its gluLookAt / gluPerspective arguments (miniworld.py:1200-1219): per env 16
 * floats -- eye[3], right s[3], up u[3], forward f[3], projection scales (cot / aspect, cot), z_clip = za w - zb. */
int mwb_debug_camera(mwb_handle* h, float* out /* host [num_envs][16] */);

/* Device address of a per-env state array (valid for the handle's lifetime; contents are stream-ordered behind
 * mwb_step / mwb_reset on the stream they were given).  Lets the host side expose what the reference's level step()s
 * put into `info` without a state copy: info["health"] (envs/collecthealth.py:100) = MWB_ARRAY_COUNTER, the same
 * counter PickupObjects keeps as num_picked_up (envs/pickupobjects.py:88); info["goal_pos"] (envs/tmaze.py:89) = rows
 * of MWB_ARRAY_ENT_X/Y/Z ([max_ents][num_envs], entity-list slot major). */
#define MWB_ARRAY_COUNTER 0      /* int32   [num_envs]            */
#define MWB_ARRAY_STEP_COUNT 1   /* int32   [num_envs]            */
#define MWB_ARRAY_ENT_X 2        /* float64 [max_ents][num_envs]  */
#define MWB_ARRAY_ENT_Y 3
#define MWB_ARRAY_ENT_Z 4
#define MWB_ARRAY_ENT_DIR 5
/* with level changes on (mwb_enable_level_changes; MWB_ESTATE otherwise): */
#define MWB_ARRAY_ENV_LEVEL 6       /* int32   [num_envs]  level of each env's current episode                   */
#define MWB_ARRAY_NEXT_LEVEL 7      /* int32   [num_envs]  pending assignment for the next reset, -1 = none      */
#define MWB_ARRAY_LEVEL_WEIGHTS 8   /* float32 [n_levels]  sampling weights of the next resets                   */
/* on every handle with device resets (params and a reset program set; MWB_ESTATE otherwise, e.g. for a handle whose
 * envs only ever get host-generated worlds through mwb_set_world), with or without level changes: */
#define MWB_ARRAY_LEVEL_PARAMS 9    /* mwb_params [n_levels]  each level's DomainParams, count = n_levels records   */
/* MWB_ARRAY_LEVEL_PARAMS: the level table's DomainParams, which mwb_set_params / mwb_set_levels fill and which the
 * caller may then rewrite in place while the batch runs (automatic domain randomisation: widen a range once the
 * policy succeeds at its edge), stream-ordered like LEVEL_WEIGHTS: a write enqueued on the stream of the next
 * mwb_step / mwb_reset is seen by it.  Level l's row is what MiniWorldEnv.params is to every env whose current episode
 * runs level l (reference miniworld.py:576-585, 677-680), and when each field is read decides when a write applies:
 *   - forward_step, forward_drift, turn_step (default, _lo, _rng): read by mwb_step at every step, so a write applies
 *     from the next step of every env of the level, mid-episode included (domain_rand on: uniform(lo, lo + rng),
 *     off: the default);
 *   - sky_color, light_pos, light_color, light_ambient, obj_color_bias, cam_height, cam_fwd_disp, cam_pitch,
 *     cam_fov_y: read only at resets, so a write applies from each env's next reset; a running episode keeps the
 *     values it drew (mwb_state_view cam / env_params, entity colours);
 *   - max_forward_step: read only at resets too.  Each env keeps the value its last reset took (self.max_forward_step,
 *     miniworld.py:581) for its near() thresholds (1.1 * max_forward_step, :975) and the carry position (:611), so an
 *     episode in progress keeps its threshold.  Whoever writes raw rows must keep it equal to forward_step's max
 *     (forward_step_lo + forward_step_rng as the reference's params.get_max("forward_step") would return it).
 * Every _rng must be the float64 difference max - min (numpy's uniform(low, high) is low + (high - low) * random(),
 * with high - low rounded once).  The domain_rand flag stays table data.  A handle whose rows are never written runs
 * exactly as before.  Snapshots carry the table and every env's max_forward_step, and a restore adopts both. */
/* with episode seeds on (mwb_enable_episode_seeds; MWB_ESTATE otherwise); ids 10 to 15 stay unknown (MWB_EINVAL), free
 * for further level-table arrays: */
#define MWB_ARRAY_NEXT_SEED 16      /* int64   [num_envs]  seed of the env's next reset, negative = none           */
#define MWB_ARRAY_EPISODE_SEED 17   /* int64   [num_envs]  seed the env's current episode started from, or -1    */
/* with maze layouts on (mwb_enable_maze_layouts; MWB_ESTATE otherwise); count = elements, rows x cols per env: */
#define MWB_ARRAY_NEXT_MAZE 18        /* uint8 [num_envs][rows][cols]  layout of the env's next reset at a Maze level */
#define MWB_ARRAY_NEXT_MAZE_CELLS 19  /* int32 [num_envs][2]  goal cell, agent cell of that layout, -1 = random       */
#define MWB_ARRAY_MAZE_PENDING 20     /* uint8 [num_envs]  nonzero = next_maze waits for a reset at a Maze level       */
#define MWB_ARRAY_EPISODE_MAZE 21     /* uint8 [num_envs][rows][cols]  layout of the env's running episode            */
/* with start poses on (mwb_enable_start_poses; MWB_ESTATE otherwise); count = elements: */
#define MWB_ARRAY_NEXT_POSE 22        /* float64 [num_envs][max_ents][3]  designed (x, z, dir) per slot, next reset   */
#define MWB_ARRAY_NEXT_AGENT_POSE 23  /* float64 [num_envs][3]  designed (x, z, dir) of the agent, next reset         */
#define MWB_ARRAY_POSE_PENDING 24     /* uint8 [num_envs]  nonzero = the designed poses wait for the next reset       */
#define MWB_ARRAY_EPISODE_START 25    /* float64 [num_envs][3]  the agent's (x, z, dir) when the episode started      */
/* with the state bank on (mwb_enable_state_bank; MWB_ESTATE otherwise): */
#define MWB_ARRAY_NEXT_STATE 26       /* int32 [num_envs]  slot the env's next reset loads, -1 = none                  */
#define MWB_ARRAY_EPISODE_STATE 27    /* int32 [num_envs]  slot the running episode was loaded from, -1 = none         */
#define MWB_ARRAY_BANK_LEVEL 28       /* int32 [slots]  level of the state each slot holds, -1 = empty                 */
/* with reset draws on (mwb_enable_reset_draws; MWB_ESTATE otherwise); count = elements, D per env: */
#define MWB_ARRAY_NEXT_DRAWS 29       /* float64 [num_envs][D]  designed outcome of each reset draw, next reset        */
#define MWB_ARRAY_DRAWS_PENDING 30    /* uint8 [num_envs]  nonzero = the designed draws wait for the next reset        */
#define MWB_ARRAY_EPISODE_DRAWS 31    /* float64 [num_envs][D]  outcome of each reset draw of the running episode      */
/* with goal distance on (mwb_enable_goal_distance; MWB_ESTATE otherwise), read-only; count = elements: */
#define MWB_ARRAY_GOAL_DIST 32        /* float64 [num_envs]  geodesic metres from the agent to the goal                 */
#define MWB_ARRAY_EXPERT_ACTION 33    /* int32 [num_envs]  action along the shortest path, -1 = none                   */
#define MWB_ARRAY_EPISODE_SHORTEST 34 /* float64 [num_envs]  goal_dist right after the running episode's reset          */
#define MWB_ARRAY_GOAL_FIELD 35       /* uint16 [num_envs][G]  distance field in units of h / 5, 0xFFFF = none          */
/* with env params on (mwb_enable_env_params; MWB_ESTATE otherwise); count = elements: */
#define MWB_ARRAY_NEXT_PARAMS 36      /* float64 [num_envs][22][3]  (default, min, max) rows of the next episode       */
#define MWB_ARRAY_PARAMS_PENDING 37   /* uint8 [num_envs]  nonzero = next_params waits for the env's next reset        */
#define MWB_ARRAY_EPISODE_PARAMS 38   /* float64 [num_envs][22][3]  rows of the running episode, NaN = the level's      */
int mwb_state_array(mwb_handle* h, int which, void** dev_ptr, int64_t* count);
/* 1 when this library keeps the handle's state arrays (mwb_state_array) in host memory -- the CPU build of the kernels
 * used by the test suite -- and 0 for libmwb.so, whose arrays are device memory. */
int mwb_state_in_host_memory(void);

/* ---- one-way completion flags for the multi-GPU observation path (SURVEY 8e) --------------
 * The reference has no counterpart (it has no multi-device path at all, README.md:34); these replace the per-step
 * rendezvous a gather collective would impose.  mwb_flag_write enqueues, on `stream`, a 32-bit store of `value` to
 * `dev_ptr` (device memory of this or -- through mwb_shared_open -- of another GPU) that becomes visible system-wide
 * only after everything enqueued before it on the stream, including a kernel's peer stores.  mwb_flag_wait_geq makes
 * `stream` wait until *dev_ptr - value >= 0 (wrap-around compare).  mwb_flag_mode: 0 = CUDA stream memory operations,
 * 1 = one-thread kernels (MWB_FLAG_MODE=kernel, or a driver without stream memory operations). */
int mwb_flag_write(void* cuda_stream, uint32_t* dev_ptr, uint32_t value);
int mwb_flag_wait_geq(void* cuda_stream, const uint32_t* dev_ptr, uint32_t value);
int mwb_flag_mode(void);

/* sizeof() of every ABI struct, in declaration order (config, params, tex_desc, mesh_desc,
 * room, quad, seg, proto, entity, op, geometry, world, rng_state, state_view, maze_desc, level, goal_grid): lets a
 * binding verify its mirror of this header.  Returns the number of entries written. */
int mwb_abi_sizes(int32_t* out, int cap);

#ifdef __cplusplus
}
#endif
#endif /* MWB_H_ */
