// state.h -- the flat structure-of-arrays holding N independent environments in HBM.
//
// Layout rule: every per-env scalar is an array [N] (env index fastest) so that the
// one-thread-per-env physics kernel reads and writes fully coalesced; per-entity fields are
// [max_ents][N].  Static room geometry is one shared template per level (levels without per-episode
// topology) followed, when some level is a Maze, by one world block per env; geom_index picks the block
// from the env's level.  Nothing here is ever
// re-laid-out between kernels: the physics kernel and the rasteriser read the same arrays.
#pragma once
#include "../../include/mwb.h"
#include "np_rng.cuh"

#define MWB_MAX_BINS 640         // half-tiles of one entity's screen box that can be binned (160x120 frame: 600)
#define MWB_BIN_REFS 6           // bin references per listed triangle the index buffer has room for

// K1 runs an env's scalar logic on all 32 lanes of a warp with identical values (every store writes the same value).
// The read-modify-write sequences on per-env state (step counter, RNG stream, entity list edits, level resolution) rely
// on the lanes not drifting apart between the loads and the stores: explicit warp barriers pin that down.
#ifdef __CUDA_ARCH__
#define MWB_WARP_SYNC() __syncwarp()
#else
#define MWB_WARP_SYNC()
#endif

// The maze layout arrays (mwb_enable_maze_layouts).  A layout is rows x cols bytes (the maxima over the handle's Maze
// levels), bit 0 of cell (j, i) opening its +x wall, bit 1 its +z wall.
struct MazeLayouts {
  uint8_t* next;                // [N][rows][cols] layout the env's next reset at a Maze level builds
  int32_t* cells;               // [N][2] goal cell, agent cell of that layout (j * cols + i), -1 = random
  uint8_t* pending;             // [N] 1 = next[i] waits for the env's next reset at a Maze level
  uint8_t* episode;             // [N][rows][cols] layout of the env's running episode (zeros: no maze)
  int32_t rows, cols;
};

// The start pose arrays (mwb_enable_start_poses).  A pose is (x, z, dir); a row applies when its x and z are finite,
// and its dir when that is finite too.
struct StartPoses {
  double* next;                 // [N][E][3] designed pose of each entity-list slot at the env's next reset
  double* next_agent;           // [N][3] designed pose of the agent at the env's next reset (wins over its slot's row)
  uint8_t* pending;             // [N] 1 = the rows wait for the env's next reset
  double* episode;              // [N][3] the agent's pose at the start of the env's running episode
};

// The reset draw arrays (mwb_enable_reset_draws).  A level's reset draws are the CHOICE and UNIFORM ops of its program,
// op.room holding draw d's index; D is the largest draw count over the handle's levels.
struct ResetDraws {
  double* next;                 // [N][D] designed outcome of draw d at the env's next reset (NaN: draw as usual)
  uint8_t* pending;             // [N] 1 = the rows wait for the env's next reset
  double* episode;              // [N][D] outcome of each draw of the env's running episode, NaN beyond the level's count
  int32_t D, pad_;
};

// The env params arrays (mwb_enable_env_params).  A row is MWB_ENV_PARAM_ELEMS element rows of (default, min, max).
#define MWB_ENV_PARAM_WORDS (MWB_ENV_PARAM_ELEMS * 3)
struct EnvParams {
  double* next;                 // [N][22][3] row the env's next reset takes
  uint8_t* pending;             // [N] 1 = next[i] waits for the env's next reset
  double* episode;              // [N][22][3] row of the env's running episode (NaN: the level's)
  mwb_params* merged;           // [N] scratch: the level row merged with episode[i], written before every read
};

// The goal distance arrays (mwb_enable_goal_distance); navigation.cuh builds and reads them.
struct GoalNav {
  const mwb_goal_grid* grids;   // [levels]
  uint16_t* field;              // [N][G] distance field of the env's running episode, units of h / 5
  uint8_t* node_class;          // [N][G] MWB_NAV_* bits of each node (the field alone does not tell a source that is not free)
  uint8_t* dirty;               // [N] 1 = reset since the last build (episode_shortest follows), other nonzero = rebuild only
  double* goal_dist;            // [N]
  int32_t* expert;              // [N]
  double* shortest;             // [N]
  int32_t G, pad_;
};

// One scalar of an env's state in a state-bank record: env i's copy lives at base + i * env_stride (a per-env row of
// the structure of arrays, or an element of an [N][k] array), the record's at byte rec_off; bytes is 1, 4 or 8.
struct BankCol {
  uint8_t* base;
  int32_t env_stride;
  int32_t rec_off;
  int32_t bytes;
  int32_t pad_;
};

// The state bank (mwb_enable_state_bank).  A record is rec_bytes bytes, 16-byte aligned: the BankCol scalars in record
// order, then, on handles with per-env worlds, the world section at world_off: int32 {rooms, quads, segments in use,
// 1 = the record holds a world}, then room, quad and segment arrays of the handle's capacities at room_off / quad_off /
// seg_off.  The geometry addresses are the handle's, which no call can replace once the bank is on.
struct StateBank {
  uint8_t* records;             // [slots][rec_bytes]
  int32_t* bank_level;          // [slots] level of the state a slot holds, -1 = empty
  int32_t* next_state;          // [N] slot the env's next reset loads, -1 = none
  int32_t* episode_state;       // [N] slot the running episode was loaded from, -1 = the level's program ran
  const BankCol* cols;          // [num_cols] in record order
  int32_t num_cols, slots;
  int64_t rec_bytes;
  int32_t world_off, room_off, quad_off, seg_off;   // world_off -1: the handle has no per-env worlds
  int32_t env_geom, R, Q, S;
  int32_t *num_rooms, *num_quads, *num_segs;
  mwb_room* rooms;
  mwb_quad* quads;
  mwb_seg* segs;
};

struct TriRec;
struct MeshSegInfo;
struct MazeDev;

// One row of the level table (mwb_set_levels): what K1 reads per env instead of per handle.  The row's DomainParams
// live apart from it, in DevState::level_params, which callers may rewrite while the batch runs.
struct LevelDev {
  int32_t rule_kind, rule_arg;
  int32_t max_episode_steps;
  int32_t op_first, num_ops;    // slice of DevState::ops
  int32_t maze;                 // index of the level's Maze templates in DevState::maze / maze_cdf, -1 = none
  int32_t env_worlds;           // 1: every env of the level has its own world (geometry block env_geom + i)
  int32_t tri_cap;              // K2: room + box triangle records one frame of the level can keep
  int32_t tris_hbm;             // K2: 1 = those records live in DevState::room_tris, 0 = in shared memory
  int32_t domain_rand;          // MiniWorldEnv(domain_rand=...) of the level: per-step and reset draws of its envs
};

struct DevState {
  int32_t N, E, R, Q, S;        // envs, entity slots, room / quad / segment capacity
  int32_t env_geom;             // geometry block of env 0's own world (after the level templates)
  int32_t obs_w, obs_h, msaa;

  // ---- dynamic per-env state ----
  int32_t* ent_proto;           // [E][N]  -1 = empty / removed
  double* ent_px;               // [E][N]
  double* ent_py;
  double* ent_pz;
  double* ent_dir;
  double* ent_col;              // [E][3][N]  Box colour after randomize
  double* ent_size;             // [E][N]  per-episode Box edge length drawn by the level (PutNext); 0 = the prototype's
  int32_t* num_slots;           // [N] entity-list length
  int32_t* agent_slot;          // [N]
  int32_t* carrying;            // [N] slot or -1
  int32_t* step_count;          // [N]
  int32_t* num_picked;          // [N]
  int32_t* needs_reset;         // [N] set by a terminated|truncated step when autoreset
  unsigned long long* episodes_done;   // [1] device counter of episode-ending steps
  int32_t* fault;               // [1] capacity faults: K2 triangle lists that overflowed or needed more than MWB_MAX_SLOTS
                                //     slots, device world generation that ran
                                //     out of room / quad / segment capacity (mwb_overflow_count; must stay 0)
  double* cam;                  // [4][N]  cam_height, cam_fwd_disp, cam_pitch, cam_fov_y
  double* envp;                 // [12][N] sky_color, light_pos, light_color, light_ambient
  double* env_mfs;              // [N] max_forward_step the env's last reset took (miniworld.py:581): near() and the
                                //     carry position read it, so an episode keeps it when its level's ranges change
  // object removed by the level rule AFTER this step's observation (pickupobjects.py:86-90)
  int32_t* ghost_slot;          // [N] -1 = none
  int32_t* ghost_proto;         // [N]
  double* ghost_pose;           // [4][N] x, y, z, dir
  double* ghost_col;            // [3][N]
  // numpy PCG64 stream
  uint64_t* rng_s_hi;
  uint64_t* rng_s_lo;
  uint64_t* rng_inc_hi;
  uint64_t* rng_inc_lo;
  int32_t* rng_has32;
  uint32_t* rng_cache;

  // ---- geometry: [env_geom + N][capacity] -- one template per level, then one world per env when some level has
  //      per-env worlds (shared_geometry = 0 handles: env_geom = 0, worlds only; template-only handles: no worlds) ----
  int32_t* num_rooms;           // [blocks]
  int32_t* num_quads;
  int32_t* num_segs;
  mwb_room* rooms;
  mwb_quad* quads;
  mwb_seg* segs;
  int32_t* room_tex;            // [N][R][3] texture id in use (domain-rand variants)

  // ---- per-frame mesh triangle lists written by mesh_setup_kernel: [N][E][mesh_cap] ----
  TriRec* mesh_tris;
  MeshSegInfo* mesh_seg;        // [N][E]
  uint2* mesh_bbox;             // [N][E][mesh_cap] packed (bx, by) of each listed triangle, coalesced for the tile scan
  // the same lists binned by half-tile of the entity's screen box (mesh_setup_kernel): bin b holds
  // mesh_bin_idx[mesh_bin_off[b] .. mesh_bin_off[b + 1]) = triangles that can touch that half-tile
  uint16_t* mesh_bin_idx;       // [N][E][MWB_BIN_REFS * mesh_cap]
  int32_t* mesh_bin_off;        // [N][E][MWB_MAX_BINS + 1]
  int32_t mesh_cap;             // 0 = the level has no mesh entities
  // per-frame trigonometry, written by frame_trig_kernel right before every render launch: the glibc-exact
  // cos / sin of the camera's three angles and of every entity slot's model rotation (one thread each), so that
  // neither K2's nor mesh_setup_kernel's blocks wait for a thread that evaluates them
  double* cam_trig;             // [6][N]  cos, sin of heading, pitch, half field of view
  float* ent_cs;                // [E][2][N]  cos, sin of the slot's glRotatef angle (the form its prototype's render() uses)
  const float* depth_lut;       // [65536] depth16 code -> metres (depth_code_to_metres of every code), or null
  TriRec* room_tris;            // [N][parts][tri_cap] room + box triangle lists in HBM for the envs of levels whose
                                //   lists do not fit shared memory (LevelDev::tris_hbm); null = no such level

  // ---- level definition ----
  const MazeDev* maze;          // [levels] Maze templates (mwb_set_maze, mwb_set_level_maze) or null
  const double* maze_cdf;       // [levels][MWB_MAZE_CDF_STRIDE] cumulative room probabilities
  const mwb_proto* protos;      // shared by all levels
  int32_t num_protos;
  const mwb_op* ops;            // every level's reset program, one after another
  const LevelDev* levels;       // [levels] rule, truncation, program slice
  const mwb_params* level_params;   // [levels] DomainParams of each level (MWB_ARRAY_LEVEL_PARAMS: writable in place,
                                    //   stream-ordered); K1 reads the step ranges per step, the rest at resets
  int32_t* env_level;           // [N] level of each env (all 0 on a one-level handle); with level changes on, the
                                //     resets rewrite it (device_reset: resolve_level)
  int32_t num_levels;
  // level changes at resets (mwb_enable_level_changes); null on a handle without them
  int32_t* next_level;          // [N] pending assignment, -1 = none
  uint32_t* level_draws;        // [N] level draws made so far (counter of the draw hash)
  const float* level_weights;   // [num_levels] sampling weights, all <= 0 = keep the level
  uint64_t level_seed;
  int32_t level_env_offset;     // global index of env 0 (sharded runs)
  // episode seeds (mwb_enable_episode_seeds); null on a handle without them
  int64_t* next_seed;           // [N] seed the env's next reset starts its stream from, negative = none
  int64_t* episode_seed;        // [N] seed the env's current episode started from, -1 = it continued its stream
  // maze layouts (mwb_enable_maze_layouts); null on a handle without them.  One pointer to a device-side record rather
  // than its fields: every byte of DevState is a kernel parameter of every launch
  const struct MazeLayouts* layouts;
  // start poses (mwb_enable_start_poses); null on a handle without them, one pointer for the same reason
  const struct StartPoses* poses;
  // reset draws (mwb_enable_reset_draws); null on a handle without them, one pointer for the same reason
  const struct ResetDraws* draws;
  // state bank (mwb_enable_state_bank); null on a handle without it, one pointer for the same reason
  const struct StateBank* bank;
  // goal distance (mwb_enable_goal_distance); null on a handle without it, one pointer for the same reason
  const struct GoalNav* nav;
  // env params (mwb_enable_env_params); null on a handle without them, one pointer for the same reason
  const struct EnvParams* envparams;
  int32_t autoreset;
  // StochasticActionWrapper on the device (reference wrappers.py:49-71): per step one uniform() draw from
  // the env's own stream; below act_prob the chosen action stands, else act_random (< 0: integers(0, 6))
  int32_t act_noise, act_random;
  double act_prob;
};

// Block of the geometry arrays env i reads while it runs level lvl: its own world, or the level's template
MWB_DEV int geom_block(const DevState& S, int i, int lvl) { return S.levels[lvl].env_worlds ? S.env_geom + i : lvl; }
MWB_DEV int geom_index(const DevState& S, int i) { return geom_block(S, i, S.env_level[i]); }
MWB_DEV const LevelDev& env_level_of(const DevState& S, int i) { return S.levels[S.env_level[i]]; }
MWB_DEV const mwb_params& env_params_of(const DevState& S, int i) { return S.level_params[S.env_level[i]]; }

// Words of element e (mwb_enable_env_params' order) in an mwb_params record viewed as doubles: its default, lo and rng.
// A vector param is [3] defaults, [3] lows, [3] spans; a scalar one default, low, span.
MWB_DEV int env_param_word(int e) { return e < 15 ? (e / 3) * 9 + e % 3 : 45 + (e - 15) * 3; }
MWB_DEV int env_param_step(int e) { return e < 15 ? 3 : 1; }

// The level row `lvl` merged with env i's episode row for elements [e0, e1) into V->merged[i] (include/mwb.h states the
// rule), and max_forward_step with them when forward_step (15) is among them.  Returns the merged record, or the level
// row when the episode row designs none of those elements.  Out of line, and given the record's address rather than its
// fields, so that handles without the mode keep their registers.
MWB_DEV_NOINLINE const mwb_params* merge_env_params(const EnvParams* V, int i, const mwb_params* lvl, int e0, int e1) {
  const double* ep = V->episode + (size_t)i * MWB_ENV_PARAM_WORDS;
  bool any = false;
#pragma unroll 1
  for (int e = e0; e < e1; ++e) any |= isfinite(ep[3 * e]) || (isfinite(ep[3 * e + 1]) && isfinite(ep[3 * e + 2]));
  if (!any) return lvl;
  const double* src = (const double*)lvl;
  mwb_params* m = V->merged + i;
  double* dst = (double*)m;
#pragma unroll 1
  for (int e = e0; e < e1; ++e) {
    const int w = env_param_word(e), s = env_param_step(e);
    const double d = ep[3 * e], lo = ep[3 * e + 1], hi = ep[3 * e + 2];
    const bool range = isfinite(lo) && isfinite(hi);
    dst[w] = isfinite(d) ? d : src[w];
    dst[w + s] = range ? lo : src[w + s];
    dst[w + 2 * s] = range ? d_sub(hi, lo) : src[w + 2 * s];
    if (e == 15) m->max_forward_step = range ? hi : lvl->max_forward_step;
  }
  MWB_WARP_SYNC();
  return m;
}

// turn_step's default of env i's running episode (its episode row's when finite, else its level's as it stands)
MWB_DEV double env_turn_step(const DevState& S, int i) {
  if (S.envparams) {
    const double t = S.envparams->episode[(size_t)i * MWB_ENV_PARAM_WORDS + 3 * 17];
    if (isfinite(t)) return t;
  }
  return env_params_of(S, i).turn_step;
}

MWB_DEV NpRng load_rng(const DevState& S, int i) {
  NpRng r;
  r.s_hi = S.rng_s_hi[i];
  r.s_lo = S.rng_s_lo[i];
  r.inc_hi = S.rng_inc_hi[i];
  r.inc_lo = S.rng_inc_lo[i];
  r.has32 = S.rng_has32[i];
  r.cache = S.rng_cache[i];
  return r;
}

MWB_DEV void store_rng(const DevState& S, int i, const NpRng& r) {
  S.rng_s_hi[i] = r.s_hi;
  S.rng_s_lo[i] = r.s_lo;
  S.rng_has32[i] = r.has32;
  S.rng_cache[i] = r.cache;
}
