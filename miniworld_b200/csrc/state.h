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

struct TriRec;
struct MeshSegInfo;
struct MazeDev;

// One row of the level table (mwb_set_levels): what K1 reads per env instead of per handle.
struct LevelDev {
  mwb_params params;
  double near_extra;            // 1.1 * max_forward_step
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
  const LevelDev* levels;       // [levels] rule, truncation, params, program slice
  int32_t* env_level;           // [N] level of each env (all 0 on a one-level handle); with level changes on, the
                                //     resets rewrite it (device_reset: resolve_level)
  int32_t num_levels;
  // level changes at resets (mwb_enable_level_changes); null on a handle without them
  int32_t* next_level;          // [N] pending assignment, -1 = none
  uint32_t* level_draws;        // [N] level draws made so far (counter of the draw hash)
  const float* level_weights;   // [num_levels] sampling weights, all <= 0 = keep the level
  uint64_t level_seed;
  int32_t level_env_offset;     // global index of env 0 (sharded runs)
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
