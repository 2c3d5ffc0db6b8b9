// reset.cuh -- device-side MiniWorldEnv.reset(): runs a lowered _gen_world() per env.
//
// Restates reference miniworld/miniworld.py:544-604 (reset), :839-909 (place_entity),
// :272-284 (Room.point_inside), :987-1003 (_gen_static_data's texture draws via
// opengl.py:113-145) and entity.py:405-407 / :505-516 (randomize), consuming the env's
// numpy PCG64 stream in exactly the reference's call order, so that an episode reset on the
// GPU lands on the same poses, colours and camera parameters as `env.reset()` in Python.
// The level's `_gen_world()` is lowered on the host into a short program of
// CHOICE / UNIFORM / PLACE / PUT / IFEQ ops (miniworld_b200/program.py); room layout comes from the
// static template of the env's level, and the program is that level's slice of the op array.  Maze levels carve a
// fresh world into the env's own geometry block (maze.cuh) from their level's templates; Maze variants whose
// templates do not reproduce the host exactly reset on the host and arrive through mwb_set_world instead.  With maze layouts
// on (mwb_enable_maze_layouts) a Maze reset can instead build a layout written into next_maze (take_maze, maze_design),
// with the goal box and the agent in the layout's cells.  With start poses on (mwb_enable_start_poses) a reset can take
// designed poses for the agent and the placed entities (take_poses, designed_pose), as place_entity(pos=..., dir=...).
// With reset draws on (mwb_enable_reset_draws) a reset can replace the outcomes of its CHOICE / UNIFORM ops with
// designed ones inside their support, and records every outcome (take_draws, designed_draw).  With env params on
// (mwb_enable_env_params) a reset can run on its level's params merged with a row of its own (take_env_params).  With the state bank on (mwb_enable_state_bank) a reset with a pending slot can instead load a saved env state
// (bank_load in bank.cuh) and return before the program runs.
#pragma once
#include "bank.cuh"
#include "maze.cuh"
#include "physics.cuh"

// the first place_entity triggers _gen_static_data: per room Texture.get(wall / floor / ceil), each one
// rng.integers(0, n_variants) under domain randomisation of the env's level (opengl.py:113-145)
MWB_DEV void draw_room_textures(const DevState& S, int i, const mwb_room* rooms, int n_rooms, bool domain_rand,
                                NpRng& rng) {
  for (int r = 0; r < n_rooms; ++r)
    for (int k = 0; k < 3; ++k) {
      int v = 0;
      if (domain_rand) v = (int)rng_integers(rng, (uint32_t)rooms[r].tex_count[k]);
      S.room_tex[((size_t)i * S.R + r) * 3 + k] = rooms[r].tex_first[k] + v;
    }
}

// splitmix64 (Steele, Lea, Flood 2014): the output at position k of the generator seeded with `seed`
MWB_DEV uint64_t splitmix64_at(uint64_t seed, uint64_t k) {
  uint64_t z = seed + (k + 1) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// The level env i runs from this reset on (mwb_enable_level_changes; include/mwb.h states the rule and the draw).
// Every lane of the warp computes the same value from the same loads; the stores follow a warp barrier, so that no
// lane reads a value another lane has already replaced.
MWB_DEV int resolve_level(const DevState& S, int i) {
  MWB_WARP_SYNC();
  const int cur = S.env_level[i];
  const int pending = S.next_level[i];
  uint32_t draws = S.level_draws[i];
  int lvl = cur;
  if (pending >= 0 && pending < S.num_levels) {
    lvl = pending;
  } else {
    float total = 0.0f;
    for (int l = 0; l < S.num_levels; ++l) {
      const float w = S.level_weights[l];
      if (w > 0.0f) total = f_add(total, w);
    }
    if (total > 0.0f) {
      const uint64_t k = ((uint64_t)((uint32_t)S.level_env_offset + (uint32_t)i) << 32) | draws;
      const uint32_t u24 = (uint32_t)(splitmix64_at(S.level_seed, k) >> 40);
      const float target = f_mul(f_mul((float)u24, 5.9604644775390625e-08f), total);   // u24 * 2^-24 * total
      float cdf = 0.0f;
      for (int l = 0; l < S.num_levels; ++l) {
        const float w = S.level_weights[l];
        if (!(w > 0.0f)) continue;
        cdf = f_add(cdf, w);
        lvl = l;
        if (cdf > target) break;
      }
      ++draws;
    }
  }
  MWB_WARP_SYNC();
  if (pending != -1) S.next_level[i] = -1;
  S.level_draws[i] = draws;
  S.env_level[i] = lvl;
  MWB_WARP_SYNC();
  return lvl;
}

// SeedSequence(seed) -> PCG64 into one env's stream.  Out of line: about a hundred dependent integer operations that
// only a reset with a pending seed runs, kept out of step_kernel's register allocation.  It takes the six addresses
// rather than the DevState, which is a kernel parameter and would be copied to the stack to be passed on.
MWB_DEV_NOINLINE void seed_stream(uint64_t seed, uint64_t* s_hi, uint64_t* s_lo, uint64_t* inc_hi, uint64_t* inc_lo,
                                  int32_t* has32, uint32_t* cache) {
  const NpRng r = rng_seed(seed);
  *s_hi = r.s_hi;
  *s_lo = r.s_lo;
  *inc_hi = r.inc_hi;
  *inc_lo = r.inc_lo;
  *has32 = r.has32;
  *cache = r.cache;
}

// The stream env i's reset starts from (mwb_enable_episode_seeds; include/mwb.h states the rule): a pending seed
// replaces the stream and is consumed, otherwise the env continues its own.  As in resolve_level, every lane computes
// the same value from the same loads, and warp barriers separate the loads from the stores.
MWB_DEV void take_seed(const DevState& S, int i) {
  MWB_WARP_SYNC();
  const int64_t seed = S.next_seed[i];
  MWB_WARP_SYNC();
  S.episode_seed[i] = seed >= 0 ? seed : -1;
  if (seed != -1) S.next_seed[i] = -1;
  if (seed >= 0)
    seed_stream((uint64_t)seed, S.rng_s_hi + i, S.rng_s_lo + i, S.rng_inc_hi + i, S.rng_inc_lo + i, S.rng_has32 + i,
                S.rng_cache + i);
  MWB_WARP_SYNC();
}

// Room of flat layout cell f (j * cols_max + i) in a level of R x C cells, -1 when f is outside the grid.
MWB_DEV int layout_cell_room(int f, int cols_max, int R, int C) {
  return f >= 0 && f / cols_max < R && f % cols_max < C ? (f / cols_max) * C + f % cols_max : -1;
}

// The layout env i's reset at a level of R x C cells builds (mwb_enable_maze_layouts; include/mwb.h states the rule; R = 0
// for a level that is not a Maze).  At a Maze level a pending layout is taken: its copy masked to the grid becomes the
// episode's layout (episode_maze, which maze_design then reads), and the return value is 1.  Otherwise it returns 0: a
// Maze level carves (maze_generate records the topology), and any other level writes zeros and leaves a pending layout
// waiting.  As in take_seed, every lane computes the same values from the same loads, and warp barriers separate the
// loads from the stores.
MWB_DEV int take_maze(uint8_t* pending_flag, const uint8_t* next, uint8_t* episode, int rows_max, int cols_max, int R,
                      int C) {
  MWB_WARP_SYNC();
  const bool take = R > 0 && *pending_flag != 0;
  if (R > 0 && !take) return 0;
  for (int j = 0; j < rows_max; ++j)
    for (int ci = 0; ci < cols_max; ++ci) {
      int b = take && j < R && ci < C ? next[j * cols_max + ci] & 3 : 0;
      if (ci + 1 >= C) b &= ~1;
      if (j + 1 >= R) b &= ~2;
      episode[j * cols_max + ci] = (uint8_t)b;
    }
  MWB_WARP_SYNC();
  if (take) *pending_flag = 0;
  MWB_WARP_SYNC();
  return take ? 1 : 0;
}

// Whether env i's reset takes the designed start poses (mwb_enable_start_poses; include/mwb.h states the rule): a pending
// flag is consumed by the next reset at any level, and the rows stay as written.  As in take_seed, every lane computes
// the same value from the same load, and warp barriers separate the load from the store.
MWB_DEV bool take_poses(uint8_t* pending_flag) {
  MWB_WARP_SYNC();
  const bool take = *pending_flag != 0;
  MWB_WARP_SYNC();
  if (take) *pending_flag = 0;
  MWB_WARP_SYNC();
  return take;
}

// The designed (x, z, dir) row of the placement that fills slot e of env i, or null when the placement runs as the
// level wrote it: the agent's call takes next_agent when its x and z are finite, then (any call) the slot's row when
// its x and z are finite.  Out of line, like seed_stream, so that handles without the mode keep their registers.
MWB_DEV_NOINLINE const double* designed_pose(const StartPoses* P, int i, int e, int E, int is_agent) {
  const double* a = P->next_agent + (size_t)3 * i;
  if (is_agent && isfinite(a[0]) && isfinite(a[1])) return a;
  const double* r = P->next + ((size_t)i * E + e) * 3;
  return isfinite(r[0]) && isfinite(r[1]) ? r : nullptr;
}

// Whether env i's reset takes the designed draws (mwb_enable_reset_draws; include/mwb.h states the rule): as take_poses,
// and the env's episode_draws row is refilled with NaN, which the level's draws then overwrite.  Out of line, like
// designed_draw, and given the record's address rather than its fields, so that handles without the mode keep their
// registers.
MWB_DEV_NOINLINE bool take_draws(const ResetDraws* R, int i) {
  MWB_WARP_SYNC();
  const bool take = R->pending[i] != 0;
  MWB_WARP_SYNC();
  if (take) R->pending[i] = 0;
  for (int d = 0; d < R->D; ++d) R->episode[(size_t)i * R->D + d] = MWB_NAN;
  MWB_WARP_SYNC();
  return take;
}

// The outcome of reset draw `op` (a CHOICE or UNIFORM, op->room = its index d) of env i, which the stream drew as v:
// with take set, next[i][d] when it lies in the draw's support (a choice over n: an integer in [0, n); a uniform over
// [lo, hi]: finite and lo <= x <= hi), else v.  The outcome is recorded in episode[i][d].  Out of line, like
// designed_pose, so that handles without the mode keep their registers.
MWB_DEV_NOINLINE double designed_draw(const ResetDraws* R, int i, const mwb_op* op, double v, int take) {
  const int d = op->room;
  if (d < 0 || d >= R->D) return v;
  if (take) {
    const double x = R->next[(size_t)i * R->D + d];
    if (op->op == MWB_OP_CHOICE ? x >= 0.0 && x < (double)op->b && x == floor(x)
                                : isfinite(x) && x >= op->f[0] && x <= op->f[1])
      v = op->op == MWB_OP_CHOICE ? (double)(int)x : x;
  }
  R->episode[(size_t)i * R->D + d] = v;
  return v;
}

// The params env i's reset at level row `lvl` runs on (mwb_enable_env_params; include/mwb.h states the rule): a pending
// row is taken into episode[i] and the flag cleared, the rows staying as written; otherwise episode[i] becomes all NaN.
// Returns the level row merged with episode[i] (merge_env_params).  As in take_draws, every lane computes the same
// flag from the same load, warp barriers separate the flag's load from its store, and it is out of line and given the
// record's address; the record row is filled by all lanes, word w by lane w % 32.
MWB_DEV_NOINLINE const mwb_params* take_env_params(const EnvParams* V, int i, const mwb_params* lvl) {
  MWB_WARP_SYNC();
  const bool take = V->pending[i] != 0;
  MWB_WARP_SYNC();
  if (take) V->pending[i] = 0;
  const double* nx = V->next + (size_t)i * MWB_ENV_PARAM_WORDS;
  double* ep = V->episode + (size_t)i * MWB_ENV_PARAM_WORDS;
  // the 66 words spread over the warp's lanes (every lane then reads them after the barrier below)
#ifdef __CUDA_ARCH__
  const int lane = threadIdx.x & 31, lanes = 32;
#else
  const int lane = 0, lanes = 1;
#endif
#pragma unroll 1
  for (int w = lane; w < MWB_ENV_PARAM_WORDS; w += lanes) ep[w] = take ? nx[w] : MWB_NAN;
  MWB_WARP_SYNC();
  return take ? merge_env_params(V, i, lvl, 0, MWB_ENV_PARAM_ELEMS) : lvl;
}

MWB_DEV void device_reset(const DevState& S, int i) {
  const size_t N = S.N;
  // the world changes: the goal distance kernel that follows rebuilds the env's field (navigation.cuh)
  if (S.nav) S.nav->dirty[i] = 1;
  // a pending saved state wins over everything else and consumes only next_state (bank.cuh)
  if (S.bank && bank_load(S.bank, i, S.env_level[i], S.next_level != nullptr)) return;
  if (S.next_seed) take_seed(S, i);
  // bit 4 of flags below: this reset takes designed draws (taken before anything below is loaded: a call while those
  // values are live costs reset_kernel registers)
  const int draw_flag = S.draws && take_draws(S.draws, i) ? 16 : 0;
  const int lvl = S.next_level ? resolve_level(S, i) : S.env_level[i];
  // the level's ranges as they stand at this reset, merged with the env's own row when it took one (env params; taken
  // before the stream is loaded, for the reason above)
  const mwb_params& P = S.envparams ? *take_env_params(S.envparams, i, S.level_params + lvl) : S.level_params[lvl];
  NpRng rng = load_rng(S, i);
  // the resolved level decides everything below, its domain_rand included: a reset that switches levels draws by the
  // new level's flag (read at each use: the row's address is live anyway, a cached copy would cost step_kernel a spill)
  const LevelDev& L = S.levels[lvl];
  const mwb_op* ops = S.ops + L.op_first;
  const int num_ops = L.num_ops;
  // the geometry of the level this episode runs: the env's own world (regenerated below by a Maze program) or the
  // level's template, so that an env leaving a Maze level stops reading its old world
  const int g = geom_block(S, i, lvl);
  const mwb_room* rooms = S.rooms + (size_t)g * S.R;
  int n_rooms = S.num_rooms[g];
  // bit 0: the rooms' textures are drawn (_gen_static_data ran); bits 1 / 2: a designed maze's goal / agent cell is
  // still to be placed; bit 3: this reset takes designed start poses; bit 4: it takes designed draws (one variable, so
  // that the designed paths add no register to the loop below)
  int flags = draw_flag;
  if (S.poses && take_poses(S.poses->pending + i)) flags |= 8;
  if (S.layouts) {
    const MazeLayouts& Y = *S.layouts;
    const size_t cells = (size_t)Y.rows * Y.cols;
    const bool maze = L.maze >= 0 && L.env_worlds;
    if (take_maze(Y.pending + i, Y.next + cells * i, Y.episode + cells * i, Y.rows, Y.cols,
                  maze ? S.maze[L.maze].rows : 0, maze ? S.maze[L.maze].cols : 0))
      flags |= 6;
  }

  S.step_count[i] = 0;
  S.carrying[i] = -1;
  S.num_picked[i] = L.rule_kind == MWB_RULE_HEALTH ? 100 : 0;   // CollectHealth: self.health = 100
  S.ghost_slot[i] = -1;
  S.num_slots[i] = 0;
  for (int e = 0; e < S.E; ++e) {
    S.ent_proto[e * N + i] = -1;
    S.ent_size[e * N + i] = 0.0;
  }
  // Agent() defaults (entity.py:459-474)
  S.cam[0 * N + i] = P.cam_height;
  S.cam[1 * N + i] = P.cam_fwd_disp;
  S.cam[2 * N + i] = P.cam_pitch;
  S.cam[3 * N + i] = P.cam_fov_y;
  // self.max_forward_step = params.get_max("forward_step") (miniworld.py:581): the episode keeps it
  S.env_mfs[i] = P.max_forward_step;

  int ireg[8];
  double freg[8];
  int slots = 0;

  for (int pc = 0; pc < num_ops; ++pc) {
    const mwb_op& op = ops[pc];
    if (op.op == MWB_OP_END) break;
    if (op.op == MWB_OP_MAZE) {          // per-episode topology: regenerate this env's rooms
      // (a Maze program's first op: flags holds only the designed bits here)
      const bool built =
          L.maze >= 0 && L.env_worlds &&
          ((flags & 6) ? maze_design(S.maze + L.maze, S.layouts->episode + (size_t)S.layouts->rows * S.layouts->cols * i,
                               S.layouts->cols, S.rooms + (size_t)g * S.R, S.quads + (size_t)g * S.Q,
                               S.segs + (size_t)g * S.S, S.R, S.Q, S.S, S.num_rooms + g, S.num_quads + g, S.num_segs + g)
                 : maze_generate(S, S.maze[L.maze], S.maze_cdf + (size_t)L.maze * MWB_MAZE_CDF_STRIDE, g, rng,
                                 S.layouts ? S.layouts->episode + (size_t)S.layouts->rows * S.layouts->cols * i : nullptr,
                                 S.layouts ? S.layouts->rows : 0, S.layouts ? S.layouts->cols : 0));
      if (built) {
        n_rooms = S.num_rooms[g];
      } else {
        // out of capacity (unreachable when the host sized the handle from a generated maze, mwb_set_maze): placing
        // entities into stale geometry could search forever, so the env is left empty and the fault is counted
#ifdef __CUDA_ARCH__
        if ((threadIdx.x & 31) == 0) atomicAdd(S.fault, 1);
#else
        *S.fault += 1;
#endif
        store_rng(S, i, rng);
        return;
      }
      continue;
    }
    if (op.op == MWB_OP_IFEQ) {
      if (ireg[op.a & 7] != op.b) ++pc;
      continue;
    }
    if (op.op == MWB_OP_PUT) {
      if (!(flags & 1) && op.b == 0) {
        draw_room_textures(S, i, rooms, n_rooms, L.domain_rand != 0, rng);
        flags |= 1;
      }
      const mwb_proto& pr = S.protos[op.a];
      // a designed pose replaces x and z (the level's y stays), and its dir when that is finite; append-only
      // entities are not placed, so they keep the level's pose
      const double* d = (flags & 8) && op.b == 0 ? designed_pose(S.poses, i, slots, S.E, 0) : nullptr;
      const double dir = d && isfinite(d[2]) ? d[2]
                         : isnan(op.f[3]) ? rng_uniform(rng, -3.141592653589793, d_sub(3.141592653589793, -3.141592653589793))
                                          : op.f[3];
      const int e = slots++;
      S.ent_proto[e * N + i] = op.a;
      S.ent_px[e * N + i] = d ? d[0] : op.f[0];
      S.ent_py[e * N + i] = op.f[1];
      S.ent_pz[e * N + i] = d ? d[1] : op.f[2];
      S.ent_dir[e * N + i] = dir;
      S.ent_size[e * N + i] = 0.0;
      for (int k = 0; k < 3; ++k) S.ent_col[((size_t)e * 3 + k) * N + i] = pr.color[k];
      S.num_slots[i] = slots;
      continue;
    }
    if (op.op == MWB_OP_CHOICE) {
      // a designed draw is drawn first, so that the stream advances as it would without the design
      int v = (int)rng_integers(rng, (uint32_t)op.b);
      if (S.draws) v = (int)designed_draw(S.draws, i, &op, (double)v, flags & 16);
      ireg[op.a & 7] = v;
    } else if (op.op == MWB_OP_UNIFORM) {
      double v = rng_uniform(rng, op.f[0], d_sub(op.f[1], op.f[0]));
      if (S.draws) v = designed_draw(S.draws, i, &op, v, flags & 16);
      freg[op.a & 7] = v;
    } else if (op.op == MWB_OP_PLACE) {
      if (!(flags & 1)) {
        draw_room_textures(S, i, rooms, n_rooms, L.domain_rand != 0, rng);
        flags |= 1;
      }
      int proto = op.a;
      if (op.ireg_a >= 0) proto += ireg[op.ireg_a & 7] * op.stride_a;
      if (op.ireg_b >= 0) proto += ireg[op.ireg_b & 7] * op.stride_b;
      const mwb_proto& pr = S.protos[proto];
      double x, z, dir;
      S.num_slots[i] = slots;   // entities placed so far
      // a Box whose edge length the level drew for this episode (op.b = 1 + freg): Box.__init__'s radius
      const double size = op.b > 0 ? freg[(op.b - 1) & 7] : 0.0;
      const double rad = size > 0.0 ? d_div(d_sqrt(d_add(d_mul(size, size), d_mul(size, size))), 2.0) : pr.radius;
      // a designed maze's cells: the agent's PLACE takes the agent cell, the first other PLACE (the goal box) the goal cell
      int room = op.room;
      if (flags & (op.is_agent ? 4 : 2)) {
        const MazeDev& M = S.maze[L.maze];
        room = layout_cell_room(S.layouts->cells[2 * (size_t)i + (op.is_agent ? 1 : 0)], S.layouts->cols, M.rows, M.cols);
        flags &= op.is_agent ? ~4 : ~2;
      }
      // a designed pose: place_entity(pos=...)'s branch (reference miniworld.py:861-867), no room, search or
      // collision check; dir is the designed one when finite, else the level's, else uniform(-pi, pi)
      const double* d = (flags & 8) ? designed_pose(S.poses, i, slots, S.E, op.is_agent) : nullptr;
      if (d) {
        x = d[0];
        z = d[1];
        dir = isfinite(d[2]) ? d[2]
              : op.dir_freg >= 0 ? freg[op.dir_freg & 7]
                                 : rng_uniform(rng, -3.141592653589793, d_sub(3.141592653589793, -3.141592653589793));
      } else {
        place_search(S, i, rng, rooms, n_rooms, room, op.f, rad, pr.radius_is_f32 != 0,
                     op.dir_freg >= 0 ? freg[op.dir_freg & 7] : MWB_NAN, x, z, dir);
      }
      int e = slots++;
      S.ent_size[e * N + i] = size;
      S.ent_proto[e * N + i] = proto;
      S.ent_px[e * N + i] = x;
      S.ent_py[e * N + i] = 0.0;
      S.ent_pz[e * N + i] = z;
      S.ent_dir[e * N + i] = dir;
      for (int k = 0; k < 3; ++k) S.ent_col[((size_t)e * 3 + k) * N + i] = pr.color[k];
      if (op.is_agent) S.agent_slot[i] = e;
      S.num_slots[i] = slots;
    }
  }
  if (S.poses) {   // where this episode starts, designed or drawn
    const int a = S.agent_slot[i];
    double* st = S.poses->episode + (size_t)3 * i;
    st[0] = S.ent_px[a * N + i];
    st[1] = S.ent_pz[a * N + i];
    st[2] = S.ent_dir[a * N + i];
  }

  // params.sample_many(rand, self, [sky_color, light_pos, light_color, light_ambient])
  const double* defs[4] = {P.sky_color, P.light_pos, P.light_color, P.light_ambient};
  const double* los[4] = {P.sky_color_lo, P.light_pos_lo, P.light_color_lo, P.light_ambient_lo};
  const double* rngs[4] = {P.sky_color_rng, P.light_pos_rng, P.light_color_rng, P.light_ambient_rng};
  for (int q = 0; q < 4; ++q)
    for (int k = 0; k < 3; ++k)
      S.envp[(size_t)(q * 3 + k) * N + i] = L.domain_rand ? rng_uniform(rng, los[q][k], rngs[q][k]) : defs[q][k];

  // for ent in self.entities: ent.randomize(params, rand).  Without randomisation a Box still adds obj_color_bias's
  // default (params.sample(None, ...), entity.py:405-407): zero unless a level row or an env's row sets it, and adding
  // zero changes no colour, so the loop runs only when there is something to draw or add
  const bool bias = P.obj_color_bias[0] != 0.0 || P.obj_color_bias[1] != 0.0 || P.obj_color_bias[2] != 0.0;
  if (L.domain_rand || bias) {
    for (int e = 0; e < slots; ++e) {
      const mwb_proto& pr = S.protos[S.ent_proto[e * N + i]];
      if (pr.kind == MWB_KIND_BOX) {
        for (int k = 0; k < 3; ++k) {
          const double b = L.domain_rand ? rng_uniform(rng, P.obj_color_bias_lo[k], P.obj_color_bias_rng[k])
                                         : P.obj_color_bias[k];
          double c = d_add(pr.color[k], b);
          S.ent_col[((size_t)e * 3 + k) * N + i] = c < 0.0 ? 0.0 : (c > 1.0 ? 1.0 : c);
        }
      } else if (L.domain_rand && pr.kind == MWB_KIND_AGENT) {
        S.cam[0 * N + i] = rng_uniform(rng, P.cam_height_lo, P.cam_height_rng);
        S.cam[1 * N + i] = rng_uniform(rng, P.cam_fwd_disp_lo, P.cam_fwd_disp_rng);
        S.cam[2 * N + i] = rng_uniform(rng, P.cam_pitch_lo, P.cam_pitch_rng);
        S.cam[3 * N + i] = rng_uniform(rng, P.cam_fov_y_lo, P.cam_fov_y_rng);
      }
    }
  }
  store_rng(S, i, rng);
}

