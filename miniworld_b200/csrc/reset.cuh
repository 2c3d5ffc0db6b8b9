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
// templates do not reproduce the host exactly reset on the host and arrive through mwb_set_world instead.
#pragma once
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

MWB_DEV void device_reset(const DevState& S, int i) {
  const size_t N = S.N;
  NpRng rng = load_rng(S, i);
  const int lvl = S.next_level ? resolve_level(S, i) : S.env_level[i];
  // the resolved level decides everything below, its domain_rand included: a reset that switches levels draws by the
  // new level's flag (read at each use: the row's address is live anyway, a cached copy would cost step_kernel a spill)
  const LevelDev& L = S.levels[lvl];
  const mwb_params& P = L.params;
  const mwb_op* ops = S.ops + L.op_first;
  const int num_ops = L.num_ops;
  // the geometry of the level this episode runs: the env's own world (regenerated below by a Maze program) or the
  // level's template, so that an env leaving a Maze level stops reading its old world
  const int g = geom_block(S, i, lvl);
  const mwb_room* rooms = S.rooms + (size_t)g * S.R;
  int n_rooms = S.num_rooms[g];

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

  int ireg[8];
  double freg[8];
  bool static_done = false;
  int slots = 0;

  for (int pc = 0; pc < num_ops; ++pc) {
    const mwb_op& op = ops[pc];
    if (op.op == MWB_OP_END) break;
    if (op.op == MWB_OP_MAZE) {          // per-episode topology: regenerate this env's rooms
      if (L.maze >= 0 && L.env_worlds && maze_generate(S, S.maze[L.maze], S.maze_cdf + (size_t)L.maze * MWB_MAZE_CDF_STRIDE, g, rng)) {
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
      if (!static_done && op.b == 0) {
        draw_room_textures(S, i, rooms, n_rooms, L.domain_rand != 0, rng);
        static_done = true;
      }
      const mwb_proto& pr = S.protos[op.a];
      const double dir = isnan(op.f[3]) ? rng_uniform(rng, -3.141592653589793, d_sub(3.141592653589793, -3.141592653589793))
                                        : op.f[3];
      const int e = slots++;
      S.ent_proto[e * N + i] = op.a;
      S.ent_px[e * N + i] = op.f[0];
      S.ent_py[e * N + i] = op.f[1];
      S.ent_pz[e * N + i] = op.f[2];
      S.ent_dir[e * N + i] = dir;
      S.ent_size[e * N + i] = 0.0;
      for (int k = 0; k < 3; ++k) S.ent_col[((size_t)e * 3 + k) * N + i] = pr.color[k];
      S.num_slots[i] = slots;
      continue;
    }
    if (op.op == MWB_OP_CHOICE) {
      ireg[op.a & 7] = (int)rng_integers(rng, (uint32_t)op.b);
    } else if (op.op == MWB_OP_UNIFORM) {
      freg[op.a & 7] = rng_uniform(rng, op.f[0], d_sub(op.f[1], op.f[0]));
    } else if (op.op == MWB_OP_PLACE) {
      if (!static_done) {
        draw_room_textures(S, i, rooms, n_rooms, L.domain_rand != 0, rng);
        static_done = true;
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
      place_search(S, i, rng, rooms, n_rooms, op.room, op.f, rad, pr.radius_is_f32 != 0,
                   op.dir_freg >= 0 ? freg[op.dir_freg & 7] : MWB_NAN, x, z, dir);
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

  // params.sample_many(rand, self, [sky_color, light_pos, light_color, light_ambient])
  const double* defs[4] = {P.sky_color, P.light_pos, P.light_color, P.light_ambient};
  const double* los[4] = {P.sky_color_lo, P.light_pos_lo, P.light_color_lo, P.light_ambient_lo};
  const double* rngs[4] = {P.sky_color_rng, P.light_pos_rng, P.light_color_rng, P.light_ambient_rng};
  for (int q = 0; q < 4; ++q)
    for (int k = 0; k < 3; ++k)
      S.envp[(size_t)(q * 3 + k) * N + i] = L.domain_rand ? rng_uniform(rng, los[q][k], rngs[q][k]) : defs[q][k];

  // for ent in self.entities: ent.randomize(params, rand)
  if (L.domain_rand) {
    for (int e = 0; e < slots; ++e) {
      const mwb_proto& pr = S.protos[S.ent_proto[e * N + i]];
      if (pr.kind == MWB_KIND_BOX) {
        for (int k = 0; k < 3; ++k) {
          double c = d_add(pr.color[k], rng_uniform(rng, P.obj_color_bias_lo[k], P.obj_color_bias_rng[k]));
          S.ent_col[((size_t)e * 3 + k) * N + i] = c < 0.0 ? 0.0 : (c > 1.0 ? 1.0 : c);
        }
      } else if (pr.kind == MWB_KIND_AGENT) {
        S.cam[0 * N + i] = rng_uniform(rng, P.cam_height_lo, P.cam_height_rng);
        S.cam[1 * N + i] = rng_uniform(rng, P.cam_fwd_disp_lo, P.cam_fwd_disp_rng);
        S.cam[2 * N + i] = rng_uniform(rng, P.cam_pitch_lo, P.cam_pitch_rng);
        S.cam[3 * N + i] = rng_uniform(rng, P.cam_fov_y_lo, P.cam_fov_y_rng);
      }
    }
  }
  store_rng(S, i, rng);
}
