// physics.cuh -- K1: one warp per environment (scalar logic in lockstep, wall tests lane-parallel), float64,
// the reference's arithmetic.
//
// Restates, operation for operation (no FMA contraction except where numpy's BLAS ddot
// itself fuses), the step path of the reference:
//   math.intersect_circle_segs      reference miniworld/math.py:30-62
//   MiniWorldEnv.intersect          reference miniworld/miniworld.py:937-963
//   MiniWorldEnv.move_agent         :620-645      MiniWorldEnv.turn_agent :647-668
//   MiniWorldEnv._get_carry_pos     :606-618      MiniWorldEnv.step       :670-730
//   MiniWorldEnv.near / _reward     :965-975, :1012-1017
//   level rules                     envs/hallway.py:67-74 (goal), envs/pickupobjects.py:83-95
// Outputs are bit-identical to the reference on this image (numpy 2.3.5, glibc 2.39):
// tests/test_gpu_physics.py compares against trajectories dumped from the reference itself.
#pragma once
#include "libm_sincos.cuh"
#include "state.h"

#define MWB_HIT_NONE (-1)
#define MWB_HIT_WALL (-2)

// intersect_circle_segs: any(dist(point, seg) < radius), strict.  numpy evaluates
// sum(ap*ab, axis=1) as (x*x' + 0) + z*z' with separate roundings (ufunc reduce, no FMA).
// On the GPU the K1 kernels run ONE WARP PER ENVIRONMENT: all 32 lanes execute the env's scalar logic in
// lockstep on identical values (so control flow never diverges and every store writes the same value), and
// this loop -- the only long one: up to 256 wall segments in an 8x8 maze -- is strided across the lanes and
// closed with a warp vote.
MWB_DEV bool circle_hits_walls(const mwb_seg* segs, int n, double px, double pz, double radius) {
#ifdef __CUDA_ARCH__
  const int first = threadIdx.x & 31, stride = 32;
#else
  const int first = 0, stride = 1;
#endif
  bool hit = false;
  for (int s = first; s < n && !hit; s += stride) {
    double ax = segs[s].ax, az = segs[s].az;
    double abx = d_sub(segs[s].bx, ax), abz = d_sub(segs[s].bz, az);
    double apx = d_sub(px, ax), apz = d_sub(pz, az);
    double apab = d_add(d_mul(apx, abx), d_mul(apz, abz));
    double abab = d_add(d_mul(abx, abx), d_mul(abz, abz));
    double t = d_div(apab, abab);
    t = t < 0.0 ? 0.0 : (t > 1.0 ? 1.0 : t);
    double cx = d_add(ax, d_mul(t, abx)), cz = d_add(az, d_mul(t, abz));
    double dx = d_sub(cx, px), dz = d_sub(cz, pz);
    double dist = d_sqrt(d_add(d_mul(dx, dx), d_mul(dz, dz)));
    if (dist < radius) hit = true;
  }
#ifdef __CUDA_ARCH__
  hit = __any_sync(0xffffffffu, hit);
#endif
  return hit;
}

// `radius + ent2.radius` as Python/numpy evaluates it: float32 arithmetic as soon as one of
// the operands is an np.float32 (MeshEnt radii under numpy >= 2, NEP 50), else float64.
MWB_DEV double sum_radii(double r0, bool r0_f32, double r1, bool r1_f32) {
  if (r0_f32 || r1_f32) return (double)f_add((float)r0, (float)r1);
  return d_add(r0, r1);
}

// Physical size of the entity in slot e: the prototype's, unless the level drew this episode's Box edge
// length itself (PutNext: Box(size=rng.uniform(0.6, 0.85))); then Box.__init__'s arithmetic applies
// (entity.py:396-403): radius = math.sqrt(sx * sx + sz * sz) / 2, height = sy.
struct EntDims {
  double radius, height, size;   // size = 0: prototype geometry
  bool f32;
};
MWB_DEV EntDims ent_dims(const DevState& S, int i, int e, const mwb_proto& pr) {
  EntDims d;
  d.f32 = pr.radius_is_f32 != 0;
  const double s = S.ent_size[(size_t)e * S.N + i];
  if (s > 0.0) {
    d.radius = d_div(d_sqrt(d_add(d_mul(s, s), d_mul(s, s))), 2.0);
    d.height = s;
    d.size = s;
  } else {
    d.radius = pr.radius;
    d.height = pr.height;
    d.size = 0.0;
  }
  return d;
}

// MiniWorldEnv.intersect: walls first, then the entity list in order (skipping `self_slot`).
// np.linalg.norm of a 1-D vector goes through BLAS ddot, which accumulates with FMA:
// sqrt(fma(dz, dz, fma(dy, dy, dx*dx))) with dy == 0 here.
MWB_DEV int world_intersect(const DevState& S, int i, int self_slot, double px, double pz, double radius,
                            bool radius_f32) {
  int g = geom_index(S, i);
  if (circle_hits_walls(S.segs + (size_t)g * S.S, S.num_segs[g], px, pz, radius)) return MWB_HIT_WALL;
  int n = S.num_slots[i];
  for (int e = 0; e < n; ++e) {
    if (e == self_slot) continue;
    int p = S.ent_proto[(size_t)e * S.N + i];
    if (p < 0) continue;
    double dx = d_sub(S.ent_px[(size_t)e * S.N + i], px);
    double dz = d_sub(S.ent_pz[(size_t)e * S.N + i], pz);
    double d = d_sqrt(d_fma(dz, dz, d_mul(dx, dx)));
    const EntDims ed = ent_dims(S, i, e, S.protos[p]);
    if (d < sum_radii(radius, radius_f32, ed.radius, ed.f32)) return e;
  }
  return MWB_HIT_NONE;
}

struct CarryPos {
  double x, y, z;
};

// _get_carry_pos(agent_pos, ent): agent_pos + dir_vec * 1.05 * dist, lifted to stay visible
MWB_DEV CarryPos carry_pos(const DevState& S, int i, double apx, double apz, double c, double s, int slot, double ar) {
  const EntDims pr = ent_dims(S, i, slot, S.protos[S.ent_proto[(size_t)slot * S.N + i]]);
  const double mfs = env_level_of(S, i).params.max_forward_step;
  double dist;   // agent.radius + ent.radius + max_forward_step, float32 as soon as ent.radius is
  if (pr.f32)
    dist = (double)f_add(f_add((float)ar, (float)pr.radius), (float)mfs);
  else
    dist = d_add(d_add(ar, pr.radius), mfs);
  CarryPos o;
  o.x = d_add(apx, d_mul(d_mul(c, 1.05), dist));
  o.z = d_add(apz, d_mul(d_mul(-s, 1.05), dist));
  double y = d_sub(d_sub(S.cam[0 * (size_t)S.N + i], pr.height), 0.3);
  o.y = y > 0.0 ? y : 0.0;
  return o;
}

// Room.point_inside: all(sum(edge_norms * (p - outline), axis=1) > 0)
MWB_DEV bool room_contains(const mwb_room& r, double px, double pz) {
  for (int e = 0; e < r.num_edges; ++e) {
    double d = d_add(d_mul(r.edge_nx[e], d_sub(px, r.edge_px[e])), d_mul(r.edge_nz[e], d_sub(pz, r.edge_pz[e])));
    if (!(d > 0.0)) return false;
  }
  return true;
}

// place_entity's search loop (miniworld.py:871-909): pick a room (fixed, or Generator.choice(n, p=room_probs) =
// searchsorted(cdf, random(), 'right')), draw a position in its (optionally overridden) extents grown by the
// entity's radius, retry until it is inside the room and free; then the heading (given, or uniform(-pi, pi)).
#define MWB_NAN (__builtin_nan(""))
MWB_DEV void place_search(const DevState& S, int i, NpRng& rng, const mwb_room* rooms, int n_rooms, int room_fixed,
                          const double bounds[4], double rad, bool rad_f32, double dir_given, double& x, double& z,
                          double& dir) {
  for (;;) {
    int r = room_fixed;
    if (r < 0) {
      double u = rng_random(rng);
      r = 0;
      while (r < n_rooms - 1 && rooms[r].cdf <= u) ++r;
    }
    const mwb_room& rm = rooms[r];
    double lx = isnan(bounds[0]) ? rm.min_x : bounds[0];
    double hx = isnan(bounds[1]) ? rm.max_x : bounds[1];
    double lz = isnan(bounds[2]) ? rm.min_z : bounds[2];
    double hz = isnan(bounds[3]) ? rm.max_z : bounds[3];
    double lox = d_sub(lx, rad), loz = d_sub(lz, rad);
    x = rng_uniform(rng, lox, d_sub(d_add(hx, rad), lox));
    (void)rng_random(rng);   // the y component: uniform(0, 0) still consumes a draw
    z = rng_uniform(rng, loz, d_sub(d_add(hz, rad), loz));
    if (!room_contains(rm, x, z)) continue;
    if (world_intersect(S, i, -1, x, z, rad, rad_f32) != MWB_HIT_NONE) continue;
    dir = isnan(dir_given) ? rng_uniform(rng, -3.141592653589793, d_sub(3.141592653589793, -3.141592653589793)) : dir_given;
    return;
  }
}

// Threshold of MiniWorldEnv.near (miniworld.py:965-975): `ent0.radius + ent1.radius + 1.1 * self.max_forward_step`,
// evaluated left to right.  Once one radius is an np.float32 (MeshEnt under numpy >= 2) the first sum is float32 and
// stays float32 when the Python float 1.1 * max_forward_step is added (NEP 50: Python scalars are weak), so the
// threshold is float32(float32(r0 + r1) + float32(extra)); with two float64 radii everything is float64.
MWB_DEV double near_threshold(double r0, bool r0_f32, double r1, bool r1_f32, double extra) {
  if (r0_f32 || r1_f32) return (double)f_add(f_add((float)r0, (float)r1), (float)extra);
  return d_add(d_add(r0, r1), extra);
}

// MiniWorldEnv.near(ent): np.linalg.norm(ent.pos - agent.pos) < ent.radius + agent.radius + 1.1 * max_forward_step
// (3-D distance through BLAS ddot, i.e. an FMA chain)
MWB_DEV bool near_agent(const DevState& S, int i, int b, int as, double ar) {
  const size_t N = S.N;
  const int bp = S.ent_proto[b * N + i];
  if (bp < 0) return false;
  const double dx = d_sub(S.ent_px[b * N + i], S.ent_px[as * N + i]);
  const double dy = d_sub(S.ent_py[b * N + i], S.ent_py[as * N + i]);
  const double dz = d_sub(S.ent_pz[b * N + i], S.ent_pz[as * N + i]);
  const double d = d_sqrt(d_fma(dz, dz, d_fma(dy, dy, d_mul(dx, dx))));
  const EntDims pr = ent_dims(S, i, b, S.protos[bp]);
  return d < near_threshold(pr.radius, pr.f32, ar, false, env_level_of(S, i).near_extra);
}

// MiniWorldEnv.near(ent0, ent1) between two entities of the list
MWB_DEV bool near_pair(const DevState& S, int i, int a, int b) {
  const size_t N = S.N;
  const int pa = S.ent_proto[a * N + i], pb = S.ent_proto[b * N + i];
  if (pa < 0 || pb < 0) return false;
  const double dx = d_sub(S.ent_px[a * N + i], S.ent_px[b * N + i]);
  const double dy = d_sub(S.ent_py[a * N + i], S.ent_py[b * N + i]);
  const double dz = d_sub(S.ent_pz[a * N + i], S.ent_pz[b * N + i]);
  const double d = d_sqrt(d_fma(dz, dz, d_fma(dy, dy, d_mul(dx, dx))));
  const EntDims da = ent_dims(S, i, a, S.protos[pa]), db = ent_dims(S, i, b, S.protos[pb]);
  return d < near_threshold(da.radius, da.f32, db.radius, db.f32, env_level_of(S, i).near_extra);
}

struct StepOut {
  double reward;
  int terminated, truncated;
};

// One MiniWorldEnv.step() (without the render) followed by the lowered level rule.
// fwd_step / fwd_drift / turn_step are the three per-step parameters of miniworld.py:677-680.
MWB_DEV StepOut physics_step(const DevState& S, int i, int action, double fwd_step, double fwd_drift,
                             double turn_step) {
  const size_t N = S.N;
  const int as = S.agent_slot[i];
  double px = S.ent_px[as * N + i], pz = S.ent_pz[as * N + i], dir = S.ent_dir[as * N + i];
  const double ar = S.protos[S.ent_proto[as * N + i]].radius;   // Agent.radius (0.4 unless the level changes it)
  int carrying = S.carrying[i];
  int sc = S.step_count[i] + 1;
#ifdef __CUDA_ARCH__
  __syncwarp();                 // every lane has read the counter before any lane writes it back
#endif
  S.step_count[i] = sc;
  S.ghost_slot[i] = -1;

  if (action == 2 || action == 3) {   // move_forward / move_back
    double fwd = action == 2 ? fwd_step : -fwd_step;
    double c = mwb_libm::cos_glibc(dir), s = mwb_libm::sin_glibc(dir);
    double nx = d_add(d_add(px, d_mul(c, fwd)), d_mul(s, fwd_drift));
    double nz = d_add(d_add(pz, d_mul(-s, fwd)), d_mul(c, fwd_drift));
    bool ok = world_intersect(S, i, as, nx, nz, ar, false) == MWB_HIT_NONE;
    if (ok && carrying >= 0) {
      CarryPos cp = carry_pos(S, i, nx, nz, c, s, carrying, ar);
      const EntDims pr = ent_dims(S, i, carrying, S.protos[S.ent_proto[carrying * N + i]]);
      ok = world_intersect(S, i, carrying, cp.x, cp.z, pr.radius, pr.f32) == MWB_HIT_NONE;
      if (ok) {
        S.ent_px[carrying * N + i] = cp.x;
        S.ent_py[carrying * N + i] = cp.y;
        S.ent_pz[carrying * N + i] = cp.z;
      }
    }
    if (ok) {
      px = nx;
      pz = nz;
      S.ent_px[as * N + i] = px;
      S.ent_pz[as * N + i] = pz;
    }
  } else if (action == 0 || action == 1) {   // turn_left / turn_right
    double ang = d_mul(action == 0 ? turn_step : -turn_step, 0.017453292519943295 /* math.pi / 180 */);
    double ndir = d_add(dir, ang);
    bool ok = true;
    if (carrying >= 0) {
      double c = mwb_libm::cos_glibc(ndir), s = mwb_libm::sin_glibc(ndir);
      CarryPos cp = carry_pos(S, i, px, pz, c, s, carrying, ar);
      const EntDims pr = ent_dims(S, i, carrying, S.protos[S.ent_proto[carrying * N + i]]);
      // the agent's dir is already updated when the reference tests this; intersect() does not read it
      ok = world_intersect(S, i, carrying, cp.x, cp.z, pr.radius, pr.f32) == MWB_HIT_NONE;
      if (ok) {
        S.ent_px[carrying * N + i] = cp.x;
        S.ent_py[carrying * N + i] = cp.y;
        S.ent_pz[carrying * N + i] = cp.z;
        S.ent_dir[carrying * N + i] = ndir;
      }
    }
    if (ok) {
      dir = ndir;
      S.ent_dir[as * N + i] = dir;
    }
  } else if (action == 4) {   // pickup
    double c = mwb_libm::cos_glibc(dir), s = mwb_libm::sin_glibc(dir);
    double tx = d_add(px, d_mul(d_mul(c, 1.5), ar));
    double tz = d_add(pz, d_mul(d_mul(-s, 1.5), ar));
    int hit = world_intersect(S, i, as, tx, tz, d_mul(1.2, ar), false);
    if (carrying < 0 && hit >= 0 && !S.protos[S.ent_proto[hit * N + i]].is_static) carrying = hit;
  } else if (action == 5) {   // drop
    if (carrying >= 0) {
      S.ent_py[carrying * N + i] = 0.0;
      carrying = -1;
    }
  }

  if (carrying >= 0) {   // carried object follows the agent
    double c = mwb_libm::cos_glibc(dir), s = mwb_libm::sin_glibc(dir);
    CarryPos cp = carry_pos(S, i, px, pz, c, s, carrying, ar);
    S.ent_px[carrying * N + i] = cp.x;
    S.ent_py[carrying * N + i] = cp.y;
    S.ent_pz[carrying * N + i] = cp.z;
    S.ent_dir[carrying * N + i] = dir;
  }

  // the env's level: its rule, rule argument and truncation length
  const LevelDev& L = env_level_of(S, i);
  const int rule_kind = L.rule_kind, rule_arg = L.rule_arg, max_steps = L.max_episode_steps;
  StepOut o;
  o.reward = 0.0;
  o.terminated = 0;
  o.truncated = sc >= max_steps ? 1 : 0;

  if (rule_kind == MWB_RULE_SIDEWALK) {
    // sidewalk.py:96-99: stepping into the street ends the episode with reward 0, before the goal test
    const mwb_room& street = S.rooms[(size_t)geom_index(S, i) * S.R + (rule_arg >> 8)];
    if (room_contains(street, px, pz)) {
      o.reward = 0.0;
      o.terminated = 1;
    }
  }
  if (rule_kind == MWB_RULE_GOAL || rule_kind == MWB_RULE_SIDEWALK) {
    if (near_agent(S, i, rule_arg & 0xFF, as, ar)) {
      o.reward = d_add(o.reward, d_sub(1.0, d_mul(0.2, d_div((double)sc, (double)max_steps))));
      o.terminated = 1;
    }
  } else if (rule_kind == MWB_RULE_SIGN) {
    // sign.py:158-173: the extra action ends the episode; touching any of the six objects ends it with
    // reward +1 for the object the sign names (colour index, kind = goal) and -1 otherwise (the last hit wins)
    if (action == 3) o.terminated = 1;
    const int colour = rule_arg & 0xFF, goal = (rule_arg >> 8) & 0xFF;
    for (int b = 0; b < 6; ++b)
      if (near_agent(S, i, b, as, ar)) {
        o.terminated = 1;
        o.reward = (b % 3 == colour && b / 3 == goal) ? 1.0 : -1.0;
      }
  } else if (rule_kind == MWB_RULE_PUTNEXT) {
    // putnext.py:61-66: done once the two boxes are next to each other and the agent has let go
    if (carrying < 0 && near_pair(S, i, rule_arg & 0xFF, (rule_arg >> 8) & 0xFF)) {
      o.reward = d_add(o.reward, d_sub(1.0, d_mul(0.2, d_div((double)sc, (double)max_steps))));
      o.terminated = 1;
    }
  } else if (rule_kind == MWB_RULE_HEALTH) {
    // collecthealth.py:62-86.  The level counter (num_picked) holds the agent's health.
    int health = S.num_picked[i] - 2;
    if (action == 4 && carrying >= 0) {
      // the kit in hand is consumed and respawned: entities.remove(kit); place_entity(kit).  This step's
      // observation was rendered before that, so the frame still shows it at its carry pose (ghost).
      const int k = carrying, n = S.num_slots[i], kp = S.ent_proto[k * N + i];
      S.ghost_slot[i] = n - 1;
      S.ghost_proto[i] = kp;
      S.ghost_pose[0 * N + i] = S.ent_px[k * N + i];
      S.ghost_pose[1 * N + i] = S.ent_py[k * N + i];
      S.ghost_pose[2 * N + i] = S.ent_pz[k * N + i];
      S.ghost_pose[3 * N + i] = S.ent_dir[k * N + i];
      for (int c = 0; c < 3; ++c) S.ghost_col[c * N + i] = S.ent_col[((size_t)k * 3 + c) * N + i];
      for (int e = k; e + 1 < n; ++e) {       // list.remove(): later entities move up one place
        S.ent_proto[e * N + i] = S.ent_proto[(e + 1) * N + i];
        S.ent_px[e * N + i] = S.ent_px[(e + 1) * N + i];
        S.ent_py[e * N + i] = S.ent_py[(e + 1) * N + i];
        S.ent_pz[e * N + i] = S.ent_pz[(e + 1) * N + i];
        S.ent_dir[e * N + i] = S.ent_dir[(e + 1) * N + i];
        S.ent_size[e * N + i] = S.ent_size[(e + 1) * N + i];
        for (int c = 0; c < 3; ++c) S.ent_col[((size_t)e * 3 + c) * N + i] = S.ent_col[((size_t)(e + 1) * 3 + c) * N + i];
      }
      int as2 = as > k ? as - 1 : as;
      S.agent_slot[i] = as2;
      S.ent_proto[(n - 1) * N + i] = -1;
      S.num_slots[i] = n - 1;
      const int g = geom_index(S, i);
      const double nob[4] = {MWB_NAN, MWB_NAN, MWB_NAN, MWB_NAN};
      NpRng rng = load_rng(S, i);
      double x, z, dir;
      place_search(S, i, rng, S.rooms + (size_t)g * S.R, S.num_rooms[g], -1, nob, S.protos[kp].radius,
                   S.protos[kp].radius_is_f32 != 0, MWB_NAN, x, z, dir);
      store_rng(S, i, rng);
      S.ent_proto[(n - 1) * N + i] = kp;      // list.append()
      S.ent_px[(n - 1) * N + i] = x;
      S.ent_py[(n - 1) * N + i] = 0.0;
      S.ent_pz[(n - 1) * N + i] = z;
      S.ent_dir[(n - 1) * N + i] = dir;
      S.ent_size[(n - 1) * N + i] = 0.0;
      S.num_slots[i] = n;
      carrying = -1;
      health = 100;
    }
    S.num_picked[i] = health;
    if (health > 0) {
      o.reward = 2.0;
    } else {
      o.reward = -100.0;
      o.terminated = 1;
    }
  } else if (rule_kind == MWB_RULE_PICKUP) {
    if (carrying >= 0) {
      // the observation of this step still shows the object at its carry position
      S.ghost_slot[i] = carrying;
      S.ghost_proto[i] = S.ent_proto[carrying * N + i];
      S.ghost_pose[0 * N + i] = S.ent_px[carrying * N + i];
      S.ghost_pose[1 * N + i] = S.ent_py[carrying * N + i];
      S.ghost_pose[2 * N + i] = S.ent_pz[carrying * N + i];
      S.ghost_pose[3 * N + i] = S.ent_dir[carrying * N + i];
      for (int k = 0; k < 3; ++k) S.ghost_col[k * N + i] = S.ent_col[((size_t)carrying * 3 + k) * N + i];
      S.ent_proto[carrying * N + i] = -1;
      carrying = -1;
      int np_ = S.num_picked[i] + 1;
      S.num_picked[i] = np_;
      o.reward = 1.0;
      if (np_ == rule_arg) o.terminated = 1;
    }
  }
  S.carrying[i] = carrying;
  return o;
}
