// navigation.cuh -- goal distance (mwb_enable_goal_distance; include/mwb.h states the definitions): a distance field
// over a fixed grid of each goal level, built per env when a reset changed its world, and the agent's geodesic
// distance to the goal, the episode's shortest path and an expert action read from it after every step and reset.
//
// One block per env.  A block whose env was reset classifies the grid's nodes into shared memory (one warp per node:
// circle_hits_walls strides the wall segments across the lanes), relaxes the integer field in place with alternating
// row and column sweeps until a sweep round changes nothing, and writes field and free flags to HBM.  Positive integer
// edge costs make the fixed point unique, so the result does not depend on the order the sweeps update the nodes in:
// the host build, which runs the same functions on one thread, gets the same bytes.  Thread 0 then reads the field.
#pragma once
#include "physics.cuh"

#define MWB_NAV_NONE 0xFFFFu          // unreachable, or not a free or source node
#define MWB_NAV_MAX 0xFFFEu           // distances saturate here
#define MWB_NAV_PASS 1                // node class bits: free or source (an edge may end here)
#define MWB_NAV_FREE 2                // free: no wall within r + h/2, no other entity within r + h/2 + its radius
#define MWB_NAV_SOURCE 4              // an agent standing here is near(goal)
#define MWB_NAV_THREADS 256

#ifdef __CUDA_ARCH__
#define MWB_NAV_TID ((int)threadIdx.x)
#define MWB_NAV_NT ((int)blockDim.x)
#define MWB_NAV_SYNC() __syncthreads()
#define MWB_NAV_SYNC_OR(x) __syncthreads_or(x)
#else
#define MWB_NAV_TID 0
#define MWB_NAV_NT 1
#define MWB_NAV_SYNC()
#define MWB_NAV_SYNC_OR(x) (x)
#endif

// Floor position of node k along an axis that starts at lo: lo + (k + 0.5) h (the product is exact)
MWB_DEV double nav_node_pos(double lo, int k) { return d_add(lo, d_mul((double)k + 0.5, MWB_GOAL_GRID_STEP)); }

// Class bits of node n of env i's grid.  Every lane of the calling warp passes the same node: the rooms, like the wall
// segments in circle_hits_walls, are strided across the lanes (an 8 x 8 Maze has 176 rooms) and closed with a vote.
MWB_DEV int nav_classify(const DevState& S, int i, const mwb_goal_grid& gr, int n, int as, double ar, double ay) {
  const size_t N = S.N;
  const int g = geom_index(S, i);
  const double x = nav_node_pos(gr.min_x, n % gr.nx), z = nav_node_pos(gr.min_z, n / gr.nx);
#ifdef __CUDA_ARCH__
  const int first = threadIdx.x & 31, stride = 32;
#else
  const int first = 0, stride = 1;
#endif
  bool inside = false;
  for (int r = first; r < S.num_rooms[g] && !inside; r += stride)
    inside = room_contains(S.rooms[(size_t)g * S.R + r], x, z);
#ifdef __CUDA_ARCH__
  inside = __any_sync(0xffffffffu, inside);
#endif
  if (!inside) return 0;
  const int cls = near_point(S, i, gr.goal_slot, x, ay, z, ar) ? MWB_NAV_PASS | MWB_NAV_SOURCE : 0;
  const double rad = d_add(ar, 0.5 * MWB_GOAL_GRID_STEP);
  if (circle_hits_walls(S.segs + (size_t)g * S.S, S.num_segs[g], x, z, rad)) return cls;
  const int n_ents = S.num_slots[i];
  for (int e = 0; e < n_ents; ++e) {   // world_intersect's entity test, without the agent and the goal
    const int p = S.ent_proto[(size_t)e * N + i];
    if (e == as || e == gr.goal_slot || p < 0) continue;
    const double dx = d_sub(S.ent_px[(size_t)e * N + i], x);
    const double dz = d_sub(S.ent_pz[(size_t)e * N + i], z);
    const EntDims ed = ent_dims(S, i, e, S.protos[p]);
    if (d_sqrt(d_fma(dz, dz, d_mul(dx, dx))) < sum_radii(rad, false, ed.radius, ed.f32)) return cls;
  }
  return cls | MWB_NAV_PASS | MWB_NAV_FREE;
}

// Whether the edge from node (k, l) to its 8-neighbour (k + dk, l + dl) exists (both ends on the grid and passable; a
// diagonal also needs the two orthogonal nodes it passes), and its cost.
MWB_DEV int nav_edge(const uint8_t* c, int nx, int nz, int k, int l, int dk, int dl) {
  const int kk = k + dk, ll = l + dl;
  if (kk < 0 || kk >= nx || ll < 0 || ll >= nz || !(c[ll * nx + kk] & MWB_NAV_PASS)) return 0;
  if (dk && dl) return (c[l * nx + kk] & MWB_NAV_PASS) && (c[ll * nx + k] & MWB_NAV_PASS) ? 7 : 0;
  return 5;
}

// One Bellman update of node (k, l): its field becomes the least of itself and every neighbour's field + edge cost.
MWB_DEV bool nav_relax_node(uint16_t* f, const uint8_t* c, int nx, int nz, int k, int l) {
  const int n = l * nx + k;
  const unsigned cur = f[n];
  if (cur == 0 || !(c[n] & MWB_NAV_PASS)) return false;
  unsigned best = cur;
  for (int dl = -1; dl <= 1; ++dl)
    for (int dk = -1; dk <= 1; ++dk) {
      if (!dk && !dl) continue;
      const int w = nav_edge(c, nx, nz, k, l, dk, dl);
      const unsigned fm = w ? f[(l + dl) * nx + k + dk] : MWB_NAV_NONE;
      if (fm == MWB_NAV_NONE) continue;
      const unsigned v = fm + w < MWB_NAV_MAX ? fm + w : MWB_NAV_MAX;
      if (v < best) best = v;
    }
  if (best == cur) return false;
  f[n] = (uint16_t)best;
  return true;
}

// Sweep `pass` (0 / 1: rows towards +x / -x, 2 / 3: columns towards +z / -z) over the lines of thread t of nt.  Each node
// is written by one thread only; a neighbour another thread updates meanwhile is read old or new, and both are upper
// bounds of its distance, so a round without a change anywhere is the fixed point.
MWB_DEV bool nav_sweep(uint16_t* f, const uint8_t* c, int nx, int nz, int pass, int t, int nt) {
  const bool rows = pass < 2, fwd = (pass & 1) == 0;
  const int lines = rows ? nz : nx, len = rows ? nx : nz;
  bool changed = false;
  for (int a = t; a < lines; a += nt)
    for (int s = 0; s < len; ++s) {
      const int b = fwd ? s : len - 1 - s;
      changed |= rows ? nav_relax_node(f, c, nx, nz, b, a) : nav_relax_node(f, c, nx, nz, a, b);
    }
  return changed;
}

// goal_dist, expert_action and (at a reset) episode_shortest of env i from its grid's field and node classes.
MWB_DEV void nav_query(const DevState& S, int i, const mwb_goal_grid& gr, const uint16_t* f, const uint8_t* c,
                       bool at_reset) {
  const GoalNav& V = *S.nav;
  double dist = MWB_NAN;
  int action = -1;
  if (gr.goal_slot >= 0) {
    const size_t N = S.N;
    const int as = S.agent_slot[i];
    const double ax = S.ent_px[as * N + i], az = S.ent_pz[as * N + i], dir = S.ent_dir[as * N + i];
    const double ar = S.protos[S.ent_proto[as * N + i]].radius;
    const bool near = near_agent(S, i, gr.goal_slot, as, ar);
    int best = -1;
    dist = near ? 0.0 : __builtin_inf();
    if (!near) {
      const int k0 = (int)floor(d_sub(d_div(d_sub(ax, gr.min_x), MWB_GOAL_GRID_STEP), 0.5));
      const int l0 = (int)floor(d_sub(d_div(d_sub(az, gr.min_z), MWB_GOAL_GRID_STEP), 0.5));
      for (int l = l0 - 1; l <= l0 + 2; ++l)
        for (int k = k0 - 1; k <= k0 + 2; ++k) {   // increasing flat index: a strict < keeps the lowest on ties
          if (k < 0 || k >= gr.nx || l < 0 || l >= gr.nz) continue;
          const int n = l * gr.nx + k;
          if (!(c[n] & MWB_NAV_FREE) || f[n] == MWB_NAV_NONE) continue;
          const double dx = d_sub(nav_node_pos(gr.min_x, k), ax), dz = d_sub(nav_node_pos(gr.min_z, l), az);
          const double v = d_add(d_mul((double)f[n], 0.05), d_sqrt(d_add(d_mul(dx, dx), d_mul(dz, dz))));
          if (v < dist) {
            dist = v;
            best = n;
          }
        }
    }
    if (near || best >= 0) {
      double wx = S.ent_px[(size_t)gr.goal_slot * N + i], wz = S.ent_pz[(size_t)gr.goal_slot * N + i];
      if (!near && f[best] != 0) {   // the neighbour of best on a shortest path
        const int k = best % gr.nx, l = best / gr.nx;
        unsigned least = 0xFFFFFFFFu;   // a reachable node with a field above 0 has a neighbour on its path
        int m = best;
        for (int dl = -1; dl <= 1; ++dl)
          for (int dk = -1; dk <= 1; ++dk) {
            const int w = dk || dl ? nav_edge(c, gr.nx, gr.nz, k, l, dk, dl) : 0;
            const unsigned fm = w ? f[(l + dl) * gr.nx + k + dk] : MWB_NAV_NONE;
            if (fm == MWB_NAV_NONE || fm + w >= least) continue;
            least = fm + w;
            m = (l + dl) * gr.nx + k + dk;
          }
        wx = nav_node_pos(gr.min_x, m % gr.nx);
        wz = nav_node_pos(gr.min_z, m / gr.nx);
      }
      const double co = mwb_libm::cos_glibc(dir), si = mwb_libm::sin_glibc(dir);
      const double vx = d_sub(wx, ax), vz = d_sub(wz, az);
      const double vf = d_add(d_mul(vx, co), d_mul(vz, -si));   // v . dir_vec, dir_vec = (cos, 0, -sin)
      const double vv = d_add(d_mul(vx, vx), d_mul(vz, vz));
      const double ch = mwb_libm::cos_glibc(d_mul(d_mul(0.5, env_turn_step(S, i)), 0.017453292519943295));
      if (vf > 0.0 && d_mul(vf, vf) >= d_mul(vv, d_mul(ch, ch)))
        action = 2;                                               // move_forward
      else                                                        // turn_left (dir grows) turns dir_vec towards
        action = d_add(d_mul(vx, -si), d_mul(vz, -co)) > 0.0 ? 0 : 1;   // (-sin, -cos)
    }
  }
  V.goal_dist[i] = dist;
  V.expert[i] = action;
  if (at_reset) V.shortest[i] = dist;
}

// The block of env i: build the field when the env was reset or restored since the last launch, then the query.
// f and c are the block's shared memory (uint16 [G], uint8 [G]).
MWB_DEV void goal_nav(const DevState& S, int i, uint16_t* f, uint8_t* c) {
  const GoalNav& V = *S.nav;
  const mwb_goal_grid gr = V.grids[S.env_level[i]];
  const int dirty = V.dirty[i];
  uint16_t* field = V.field + (size_t)i * V.G;
  uint8_t* node_class = V.node_class + (size_t)i * V.G;
  if (dirty) {
    const int nodes = gr.goal_slot >= 0 ? gr.nx * gr.nz : 0;
    const size_t N = S.N;
    const int t = MWB_NAV_TID, nt = MWB_NAV_NT;
    for (int n = t; n < V.G; n += nt) c[n] = 0;
    MWB_NAV_SYNC();
    if (nodes) {
      const int as = S.agent_slot[i];
      const double ar = S.protos[S.ent_proto[as * N + i]].radius, ay = S.ent_py[as * N + i];
#ifdef __CUDA_ARCH__
      const int lane = t & 31, warp = t >> 5, warps = nt >> 5;
#else
      const int lane = 0, warp = 0, warps = 1;
#endif
      for (int n = warp; n < nodes; n += warps) {
        const int cls = nav_classify(S, i, gr, n, as, ar, ay);
        if (lane == 0) c[n] = (uint8_t)cls;
      }
    }
    MWB_NAV_SYNC();
    for (int n = t; n < V.G; n += nt) f[n] = c[n] & MWB_NAV_SOURCE ? 0 : MWB_NAV_NONE;
    MWB_NAV_SYNC();
    for (;;) {
      bool changed = false;
      for (int pass = 0; pass < 4; ++pass) {
        changed |= nav_sweep(f, c, gr.nx, gr.nz, pass, t, nt);
        if (pass < 3) MWB_NAV_SYNC();
      }
      if (!MWB_NAV_SYNC_OR(changed)) break;
    }
    for (int n = t; n < V.G; n += nt) {
      field[n] = f[n];
      node_class[n] = c[n];
    }
    MWB_NAV_SYNC();
  }
  if (MWB_NAV_TID == 0) {
    nav_query(S, i, gr, field, node_class, dirty == 1);
    if (dirty) V.dirty[i] = 0;
  }
}
