// maze.cuh -- device-side Maze._gen_world(): recursive-backtracker topology on the env's numpy
// stream + geometry assembled from translated templates (reference envs/maze.py:73-153,
// miniworld.py:768-837 connect_rooms, :286-399 Room._gen_static_data).
//
// The random part of a Maze episode is only WHICH neighbouring cells get connected and in what
// order: `visit(i, j)` shuffles the four neighbour offsets with choice(4), choice(3), choice(2),
// choice(1) (the last one consumes nothing) and recurses into unvisited neighbours, calling
// connect_rooms on the way.  Every room, wall quad and collision segment is then a translate of
// a template (miniworld_b200/maze_lowering.py cuts them out of host-built worlds and verifies
// that the assembly reproduces a host-generated maze field for field).
#pragma once
#include "state.h"

struct MazeDev {
  int32_t rows, cols;
  double pitch;
  mwb_room cell_room;
  mwb_quad cell_quads[6];
  mwb_seg cell_segs[4];
  int32_t open_a[4], open_b[4];
  mwb_room conn_room[4];
  mwb_quad conn_quads[4][4];
  mwb_seg conn_segs[4][2];
};

#define MWB_MAZE_MAX_CELLS 256
#define MWB_MAZE_CDF_STRIDE (2 * MWB_MAZE_MAX_CELLS)   // doubles per level in DevState::maze_cdf (2 cells - 1 used)

MWB_DEV void maze_put_room(mwb_room* dst, const mwb_room& src, double dx, double dz, double cdf) {
  mwb_room r = src;
  r.min_x = d_add(r.min_x, dx);
  r.max_x = d_add(r.max_x, dx);
  r.min_z = d_add(r.min_z, dz);
  r.max_z = d_add(r.max_z, dz);
  for (int e = 0; e < r.num_edges; ++e) {
    r.edge_px[e] = d_add(r.edge_px[e], dx);
    r.edge_pz[e] = d_add(r.edge_pz[e], dz);
  }
  r.cdf = cdf;
  for (int k = 0; k < 3; ++k) r.tex_id[k] = r.tex_first[k];
  *dst = r;
}

MWB_DEV void maze_put_quad(mwb_quad* dst, const mwb_quad& src, double dx, double dz, int room, bool floor_like) {
  mwb_quad q = src;
  for (int k = 0; k < q.num_verts; ++k) {
    q.pos[k][0] = (float)d_add((double)q.pos[k][0], dx);
    q.pos[k][2] = (float)d_add((double)q.pos[k][2], dz);
    if (floor_like) {   // floor / ceiling texcoords are world (x, z)
      q.uvm[k][0] = d_add(q.uvm[k][0], dx);
      q.uvm[k][1] = d_add(q.uvm[k][1], dz);
    }
  }
  q.room = room;
  *dst = q;
}

MWB_DEV void maze_put_seg(mwb_seg* dst, const mwb_seg& src, double dx, double dz) {
  dst->ax = d_add(src.ax, dx);
  dst->bx = d_add(src.bx, dx);
  dst->az = d_add(src.az, dz);
  dst->bz = d_add(src.bz, dz);
}

// Generates an env's rooms / quads / segments into geometry block g (the env's own world) from its level's
// templates M and room cdf.  Returns false if the capacities of the handle are too small.
MWB_DEV bool maze_generate(const DevState& S, const MazeDev& M, const double* cdf, int g, NpRng& rng) {
  const int R = M.rows, C = M.cols, cells = R * C;
  if (cells > MWB_MAZE_MAX_CELLS || 2 * cells - 1 > S.R) return false;
  // ---- topology: iterative form of visit() -------------------------------------------------
  uint8_t visited[MWB_MAZE_MAX_CELLS];
  uint8_t opened[MWB_MAZE_MAX_CELLS];          // bit e: wall (edge) e of the cell is open
  uint8_t frame_order[MWB_MAZE_MAX_CELLS];     // per stack level: the shuffled neighbour order, 2 bits each
  uint8_t frame_next[MWB_MAZE_MAX_CELLS];
  uint16_t frame_cell[MWB_MAZE_MAX_CELLS];
  uint16_t conn_cell[MWB_MAZE_MAX_CELLS];
  uint8_t conn_dir[MWB_MAZE_MAX_CELLS];
  for (int c = 0; c < cells; ++c) visited[c] = opened[c] = 0;
  const int DJ[4] = {0, 0, -1, 1}, DI[4] = {1, -1, 0, 0};
  int depth = 0, n_conn = 0;
  frame_cell[0] = 0;
  frame_next[0] = 255;   // 255: order not drawn yet
  while (depth >= 0) {
    const int cell = frame_cell[depth], ci = cell % C, cj = cell / C;
    if (frame_next[depth] == 255) {
      visited[cell] = 1;
      // orders.remove(orders[choice(len(orders))]) four times
      int left[4] = {0, 1, 2, 3};
      uint8_t packed = 0;
      for (int n = 4; n >= 1; --n) {
        const int pick = (int)rng_integers(rng, (uint32_t)n);
        packed |= (uint8_t)(left[pick] << (2 * (4 - n)));
        for (int q = pick; q + 1 < n; ++q) left[q] = left[q + 1];
      }
      frame_order[depth] = packed;
      frame_next[depth] = 0;
    }
    bool pushed = false;
    while (frame_next[depth] < 4) {
      const int d = (frame_order[depth] >> (2 * frame_next[depth])) & 3;
      frame_next[depth]++;
      const int ni = ci + DI[d], nj = cj + DJ[d];
      if (nj < 0 || nj >= R || ni < 0 || ni >= C) continue;
      const int ncell = nj * C + ni;
      if (visited[ncell]) continue;
      conn_cell[n_conn] = (uint16_t)cell;      // connect_rooms(room, neighbor, ...)
      conn_dir[n_conn] = (uint8_t)d;
      ++n_conn;
      opened[cell] |= (uint8_t)(1u << M.open_a[d]);
      opened[ncell] |= (uint8_t)(1u << M.open_b[d]);
      ++depth;
      frame_cell[depth] = (uint16_t)ncell;
      frame_next[depth] = 255;
      pushed = true;
      break;
    }
    if (!pushed) --depth;
  }
  // ---- geometry, in the reference's list order: grid rooms row by row, then connectors ---------
  mwb_room* rooms = S.rooms + (size_t)g * S.R;
  mwb_quad* quads = S.quads + (size_t)g * S.Q;
  mwb_seg* segs = S.segs + (size_t)g * S.S;
  int nr = 0, nq = 0, ns = 0;
  for (int cj = 0; cj < R; ++cj)
    for (int ci = 0; ci < C; ++ci) {
      const double dx = d_mul((double)ci, M.pitch), dz = d_mul((double)cj, M.pitch);
      const int cell = cj * C + ci;
      if (nq + 6 > S.Q || ns + 4 > S.S) return false;
      maze_put_room(rooms + nr, M.cell_room, dx, dz, cdf[nr]);
      maze_put_quad(quads + nq++, M.cell_quads[0], dx, dz, nr, true);
      maze_put_quad(quads + nq++, M.cell_quads[1], dx, dz, nr, true);
      for (int e = 0; e < 4; ++e)
        if (!((opened[cell] >> e) & 1)) {
          maze_put_quad(quads + nq++, M.cell_quads[2 + e], dx, dz, nr, false);
          maze_put_seg(segs + ns++, M.cell_segs[e], dx, dz);
        }
      ++nr;
    }
  for (int k = 0; k < n_conn; ++k) {
    const int cell = conn_cell[k], d = conn_dir[k];
    const double dx = d_mul((double)(cell % C), M.pitch), dz = d_mul((double)(cell / C), M.pitch);
    if (nq + 4 > S.Q || ns + 2 > S.S || nr + 1 > S.R) return false;
    maze_put_room(rooms + nr, M.conn_room[d], dx, dz, cdf[nr]);
    for (int q = 0; q < 4; ++q) maze_put_quad(quads + nq++, M.conn_quads[d][q], dx, dz, nr, q < 2);
    maze_put_seg(segs + ns++, M.conn_segs[d][0], dx, dz);
    maze_put_seg(segs + ns++, M.conn_segs[d][1], dx, dz);
    ++nr;
  }
  S.num_rooms[g] = nr;
  S.num_quads[g] = nq;
  S.num_segs[g] = ns;
  return true;
}
