// maze.cuh -- device-side Maze._gen_world(): recursive-backtracker topology on the env's numpy
// stream + geometry assembled from translated templates (reference envs/maze.py:73-153,
// miniworld.py:768-837 connect_rooms, :286-399 Room._gen_static_data).
//
// The random part of a Maze episode is only WHICH neighbouring cells get connected and in what
// order: `visit(i, j)` shuffles the four neighbour offsets with choice(4), choice(3), choice(2),
// choice(1) (the last one consumes nothing) and recurses into unvisited neighbours, calling
// connect_rooms on the way.  Every room, wall quad and collision segment is then a translate of
// a template (miniworld_b200/maze_lowering.py cuts them out of host-built worlds and verifies
// that the assembly reproduces a host-generated maze field for field).  A designed maze (maze_design) assembles
// the same templates from a layout instead of a carve.
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
  *dst = src;   // then the translated fields in place: no local copy of the record
  dst->min_x = d_add(src.min_x, dx);
  dst->max_x = d_add(src.max_x, dx);
  dst->min_z = d_add(src.min_z, dz);
  dst->max_z = d_add(src.max_z, dz);
  for (int e = 0; e < src.num_edges; ++e) {
    dst->edge_px[e] = d_add(src.edge_px[e], dx);
    dst->edge_pz[e] = d_add(src.edge_pz[e], dz);
  }
  dst->cdf = cdf;
  for (int k = 0; k < 3; ++k) dst->tex_id[k] = src.tex_first[k];
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

// Grid cell `cell` (its room, floor, ceiling, and the walls of the edges not set in `opened`) appended to a world.
MWB_DEV bool maze_put_cell(const MazeDev& M, int cell, int opened, double cdf, mwb_room* rooms, mwb_quad* quads,
                           mwb_seg* segs, int cap_q, int cap_s, int& nr, int& nq, int& ns) {
  const double dx = d_mul((double)(cell % M.cols), M.pitch), dz = d_mul((double)(cell / M.cols), M.pitch);
  if (nq + 6 > cap_q || ns + 4 > cap_s) return false;
  maze_put_room(rooms + nr, M.cell_room, dx, dz, cdf);
  maze_put_quad(quads + nq++, M.cell_quads[0], dx, dz, nr, true);
  maze_put_quad(quads + nq++, M.cell_quads[1], dx, dz, nr, true);
  for (int e = 0; e < 4; ++e)
    if (!((opened >> e) & 1)) {
      maze_put_quad(quads + nq++, M.cell_quads[2 + e], dx, dz, nr, false);
      maze_put_seg(segs + ns++, M.cell_segs[e], dx, dz);
    }
  ++nr;
  return true;
}

// The connector connect_rooms(cell, its neighbour in direction d) creates, appended to a world.
MWB_DEV bool maze_put_conn(const MazeDev& M, int cell, int d, double cdf, mwb_room* rooms, mwb_quad* quads,
                           mwb_seg* segs, int cap_r, int cap_q, int cap_s, int& nr, int& nq, int& ns) {
  const double dx = d_mul((double)(cell % M.cols), M.pitch), dz = d_mul((double)(cell / M.cols), M.pitch);
  if (nq + 4 > cap_q || ns + 2 > cap_s || nr + 1 > cap_r) return false;
  maze_put_room(rooms + nr, M.conn_room[d], dx, dz, cdf);
  for (int q = 0; q < 4; ++q) maze_put_quad(quads + nq++, M.conn_quads[d][q], dx, dz, nr, q < 2);
  maze_put_seg(segs + ns++, M.conn_segs[d][0], dx, dz);
  maze_put_seg(segs + ns++, M.conn_segs[d][1], dx, dz);
  ++nr;
  return true;
}

// Generates an env's rooms / quads / segments into geometry block g (the env's own world) from its level's
// templates M and room cdf.  Returns false if the capacities of the handle are too small.  With `record` (the env's
// episode_maze row, rec_rows x rec_cols) the carved topology is written there as a layout (mwb_enable_maze_layouts).
MWB_DEV bool maze_generate(const DevState& S, const MazeDev& M, const double* cdf, int g, NpRng& rng, uint8_t* record,
                           int rec_rows, int rec_cols) {
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
  if (record) {   // the topology as a layout: a connector in direction d opens the east or south bit of one cell
    for (int k = 0; k < rec_rows * rec_cols; ++k) {
      const int cj = k / rec_cols, ci = k % rec_cols;
      uint8_t v = 0;
      if (cj < R && ci < C) {
        const int o = opened[cj * C + ci];
        v = (uint8_t)(((o >> M.open_a[0]) & 1) | (((o >> M.open_a[3]) & 1) << 1));
      }
      record[k] = v;
    }
  }
  // ---- geometry, in the reference's list order: grid rooms row by row, then connectors ---------
  mwb_room* rooms = S.rooms + (size_t)g * S.R;
  mwb_quad* quads = S.quads + (size_t)g * S.Q;
  mwb_seg* segs = S.segs + (size_t)g * S.S;
  int nr = 0, nq = 0, ns = 0;
  for (int cell = 0; cell < cells; ++cell)
    if (!maze_put_cell(M, cell, opened[cell], cdf[nr], rooms, quads, segs, S.Q, S.S, nr, nq, ns)) return false;
  for (int k = 0; k < n_conn; ++k)
    if (!maze_put_conn(M, conn_cell[k], conn_dir[k], cdf[nr], rooms, quads, segs, S.R, S.Q, S.S, nr, nq, ns)) return false;
  S.num_rooms[g] = nr;
  S.num_quads[g] = nq;
  S.num_segs[g] = ns;
  return true;
}

// numpy's pairwise summation of float64 (np.sum of a contiguous array: 0.0 + pairwise_sum_DOUBLE over all n entries,
// numpy/_core/src/umath/loops_utils.h.src): blocks of fewer than 8 entries are summed in order; blocks of up to 128
// in 8 interleaved partial sums, combined as ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)), then the entries past
// the last multiple of 8 in order; larger blocks split at n / 2 rounded down to a multiple of 8 into left + right.
// The recursion is unrolled with a stack of pending right halves (8 levels: up to 32768 entries).
template <class At>
MWB_DEV double np_pairwise_block(const At& at, int lo, int n) {
  if (n < 8) {
    double res = 0.0;
    for (int i = 0; i < n; ++i) res = d_add(res, at(lo + i));
    return res;
  }
  double r[8];
  for (int j = 0; j < 8; ++j) r[j] = at(lo + j);
  int i = 8;
  for (; i < n - (n % 8); i += 8)
    for (int j = 0; j < 8; ++j) r[j] = d_add(r[j], at(lo + i + j));
  double res = d_add(d_add(d_add(r[0], r[1]), d_add(r[2], r[3])), d_add(d_add(r[4], r[5]), d_add(r[6], r[7])));
  for (; i < n; ++i) res = d_add(res, at(lo + i));
  return res;
}

template <class At>
MWB_DEV double np_pairwise_sum(const At& at, int n) {
  int right_lo[8], right_n[8];
  double left[8];
  bool in_right[8];
  int sp = 0, lo = 0, len = n;
  for (;;) {
    while (len > 128) {
      int n2 = len / 2;
      n2 -= n2 % 8;
      right_lo[sp] = lo + n2;
      right_n[sp] = len - n2;
      in_right[sp] = false;
      ++sp;
      len = n2;
    }
    double v = np_pairwise_block(at, lo, len);
    for (;;) {
      if (sp == 0) return d_add(0.0, v);
      if (!in_right[sp - 1]) {
        left[sp - 1] = v;
        in_right[sp - 1] = true;
        lo = right_lo[sp - 1];
        len = right_n[sp - 1];
        break;
      }
      v = d_add(left[sp - 1], v);
      --sp;
    }
  }
}

// Room.area of the reference (miniworld.py): (max_x - min_x) * (max_z - min_z)
struct RoomAreaAt {
  const mwb_room* rooms;
  MWB_DEVM double operator()(int r) const {
    return d_mul(d_sub(rooms[r].max_x, rooms[r].min_x), d_sub(rooms[r].max_z, rooms[r].min_z));
  }
};

// The rooms' cdf fields as _gen_static_data and Generator.choice(p=...) make them: p = areas / np.sum(areas), then
// p.cumsum() / p.cumsum()[-1].  Out of line: only designed resets run it.
MWB_DEV_NOINLINE void maze_room_cdf(mwb_room* rooms, int n) {
  const RoomAreaAt area{rooms};
  const double total = np_pairwise_sum(area, n);
  double c = 0.0;
  for (int r = 0; r < n; ++r) {
    c = d_add(c, d_div(area(r), total));
    rooms[r].cdf = c;
  }
  for (int r = 0; r < n; ++r) rooms[r].cdf = d_div(rooms[r].cdf, c);
}

// A designed maze (mwb_enable_maze_layouts) into one env's world: the grid rooms row by row, then for each cell in
// row-major order the connector to its +x neighbour (bit 0 of the layout byte, connect_rooms(..., min_z, max_z):
// template direction 0) and then to its +z neighbour (bit 1, connect_rooms(..., min_x, max_x): direction 3).  `layout`
// (row stride `lcols`) is already masked to the level's grid.  The walls a cell opens follow from its own bits and from
// those of its -x and -z neighbours.  Returns false if the capacities are too small.  Inlined like maze_generate: as an
// out-of-line call it cost step_kernel's register allocation spills on every handle.
MWB_DEV bool maze_design(const MazeDev* Mp, const uint8_t* layout, int lcols, mwb_room* rooms, mwb_quad* quads,
                                  mwb_seg* segs, int cap_r, int cap_q, int cap_s, int32_t* n_rooms, int32_t* n_quads,
                                  int32_t* n_segs) {
  const MazeDev& M = *Mp;
  const int R = M.rows, C = M.cols, cells = R * C;
  int n_conn = 0;
  for (int cell = 0; cell < cells; ++cell) {
    const int b = layout[(cell / C) * lcols + cell % C];
    n_conn += (b & 1) + ((b >> 1) & 1);
  }
  if (cells + n_conn > cap_r) return false;
  int nr = 0, nq = 0, ns = 0;
  for (int cell = 0; cell < cells; ++cell) {
    const int cj = cell / C, ci = cell % C, b = layout[cj * lcols + ci];
    const int west = ci > 0 ? layout[cj * lcols + ci - 1] & 1 : 0;
    const int north = cj > 0 ? (layout[(cj - 1) * lcols + ci] >> 1) & 1 : 0;
    const int opened = ((b & 1) << M.open_a[0]) | (west << M.open_b[0]) | (((b >> 1) & 1) << M.open_a[3]) |
                       (north << M.open_b[3]);
    if (!maze_put_cell(M, cell, opened, 0.0, rooms, quads, segs, cap_q, cap_s, nr, nq, ns)) return false;
  }
  for (int cell = 0; cell < cells; ++cell) {
    const int b = layout[(cell / C) * lcols + cell % C];
    if ((b & 1) && !maze_put_conn(M, cell, 0, 0.0, rooms, quads, segs, cap_r, cap_q, cap_s, nr, nq, ns)) return false;
    if ((b & 2) && !maze_put_conn(M, cell, 3, 0.0, rooms, quads, segs, cap_r, cap_q, cap_s, nr, nq, ns)) return false;
  }
  maze_room_cdf(rooms, nr);
  *n_rooms = nr;
  *n_quads = nq;
  *n_segs = ns;
  return true;
}
