// visibility.cuh -- get_visible_ents: which entities would pass an occlusion query.
//
// Replaces MiniWorldEnv.get_visible_ents (miniworld.py:1238-1333).  The reference clears the
// observation frame buffer, draws every room (depth only matters), then for each entity of the
// list except the agent draws drawBox(pos.x -/+ 0.1, pos.y .. pos.y + 0.2, pos.z -/+ 0.1) -- in
// world space, no model transform -- inside a GL_ANY_SAMPLES_PASSED query, with GL_LESS depth
// testing and depth writes on.  An entity is reported visible iff at least one sample of its box
// passed the depth test at the time it was drawn.
//
// Order-free restatement used here: for one sample let room = nearest room depth code and m_k =
// nearest code of entity k's box.  Within a box the first-drawn fragment that beats the buffer
// passes, so box k passes at that sample iff m_k < min(room, m_j for j < k).  One thread walks one
// sample through the entities in list order with a running minimum; the per-entity results are
// OR-ed over all samples of the frame.  Coverage, z and the 16-bit depth code come from the same
// exact float32 functions as the rasteriser (raster_core.cuh: finish_triangle, sample_key).
#pragma once
#include "raster_core.cuh"

// triangle t (0..11) of the query box of an entity at P: drawBox's face / corner order (opengl.py:460-503)
MWB_DEV void query_box_triangle(const EntPose& P, int t, TriInput& in) {
  const int f = t >> 1, half = t & 1;
  const float x0 = (float)d_sub(P.x, 0.1), x1 = (float)d_add(P.x, 0.1);
  const float y0 = (float)P.y, y1 = (float)d_add(P.y, 0.2);
  const float z0 = (float)d_sub(P.z, 0.1), z1 = (float)d_add(P.z, 0.1);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int v = k == 0 ? 0 : k + half;
    int sx, sy, sz;
    box_corner(f, v, sx, sy, sz);
    in.pos[k][0] = sx > 0 ? x1 : x0;
    in.pos[k][1] = sy ? y1 : y0;
    in.pos[k][2] = sz > 0 ? z1 : z0;
    in.uv[k][0] = in.uv[k][1] = 0.0f;
    in.nrm[k][0] = 0.0f; in.nrm[k][1] = 1.0f; in.nrm[k][2] = 0.0f;   // colour is irrelevant to the query
    in.mat[k][0] = in.mat[k][1] = in.mat[k][2] = 1.0f;
  }
  in.tex = -1;
}

// nearest depth code of `count` set-up triangles at sample (xs, ys) of pixel (px, py); 65535 = none
MWB_DEV uint32_t nearest_code(const TriRec* tris, int count, int px, int py, float xs, float ys) {
  uint32_t best = 65535u;
  for (int t = 0; t < count; ++t) {
    const TriRec& T = tris[t];
    if ((T.bx & 0xFFFF) > px || (T.bx >> 16) < px || (T.by & 0xFFFF) > py || (T.by >> 16) < py) continue;
    const uint32_t key = sample_key(load_hot(&T), 0, xs, ys, false);
    if (key != 0xFFFFFFFFu) {
      const uint32_t code = key >> 16;
      best = code < best ? code : best;
    }
  }
  return best;
}

// Entities whose query box passes at one sample: bit = entity-list slot.  tris[0 .. n_room) are the
// room triangles, tris[box0 + 12 k ..] the box of the k-th queried entity (culled ones have an
// empty bbox), ent_slot[k] its slot.
MWB_DEV uint32_t visible_at_sample(const TriRec* tris, int n_room, int box0, int n_query, const int* ent_slot, int px,
                                   int py, float xs, float ys) {
  uint32_t cur = nearest_code(tris, n_room, px, py, xs, ys);   // cleared depth 1.0 = code 65535
  uint32_t vis = 0;
  for (int k = 0; k < n_query; ++k) {
    const uint32_t m = nearest_code(tris + box0 + 12 * k, 12, px, py, xs, ys);
    if (m < cur) {               // GL_LESS against rooms + every box drawn before
      vis |= 1u << ent_slot[k];
      cur = m;
    }
  }
  return vis;
}

// entity-list slots the reference loops over: every entity except the agent (miniworld.py:1299-1301)
MWB_DEV int queried_entities(const DevState& S, int i, int* ent_slot) {
  const size_t N = S.N;
  int n = 0;
  const int slots = S.num_slots[i], as = S.agent_slot[i];
  for (int e = 0; e < slots && n < 32; ++e) {
    if (e == as || e == S.ghost_slot[i]) continue;
    if (S.ent_proto[e * N + i] < 0) continue;
    ent_slot[n++] = e;
  }
  return n;
}

MWB_DEV void empty_bbox(TriRec& r) {
  r.bx = 1;      // x0 = 1 > x1 = 0: never hit
  r.by = 1;
}

#ifdef __CUDACC__
// rows: null = the agent's camera; else [N][ROW_WIDTH] designed cameras (x, z, dir[, cam_height, cam_fwd_disp,
// cam_pitch, cam_fov_y]), a skipped row leaves mask[i] as it is.  ROW_WIDTH is a template parameter so that the
// instances for the agent's camera and 3-column rows are the code they were before 7-column rows existed.
template <int MSAA, int ROW_WIDTH>
__global__ void __launch_bounds__(256) visible_ents_kernel(DevState S, RenderAssets A, TriRec* __restrict__ scratch, int cap,
                                                           int box0, uint32_t* __restrict__ mask, const double* __restrict__ rows) {
  const int i = blockIdx.x, tid = threadIdx.x;
  const int W = S.obs_w, H = S.obs_h;
  if (rows && view_row_skipped(rows + (size_t)i * ROW_WIDTH, ROW_WIDTH)) return;     // uniform across the block
  __shared__ Camera cam;
  __shared__ int ent_slot[32];
  __shared__ int n_query, n_room;
  __shared__ uint32_t vis_all;
  TriRec* tris = scratch + (size_t)i * cap;
  if (tid == 0) {
    cam = rows ? make_row_camera(S, i, rows + (size_t)i * ROW_WIDTH, ROW_WIDTH) : make_camera(S, i);
    n_query = queried_entities(S, i, ent_slot);
    n_room = 0;
    vis_all = 0;
  }
  __syncthreads();
  const mwb_quad* quads = env_quads(S, i);
  const int nq = S.num_quads[geom_index(S, i)];
  for (int task = tid; task < 2 * nq; task += 256) {
    TriInput in;
    TriRec rec;
    if (room_triangle(S, A, quads, i, task >> 1, task & 1, in) && finish_triangle(cam, in, W, H, rec))
      tris[atomicAdd(&n_room, 1)] = rec;          // depth only: the order of the room triangles is irrelevant
  }
  for (int j = tid; j < 12 * n_query; j += 256) {
    TriInput in;
    TriRec rec;
    query_box_triangle(entity_pose(S, i, ent_slot[j / 12]), j % 12, in);
    if (!finish_triangle(cam, in, W, H, rec)) empty_bbox(rec);
    tris[box0 + j] = rec;
  }
  __syncthreads();
  uint32_t vis = 0;
  const int total = W * H * MSAA;
  for (int idx = tid; idx < total; idx += 256) {
    const int s = idx % MSAA, pix = idx / MSAA;
    const int px = pix % W, py = pix / W;
    float ox, oy;
    sample_xy_dyn<MSAA>(s, ox, oy);
    vis |= visible_at_sample(tris, n_room, box0, n_query, ent_slot, px, py, (float)px + ox, (float)py + oy);
  }
  vis = __reduce_or_sync(0xffffffffu, vis);
  if ((tid & 31) == 0 && vis) atomicOr(&vis_all, vis);
  __syncthreads();
  if (tid == 0) mask[i] = vis_all;
}
#endif
