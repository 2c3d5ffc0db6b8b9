// bank.cuh -- the state bank (mwb_enable_state_bank): per-env state records in device memory.
//
// A record (StateBank in state.h) is everything a running episode is, gathered from the structure-of-arrays rows of
// one env: the BankCol scalars, then, on handles with per-env worlds, the env's world block.  One warp moves one
// record: the lanes split the scalars (the table is in record order, so the record side of each round is one
// contiguous run) and the world block's rooms, quads and segments in use, copied in 16-byte words where source and
// destination share their 16-byte phase and in 8-byte words otherwise.  bank_save_kernel (mwb.cu) saves; bank_load
// runs at the top of device_reset.
#pragma once
#include "state.h"

#ifndef __CUDACC__
struct uint4 { unsigned int x, y, z, w; };
#endif

#ifdef __CUDA_ARCH__
#define MWB_LANE() ((int)(threadIdx.x & 31))
#define MWB_LANES 32
#else
#define MWB_LANE() 0
#define MWB_LANES 1
#endif

// `bytes` (a multiple of 8) from src to dst by the lanes of a warp, four words in flight per lane
MWB_DEV void bank_copy_bytes(uint8_t* dst, const uint8_t* src, size_t bytes, int lane, int lanes) {
  size_t head = 0;
  if ((((uintptr_t)dst ^ (uintptr_t)src) & 15) == 0) {
    head = (16 - ((uintptr_t)src & 15)) & 15;
    if (head > bytes) head = bytes;
    if (head && lane == 0) *(uint2*)dst = *(const uint2*)src;   // the 8-byte word before the first 16-byte boundary
    const size_t body = (bytes - head) / 16;
    const uint4* s4 = (const uint4*)(src + head);
    uint4* d4 = (uint4*)(dst + head);
    size_t k = lane;
    for (; k + 3 * lanes < body; k += 4 * lanes) {
      const uint4 a = s4[k], b = s4[k + lanes], c = s4[k + 2 * lanes], d = s4[k + 3 * lanes];
      d4[k] = a;
      d4[k + lanes] = b;
      d4[k + 2 * lanes] = c;
      d4[k + 3 * lanes] = d;
    }
    for (; k < body; k += lanes) d4[k] = s4[k];
    head += body * 16;
    if (head < bytes && lane == 0) *(uint2*)(dst + head) = *(const uint2*)(src + head);   // the 8-byte tail
    return;
  }
  const size_t words = bytes / 8;
  const uint2* s2 = (const uint2*)src;
  uint2* d2 = (uint2*)dst;
  size_t k = lane;
  for (; k + 3 * lanes < words; k += 4 * lanes) {
    const uint2 a = s2[k], b = s2[k + lanes], c = s2[k + 2 * lanes], d = s2[k + 3 * lanes];
    d2[k] = a;
    d2[k + lanes] = b;
    d2[k + 2 * lanes] = c;
    d2[k + 3 * lanes] = d;
  }
  for (; k < words; k += lanes) d2[k] = s2[k];
}

// Env i's state <-> record `rec` (save: into the record), by the lanes of one warp.  `world`: env i's world block
// takes part (on a save, the env's level has per-env worlds; on a load, the record holds a world).  The scalars move as
// integers of their width, so every value, NaNs included, arrives bit for bit.
MWB_DEV void bank_move(const StateBank* B, int i, uint8_t* rec, bool save, bool world) {
  const int lane = MWB_LANE(), lanes = MWB_LANES;
  for (int c = lane; c < B->num_cols; c += lanes) {
    const BankCol col = B->cols[c];
    uint8_t* e = col.base + (size_t)i * col.env_stride;
    uint8_t* r = rec + col.rec_off;
    uint8_t* dst = save ? r : e;
    const uint8_t* src = save ? e : r;
    if (col.bytes == 8) *(uint64_t*)dst = *(const uint64_t*)src;
    else if (col.bytes == 4) *(uint32_t*)dst = *(const uint32_t*)src;
    else *dst = *src;
  }
  if (!world || B->world_off < 0) return;
  const size_t g = (size_t)B->env_geom + i;
  int32_t* head = (int32_t*)(rec + B->world_off);
  int n[3];   // rooms, quads, segments in use
  if (save) {
    n[0] = B->num_rooms[g];
    n[1] = B->num_quads[g];
    n[2] = B->num_segs[g];
    if (lane == 0) {
      head[0] = n[0];
      head[1] = n[1];
      head[2] = n[2];
      head[3] = 1;
    }
  } else {
    n[0] = head[0];
    n[1] = head[1];
    n[2] = head[2];
    if (lane == 0) {
      B->num_rooms[g] = n[0];
      B->num_quads[g] = n[1];
      B->num_segs[g] = n[2];
    }
  }
  uint8_t* env = (uint8_t*)(B->rooms + g * B->R);
  uint8_t* own = rec + B->room_off;
  bank_copy_bytes(save ? own : env, save ? env : own, (size_t)n[0] * sizeof(mwb_room), lane, lanes);
  env = (uint8_t*)(B->quads + g * B->Q);
  own = rec + B->quad_off;
  bank_copy_bytes(save ? own : env, save ? env : own, (size_t)n[1] * sizeof(mwb_quad), lane, lanes);
  env = (uint8_t*)(B->segs + g * B->S);
  own = rec + B->seg_off;
  bank_copy_bytes(save ? own : env, save ? env : own, (size_t)n[2] * sizeof(mwb_seg), lane, lanes);
}

// Save env i into slot s (bank_save_kernel's warp t, which won slot s).
MWB_DEV void bank_save(const StateBank* B, const int32_t* env_level, const LevelDev* levels, int i, int s) {
  const int lvl = env_level[i];
  uint8_t* rec = B->records + (size_t)s * B->rec_bytes;
  const bool world = B->world_off >= 0 && levels[lvl].env_worlds;
  bank_move(B, i, rec, true, world);
  if (B->world_off >= 0 && !world && MWB_LANE() == 0) ((int32_t*)(rec + B->world_off))[3] = 0;
  if (MWB_LANE() == 0) B->bank_level[s] = lvl;
}

// The load rule of env i's reset (include/mwb.h, mwb_enable_state_bank): a pending slot is consumed; when it is filled
// and its level is the env's, or level changes are on (`any_level`), env i becomes the record and the function returns
// 1, and device_reset returns without running the level's program.  Otherwise it returns 0 and the reset runs as it
// would have.  episode_state names the loaded slot or -1.  Out of line, like seed_stream: only the bank's handles
// reach it.  As in take_seed, every lane computes the same values from the same loads, and warp barriers separate the
// loads from the stores.
MWB_DEV_NOINLINE int bank_load(const StateBank* B, int i, int cur_level, int any_level) {
  MWB_WARP_SYNC();
  const int s = B->next_state[i];
  const int lvl = s >= 0 && s < B->slots ? B->bank_level[s] : -1;
  const bool take = lvl >= 0 && (lvl == cur_level || any_level);
  MWB_WARP_SYNC();
  if (s != -1) B->next_state[i] = -1;
  B->episode_state[i] = take ? s : -1;
  if (take) {
    const uint8_t* rec = B->records + (size_t)s * B->rec_bytes;
    bank_move(B, i, (uint8_t*)rec, false, B->world_off >= 0 && ((const int32_t*)(rec + B->world_off))[3] != 0);
  }
  MWB_WARP_SYNC();
  return take ? 1 : 0;
}
