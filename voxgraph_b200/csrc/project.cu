// Projected global TSDF map on the device (SURVEY §8 visualisation rows):
//   cblox SubmapCollection::getProjectedMap = for every submap S in increasing id order
//   voxblox mergeLayerAintoLayerB(S.layer, T_M_S, &global) (merge_integration.h), i.e. transformLayer
//   into a fresh layer, then the untransformed merge.  cblox's generateCombinedMesh and voxgraph's
//   save_combined_mesh / ProjectedMapServer consume the result.
//
// The rule (restated from the published voxblox / cblox sources, not checked against a compiled
// voxblox; the CPU restatement tests/project_oracle.c pins it bit for bit):
//   1. candidate output blocks (transformLayer): for every allocated block b of S, c_out = T_M_S *
//      ((b + 0.5) * block_size), offset = sqrt(3) * block_size * 0.5; per axis a float x steps from
//      c_out - offset while x < c_out + offset by block_size (two samples), and each of the 8 sample
//      points names the block floor(p / block_size + 1e-6).  The enumeration can miss output blocks at
//      the edge of a rotated submap; the port keeps that.
//   2. resampling: every voxel centre of a candidate block (origin + (v + 0.5) * voxel_size) is mapped by
//      T_S_M = T_M_S.inverse() and interpolated trilinearly in S (Interpolator::getVoxel, all 8
//      neighbours observed, ex_interp_voxel); a voxel that fails stays (0, 0), and a candidate block none
//      of whose voxels succeeds does not exist in S's transformed layer.
//   3. merge (mergeVoxelAIntoVoxelB): every voxel of every existing transformed block, (0, 0) ones
//      included: w = wA + wB; if w > 0: d = (dA * wA + dB * wB) / w, weight w.  Float, no FMA.
//   4. colour, when any input has a colour channel (then the output gets one; otherwise the launches and
//      the output are the colour-free ones): the resampling interpolates every channel like the distance
//      and truncates (ex_interp_voxel_impl<true>, layer_access.cuh); inside the merge's if (w > 0):
//      colourB = blendTwoColors(colourA, wA, colourB, wB) (colour.cuh).  An input without a channel
//      contributes colour 0 with its weight, as voxblox's default-coloured voxels do.  Same id-ordered
//      fold, so the colour is as order independent as the distance.
// Output blocks in ascending packed key ((z + 2^20) << 42 | (y + 2^20) << 21 | (x + 2^20)).
//
// Passes: candidates (one thread per input block, 8 (key, submap rank) pairs, rank = position in id
// order) -> stable cub radix sort by key, so each key's submaps come out in id order -> unique adjacent
// (key, rank) and keys (flags, two scans, scatter) -> occupancy (one CTA per key: does any submap's
// transformed block exist there) -> scan -> gather-and-fold (one CTA per kept key, each thread folds its
// voxels over the key's submaps in id order, a __syncthreads_or per submap decides whether its block
// exists) straight into the new submap's bricks -> the upload path of submap.cu.  No float atomics: the
// result does not depend on thread order.  Compiled with -fmad=false.
//
// vgx_submap_transform (voxblox transformLayer into the submap's own, uncleared layer; see the header)
// runs the same passes on one submap with two differences: every old block also enters as its own
// candidate key and is always kept (occupancy), and the fold is transform_fold_kernel: per voxel the
// interpolated (d, w) where the interpolation succeeds, else the old voxel where the block existed, else
// (0, 0).  The result goes to a scratch submap that then takes the transformed submap's id.
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <utility>
#include <vector>

#include <cub/cub.cuh>

#include "colour.cuh"
#include "layer_access.cuh"

// 63 bits set: a packed key never reaches it (each 21-bit field is at most 2^21 - 2), so it sorts last
#define PROJ_NO_KEY 0x7FFFFFFFFFFFFFFFull
#define PROJ_KEY_BITS 63
#define PROJ_THREADS 256

// voxblox kUnitCubeDiagonalLength = std::sqrt(3.0) as FloatingPoint
static constexpr float kUnitCubeDiagonalLength = 1.7320508075688772f;

struct ProjSrc {
  LayerDev L;
  float T[7];        // T_M_S [qw qx qy qz tx ty tz]
  float T_inv[7];    // T_S_M = T_M_S.inverse()
  int first_block;   // this submap's first block in the rank-ordered list of all input blocks
};

// voxel v of output block b (geometry of S), moved into S's frame
__device__ __forceinline__ void proj_voxel_in_submap(const ProjSrc& S, const int b[3], int v, float p[3]) {
  const LayerDev& L = S.L;
  int x[3];
  vgx_voxel_xyz(v, L.sh, x);
  float c[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) c[a] = vgx_voxel_centre(b[a], x[a], L.block_size, L.voxel_size);
  ov_transform(S.T_inv, c, p);
}

// does output block b exist in S's transformed layer: any of its voxels interpolates.  Called by every
// thread of the CTA; stops at the first chunk of voxels with a success.
__device__ __forceinline__ bool proj_block_exists(const ProjSrc& S, const int b[3]) {
  const int vpb = vgx_voxels_per_block(S.L.sh);
  for (int base = 0; base < vpb; base += blockDim.x) {
    const int v = base + (int)threadIdx.x;
    bool ok = false;
    if (v < vpb) {
      float p[3], d, w;
      proj_voxel_in_submap(S, b, v, p);
      ok = ex_interp_voxel(S.L, p[0], p[1], p[2], d, w);
    }
    if (__syncthreads_or(ok)) return true;
  }
  return false;
}

// pass 1: the 8 candidate (key, rank) pairs of every input block; unused slots get PROJ_NO_KEY.
// err: bit 1 = a candidate block index outside [VGX_BLOCK_INDEX_MIN, VGX_BLOCK_INDEX_MAX],
//      bit 2 = more than two samples on an axis (cannot happen for finite poses)
__global__ void __launch_bounds__(128)
project_candidate_kernel(const ProjSrc* __restrict__ src, int n_src, int n_blocks, bool own, uint64_t* __restrict__ keys,
                         uint32_t* __restrict__ ranks, int* __restrict__ err) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_blocks) return;
  int lo = 0, hi = n_src - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (src[mid].first_block <= g) lo = mid; else hi = mid - 1;
  }
  const ProjSrc& S = src[lo];
  const int slot = g - S.first_block;
  const float bs = S.L.block_size, inv = S.L.block_size_inv;
  float c_in[3], c_out[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) c_in[a] = ((float)S.L.block_idx[3 * slot + a] + 0.5f) * bs;
  ov_transform(S.T, c_in, c_out);
  const float offset = kUnitCubeDiagonalLength * bs * 0.5f;
  float smp[3][2];
  int ns[3];
  int bad = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {   // for (x = c - offset; x < c + offset; x += block_size), at most 2 samples
    const float x0 = c_out[a] - offset, x1 = x0 + bs;
    smp[a][0] = x0;
    smp[a][1] = x1;
    ns[a] = !(x0 < c_out[a] + offset) ? 0 : !(x1 < c_out[a] + offset) ? 1 : 2;
    if (ns[a] == 2 && x1 + bs < c_out[a] + offset) bad |= 4;
  }
  uint64_t* ko = keys + 8 * (size_t)g;
  uint32_t* ro = ranks + 8 * (size_t)g;
#pragma unroll
  for (int k = 0; k < 8; ++k) {   // sample (k >> 2, (k >> 1) & 1, k & 1) of the x, y, z lists
    const int i[3] = {k >> 2, (k >> 1) & 1, k & 1};
    uint64_t key = PROJ_NO_KEY;
    if (i[0] < ns[0] && i[1] < ns[1] && i[2] < ns[2]) {
      int q[3];
      bool in_range = true;
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        const float f = floorf(smp[a][i[a]] * inv + 1e-6f);   // getGridIndexFromPoint
        in_range = in_range && f >= (float)VGX_BLOCK_INDEX_MIN && f <= (float)VGX_BLOCK_INDEX_MAX;
        q[a] = in_range ? (int)f : 0;
      }
      if (in_range) key = vgx_pack_key(q[0], q[1], q[2]);
      else bad |= 2;
    }
    ko[k] = key;
    ro[k] = (uint32_t)lo;
  }
  if (own) {   // vgx_submap_transform: the old block itself, after all 8 n_blocks samples
    keys[8 * (size_t)n_blocks + g] =
        vgx_pack_key(S.L.block_idx[3 * slot], S.L.block_idx[3 * slot + 1], S.L.block_idx[3 * slot + 2]);
    ranks[8 * (size_t)n_blocks + g] = (uint32_t)lo;
  }
  if (bad) atomicOr(err, bad);
}

// pass 3a: heads of the distinct (key, rank) pairs and of the distinct keys in the sorted list
__global__ void __launch_bounds__(256)
project_flag_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ ranks, size_t n,
                    unsigned* __restrict__ pair_head, unsigned* __restrict__ key_head) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t k = keys[i];
  const bool live = k != PROJ_NO_KEY;
  const bool new_key = i == 0 || keys[i - 1] != k;
  pair_head[i] = (live && (new_key || ranks[i - 1] != ranks[i])) ? 1u : 0u;
  key_head[i] = (live && new_key) ? 1u : 0u;
}

// pass 3b: the distinct ranks of every key (in id order), the distinct keys and their segments
__global__ void __launch_bounds__(256)
project_scatter_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ ranks, size_t n,
                       const unsigned* __restrict__ pair_head, const unsigned* __restrict__ key_head,
                       const unsigned* __restrict__ pair_pos, const unsigned* __restrict__ key_pos,
                       uint64_t* __restrict__ ukey, uint32_t* __restrict__ urank, uint32_t* __restrict__ useg) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) useg[key_pos[n]] = pair_pos[n];
  if (i >= n) return;
  if (pair_head[i]) urank[pair_pos[i]] = ranks[i];
  if (key_head[i]) {
    ukey[key_pos[i]] = keys[i];
    useg[key_pos[i]] = pair_pos[i];
  }
}

// pass 4: keep[k] = 1 when any submap's transformed block exists at key k (keep_own, vgx_submap_transform:
// or the single source already has a block there)
__global__ void __launch_bounds__(PROJ_THREADS, 1)   // (256) alone spills 12 bytes at 48 registers
project_occupancy_kernel(const ProjSrc* __restrict__ src, const uint64_t* __restrict__ ukey,
                         const uint32_t* __restrict__ urank, const uint32_t* __restrict__ useg, bool keep_own,
                         unsigned* __restrict__ keep) {
  const int k = blockIdx.x;
  int b[3];
  vgx_unpack_key(ukey[k], b);
  unsigned any = keep_own && vgx_hash_find(src[0].L.hash, b[0], b[1], b[2]) >= 0 ? 1u : 0u;
  for (uint32_t j = useg[k]; !any && j < useg[k + 1]; ++j)
    if (proj_block_exists(src[urank[j]], b)) { any = 1; break; }
  if (threadIdx.x == 0) keep[k] = any;
}

__device__ __forceinline__ void proj_fold(float dA, float wA, float& dB, float& wB) {
  const float w = wA + wB;
  if (w > 0) {
    dB = (dA * wA + dB * wB) / w;
    wB = w;
  }
}

// pass 6: one CTA per key; thread t owns voxels t + j * blockDim.x (j < VPT), folded over the key's
// submaps in id order.  kRegs: the running (d, w) in registers; otherwise (vps 32) in the output brick,
// which only the owning thread reads and writes.  kColour: the running colour beside them (rule 4).
template <int VPT, bool kRegs, bool kColour>
__global__ void __launch_bounds__(PROJ_THREADS)
project_fold_kernel(const ProjSrc* __restrict__ src, const uint64_t* __restrict__ ukey,
                    const uint32_t* __restrict__ urank, const uint32_t* __restrict__ useg,
                    const unsigned* __restrict__ out_slot, float2* __restrict__ out_dw, int32_t* __restrict__ out_idx,
                    uint32_t* __restrict__ out_rgba) {
  const int k = blockIdx.x;
  const unsigned s = out_slot[k];
  if (out_slot[k + 1] == s) return;
  int b[3];
  vgx_unpack_key(ukey[k], b);
  if (threadIdx.x == 0) {
    out_idx[3 * (size_t)s] = b[0];
    out_idx[3 * (size_t)s + 1] = b[1];
    out_idx[3 * (size_t)s + 2] = b[2];
  }
  const int vpb = VPT * (int)blockDim.x;
  float2* brick = out_dw + (size_t)s * vpb;
  uint32_t* cbrick = kColour ? out_rgba + (size_t)s * vpb : nullptr;
  float ad[kRegs ? VPT : 1], aw[kRegs ? VPT : 1];
  uint32_t ac[kRegs && kColour ? VPT : 1];
#pragma unroll
  for (int t = 0; t < (kRegs ? VPT : 1); ++t) ad[t] = aw[t] = 0.0f;
#pragma unroll
  for (int t = 0; t < (kRegs && kColour ? VPT : 1); ++t) ac[t] = 0u;
  if (!kRegs)
    for (int t = 0; t < VPT; ++t) {
      brick[threadIdx.x + t * blockDim.x] = make_float2(0.0f, 0.0f);
      if (kColour) cbrick[threadIdx.x + t * blockDim.x] = 0u;
    }
  for (uint32_t j = useg[k]; j < useg[k + 1]; ++j) {
    const ProjSrc& S = src[urank[j]];
    if (!proj_block_exists(S, b)) continue;
#pragma unroll
    for (int t = 0; t < VPT; ++t) {
      const int v = (int)threadIdx.x + t * (int)blockDim.x;
      float p[3], dA = 0.0f, wA = 0.0f;
      proj_voxel_in_submap(S, b, v, p);
      uint32_t cA = 0u;
      bool ok;
      if (kColour && S.L.rgba) ok = ex_interp_voxel_impl<true>(S.L, p[0], p[1], p[2], dA, wA, cA);
      else ok = ex_interp_voxel(S.L, p[0], p[1], p[2], dA, wA);
      if (!ok) { dA = wA = 0.0f; cA = 0u; }
      if (kRegs) {
        if (kColour && wA + aw[t] > 0) ac[t] = vgx_colour_blend(cA, wA, ac[t], aw[t]);
        proj_fold(dA, wA, ad[t], aw[t]);
      } else {
        float2 q = brick[v];
        if (kColour && wA + q.y > 0) cbrick[v] = vgx_colour_blend(cA, wA, cbrick[v], q.y);
        proj_fold(dA, wA, q.x, q.y);
        brick[v] = q;
      }
    }
  }
  if (kRegs)
#pragma unroll
    for (int t = 0; t < VPT; ++t) {
      brick[threadIdx.x + t * blockDim.x] = make_float2(ad[t], aw[t]);
      if (kColour) cbrick[threadIdx.x + t * blockDim.x] = ac[t];
    }
}

// vgx_submap_transform, pass 6: one CTA per kept key of the single source S (the old copy).  Every voxel
// centre is moved by T_old_new = T_new_old.inverse() and interpolated in S; a success takes the interpolated
// (d, w), a failure keeps the old voxel where S has the block and is (0, 0) otherwise.  No merge.
__global__ void __launch_bounds__(PROJ_THREADS)
transform_fold_kernel(const ProjSrc* __restrict__ src, const uint64_t* __restrict__ ukey,
                      const unsigned* __restrict__ out_slot, float2* __restrict__ out_dw,
                      int32_t* __restrict__ out_idx) {
  const int k = blockIdx.x;
  const unsigned s = out_slot[k];
  if (out_slot[k + 1] == s) return;
  int b[3];
  vgx_unpack_key(ukey[k], b);
  if (threadIdx.x == 0) {
    out_idx[3 * (size_t)s] = b[0];
    out_idx[3 * (size_t)s + 1] = b[1];
    out_idx[3 * (size_t)s + 2] = b[2];
  }
  const ProjSrc& S = src[0];
  const int old = vgx_hash_find(S.L.hash, b[0], b[1], b[2]);
  const int vpb = vgx_voxels_per_block(S.L.sh);
  float2* brick = out_dw + (size_t)s * vpb;
  for (int v = threadIdx.x; v < vpb; v += blockDim.x) {
    float p[3], d = 0.0f, w = 0.0f;
    proj_voxel_in_submap(S, b, v, p);
    float2 q;
    if (ex_interp_voxel(S.L, p[0], p[1], p[2], d, w)) q = make_float2(d, w);
    else q = old >= 0 ? S.L.dw[vgx_voxel_index(old, v, S.L.sh)] : make_float2(0.0f, 0.0f);
    brick[v] = q;
  }
}

// ------------------------------------------------------------------ host
static int launch_fold(vgx_ctx* c, int vps, unsigned n_keys, const ProjSrc* d_src, const uint64_t* ukey,
                       const uint32_t* urank, const uint32_t* useg, const unsigned* slot, VgxSubmap* s) {
  uint32_t* rgba = s->d_rgba.get();   // the output has a channel iff an input has one
  switch (vps) {
#define PROJ_FOLD(VPT, REGS, THREADS)                                                                              \
  return vgx_launch(c, rgba ? project_fold_kernel<VPT, REGS, true> : project_fold_kernel<VPT, REGS, false>, n_keys, \
                    THREADS, 0, VgxLaunch::plain, d_src, ukey, urank, useg, slot, s->d_dw.get(),                    \
                    s->d_block_idx.get(), rgba);
    case 2: PROJ_FOLD(1, true, 8)
    case 4: PROJ_FOLD(1, true, 64)
    case 8: PROJ_FOLD(2, true, 256)
    case 16: PROJ_FOLD(16, true, 256)
    case 32: PROJ_FOLD(128, false, 256)
#undef PROJ_FOLD
    default: VGX_FAIL(c, VGX_ERR_INVALID, "unsupported voxels_per_side");
  }
}

// subs / poses in rank (id) order; creates out_id on success.  transform (one submap, vgx_submap_transform):
// the old blocks are candidates and kept as well, and the fold is transform_fold_kernel.
static int project(vgx_ctx* c, const std::vector<VgxSubmap*>& subs, const std::vector<const float*>& poses,
                   uint32_t out_id, int* n_out_blocks, bool transform = false) {
  const int ns = (int)subs.size();
  const VgxSubmap& g0 = *subs[0];
  std::vector<ProjSrc> h((size_t)ns);
  size_t n_in = 0;
  for (int r = 0; r < ns; ++r) {
    memset(&h[r], 0, sizeof(ProjSrc));
    h[r].L = layer_of(subs[r]);
    memcpy(h[r].T, poses[r], 7 * sizeof(float));
    ov_inverse(h[r].T, h[r].T_inv);
    h[r].first_block = (int)n_in;
    n_in += (size_t)subs[r]->n_blocks;
  }
  const size_t per_block = transform ? 9 : 8;   // candidate pairs per input block
  if (n_in > (size_t)INT32_MAX / per_block)
    VGX_FAIL(c, VGX_ERR_CAPACITY, transform ? "more than 2^31 / 9 input blocks"
                                            : "more than 2^28 input blocks");
  const size_t P = per_block * n_in;
  cudaStream_t st = c->stream;
  unsigned n_keys = 0, n_out = 0;
  // scratch in d_work: pairs (double-buffered for the sort), flags, scans, segments, source table
  size_t sort_tmp = 0;
  if (P > 0)
    VGX_CUDA(c, cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (unsigned long long*)nullptr,
                                                (unsigned long long*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr,
                                                (int)P, 0, PROJ_KEY_BITS, st));
  uint64_t* keys_a;     // candidates, then the distinct keys
  uint64_t* keys_b;     // sorted keys
  uint32_t* ranks_a;    // candidates, then the distinct ranks per key
  uint32_t* ranks_b;    // sorted ranks
  unsigned* pair_head;  // then keep flags
  unsigned *key_head, *pair_pos /* then output slots */, *key_pos, *scan_tmp;
  uint32_t* useg;
  ProjSrc* d_src;
  int* d_ctl;
  char* d_sort_tmp;
  VGX_TRY(vgx_carve(c, c->d_work, vgx_part(keys_a, P + 1), vgx_part(keys_b, P + 1), vgx_part(ranks_a, P + 1),
                    vgx_part(ranks_b, P + 1), vgx_part(pair_head, P + 1), vgx_part(key_head, P + 1),
                    vgx_part(pair_pos, P + 1), vgx_part(key_pos, P + 1), vgx_part(useg, P + 1),
                    vgx_part(scan_tmp, vgx_scan_tmp_count(P + 1)), vgx_part(d_src, (size_t)ns), vgx_part(d_ctl, 1),
                    vgx_part(d_sort_tmp, sort_tmp)));
  if (P > 0) {
    VGX_TRY(vgx_upload(c, d_src, h.data(), (size_t)ns));
    VGX_TRY(vgx_fill(c, d_ctl, 1));
    {
      VgxProfileScope scope(c, VGX_SLOT_PROJECT);
      VGX_TRY(vgx_launch(c, project_candidate_kernel, (unsigned)((n_in + 127) / 128), 128, 0, VgxLaunch::plain, d_src, ns,
                         (int)n_in, transform, keys_a, ranks_a, d_ctl));
    }
    {
      VgxProfileScope scope(c, VGX_SLOT_PROJECT);
      VGX_CUDA(c, cub::DeviceRadixSort::SortPairs(d_sort_tmp, sort_tmp, (unsigned long long*)keys_a,
                                                  (unsigned long long*)keys_b, ranks_a, ranks_b, (int)P, 0,
                                                  PROJ_KEY_BITS, st));
      vgx_count_launch(c);
    }
    const unsigned gp = (unsigned)((P + 255) / 256);
    {
      VgxProfileScope scope(c, VGX_SLOT_PROJECT);
      VGX_TRY(vgx_launch(c, project_flag_kernel, gp, 256, 0, VgxLaunch::plain, keys_b, ranks_b, P, pair_head, key_head));
    }
    {
      VgxProfileScope scope(c, VGX_SLOT_PROJECT);
      VGX_TRY(vgx_exclusive_scan_u32(c, pair_head, pair_pos, P, scan_tmp));
      VGX_TRY(vgx_exclusive_scan_u32(c, key_head, key_pos, P, scan_tmp));
    }
    {
      VgxProfileScope scope(c, VGX_SLOT_PROJECT);
      VGX_TRY(vgx_launch(c, project_scatter_kernel, gp, 256, 0, VgxLaunch::plain, keys_b, ranks_b, P, pair_head, key_head,
                         pair_pos, key_pos, keys_a, ranks_a, useg));
    }
    int ctl = 0;
    VGX_TRY(vgx_download(c, &ctl, d_ctl, 1));
    VGX_TRY(vgx_download(c, &n_keys, key_pos + P, 1));
    VGX_TRY(vgx_sync(c));
    if (ctl & 2)
      VGX_FAIL(c, VGX_ERR_INVALID, "a projected block index lies outside the accepted range");
    if (ctl & 4)
      VGX_FAIL(c, VGX_ERR_INVALID, "more than two candidate samples on an axis");
  }
  unsigned* keep = pair_head;
  unsigned* slot = pair_pos;
  if (n_keys > 0) {
    {
      VgxProfileScope scope(c, VGX_SLOT_PROJECT);
      VGX_TRY(vgx_launch(c, project_occupancy_kernel, n_keys, std::min(PROJ_THREADS, g0.vox_per_block), 0,
                         VgxLaunch::plain, d_src, keys_a, ranks_a, useg, transform, keep));
    }
    {
      VgxProfileScope scope(c, VGX_SLOT_PROJECT);
      VGX_TRY(vgx_exclusive_scan_u32(c, keep, slot, n_keys, scan_tmp));
    }
    VGX_TRY(vgx_read(c, &n_out, slot + n_keys));
  }
  VgxSubmap* s = nullptr;
  VGX_TRY(vgx_submap_alloc(c, out_id, g0.voxel_size, g0.vps, (int)n_out, true, &s));
  s->n_blocks = (int)n_out;
  s->finished = true;
  if (n_out > 0 && transform) {
    VgxProfileScope scope(c, VGX_SLOT_EVAL);
    VGX_TRY(vgx_launch(c, transform_fold_kernel, n_keys, std::min(PROJ_THREADS, g0.vox_per_block), 0, VgxLaunch::plain,
                       d_src, keys_a, slot, s->d_dw.get(), s->d_block_idx.get()));
  } else if (n_out > 0) {
    bool coloured = false;
    for (const VgxSubmap* in : subs) coloured = coloured || in->d_rgba.get();
    if (coloured) VGX_TRY(vgx_submap_ensure_colour(c, s));
    VgxProfileScope scope(c, VGX_SLOT_PROJECT);
    VGX_TRY(launch_fold(c, g0.vps, n_keys, d_src, keys_a, ranks_a, useg, slot, s));
  }
  VGX_TRY(vgx_submap_upload_finish(c, s));
  *n_out_blocks = (int)n_out;
  return VGX_OK;
}

extern "C" int vgx_project_map(vgx_ctx* c, int n, const uint32_t* ids, const float* T_M_S, uint32_t out_id,
                               int* n_blocks) {
  return vgx_entry(c, __func__, [&] {
    if (n_blocks) *n_blocks = 0;
    if (n < 1 || !ids || !T_M_S) VGX_FAIL(c, VGX_ERR_INVALID, "invalid argument");
    std::vector<std::pair<uint32_t, int>> order;   // (id, row of ids / T_M_S)
    for (int k = 0; k < n; ++k) {
      if (ids[k] == out_id) VGX_FAIL(c, VGX_ERR_INVALID, "out_id is one of the inputs");
      order.emplace_back(ids[k], k);
    }
    std::sort(order.begin(), order.end());
    for (int k = 1; k < n; ++k)
      if (order[k].first == order[k - 1].first)
        VGX_FAIL(c, VGX_ERR_INVALID, "repeated submap " + std::to_string(order[k].first));
    std::vector<VgxSubmap*> subs((size_t)n);
    std::vector<const float*> poses((size_t)n);
    for (int r = 0; r < n; ++r) {
      VGX_TRY(vgx_submap_get(c, order[r].first, &subs[r]));
      poses[r] = T_M_S + 7 * (size_t)order[r].second;
    }
    if (c->submaps.count(out_id)) VGX_FAIL(c, VGX_ERR_INVALID, "out_id already exists");
    for (int r = 1; r < n; ++r)
      if (subs[r]->voxel_size != subs[0]->voxel_size || subs[r]->vps != subs[0]->vps)
        VGX_FAIL(c, VGX_ERR_INVALID, "the submaps differ in voxel size or voxels_per_side");
    VGX_TRY(vgx_sync(c));   // n_blocks of an active submap is final after its integration
    int nb = 0;
    const int rc = project(c, subs, poses, out_id, &nb);
    if (rc != VGX_OK) {
      vgx_submap_drop(c, out_id);   // a failure after the allocation leaves a half-built submap
      return rc;
    }
    if (n_blocks) *n_blocks = nb;
    return VGX_OK;
  });
}

extern "C" int vgx_mesh_build_combined(vgx_ctx* c, int n, const uint32_t* ids, const float* T_M_S,
                                       const vgx_mesh_config* cfg) {
  return vgx_entry(c, __func__, [&] {
    const uint32_t pid = vgx_scratch_id(c);
    VGX_TRY(vgx_project_map(c, n, ids, T_M_S, pid, nullptr));
    const int rc = vgx_mesh_build(c, 1, &pid, nullptr, cfg, nullptr, nullptr);
    vgx_submap_drop(c, pid);
    return rc;
  });
}

extern "C" int vgx_submap_transform(vgx_ctx* c, uint32_t id, const float* T_new_old) {
  return vgx_entry(c, __func__, [&] {
    if (!T_new_old) VGX_FAIL(c, VGX_ERR_INVALID, "invalid argument");
    VgxSubmap* s;
    VGX_TRY(vgx_submap_get(c, id, &s));
    VGX_TRY(vgx_sync(c));   // n_blocks of an active submap is final after its integration
    // the result is built in a scratch submap next to the old copy, then takes the submap's id
    const uint32_t tmp = vgx_scratch_id(c);
    int nb = 0;
    const int rc = project(c, {s}, {T_new_old}, tmp, &nb, true);
    if (rc != VGX_OK) {
      vgx_submap_drop(c, tmp);
      return rc;
    }
    return vgx_submap_move(c, tmp, id);
  });
}
