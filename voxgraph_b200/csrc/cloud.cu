// Point-cloud messages on the device: the first half of PointcloudIntegrator::integratePointcloud
// (voxgraph/src/frontend/measurement_processors/pointcloud_integrator.cpp:29-63), i.e. pcl::fromROSMsg +
// voxblox::convertPointcloud, restated from the published message definition and sources (the rules are in
// include/voxgraph_b200.h; nothing here was checked against a compiled PCL or voxblox).
// Compiled with -fmad=false like the integration it feeds.
//
// One kernel.  A warp takes 32 consecutive records of one row: they are contiguous in the message
// (32 * point_step bytes), so the warp copies the 16-byte-aligned window around them into shared memory with
// coalesced 16-byte loads and every lane then picks its record's fields out of shared memory, at any byte
// offset.  One strided 4-byte load per field per lane would touch the same sectors once per field instead.
// The window may start up to 15 bytes before the records and end up to 15 bytes after them: the kernel only
// ever reads the library's own copy of the message, which starts 256-byte aligned in a scratch part whose size is
// rounded up to 256 bytes (vgx_carve), so the window never leaves the part.  Records longer than
// CLOUD_STAGE_STEP bytes are not staged; their fields are read from global memory directly.
//
// The integrate path leaves dropped records in place: their coordinates are written as they are, and the
// integration kernels skip a point with a non-finite coordinate without counting it, so no compaction and no
// count is needed on the host before the integration kernels launch.  vgx_cloud_decode compacts
// (flag -> exclusive scan -> scatter), because its caller wants convertPointcloud's arrays.
#include <limits.h>
#include <math.h>
#include <string.h>

#include "vgx_internal.h"

#define CLOUD_WARPS 4            // warps per CTA
#define CLOUD_STAGE_STEP 128     // longest record staged through shared memory

struct CloudParams {
  vgx_cloud_layout L;
  unsigned warps_per_row;        // ceil(width / 32)
  unsigned n_warps;              // height * warps_per_row
  unsigned stage_bytes;          // shared memory per warp: 32 * point_step + 32, or 0 (unstaged)
  float colour_max;
};

// 4 bytes at any alignment, little endian; p is a shared or global address
__device__ __forceinline__ uint32_t cloud_word(const uint8_t* p) {
  if ((reinterpret_cast<uintptr_t>(p) & 3) == 0) return *reinterpret_cast<const uint32_t*>(p);
  return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

// GrayscaleColorMap::colorLookup -> r, g, b, a bytes in memory order.  The clamp is voxblox's
// std::min(max, std::max(0, value)) written out, so a NaN intensity gives 0.
__device__ __forceinline__ uint32_t cloud_gray(float value, float max_value) {
  float v = 0.0f < value ? value : 0.0f;
  v = v < max_value ? v : max_value;
  const float h = v / max_value;
  const uint32_t g = (uint32_t)floor((double)h * 255.0 + 0.5);
  return g | (g << 8) | (g << 16) | 0xff000000u;
}

// pts: 3 floats per slot; rgba (may be NULL): r, g, b, a bytes per slot; flags (may be NULL): 1 = kept;
// n_kept: += the kept records
__global__ void __launch_bounds__(CLOUD_WARPS * 32)
cloud_decode_kernel(CloudParams P, const uint8_t* __restrict__ data, float* __restrict__ pts,
                    uint32_t* __restrict__ rgba, unsigned* __restrict__ flags, unsigned long long* __restrict__ n_kept) {
  extern __shared__ uint4 cloud_stage[];
  const unsigned lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const unsigned warp = blockIdx.x * CLOUD_WARPS + wib;
  if (warp >= P.n_warps) return;          // whole warps leave; the kernel has no CTA-wide barrier
  const unsigned row = warp / P.warps_per_row, col0 = (warp % P.warps_per_row) * 32;
  const unsigned cnt = min(32u, P.L.width - col0);
  const uint8_t* src = data + (size_t)row * P.L.row_step + (size_t)col0 * P.L.point_step;
  const uint8_t* rec;
  if (P.stage_bytes) {
    uint8_t* stage = reinterpret_cast<uint8_t*>(cloud_stage) + (size_t)wib * P.stage_bytes;
    const unsigned lead = (unsigned)(reinterpret_cast<uintptr_t>(src) & 15);
    const uint4* window = reinterpret_cast<const uint4*>(src - lead);
    const unsigned n_vec = (lead + cnt * P.L.point_step + 15) >> 4;
    for (unsigned v = lane; v < n_vec; v += 32) reinterpret_cast<uint4*>(stage)[v] = __ldg(window + v);
    __syncwarp();
    rec = stage + lead + (size_t)lane * P.L.point_step;
  } else {
    rec = src + (size_t)lane * P.L.point_step;
  }
  bool keep = false;
  if (lane < cnt) {
    const float x = __uint_as_float(cloud_word(rec + P.L.x_offset));
    const float y = __uint_as_float(cloud_word(rec + P.L.y_offset));
    const float z = __uint_as_float(cloud_word(rec + P.L.z_offset));
    keep = isfinite(x) && isfinite(y) && isfinite(z);
    const size_t i = (size_t)row * P.L.width + col0 + lane;
    pts[3 * i] = x; pts[3 * i + 1] = y; pts[3 * i + 2] = z;
    if (rgba) {
      uint32_t c = 0xff000000u;                                          // colorLookup(0)
      if (P.L.rgb_offset >= 0) c = __byte_perm(cloud_word(rec + P.L.rgb_offset), 0, 0x3012);   // b g r a -> r g b a
      else if (P.L.intensity_offset >= 0)
        c = cloud_gray(__uint_as_float(cloud_word(rec + P.L.intensity_offset)), P.colour_max);
      rgba[i] = c;
    }
    if (flags) flags[i] = keep ? 1u : 0u;
  }
  const unsigned kept = __popc(__ballot_sync(0xffffffffu, keep));
  if (lane == 0 && kept) atomicAdd(n_kept, (unsigned long long)kept);
}

__global__ void __launch_bounds__(256)
cloud_compact_kernel(int n, const float* __restrict__ pts, const uint32_t* __restrict__ rgba,
                     const unsigned* __restrict__ flags, const unsigned* __restrict__ offsets,
                     float* __restrict__ out_pts, uint32_t* __restrict__ out_rgba) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !flags[i]) return;
  const size_t o = offsets[i];
  out_pts[3 * o] = pts[3 * (size_t)i]; out_pts[3 * o + 1] = pts[3 * (size_t)i + 1]; out_pts[3 * o + 2] = pts[3 * (size_t)i + 2];
  out_rgba[o] = rgba[i];
}

// the validation rules of the header -> the record count
static int cloud_check(vgx_ctx* c, const vgx_cloud_layout* L, const uint8_t* data, uint64_t n_bytes, float colour_max,
                       int* n) {
  if (!L) VGX_FAIL(c, VGX_ERR_INVALID, "point cloud: no layout");
  if (L->point_step == 0) VGX_FAIL(c, VGX_ERR_INVALID, "point cloud: point_step is 0");
  const auto inside = [&](int32_t off) { return off >= 0 && (uint64_t)off + 4 <= L->point_step; };
  if (!inside(L->x_offset) || !inside(L->y_offset) || !inside(L->z_offset))
    VGX_FAIL(c, VGX_ERR_INVALID, "point cloud: an x, y or z field does not lie inside the record");
  if ((L->rgb_offset != -1 && !inside(L->rgb_offset)) || (L->intensity_offset != -1 && !inside(L->intensity_offset)))
    VGX_FAIL(c, VGX_ERR_INVALID, "point cloud: the rgb or intensity field does not lie inside the record");
  if ((uint64_t)L->row_step < (uint64_t)L->width * L->point_step)
    VGX_FAIL(c, VGX_ERR_INVALID, "point cloud: row_step is shorter than width * point_step");
  if (n_bytes < (uint64_t)L->height * L->row_step)
    VGX_FAIL(c, VGX_ERR_INVALID, "point cloud: fewer bytes than height * row_step");
  const uint64_t records = (uint64_t)L->width * L->height;
  if (records > (uint64_t)INT_MAX) VGX_FAIL(c, VGX_ERR_INVALID, "point cloud: more than INT_MAX records");
  if (records > 0 && !data) VGX_FAIL(c, VGX_ERR_INVALID, "point cloud: no data");
  if (!(colour_max > 0.0f) || !isfinite(colour_max))
    VGX_FAIL(c, VGX_ERR_INVALID, "point cloud: colour_map_max must be a finite value > 0");
  *n = (int)records;
  return VGX_OK;
}

// Uploads the message (height * row_step bytes, one asynchronous copy from the caller's pageable buffer, the way
// vgx_tsdf_integrate sends its points) into d_raw and decodes it into the slot arrays.
static int cloud_decode_launch(vgx_ctx* c, const vgx_cloud_layout& L, const uint8_t* data, float colour_max,
                               uint8_t* d_raw, float* d_pts, uint32_t* d_rgba, unsigned* d_flags,
                               unsigned long long* d_kept) {
  CloudParams P;
  P.L = L;
  P.warps_per_row = (L.width + 31) / 32;
  P.n_warps = L.height * P.warps_per_row;      // <= records <= INT_MAX
  P.stage_bytes = L.point_step <= CLOUD_STAGE_STEP ? 32 * L.point_step + 32 : 0;
  P.colour_max = colour_max;
  VGX_TRY(vgx_upload(c, d_raw, data, (size_t)L.height * L.row_step));
  VgxProfileScope scope(c, VGX_SLOT_CLOUD_DECODE);
  return vgx_launch(c, cloud_decode_kernel, (P.n_warps + CLOUD_WARPS - 1) / CLOUD_WARPS, CLOUD_WARPS * 32,
                    CLOUD_WARPS * (size_t)P.stage_bytes, VgxLaunch::plain, P, d_raw, d_pts, d_rgba, d_flags, d_kept);
}

extern "C" int vgx_cloud_decode(vgx_ctx* c, const vgx_cloud_layout* L, const uint8_t* data, uint64_t n_bytes,
                                float colour_max, int max_points, float* points_C, uint8_t* rgba, int* n_points) {
  return vgx_entry(c, __func__, [&] {
    int n = 0;
    VGX_TRY(cloud_check(c, L, data, n_bytes, colour_max, &n));
    if (max_points < 0) VGX_FAIL(c, VGX_ERR_INVALID, "negative max_points");
    if (n_points) *n_points = 0;
    if (n == 0) return VGX_OK;
    uint8_t* d_raw;
    float *d_pts, *d_out_pts;
    uint32_t *d_rgba, *d_out_rgba;
    unsigned long long* d_kept;
    unsigned *d_flags, *d_offsets, *d_scan_tmp;
    VGX_TRY(vgx_carve(c, c->d_scratch, vgx_part(d_raw, (size_t)L->height * L->row_step), vgx_part(d_pts, 3 * (size_t)n),
                      vgx_part(d_rgba, (size_t)n), vgx_part(d_out_pts, 3 * (size_t)n), vgx_part(d_out_rgba, (size_t)n),
                      vgx_part(d_kept, 1)));
    VGX_TRY(vgx_carve(c, c->d_work, vgx_part(d_flags, (size_t)n + 2), vgx_part(d_offsets, (size_t)n + 2),
                      vgx_part(d_scan_tmp, vgx_scan_tmp_count((size_t)n))));
    VGX_TRY(vgx_fill(c, d_kept, 1));
    VGX_TRY(cloud_decode_launch(c, *L, data, colour_max, d_raw, d_pts, d_rgba, d_flags, d_kept));
    {
      VgxProfileScope scope(c, VGX_SLOT_CLOUD_DECODE);
      VGX_TRY(vgx_exclusive_scan_u32(c, d_flags, d_offsets, (size_t)n, d_scan_tmp));
      VGX_TRY(vgx_launch(c, cloud_compact_kernel, (unsigned)((n + 255) / 256), 256, 0, VgxLaunch::plain, n, d_pts, d_rgba,
                         d_flags, d_offsets, d_out_pts, d_out_rgba));
    }
    unsigned kept = 0;
    VGX_TRY(vgx_read(c, &kept, d_offsets + n));
    if (n_points) *n_points = (int)kept;
    if ((points_C || rgba) && kept > (unsigned)max_points)
      VGX_FAIL(c, VGX_ERR_CAPACITY, "more kept points than max_points");
    if (points_C) VGX_TRY(vgx_download(c, points_C, d_out_pts, 3 * (size_t)kept));
    // the caller's r, g, b, a bytes against the device's colour words: written in bytes
    if (rgba) VGX_TRY(vgx_download(c, rgba, reinterpret_cast<const uint8_t*>(d_out_rgba), 4 * (size_t)kept));
    return vgx_sync(c);
  });
}

extern "C" int vgx_tsdf_integrate_cloud(vgx_ctx* c, uint32_t id, const float T_G_C[7], const vgx_cloud_layout* L,
                                        const uint8_t* data, uint64_t n_bytes, int colours, float colour_max,
                                        const vgx_tsdf_config* cfg, vgx_tsdf_stats* stats, int* n_points) {
  return vgx_entry(c, __func__, [&] {
    int n = 0;
    VGX_TRY(cloud_check(c, L, data, n_bytes, colour_max, &n));
    VgxSubmap* s;
    vgx_tsdf_config rcfg;
    VGX_TRY(vgx_tsdf_check(c, id, T_G_C, cfg, &s, &rcfg));
    if (n == 0) {
      if (stats) memset(stats, 0, sizeof(*stats));
      if (n_points) *n_points = 0;
      return VGX_OK;
    }
    // scratch: message bytes | point slots | stats | (fast) the two approximate sets | colour slots
    uint8_t* d_raw;
    float* d_pts;
    unsigned long long *d_stats, *d_sets;
    uint32_t* d_rgba;
    VGX_TRY(vgx_carve(c, c->d_scratch, vgx_part(d_raw, (size_t)L->height * L->row_step), vgx_part(d_pts, 3 * (size_t)n),
                      vgx_part(d_stats, VGX_TSDF_STAT_WORDS), vgx_part(d_sets, vgx_tsdf_set_words(rcfg)),
                      vgx_part(d_rgba, colours ? (size_t)n : 0)));
    VGX_TRY(vgx_fill(c, d_stats, VGX_TSDF_STAT_WORDS));
    VGX_TRY(cloud_decode_launch(c, *L, data, colour_max, d_raw, d_pts, colours ? d_rgba : nullptr, nullptr,
                                d_stats + VGX_TSDF_STAT_CALLER));
    return vgx_tsdf_integrate_resident(c, s, T_G_C, rcfg, n, d_pts, colours ? d_rgba : nullptr, d_stats, d_sets, stats,
                                       n_points);
  });
}
