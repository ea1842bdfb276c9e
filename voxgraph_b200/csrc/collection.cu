// cblox SubmapCollection byte stream <-> resident bricks (cblox::SubmapCollection::saveToFile,
// cblox::io::LoadSubmapCollection + VoxgraphSubmap::LoadFromStream, TSDF layer only).
//
// The host walks message framing and the header fields of every message; it never touches the voxel
// payload.  The payload (BlockProto.voxel_data, 3 uint32 varints per voxel) is decoded and encoded on
// the device, one CTA per block, straight from / into the resident (distance, weight) bricks.
//
// Wire format: restated from the published voxblox / cblox sources (utils::writeProtoMsgToStream,
// Block<TsdfVoxel>::serializeToIntegers, SubmapCollection::saveToFile and the Block, Submap,
// SubmapCollection and QuatTransformation .proto files, all proto2).  UNVERIFIED against a file
// written by cblox.  Every field number and wire type the library knows is in the table below and
// nowhere else; the parser is strict so that a wrong guess fails (VGX_ERR_INVALID) instead of
// producing a silently wrong map:
//   * a known field with another wire type is an error; unknown fields are skipped;
//   * tags, lengths and the integer fields read here are varints of at most 5 bytes that fit in 32 bits;
//   * voxel_data (packed or unpacked) must be the last field of a BlockProto, with exactly 3 vps^3 values;
//   * every block's voxels_per_side and voxel_size equal the collection header's;
//   * the stream ends right after the last block message.
// Colour: the third word of a voxel is kept as the file has it (uint32, never interpreted here).  The
// writer emits the word of a submap that has a colour channel and 0 (voxblox's default Color()) otherwise;
// the reader drops it (vgx_collection_load, vgx_layer_load) or, with VGX_COLLECTION_KEEP_COLOUR, stores it
// and keeps the channel of the submaps in which some word is non-zero.
//
// vgx_layer_load reads voxblox layer files (io::LoadLayer<TsdfVoxel>) through the same block parser, decode
// kernel and upload path: a varint32 message count, LayerProto {voxel_size, voxels_per_side, type "tsdf"},
// count - 1 BlockProto.  Also restated from the published voxblox sources and UNVERIFIED against a file
// written by voxblox.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <set>
#include <string>
#include <vector>

#include "layer_access.cuh"

// ------------------------------------------------------------------ format table
namespace {

enum : uint32_t { kWireVarint = 0, kWireFixed64 = 1, kWireLen = 2, kWireFixed32 = 5 };
struct FieldSpec {
  uint32_t number, wire;
};
__host__ __device__ constexpr uint32_t tag_of(FieldSpec f) { return (f.number << 3) | f.wire; }

// SubmapCollectionProto (the first message of a stream)
constexpr FieldSpec kCollVoxelSize{1, kWireFixed64};      // double
constexpr FieldSpec kCollVoxelsPerSide{2, kWireVarint};   // uint32
constexpr FieldSpec kCollNumSubmaps{3, kWireVarint};      // uint32
// SubmapProto (one per submap, followed by num_blocks BlockProto messages)
constexpr FieldSpec kSubmapId{1, kWireVarint};            // uint32
constexpr FieldSpec kSubmapNumBlocks{2, kWireVarint};     // uint32
constexpr FieldSpec kSubmapTransform{3, kWireLen};        // QuatTransformationProto (T_M_S)
// QuatTransformationProto
constexpr FieldSpec kTransformPosition{1, kWireLen};      // PositionProto {1 x, 2 y, 3 z: double}
constexpr FieldSpec kTransformRotation{2, kWireLen};      // QuaternionProto {1 w, 2 x, 3 y, 4 z: double}
constexpr uint32_t kPositionFields = 3, kRotationFields = 4;   // fields 1..n, all kWireFixed64
// voxblox layer files (io::LoadLayer): a varint32 message count (utils::writeProtoMsgCountToStream, not a
// delimited message), then LayerProto and count - 1 BlockProto messages
constexpr FieldSpec kLayerVoxelSize{1, kWireFixed64};     // double
constexpr FieldSpec kLayerVoxelsPerSide{2, kWireVarint};  // uint32
constexpr FieldSpec kLayerType{3, kWireLen};              // string: "tsdf" for a TsdfVoxel layer
// BlockProto
constexpr FieldSpec kBlockVoxelsPerSide{1, kWireVarint};  // int32
constexpr FieldSpec kBlockVoxelSize{2, kWireFixed64};     // double
constexpr FieldSpec kBlockOrigin[3] = {{3, kWireFixed64}, {4, kWireFixed64}, {5, kWireFixed64}};
constexpr FieldSpec kBlockHasData{6, kWireVarint};        // bool
constexpr FieldSpec kBlockVoxelData{7, kWireVarint};      // repeated uint32: 3 words per voxel
constexpr FieldSpec kBlockVoxelDataPacked{7, kWireLen};   //   (the same field, packed)
constexpr uint32_t kWordsPerVoxel = 3;                    // distance bits, weight bits, rgba colour

constexpr uint8_t kTagVoxelData = (uint8_t)tag_of(kBlockVoxelData);              // 0x38
constexpr uint8_t kTagVoxelDataPacked = (uint8_t)tag_of(kBlockVoxelDataPacked);  // 0x3A
// the BlockProto header fields the emit pass writes
constexpr uint8_t kTagBlockVoxelsPerSide = (uint8_t)tag_of(kBlockVoxelsPerSide);
constexpr uint8_t kTagBlockVoxelSize = (uint8_t)tag_of(kBlockVoxelSize);
constexpr uint8_t kTagBlockOriginX = (uint8_t)tag_of(kBlockOrigin[0]);
constexpr uint8_t kTagBlockOriginY = (uint8_t)tag_of(kBlockOrigin[1]);
constexpr uint8_t kTagBlockOriginZ = (uint8_t)tag_of(kBlockOrigin[2]);
constexpr uint8_t kTagBlockHasData = (uint8_t)tag_of(kBlockHasData);
static_assert(kTagVoxelData == 0x38 && kTagVoxelDataPacked == 0x3A, "one-byte voxel_data tags");

}  // namespace

// One block's voxel_data region: [first field-7 tag, end of the block message).
struct CollBlockRef {
  uint64_t off, len;
  int32_t packed;
  int32_t pad;
};

// ------------------------------------------------------------------ device codec
#define COLL_THREADS 256
#define COLL_DEC_BPT 16                                  // bytes per thread per tile
#define COLL_DEC_TILE (COLL_THREADS * COLL_DEC_BPT)
#define COLL_DEC_APRON 8                                 // bytes of the previous tile kept in front
#define COLL_ENC_VPT 16                                  // voxels per thread per tile

// error bits of the per-call error word
#define COLL_ERR_TAG 1        // a tag inside voxel_data other than 0x38 (unpacked) / a bad packed header
#define COLL_ERR_VARINT 2     // a varint of more than 5 bytes or above 32 bits, or a truncated one
#define COLL_ERR_COUNT 4      // not exactly 3 vps^3 values
#define COLL_ERR_LENGTH 8     // packed length does not cover the region exactly

// exclusive scan over the CTA (COLL_THREADS threads); *total = sum of all v
__device__ __forceinline__ unsigned coll_block_scan(unsigned v, unsigned* total) {
  __shared__ unsigned warp_sums[COLL_THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned x = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned y = __shfl_up_sync(0xffffffffu, x, d);
    if (lane >= d) x += y;
  }
  if (lane == 31) warp_sums[warp] = x;
  __syncthreads();
  unsigned before = 0, all = 0;
#pragma unroll
  for (int w = 0; w < COLL_THREADS / 32; ++w) {
    const unsigned s = warp_sums[w];
    if (w < warp) before += s;
    all += s;
  }
  __syncthreads();   // warp_sums is reused by the next call
  *total = all;
  return before + x - v;
}

// One CTA per block.  Every byte < 0x80 ends a varint; a CTA scan of those terminators numbers the
// varints of the region, and the terminator's thread assembles the value from at most 4 preceding
// bytes.  Unpacked: varint 2k is a tag (must be 0x38), 2k+1 is value k.  Packed: varint 0 is the 0x3A
// tag, varint 1 the length (must reach exactly to the region's end), 2 + k is value k.  Value k goes to
// voxel k / 3: word 0 = distance bits, 1 = weight bits, 2 (colour) goes to rgba and, when non-zero, raises
// *any_colour; with rgba == NULL it is dropped.
__global__ void __launch_bounds__(COLL_THREADS)
collection_decode_kernel(const uint8_t* __restrict__ bytes, const CollBlockRef* __restrict__ regions,
                         int vox_per_block, float* __restrict__ dw, uint32_t* __restrict__ rgba,
                         int* __restrict__ any_colour, int* __restrict__ err) {
  __shared__ uint8_t sb[COLL_DEC_APRON + COLL_DEC_TILE];
  const CollBlockRef r = regions[blockIdx.x];
  const unsigned n_values = kWordsPerVoxel * (unsigned)vox_per_block;
  const unsigned n_varints = r.packed ? n_values + 2 : 2 * n_values;
  float* out = dw + (size_t)blockIdx.x * vox_per_block * 2;
  const uint8_t* src = bytes + r.off;
  unsigned ord_base = 0;
  int bad = 0;
  bool coloured = false;
  for (uint64_t t0 = 0; t0 < r.len; t0 += COLL_DEC_TILE) {
    // bytes before the region read as 0 (a terminator), so no varint reaches across its start
    for (int k = threadIdx.x; k < COLL_DEC_APRON + COLL_DEC_TILE; k += COLL_THREADS) {
      const int64_t pos = (int64_t)t0 + k - COLL_DEC_APRON;
      sb[k] = (pos >= 0 && (uint64_t)pos < r.len) ? __ldg(src + pos) : 0;
    }
    __syncthreads();
    const int my0 = threadIdx.x * COLL_DEC_BPT;
    unsigned cnt = 0;
#pragma unroll
    for (int j = 0; j < COLL_DEC_BPT; ++j)
      if (t0 + my0 + j < r.len && sb[COLL_DEC_APRON + my0 + j] < 0x80) cnt++;
    unsigned total = 0;
    unsigned ord = ord_base + coll_block_scan(cnt, &total);
    for (int j = 0; j < COLL_DEC_BPT; ++j) {
      const uint64_t p = t0 + my0 + j;
      if (p >= r.len) break;
      const int q = COLL_DEC_APRON + my0 + j;
      const uint8_t b = sb[q];
      if (b >= 0x80) {
        if (p == r.len - 1) bad |= COLL_ERR_VARINT;   // the region ends inside a varint
        continue;
      }
      // assemble from the terminator backwards: at most 4 continuation bytes (5-byte varint)
      uint64_t v = b;
      int nb = 1;
      for (;;) {
        const uint8_t c = sb[q - nb];
        if (c < 0x80) break;
        if (nb == 5) { bad |= COLL_ERR_VARINT; break; }
        v = (v << 7) | (c & 0x7f);
        nb++;
      }
      if (v >> 32) bad |= COLL_ERR_VARINT;
      unsigned k;   // value index, or a framing varint
      if (r.packed) {
        if (ord == 0) {
          if (v != kTagVoxelDataPacked) bad |= COLL_ERR_TAG;
          ord++;
          continue;
        }
        if (ord == 1) {
          if (v != r.len - p - 1) bad |= COLL_ERR_LENGTH;
          ord++;
          continue;
        }
        k = ord - 2;
      } else {
        if ((ord & 1) == 0) {
          if (v != kTagVoxelData) bad |= COLL_ERR_TAG;
          ord++;
          continue;
        }
        k = ord >> 1;
      }
      ord++;
      if (k >= n_values) { bad |= COLL_ERR_COUNT; continue; }
      const unsigned voxel = k / kWordsPerVoxel, word = k - voxel * kWordsPerVoxel;
      if (word < 2) out[2 * (size_t)voxel + word] = __uint_as_float((uint32_t)v);
      else if (rgba) {
        rgba[(size_t)blockIdx.x * vox_per_block + voxel] = (uint32_t)v;
        coloured |= (uint32_t)v != 0;
      }
    }
    ord_base += total;
    __syncthreads();   // sb is refilled
  }
  if (threadIdx.x == 0 && ord_base != n_varints) bad |= COLL_ERR_COUNT;
  if (bad) atomicOr(err, bad);
  if (coloured && any_colour) *any_colour = 1;
}

__device__ __forceinline__ unsigned coll_varint_len(uint32_t v) {
  const unsigned bits = 32 - __clz(v | 1u);
  return (bits + 6) / 7;
}
__device__ __forceinline__ uint8_t* coll_put_varint(uint8_t* p, uint32_t v) {
  while (v >= 0x80) {
    *p++ = (uint8_t)(v | 0x80);
    v >>= 7;
  }
  *p++ = (uint8_t)v;
  return p;
}
__device__ __forceinline__ uint8_t* coll_put_double(uint8_t* p, uint8_t tag, double d) {
  *p++ = tag;
  const unsigned long long u = (unsigned long long)__double_as_longlong(d);
#pragma unroll
  for (int i = 0; i < 8; ++i) *p++ = (uint8_t)(u >> (8 * i));
  return p;
}
// bytes of one voxel in the unpacked form: 3 x (tag 0x38 + varint)
__device__ __forceinline__ unsigned coll_voxel_bytes(float2 v, uint32_t colour) {
  return 3 + coll_varint_len(__float_as_uint(v.x)) + coll_varint_len(__float_as_uint(v.y)) + coll_varint_len(colour);
}

struct CollEncodeArgs {
  const float2* dw;           // the submap's bricks
  const uint32_t* rgba;       // its colour channel, or NULL: every colour word is 0
  const int32_t* block_idx;   // n x 3
  int vox_per_block;
  int vps;
  float voxel_size, block_size;
  const uint32_t* sizes;      // EMIT: voxel_data bytes of each block (from the size pass)
  uint32_t* out_sizes;        // !EMIT
  const uint64_t* offsets;    // EMIT: where each framed block message starts in dst
  uint8_t* dst;
  uint32_t header_bytes;      // BlockProto fields 1-6
};

// One CTA per block.  Size pass (EMIT = false): the bytes of the block's voxel_data, by a CTA scan of
// per-voxel sizes.  Emit pass: the whole delimited BlockProto (length, fields 1-6, then voxel_data
// unpacked in linear voxel order), at the offset the host laid out.
template <bool EMIT>
__global__ void __launch_bounds__(COLL_THREADS) collection_encode_kernel(CollEncodeArgs a) {
  const int blk = blockIdx.x;
  const float2* src = a.dw + (size_t)blk * a.vox_per_block;
  const uint32_t* col = a.rgba ? a.rgba + (size_t)blk * a.vox_per_block : nullptr;
  uint8_t* payload = nullptr;
  if (EMIT) {
    uint8_t* p = a.dst + a.offsets[blk];
    const uint32_t msg = a.header_bytes + a.sizes[blk];
    int hdr = 0;
    for (uint32_t m = msg; m >= 0x80; m >>= 7) hdr++;
    payload = p + hdr + 1 + a.header_bytes;
    if (threadIdx.x == 0) {
      p = coll_put_varint(p, msg);
      *p++ = kTagBlockVoxelsPerSide;
      p = coll_put_varint(p, (uint32_t)a.vps);
      p = coll_put_double(p, kTagBlockVoxelSize, (double)a.voxel_size);
      // Block origin = index * block_size (float), stored as double
      const int32_t* bi = a.block_idx + 3 * blk;
      p = coll_put_double(p, kTagBlockOriginX, (double)__fmul_rn((float)bi[0], a.block_size));
      p = coll_put_double(p, kTagBlockOriginY, (double)__fmul_rn((float)bi[1], a.block_size));
      p = coll_put_double(p, kTagBlockOriginZ, (double)__fmul_rn((float)bi[2], a.block_size));
      *p++ = kTagBlockHasData;
      *p++ = 1;
    }
  }
  unsigned base = 0;
  for (int v0 = 0; v0 < a.vox_per_block; v0 += COLL_THREADS * COLL_ENC_VPT) {
    const int my0 = v0 + threadIdx.x * COLL_ENC_VPT;
    unsigned cnt = 0;
    for (int j = 0; j < COLL_ENC_VPT; ++j)
      if (my0 + j < a.vox_per_block) cnt += coll_voxel_bytes(src[my0 + j], col ? col[my0 + j] : 0u);
    unsigned total = 0;
    const unsigned excl = coll_block_scan(cnt, &total);
    if (EMIT) {
      uint8_t* p = payload + base + excl;
      for (int j = 0; j < COLL_ENC_VPT; ++j) {
        if (my0 + j >= a.vox_per_block) break;
        const float2 v = src[my0 + j];
        *p++ = kTagVoxelData;
        p = coll_put_varint(p, __float_as_uint(v.x));
        *p++ = kTagVoxelData;
        p = coll_put_varint(p, __float_as_uint(v.y));
        *p++ = kTagVoxelData;
        p = coll_put_varint(p, col ? col[my0 + j] : 0u);
      }
    }
    base += total;
  }
  if (!EMIT && threadIdx.x == 0) a.out_sizes[blk] = base;
}

// ------------------------------------------------------------------ host framing
namespace {

struct Cursor {
  const uint8_t* p;
  const uint8_t* end;
};

// a varint of at most max_bytes; *nbytes = its length
bool get_varint(Cursor& c, int max_bytes, uint64_t* v, int* nbytes) {
  uint64_t x = 0;
  for (int i = 0; i < max_bytes; ++i) {
    if (c.p >= c.end) return false;
    const uint8_t b = *c.p++;
    x |= (uint64_t)(b & 0x7f) << (7 * i);
    if (b < 0x80) {
      *v = x;
      *nbytes = i + 1;
      return true;
    }
  }
  return false;
}
bool get_varint32(Cursor& c, uint32_t* v) {
  uint64_t x = 0;
  int nb = 0;
  if (!get_varint(c, 5, &x, &nb) || (x >> 32)) return false;
  *v = (uint32_t)x;
  return true;
}

struct Field {
  uint32_t number, wire;
  uint64_t value;       // varint / fixed
  bool narrow;          // varint: at most 5 bytes and within 32 bits
  Cursor sub;           // length-delimited payload
  const uint8_t* start; // position of the tag
};

// next field of a message; unknown-field payloads are consumed as protobuf skips them
bool next_field(Cursor& c, Field* f) {
  f->start = c.p;
  uint32_t tag = 0;
  if (!get_varint32(c, &tag)) return false;
  f->number = tag >> 3;
  f->wire = tag & 7;
  if (f->number == 0) return false;
  int nb = 0;
  switch (f->wire) {
    case kWireVarint:
      if (!get_varint(c, 10, &f->value, &nb)) return false;
      f->narrow = nb <= 5 && (f->value >> 32) == 0;
      return true;
    case kWireFixed64:
    case kWireFixed32: {
      const int n = f->wire == kWireFixed64 ? 8 : 4;
      if (c.end - c.p < n) return false;
      f->value = 0;
      for (int i = 0; i < n; ++i) f->value |= (uint64_t)c.p[i] << (8 * i);
      c.p += n;
      return true;
    }
    case kWireLen: {
      uint32_t len = 0;
      if (!get_varint32(c, &len) || (uint64_t)(c.end - c.p) < len) return false;
      f->sub = Cursor{c.p, c.p + len};
      c.p += len;
      return true;
    }
    default:   // groups (3, 4) and undefined wire types
      return false;
  }
}

bool is(const Field& f, FieldSpec s, bool* wire_ok) {
  if (f.number != s.number) return false;
  *wire_ok = f.wire == s.wire;
  return true;
}
double as_double(uint64_t bits) {
  double d;
  memcpy(&d, &bits, sizeof d);
  return d;
}

struct CollSubmapRef {
  uint32_t id, n_blocks;
  float T[7];   // qw qx qy qz tx ty tz
  size_t first_block;
};
struct CollLayout {
  double voxel_size = 0;
  uint32_t vps = 0;
  std::vector<CollSubmapRef> submaps;
  std::vector<CollBlockRef> blocks;
  std::vector<int32_t> block_idx;   // 3 per block
};

struct Parser {
  const uint8_t* base;
  Cursor c;
  std::string err;

  bool fail(const std::string& e) {
    err = "collection stream at byte " + std::to_string((long long)(c.p - base)) + ": " + e;
    return false;
  }
  // next delimited message of the stream
  bool message(Cursor* m, const char* what) {
    if (c.p >= c.end) return fail(std::string("stream ends before the ") + what);
    uint32_t len = 0;
    if (!get_varint32(c, &len)) return fail(std::string("bad length of the ") + what);
    if ((uint64_t)(c.end - c.p) < len) return fail(std::string("truncated ") + what);
    *m = Cursor{c.p, c.p + len};
    c.p += len;
    return true;
  }

  bool header(CollLayout* L, uint32_t* num_submaps) {
    Cursor m;
    if (!message(&m, "SubmapCollectionProto")) return false;
    bool have[3] = {false, false, false};
    Field f;
    while (m.p < m.end) {
      if (!next_field(m, &f)) return fail("malformed SubmapCollectionProto field");
      bool ok = true;
      if (is(f, kCollVoxelSize, &ok)) {
        if (!ok) return fail("SubmapCollectionProto.voxel_size: wrong wire type");
        L->voxel_size = as_double(f.value);
        have[0] = true;
      } else if (is(f, kCollVoxelsPerSide, &ok)) {
        if (!ok || !f.narrow) return fail("SubmapCollectionProto.voxels_per_side: wrong wire type or width");
        L->vps = (uint32_t)f.value;
        have[1] = true;
      } else if (is(f, kCollNumSubmaps, &ok)) {
        if (!ok || !f.narrow) return fail("SubmapCollectionProto.num_submaps: wrong wire type or width");
        *num_submaps = (uint32_t)f.value;
        have[2] = true;
      }
    }
    if (!(have[0] && have[1] && have[2])) return fail("SubmapCollectionProto lacks a field");
    if (*num_submaps == 0) return true;   // no layer: the geometry is not used
    return geometry(*L);
  }

  // the layer geometry of the header, as the upload path accepts it
  bool geometry(const CollLayout& L) {
    if (!vgx_vps_ok(L.vps))
      return fail("voxels_per_side must be a power of two in [2, 32]");
    if (!(L.voxel_size > 0) || !((float)L.voxel_size > 0) || !isfinite((float)L.voxel_size))
      return fail("voxel_size must be positive and finite");
    return true;
  }

  bool doubles(Cursor m, uint32_t n_fields, double* out, const char* what) {
    Field f;
    while (m.p < m.end) {
      if (!next_field(m, &f)) return fail(std::string("malformed ") + what + " field");
      if (f.number >= 1 && f.number <= n_fields) {
        if (f.wire != kWireFixed64) return fail(std::string(what) + ": wrong wire type");
        out[f.number - 1] = as_double(f.value);
      }
    }
    return true;
  }

  bool submap(CollSubmapRef* s) {
    Cursor m;
    if (!message(&m, "SubmapProto")) return false;
    bool have_id = false, have_nb = false;
    double pos[3] = {0, 0, 0}, rot[4] = {0, 0, 0, 0};
    Field f, g;
    while (m.p < m.end) {
      if (!next_field(m, &f)) return fail("malformed SubmapProto field");
      bool ok = true;
      if (is(f, kSubmapId, &ok)) {
        if (!ok || !f.narrow) return fail("SubmapProto.id: wrong wire type or width");
        s->id = (uint32_t)f.value;
        have_id = true;
      } else if (is(f, kSubmapNumBlocks, &ok)) {
        if (!ok || !f.narrow) return fail("SubmapProto.num_blocks: wrong wire type or width");
        s->n_blocks = (uint32_t)f.value;
        have_nb = true;
      } else if (is(f, kSubmapTransform, &ok)) {
        if (!ok) return fail("SubmapProto.transform: wrong wire type");
        Cursor t = f.sub;
        while (t.p < t.end) {
          if (!next_field(t, &g)) return fail("malformed QuatTransformationProto field");
          if (is(g, kTransformPosition, &ok)) {
            if (!ok) return fail("QuatTransformationProto.position: wrong wire type");
            if (!doubles(g.sub, kPositionFields, pos, "PositionProto")) return false;
          } else if (is(g, kTransformRotation, &ok)) {
            if (!ok) return fail("QuatTransformationProto.rotation: wrong wire type");
            if (!doubles(g.sub, kRotationFields, rot, "QuaternionProto")) return false;
          }
        }
      }
    }
    if (!have_id || !have_nb) return fail("SubmapProto lacks its id or num_blocks");
    if (s->n_blocks > (uint32_t)INT32_MAX) return fail("SubmapProto.num_blocks too large");
    for (int k = 0; k < 4; ++k) s->T[k] = (float)rot[k];
    for (int k = 0; k < 3; ++k) s->T[4 + k] = (float)pos[k];
    return true;
  }

  bool block(const CollLayout& L, CollBlockRef* b, int32_t idx[3]) {
    Cursor m;
    if (!message(&m, "BlockProto")) return false;
    bool have_vps = false, have_vs = false, have_o[3] = {false, false, false}, have_data = false;
    int64_t vps = 0;
    double vs = 0, origin[3] = {0, 0, 0};
    Field f;
    while (m.p < m.end) {
      const uint8_t* at = m.p;
      if (!next_field(m, &f)) return fail("malformed BlockProto field");
      bool ok = true;
      if (f.number == kBlockVoxelData.number) {   // the last field: the device walks the rest
        if (f.wire != kBlockVoxelData.wire && f.wire != kBlockVoxelDataPacked.wire)
          return fail("BlockProto.voxel_data: wrong wire type");
        b->off = (uint64_t)(at - base);
        b->len = (uint64_t)(m.end - at);
        b->packed = f.wire == kBlockVoxelDataPacked.wire;
        have_data = true;
        break;
      }
      if (is(f, kBlockVoxelsPerSide, &ok)) {
        if (!ok || !f.narrow) return fail("BlockProto.voxels_per_side: wrong wire type or width");
        vps = (int64_t)f.value;
        have_vps = true;
      } else if (is(f, kBlockVoxelSize, &ok)) {
        if (!ok) return fail("BlockProto.voxel_size: wrong wire type");
        vs = as_double(f.value);
        have_vs = true;
      } else if (is(f, kBlockHasData, &ok)) {
        if (!ok || !f.narrow) return fail("BlockProto.has_data: wrong wire type or width");
      } else {
        for (int a = 0; a < 3; ++a)
          if (is(f, kBlockOrigin[a], &ok)) {
            if (!ok) return fail("BlockProto.origin: wrong wire type");
            origin[a] = as_double(f.value);
            have_o[a] = true;
          }
      }
    }
    if (!have_data) return fail("BlockProto without voxel_data");
    if (b->len > 2ull * 5 * kWordsPerVoxel * L.vps * L.vps * L.vps + 6)   // a bound for both forms
      return fail("BlockProto.voxel_data longer than 3 vps^3 varints");
    if (!have_vps || vps != (int64_t)L.vps) return fail("BlockProto.voxels_per_side differs from the collection's");
    if (!have_vs || vs != L.voxel_size) return fail("BlockProto.voxel_size differs from the collection's");
    if (!(have_o[0] && have_o[1] && have_o[2])) return fail("BlockProto lacks an origin coordinate");
    // voxblox getGridIndexFromOriginPoint: round(float(origin) * block_size_inv), in float
    const float block_size = (float)L.voxel_size * (float)L.vps;
    const float block_size_inv = (float)(1.0 / (double)block_size);
    for (int a = 0; a < 3; ++a) {
      const float q = (float)origin[a] * block_size_inv;
      if (!(fabsf(q) < 1073741824.0f)) return fail("BlockProto.origin out of range");
      idx[a] = (int32_t)roundf(q);
    }
    return true;
  }

  // the next n BlockProtos, appended to L's blocks
  bool blocks(CollLayout* L, uint32_t n) {
    for (uint32_t k = 0; k < n; ++k) {
      CollBlockRef b{};
      int32_t idx[3];
      if (!block(*L, &b, idx)) return false;
      L->blocks.push_back(b);
      L->block_idx.insert(L->block_idx.end(), idx, idx + 3);
    }
    return true;
  }

  // a voxblox layer file (vgx_layer_load): the whole stream is one layer, held as one submap entry
  bool layer_stream(CollLayout* L) {
    uint32_t count = 0;
    if (!get_varint32(c, &count)) return fail("bad message count");
    if (count == 0) return fail("message count 0: no LayerProto");
    Cursor m;
    if (!message(&m, "LayerProto")) return false;
    bool have[3] = {false, false, false};
    std::string type;
    Field f;
    while (m.p < m.end) {
      if (!next_field(m, &f)) return fail("malformed LayerProto field");
      bool ok = true;
      if (is(f, kLayerVoxelSize, &ok)) {
        if (!ok) return fail("LayerProto.voxel_size: wrong wire type");
        L->voxel_size = as_double(f.value);
        have[0] = true;
      } else if (is(f, kLayerVoxelsPerSide, &ok)) {
        if (!ok || !f.narrow) return fail("LayerProto.voxels_per_side: wrong wire type or width");
        L->vps = (uint32_t)f.value;
        have[1] = true;
      } else if (is(f, kLayerType, &ok)) {
        if (!ok) return fail("LayerProto.type: wrong wire type");
        type.assign((const char*)f.sub.p, (size_t)(f.sub.end - f.sub.p));
        have[2] = true;
      }
    }
    if (!(have[0] && have[1] && have[2])) return fail("LayerProto lacks a field");
    if (type != "tsdf") return fail("LayerProto.type is not \"tsdf\"");
    if (!geometry(*L)) return false;
    CollSubmapRef s{};
    s.n_blocks = count - 1;
    s.first_block = 0;
    if (s.n_blocks > (uint32_t)INT32_MAX) return fail("too many blocks");
    if (!blocks(L, s.n_blocks)) return false;
    L->submaps.push_back(s);
    if (c.p != c.end) return fail("trailing bytes after the last block");
    return true;
  }

  bool stream(CollLayout* L) {
    uint32_t num_submaps = 0;
    if (!header(L, &num_submaps)) return false;
    std::set<uint32_t> ids;
    for (uint32_t i = 0; i < num_submaps; ++i) {
      CollSubmapRef s{};
      if (!submap(&s)) return false;
      if (!ids.insert(s.id).second) return fail("submap id " + std::to_string(s.id) + " appears twice");
      s.first_block = L->blocks.size();
      if (!blocks(L, s.n_blocks)) return false;
      L->submaps.push_back(s);
    }
    if (c.p != c.end) return fail("trailing bytes after the last block");
    if (L->blocks.size() > (size_t)INT32_MAX) return fail("too many blocks");
    return true;
  }
};

// layer: a voxblox layer file (one submap entry) instead of a submap collection
bool parse_stream(const uint8_t* bytes, uint64_t n, bool layer, CollLayout* L, std::string* err) {
  Parser p{bytes, Cursor{bytes, bytes + n}, std::string()};
  if (!bytes && n) {
    *err = "null stream";
    return false;
  }
  const bool ok = layer ? p.layer_stream(L) : p.stream(L);
  if (!ok) *err = p.err;
  return ok;
}

// host-side writers of the framing the host lays out
void put_varint(std::vector<uint8_t>& o, uint64_t v) {
  while (v >= 0x80) {
    o.push_back((uint8_t)(v | 0x80));
    v >>= 7;
  }
  o.push_back((uint8_t)v);
}
unsigned varint_len(uint64_t v) {
  unsigned n = 1;
  while (v >= 0x80) { v >>= 7; n++; }
  return n;
}
void put_tag(std::vector<uint8_t>& o, FieldSpec f) { put_varint(o, tag_of(f)); }
void put_double(std::vector<uint8_t>& o, FieldSpec f, double d) {
  put_tag(o, f);
  uint64_t u;
  memcpy(&u, &d, sizeof u);
  for (int i = 0; i < 8; ++i) o.push_back((uint8_t)(u >> (8 * i)));
}
void put_delimited(std::vector<uint8_t>& o, const std::vector<uint8_t>& msg) {
  put_varint(o, msg.size());
  o.insert(o.end(), msg.begin(), msg.end());
}
void put_submessage(std::vector<uint8_t>& o, FieldSpec f, const std::vector<uint8_t>& msg) {
  put_tag(o, f);
  put_delimited(o, msg);
}
std::vector<uint8_t> collection_header(double voxel_size, uint32_t vps, uint32_t n) {
  std::vector<uint8_t> m;
  put_double(m, kCollVoxelSize, voxel_size);
  put_tag(m, kCollVoxelsPerSide);
  put_varint(m, vps);
  put_tag(m, kCollNumSubmaps);
  put_varint(m, n);
  return m;
}
std::vector<uint8_t> submap_message(uint32_t id, uint32_t n_blocks, const float T[7]) {
  std::vector<uint8_t> pos, rot, tf, m;
  for (uint32_t k = 0; k < kPositionFields; ++k) put_double(pos, FieldSpec{k + 1, kWireFixed64}, (double)T[4 + k]);
  for (uint32_t k = 0; k < kRotationFields; ++k) put_double(rot, FieldSpec{k + 1, kWireFixed64}, (double)T[k]);
  put_submessage(tf, kTransformPosition, pos);
  put_submessage(tf, kTransformRotation, rot);
  put_tag(m, kSubmapId);
  put_varint(m, id);
  put_tag(m, kSubmapNumBlocks);
  put_varint(m, n_blocks);
  put_submessage(m, kSubmapTransform, tf);
  return m;
}
// BlockProto fields 1-6 as the emit pass writes them
uint32_t block_header_bytes(int vps) { return 1 + varint_len((uint64_t)vps) + 4 * 9 + 2; }

// Host <-> device copies of the stream through two pinned staging halves, so the host-side memcpy of
// one chunk overlaps the DMA of the other.
constexpr size_t kChunk = (size_t)8 << 20;
struct EventPair {
  cudaEvent_t e[2] = {nullptr, nullptr};
  ~EventPair() {
    for (auto& x : e)
      if (x) cudaEventDestroy(x);
  }
  int init(vgx_ctx* c) {
    for (auto& x : e) VGX_CUDA(c, cudaEventCreateWithFlags(&x, cudaEventDisableTiming));
    return VGX_OK;
  }
};

int copy_h2d_chunked(vgx_ctx* c, uint8_t* d, const uint8_t* h, uint64_t n) {
  if (n == 0) return VGX_OK;
  uint8_t* stage;
  VGX_TRY(vgx_carve(c, c->h_pinned, vgx_part(stage, 2 * kChunk)));
  EventPair ev;
  VGX_TRY(ev.init(c));
  uint64_t off = 0;
  for (int k = 0; off < n; ++k) {
    const size_t len = (size_t)std::min<uint64_t>(kChunk, n - off);
    uint8_t* half = stage + (k & 1) * kChunk;
    if (k >= 2) VGX_CUDA(c, cudaEventSynchronize(ev.e[k & 1]));
    memcpy(half, h + off, len);
    VGX_TRY(vgx_upload(c, d + off, half, len));
    VGX_CUDA(c, cudaEventRecord(ev.e[k & 1], c->stream));
    off += len;
  }
  return vgx_sync(c);   // the staging buffer is reused by the next call
}

int copy_d2h_chunked(vgx_ctx* c, uint8_t* h, const uint8_t* d, uint64_t n) {
  if (n == 0) return VGX_OK;
  uint8_t* stage;
  VGX_TRY(vgx_carve(c, c->h_pinned, vgx_part(stage, 2 * kChunk)));
  EventPair ev;
  VGX_TRY(ev.init(c));
  const uint64_t chunks = (n + kChunk - 1) / kChunk;
  for (uint64_t k = 0; k <= chunks; ++k) {
    if (k < chunks) {   // enqueue chunk k, then drain chunk k - 1 while it runs
      const size_t len = (size_t)std::min<uint64_t>(kChunk, n - k * kChunk);
      VGX_TRY(vgx_download(c, stage + (k & 1) * kChunk, d + k * kChunk, len));
      VGX_CUDA(c, cudaEventRecord(ev.e[k & 1], c->stream));
    }
    if (k >= 1) {
      const uint64_t j = k - 1;
      const size_t len = (size_t)std::min<uint64_t>(kChunk, n - j * kChunk);
      VGX_CUDA(c, cudaEventSynchronize(ev.e[j & 1]));
      memcpy(h + j * kChunk, stage + (j & 1) * kChunk, len);
    }
  }
  return VGX_OK;
}

}  // namespace

// ------------------------------------------------------------------ C-ABI
extern "C" int vgx_collection_scan(const uint8_t* bytes, uint64_t n, int max_submaps, vgx_collection_entry* out,
                                   int* n_submaps) {
  return vgx_entry_noctx([&] {
    if (!n_submaps || max_submaps < 0 || (max_submaps > 0 && !out)) return VGX_ERR_INVALID;
    *n_submaps = 0;
    CollLayout L;
    std::string err;
    if (!parse_stream(bytes, n, false, &L, &err)) return VGX_ERR_INVALID;
    if (L.submaps.size() > (size_t)INT32_MAX) return VGX_ERR_INVALID;
    *n_submaps = (int)L.submaps.size();
    if (L.submaps.size() > (size_t)max_submaps) return VGX_ERR_CAPACITY;
    for (size_t i = 0; i < L.submaps.size(); ++i) {
      const CollSubmapRef& s = L.submaps[i];
      out[i].id = s.id;
      out[i].num_blocks = s.n_blocks;
      out[i].voxel_size = (float)L.voxel_size;
      out[i].voxels_per_side = (int32_t)L.vps;
      for (int k = 0; k < 7; ++k) out[i].T_M_S[k] = s.T[k];
    }
    return VGX_OK;
  });
}

// Decodes a parsed stream into new submaps, one per entry of L.submaps under the entry's id, then runs the
// upload path (block hash, registration view, block-index rules, grid) on each.
// keep_colour: every submap gets a colour channel for the decode, and keeps it iff a colour word is non-zero
// (a colourless file loaded with the flag pays a transient 4 B per voxel and its clearing: whether a word is
// non-zero is only known once the varints are decoded, which is the decode pass itself).
static int decode_layout(vgx_ctx* c, const CollLayout& L, const uint8_t* bytes, uint64_t n, bool keep_colour) {
  const int vpb = (int)(L.vps * L.vps * L.vps);
  CollBlockRef* d_regions;
  int *d_err, *d_any;   // d_any: one flag per submap
  uint8_t* d_bytes;
  VGX_TRY(vgx_carve(c, c->d_scratch, vgx_part(d_regions, L.blocks.size()), vgx_part(d_err, 1),
                    vgx_part(d_any, keep_colour ? L.submaps.size() : 0), vgx_part(d_bytes, (size_t)n)));
  if (keep_colour && !L.submaps.empty())
    VGX_TRY(vgx_fill(c, d_any, L.submaps.size()));
  {
    VgxProfileScope copies(c, VGX_SLOT_COLL_COPY);
    if (!L.blocks.empty())
      VGX_TRY(vgx_upload(c, d_regions, L.blocks.data(), L.blocks.size()));
    VGX_TRY(vgx_fill(c, d_err, 1));
    VGX_TRY(copy_h2d_chunked(c, d_bytes, bytes, n));
  }
  for (size_t k = 0; k < L.submaps.size(); ++k) {
    const CollSubmapRef& s = L.submaps[k];
    VgxSubmap* sm = nullptr;
    VGX_TRY(vgx_submap_alloc(c, s.id, (float)L.voxel_size, (int)L.vps, (int)s.n_blocks, true, &sm));
    sm->n_blocks = (int)s.n_blocks;
    sm->finished = true;
    if (s.n_blocks == 0) continue;
    if (keep_colour) VGX_TRY(vgx_submap_ensure_colour(c, sm));
    {
      VgxProfileScope copies(c, VGX_SLOT_COLL_COPY);
      VGX_TRY(vgx_upload(c, sm->d_block_idx.get(), L.block_idx.data() + 3 * s.first_block, 3 * (size_t)s.n_blocks));
    }
    VgxProfileScope scope(c, VGX_SLOT_COLL_CODEC);
    VGX_TRY(vgx_launch(c, collection_decode_kernel, s.n_blocks, COLL_THREADS, 0, VgxLaunch::plain, d_bytes,
                       d_regions + s.first_block, vpb, reinterpret_cast<float*>(sm->d_dw.get()), sm->d_rgba.get(),
                       keep_colour ? d_any + k : nullptr, d_err));
  }
  int h_err = 0;
  std::vector<int> h_any(keep_colour ? L.submaps.size() : 0);
  VGX_TRY(vgx_download(c, &h_err, d_err, 1));
  if (!h_any.empty()) VGX_TRY(vgx_download(c, h_any.data(), d_any, h_any.size()));
  VGX_TRY(vgx_sync(c));
  if (h_err) {
    c->set_error(std::string("voxel_data: ") +
                 ((h_err & COLL_ERR_TAG) ? "unexpected tag; " : "") +
                 ((h_err & COLL_ERR_VARINT) ? "varint longer than 5 bytes, above 32 bits or truncated; " : "") +
                 ((h_err & COLL_ERR_COUNT) ? "not 3 vps^3 values; " : "") +
                 ((h_err & COLL_ERR_LENGTH) ? "packed length does not match the block; " : ""));
    return VGX_ERR_INVALID;
  }
  for (size_t k = 0; k < L.submaps.size(); ++k) {
    VgxSubmap* sm = c->find(L.submaps[k].id);
    if (keep_colour && !h_any[k]) sm->d_rgba.reset();   // all words zero: a colour-free submap (synchronised above)
    VgxProfileScope scope(c, VGX_SLOT_COLL_UPLOAD);
    VGX_TRY(vgx_submap_upload_finish(c, sm));
  }
  return VGX_OK;
}

// decode_layout for ids none of which exists yet: on failure no submap of L is left
static int load_layout(vgx_ctx* c, const CollLayout& L, const uint8_t* bytes, uint64_t n, bool keep_colour) {
  const int rc = decode_layout(c, L, bytes, n, keep_colour);
  if (rc != VGX_OK)
    for (const CollSubmapRef& s : L.submaps) vgx_submap_drop(c, s.id);
  return rc;
}

extern "C" int vgx_collection_load_ex(vgx_ctx* c, const uint8_t* bytes, uint64_t n, int flags, int* n_submaps) {
  return vgx_entry(c, __func__, [&] {
    if (n_submaps) *n_submaps = 0;
    if (flags & ~VGX_COLLECTION_KEEP_COLOUR) VGX_FAIL(c, VGX_ERR_INVALID, "unknown flag");
    CollLayout L;
    std::string err;
    if (!parse_stream(bytes, n, false, &L, &err)) VGX_FAIL(c, VGX_ERR_INVALID, err);
    for (const CollSubmapRef& s : L.submaps)
      if (c->submaps.count(s.id))
        VGX_FAIL(c, VGX_ERR_INVALID, "submap " + std::to_string(s.id) + " already exists");
    const int rc = load_layout(c, L, bytes, n, (flags & VGX_COLLECTION_KEEP_COLOUR) != 0);
    if (rc == VGX_OK && n_submaps) *n_submaps = (int)L.submaps.size();
    return rc;
  });
}

extern "C" int vgx_collection_load(vgx_ctx* c, const uint8_t* bytes, uint64_t n, int* n_submaps) {
  return vgx_entry(c, __func__, [&] { return vgx_collection_load_ex(c, bytes, n, 0, n_submaps); });
}

extern "C" int vgx_collection_save(vgx_ctx* c, int n, const uint32_t* ids, const float* T_M_S, uint8_t* out,
                                   uint64_t capacity, uint64_t* size) {
  return vgx_entry(c, __func__, [&] {
    if (n < 0 || !size || (n > 0 && (!ids || !T_M_S))) VGX_FAIL(c, VGX_ERR_INVALID, "invalid argument");
    *size = 0;
    std::vector<int> order((size_t)n);
    for (int i = 0; i < n; ++i) order[i] = i;
    std::sort(order.begin(), order.end(), [&](int a, int b) { return ids[a] < ids[b]; });   // cblox: std::map order
    std::vector<VgxSubmap*> subs;
    for (int k = 0; k < n; ++k) {
      const uint32_t id = ids[order[k]];
      if (k > 0 && ids[order[k - 1]] == id) VGX_FAIL(c, VGX_ERR_INVALID, "repeated submap id");
      VgxSubmap* s;
      VGX_TRY(vgx_submap_get(c, id, &s));
      if (!subs.empty() && (s->voxel_size != subs[0]->voxel_size || s->vps != subs[0]->vps))
        VGX_FAIL(c, VGX_ERR_INVALID, "a collection has one voxel size and voxels_per_side");
      subs.push_back(s);
    }
    VGX_TRY(vgx_sync(c));   // n_blocks of an active submap is final after its integration
    const double voxel_size = subs.empty() ? 0.0 : (double)subs[0]->voxel_size;
    const int vps = subs.empty() ? 16 : subs[0]->vps;
    const uint32_t hdr = block_header_bytes(vps);
    size_t total_blocks = 0;
    for (VgxSubmap* s : subs) total_blocks += (size_t)s->n_blocks;
    // scratch: [payload sizes | block offsets | block messages]
    uint32_t* d_sizes;
    uint64_t* d_offs;
    uint8_t* d_msgs;
    VGX_TRY(vgx_carve(c, c->d_scratch, vgx_part(d_sizes, total_blocks), vgx_part(d_offs, total_blocks)));
    CollEncodeArgs a{};
    a.vps = vps;
    a.header_bytes = hdr;
    size_t first = 0;
    for (VgxSubmap* s : subs) {
      if (s->n_blocks > 0) {
        a.dw = s->d_dw.get();
        a.rgba = s->d_rgba.get();
        a.block_idx = s->d_block_idx.get();
        a.vox_per_block = s->vox_per_block;
        a.out_sizes = d_sizes + first;
        VgxProfileScope scope(c, VGX_SLOT_COLL_CODEC);
        VGX_TRY(vgx_launch(c, collection_encode_kernel<false>, s->n_blocks, COLL_THREADS, 0, VgxLaunch::plain, a));
      }
      first += (size_t)s->n_blocks;
    }
    std::vector<uint32_t> sizes(total_blocks);
    if (total_blocks) VGX_TRY(vgx_download(c, sizes.data(), d_sizes, total_blocks));
    VGX_TRY(vgx_sync(c));
    // layout: header, then per submap its SubmapProto and its blocks; block messages are contiguous per
    // submap in the device buffer
    std::vector<std::vector<uint8_t>> framing((size_t)n + 1);
    put_delimited(framing[0], collection_header(voxel_size, (uint32_t)vps, (uint32_t)n));
    std::vector<uint64_t> offsets(total_blocks), span((size_t)n);
    uint64_t total = framing[0].size(), dev_bytes = 0;
    first = 0;
    for (int k = 0; k < n; ++k) {
      VgxSubmap* s = subs[k];
      put_delimited(framing[k + 1], submap_message(s->id, (uint32_t)s->n_blocks, T_M_S + 7 * (size_t)order[k]));
      const uint64_t start = dev_bytes;
      for (int b = 0; b < s->n_blocks; ++b) {
        const uint64_t msg = (uint64_t)hdr + sizes[first + b];
        offsets[first + b] = dev_bytes;
        dev_bytes += varint_len(msg) + msg;
      }
      span[k] = dev_bytes - start;
      total += framing[k + 1].size() + span[k];
      first += (size_t)s->n_blocks;
    }
    *size = total;
    if (!out) return VGX_OK;
    if (capacity < total) VGX_FAIL(c, VGX_ERR_CAPACITY, "capacity too small");
    // the second carve of d_scratch may move it: the sizes are re-sent
    VGX_TRY(vgx_carve(c, c->d_scratch, vgx_part(d_sizes, total_blocks), vgx_part(d_offs, total_blocks),
                      vgx_part(d_msgs, (size_t)dev_bytes)));
    if (total_blocks) {
      VgxProfileScope copies(c, VGX_SLOT_COLL_COPY);
      VGX_TRY(vgx_upload(c, d_sizes, sizes.data(), total_blocks));
      VGX_TRY(vgx_upload(c, d_offs, offsets.data(), total_blocks));
    }
    a.dst = d_msgs;
    first = 0;
    for (VgxSubmap* s : subs) {
      if (s->n_blocks > 0) {
        a.dw = s->d_dw.get();
        a.rgba = s->d_rgba.get();
        a.block_idx = s->d_block_idx.get();
        a.vox_per_block = s->vox_per_block;
        a.voxel_size = s->voxel_size;
        a.block_size = s->block_size;
        a.sizes = d_sizes + first;
        a.offsets = d_offs + first;
        VgxProfileScope scope(c, VGX_SLOT_COLL_CODEC);
        VGX_TRY(vgx_launch(c, collection_encode_kernel<true>, s->n_blocks, COLL_THREADS, 0, VgxLaunch::plain, a));
      }
      first += (size_t)s->n_blocks;
    }
    VgxProfileScope copies(c, VGX_SLOT_COLL_COPY);
    uint8_t* o = out;
    uint64_t dev_off = 0;
    memcpy(o, framing[0].data(), framing[0].size());
    o += framing[0].size();
    for (int k = 0; k < n; ++k) {
      memcpy(o, framing[k + 1].data(), framing[k + 1].size());
      o += framing[k + 1].size();
      VGX_TRY(copy_d2h_chunked(c, o, d_msgs + dev_off, span[k]));
      o += span[k];
      dev_off += span[k];
    }
    return vgx_sync(c);
  });
}

extern "C" int vgx_layer_load(vgx_ctx* c, uint32_t id, const uint8_t* bytes, uint64_t n, int* n_blocks) {
  return vgx_entry(c, __func__, [&] {
    if (n_blocks) *n_blocks = 0;
    CollLayout L;
    std::string err;
    if (!parse_stream(bytes, n, true, &L, &err)) VGX_FAIL(c, VGX_ERR_INVALID, err);
    if (c->submaps.count(id)) VGX_FAIL(c, VGX_ERR_INVALID, "submap " + std::to_string(id) + " already exists");
    // the layer is the single submap entry; a repeated block index is refused by the upload path
    // (voxblox BlockMergingStrategy::kProhibit)
    L.submaps[0].id = id;
    const int rc = load_layout(c, L, bytes, n, false);
    if (rc == VGX_OK && n_blocks) *n_blocks = (int)L.submaps[0].n_blocks;
    return rc;
  });
}
