// pool_rehash.cuh — moving every claimed brick of a live volume into a brick pool of another size (b200tsdf_resize_pool).
//
// The payload slot is the hash slot (tsdf_core.cuh), so a pool of another size means a new directory: each claimed brick
// claims its slot in the new one with find_or_insert_brick and then carries its whole payload there.  The new pool starts
// fresh, so every slot nobody claims stays fresh and the invariant of tsdf_core.cuh holds in it.  k_pool_rehash (engine.cu)
// runs these routines one warp per brick; tests/emu runs the same code on the host, one brick at a time.
#pragma once
#include "tsdf_core.cuh"

namespace b2 {

// Every per-brick payload array is a whole number of 16-byte words per brick (nodes 292, split 5, rgb / M / ns 146, rgbn
// 584), and brick b of each starts at a multiple of 16 bytes, so a brick moves as 16-byte vector loads and stores.
struct alignas (16) Word16 { uint32_t v[4]; };

// The load limit of a resize: n claimed bricks fit a pool of cap slots when n <= 7/8 cap.  Linear probing at that load still
// finds every key far inside MAX_PROBE, and the volume keeps a little room to grow before the caller resizes again.
B2_HD bool rehash_fits (long long n, long long cap) { return n * 8 <= cap * 7; }

template <typename T, int N>
B2_HD void rehash_words (const T* src, T* dst, uint32_t s, uint32_t d, int lane, int lanes)
{
  static_assert ((N * sizeof (T)) % sizeof (Word16) == 0, "brick payload is not a whole number of 16-byte words");
  constexpr int W = (int) (N * sizeof (T) / sizeof (Word16));
  const Word16* a = reinterpret_cast<const Word16*> (src + (size_t) s * N);
  Word16* b = reinterpret_cast<Word16*> (dst + (size_t) d * N);
  for (int i = lane; i < W; i += lanes) b[i] = a[i];
}

// the slot of old slot s's brick in the pool of `to`: its key, claimed with find_or_insert_brick.  -1 when the probe reaches
// MAX_PROBE (ERR_POOL_FULL is then raised on to.err)
B2_HD int rehash_claim (const Params& from, const Params& to, uint32_t s)
{
  int t, bx, by, bz;
  brick_key_decode (from.keys[s], t, bx, by, bz);
  return find_or_insert_brick (to, t, bx, by, bz);
}

// the payload of old slot s into slot d of `to`: {d, w} nodes, split words, and the rgb, rgbn, M / ns and work arrays the
// volume carries.  The lanes lane, lane + lanes, ... of one brick share the words among them.
B2_HD void rehash_brick (const Params& from, const Params& to, uint32_t s, uint32_t d, int lane, int lanes)
{
  rehash_words<float2, BRICK_NODES> (from.nodes, to.nodes, s, d, lane, lanes);
  rehash_words<uint32_t, BRICK_SPLIT_WORDS> (from.split, to.split, s, d, lane, lanes);
  if (from.rgb) rehash_words<uchar4, BRICK_NODES> (from.rgb, to.rgb, s, d, lane, lanes);
  if (from.rgbn) rehash_words<float4, BRICK_NODES> (from.rgbn, to.rgbn, s, d, lane, lanes);
  if (from.M)
  {
    rehash_words<float, BRICK_NODES> (from.M, to.M, s, d, lane, lanes);
    rehash_words<int, BRICK_NODES> (from.ns, to.ns, s, d, lane, lanes);
  }
  if (from.work && lane == 0) to.work[d] = from.work[s];
}

} // namespace b2
