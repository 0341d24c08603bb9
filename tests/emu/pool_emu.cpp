// tests/emu/pool_emu.cpp — HOST EMULATION of b200tsdf_resize_pool (k_pool_rehash in engine.cu).  TEST HARNESS ONLY.
//
// Compiles the emulation of emu.cpp and adds emu_resize_pool, which moves every claimed brick into a fresh pool of another
// size through the same __host__ __device__ routines the kernel runs (rehash_claim, rehash_brick in pool_rehash.cuh), with
// the 32 lanes of the kernel's warp run one after another; and the raw storage accessors the tests compare.
#include "emu.cpp"
#include "../../cpu_tsdf_b200/csrc/pool_rehash.cuh"

#include <cmath>

extern "C" {

// The volume into a pool of pool_log2 (0: the default size): 0 installed; 1 the claimed bricks exceed the load limit
// (rehash_fits; only checked when check_fit); 2 a brick found no slot within MAX_PROBE; 3 pool_log2 out of range.  On any
// refusal the volume is unchanged and so is its error word (the rehash raises on a flag of its own).
int emu_resize_pool (Emu* e, int pool_log2, int check_fit)
{
  const size_t pool = pool_capacity_of (pool_log2);
  if (!pool) return 3;
  Params& p = e->p;
  long long nb = 0;
  for (size_t s = 0; s <= p.pool_mask; ++s) nb += p.keys[s] != KEY_EMPTY;
  if (check_fit && !rehash_fits (nb, (long long) pool)) return 1;
  const size_t nn = pool * BRICK_NODES;
  std::vector<uint64_t> keys (pool, KEY_EMPTY);
  std::vector<float2> nodes (nn, make_float2 (-1.f, 0.f));
  std::vector<uint32_t> split (pool * BRICK_SPLIT_WORDS, 0u);
  std::vector<uchar4> rgb; std::vector<float> M; std::vector<int> ns;
  Params to = p;
  to.keys = keys.data (); to.nodes = nodes.data (); to.split = split.data (); to.pool_mask = (uint32_t) (pool - 1);
  if (p.rgb) { rgb.assign (nn, make_uchar4 (0, 0, 0, 0)); to.rgb = rgb.data (); }
  if (p.M) { M.assign (nn, 0.f); ns.assign (nn, 0); to.M = M.data (); to.ns = ns.data (); }
  int rerr = 0;
  to.err = &rerr;
  for (uint32_t s = 0; s <= p.pool_mask; ++s)
  {
    if (p.keys[s] == KEY_EMPTY) continue;
    const int d = rehash_claim (p, to, s);
    if (d < 0) continue;
    for (int lane = 0; lane < 32; ++lane) rehash_brick (p, to, s, (uint32_t) d, lane, 32);
  }
  if (rerr & ERR_POOL_FULL) return 2;
  e->keys.swap (keys); e->nodes.swap (nodes); e->split.swap (split); e->rgb.swap (rgb); e->M.swap (M); e->ns.swap (ns);
  to.err = &e->err;
  p = to;
  return 0;
}

long long emu_pool_capacity (const Emu* e) { return (long long) e->p.pool_mask + 1; }

// the claimed slots in slot order: their numbers, keys and payload arrays (a null pointer skips that array; rgb / M / ns only
// when the volume carries them).  Returns their count.
long long emu_pool_claimed (const Emu* e, int* slots, uint64_t* keys, float2* nodes, uint32_t* split, uchar4* rgb, float* M, int* ns)
{
  const Params& p = e->p;
  long long n = 0;
  for (size_t s = 0; s <= p.pool_mask; ++s)
  {
    if (p.keys[s] == KEY_EMPTY) continue;
    const size_t a = s * BRICK_NODES, b = (size_t) n * BRICK_NODES;
    if (slots) slots[n] = (int) s;
    if (keys) keys[n] = p.keys[s];
    if (nodes) std::copy (p.nodes + a, p.nodes + a + BRICK_NODES, nodes + b);
    if (split) std::copy (p.split + s * BRICK_SPLIT_WORDS, p.split + (s + 1) * BRICK_SPLIT_WORDS, split + (size_t) n * BRICK_SPLIT_WORDS);
    if (rgb && p.rgb) std::copy (p.rgb + a, p.rgb + a + BRICK_NODES, rgb + b);
    if (M && p.M) { std::copy (p.M + a, p.M + a + BRICK_NODES, M + b); std::copy (p.ns + a, p.ns + a + BRICK_NODES, ns + b); }
    ++n;
  }
  return n;
}

// the unclaimed slots whose storage is not fresh ({-1, 0} nodes, no split bit, zero rgb / M / ns)
long long emu_unclaimed_not_fresh (const Emu* e)
{
  const Params& p = e->p;
  long long bad = 0;
  for (size_t s = 0; s <= p.pool_mask; ++s)
  {
    if (p.keys[s] != KEY_EMPTY) continue;
    bool fresh = true;
    for (int w = 0; w < BRICK_SPLIT_WORDS; ++w) fresh = fresh && p.split[s * BRICK_SPLIT_WORDS + w] == 0;
    for (size_t i = s * BRICK_NODES; i < (s + 1) * BRICK_NODES; ++i)
    {
      const float2 dw = p.nodes[i];
      fresh = fresh && dw.x == -1.f && !std::signbit (dw.y) && dw.y == 0.f;
      if (p.rgb) fresh = fresh && !p.rgb[i].x && !p.rgb[i].y && !p.rgb[i].z && !p.rgb[i].w;
      if (p.M) fresh = fresh && p.M[i] == 0.f && !std::signbit (p.M[i]) && p.ns[i] == 0;
    }
    bad += !fresh;
  }
  return bad;
}

// the slot of each key through find_brick (-1: not found within MAX_PROBE)
void emu_find_keys (const Emu* e, const uint64_t* keys, long long n, int* slots)
{
  for (long long i = 0; i < n; ++i)
  {
    int t, bx, by, bz;
    brick_key_decode (keys[i], t, bx, by, bz);
    slots[i] = find_brick (e->p, t, bx, by, bz);
  }
}

int emu_err (const Emu* e) { return e->err; }

} // extern "C"
