// rbk_group_plan.h — the copy plan of rbk_group_compact (rbk_group.cu): which staged rows go where, chunk by chunk.
// Pure host code with no CUDA include, so that tests/test_group_compact_host.py compiles it with g++ and replays the
// plan against a model of the block-cyclic layout.
//
// Layout: global slot s lives on device (s / block) % G at local row (s / block / G) * block + s % block, before and
// after compaction alike.  Compaction sends every survivor to its stable rank among the survivors, so a row only moves
// to a lower global slot.  Chunks of whole global blocks are planned in ascending order; chunk [s0, s1) sends its
// survivors to new slots [d0, d1) with d1 <= s1, so its writes land in the storage of old slots below s1 - all of them
// staged by this chunk or an earlier one - and never in a source of a later chunk.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <vector>

namespace rbk {
namespace group_plan {

// local row of global slot s on its device
inline int64_t local_row(int G, int64_t block, int64_t s) { return (s / block / G) * block + s % block; }

// rows that device d holds of global slots [0, n): monotone in n, so a compacted member never grows
inline int64_t member_rows(int G, int64_t block, int64_t n, int d) {
  const int64_t full = n / block, rem = n % block;
  return (full / G) * block + (d < full % G ? block : 0) + (d == full % G ? rem : 0);
}

// len rows from staging rows [src_off, src_off + len) of member src to local rows [dst_row, dst_row + len) of member dst
struct Segment {
  int src;
  int64_t src_off;
  int dst;
  int64_t dst_row;
  int64_t len;
};

struct Chunk {
  int64_t s0, s1;               // old global slots
  int64_t d0, d1;               // new global slots of their survivors
  // per member: gather of local rows [g0, g0 + gn) (gn == 0: the member has no rows in the chunk), whose survivors
  // are staged in local order from staging row 0; rank0 = the member's survivors before local row g0
  std::vector<int64_t> g0, gn, rank0, staged;
  std::vector<Segment> segs;
};

struct Plan {
  std::vector<int64_t> base;    // per global block: the new global slot of its first survivor
  int64_t n_live = 0;
  std::vector<Chunk> chunks;    // the chunks that move rows, in ascending order
};

// block_live[b]: survivors of global block b, for every block of global slots [0, n_slots).  chunk_blocks: global
// blocks per chunk; a member stages at most ceil(chunk_blocks / G) blocks of rows per chunk.
inline Plan make_plan(int G, int64_t block, int64_t n_slots, const std::vector<int64_t>& block_live,
                      int64_t chunk_blocks) {
  Plan p;
  const int64_t nb = (n_slots + block - 1) / block;
  p.base.resize(static_cast<size_t>(nb));
  for (int64_t b = 0; b < nb; ++b) {
    p.base[b] = p.n_live;
    p.n_live += block_live[b];
  }
  std::vector<int64_t> rank(G, 0);   // survivors of each member before the current chunk
  for (int64_t b0 = 0; b0 < nb; b0 += chunk_blocks) {
    const int64_t b1 = std::min(nb, b0 + chunk_blocks);
    Chunk c;
    c.s0 = b0 * block;
    c.s1 = std::min(n_slots, b1 * block);
    c.d0 = p.base[b0];
    c.d1 = b1 < nb ? p.base[b1] : p.n_live;
    c.g0.assign(G, 0);
    c.gn.assign(G, 0);
    c.rank0 = rank;
    c.staged.assign(G, 0);
    for (int64_t b = b0; b < b1; ++b) {   // a member's blocks in the chunk are consecutive local blocks
      const int e = static_cast<int>(b % G);
      const int64_t first = (b / G) * block, rows = std::min(block, n_slots - b * block);
      if (c.gn[e] == 0) c.g0[e] = first;
      c.gn[e] = first + rows - c.g0[e];
    }
    for (int64_t b = b0; b < b1; ++b) {
      const int e = static_cast<int>(b % G);
      int64_t t = p.base[b], off = c.staged[e], left = block_live[b];
      c.staged[e] += left;
      while (left > 0) {   // a block's survivors cross at most one destination block boundary
        const int64_t len = std::min(left, block - t % block);
        const Segment s{e, off, static_cast<int>((t / block) % G), local_row(G, block, t), len};
        Segment* prev = c.segs.empty() ? nullptr : &c.segs.back();
        if (prev && prev->src == s.src && prev->dst == s.dst && prev->src_off + prev->len == s.src_off &&
            prev->dst_row + prev->len == s.dst_row)
          prev->len += len;
        else
          c.segs.push_back(s);
        t += len;
        off += len;
        left -= len;
      }
    }
    for (int e = 0; e < G; ++e) rank[e] += c.staged[e];
    const bool in_place = c.d0 == c.s0 && c.d1 == c.s1;   // before the first tombstone: nothing moves
    if (!in_place && c.d1 > c.d0) p.chunks.push_back(std::move(c));
  }
  return p;
}

// old_to_new of every global slot below n_slots: its block's base plus its rank within the block, or -1.  rank[e]:
// member e's live rank of each local row (-1: tombstoned); block_pref[e]: its live rows before each local block.
inline void fill_old_to_new(int G, int64_t block, int64_t n_slots, const Plan& p,
                            const std::vector<const int64_t*>& rank, const std::vector<const int*>& block_pref,
                            int64_t* old_to_new) {
  const int64_t nb = (n_slots + block - 1) / block;
  for (int64_t b = 0; b < nb; ++b) {
    const int e = static_cast<int>(b % G);
    const int64_t rows = std::min(block, n_slots - b * block), r0 = block_pref[e][b / G];
    const int64_t* m = rank[e] + (b / G) * block;
    for (int64_t i = 0; i < rows; ++i) old_to_new[b * block + i] = m[i] < 0 ? -1 : p.base[b] + m[i] - r0;
  }
}

}  // namespace group_plan
}  // namespace rbk
