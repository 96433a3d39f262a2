// arena_packer.hpp -- liveness-packed layout of a plan's arena.  Pure host code: no device calls, so that it can be
// tested on its own (tests/test_arena_packing.py).
//
// Input: the plan's steps in issue order (stream, and the earlier steps each one waits on) and its buffers (size, the
// step that first touches it, the steps that read it, pinned = lives for the whole plan).  Output: a word offset per
// buffer, the extra waits that make storage reuse safe, and the peak.
//
// Invariant: two buffers share words only if every access of the earlier one (its writer and its readers)
// happens-before the writer of the later one, where happens-before is stream order plus waits (including the waits
// added here).  Pinned buffers sit below every other buffer and are never reused.
//
// Policy: steps are walked in issue order with a vector clock per step (the last step of every stream known to be
// complete when it starts).  A buffer is freed after its last access; a free block remembers, per stream, the last
// step that accessed it.  A buffer is placed in the run of adjacent free blocks that (1) does not raise the peak,
// (2) needs the fewest new waits (a block last used on the writer's own stream, or one already ordered by the plan's
// events, needs none) and (3) wastes the fewest words; if every run raises the peak, the top of the arena is used.
#pragma once
#include <algorithm>
#include <cstddef>
#include <stdexcept>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

namespace evab {

struct PackStep {
  int stream = 0;
  std::vector<int> waits;   // earlier steps (issue order) this step waits on
};
struct PackBuffer {
  std::size_t words = 0;
  int writer = 0;            // the step that first writes it
  std::vector<int> readers;  // the steps that read it
  bool pinned = false;       // program inputs, outputs, plan-time constants, workspaces: never reused
};
struct PackResult {
  std::vector<std::size_t> offsets;            // per buffer
  std::vector<std::pair<int, int>> waits;      // (step, earlier step it must wait on), in addition to PackStep::waits
  std::size_t peak = 0;                        // words
};

inline PackResult packArena(const std::vector<PackStep> &steps, const std::vector<PackBuffer> &bufs) {
  const int n = (int)steps.size();
  int S = 1;
  for (int i = 0; i < n; i++) {
    if (steps[i].stream < 0) throw std::invalid_argument("packArena: negative stream id");
    S = std::max(S, steps[i].stream + 1);
    for (int w : steps[i].waits)
      if (w < 0 || w >= i) throw std::invalid_argument("packArena: step " + std::to_string(i) + " waits on a step that is not earlier");
  }
  PackResult res;
  res.offsets.assign(bufs.size(), 0);
  std::size_t top = 0;
  for (std::size_t b = 0; b < bufs.size(); b++)   // pinned buffers: the bottom of the arena, in order
    if (bufs[b].pinned) { res.offsets[b] = top; top += bufs[b].words; }

  // lifetime of every other buffer: [first access, last access]; guard = last accessing step per stream
  std::vector<std::vector<int>> startAt(n), endAt(n);
  std::vector<std::vector<int>> guardOf(bufs.size());
  for (std::size_t b = 0; b < bufs.size(); b++) {
    const PackBuffer &B = bufs[b];
    if (B.pinned || B.words == 0) continue;
    if (B.writer < 0 || B.writer >= n) throw std::invalid_argument("packArena: buffer " + std::to_string(b) + " has no valid writer step");
    int first = B.writer, last = B.writer;
    std::vector<int> g(S, -1);
    g[steps[B.writer].stream] = B.writer;
    for (int r : B.readers) {
      if (r < 0 || r >= n) throw std::invalid_argument("packArena: buffer " + std::to_string(b) + " has a reader out of range");
      first = std::min(first, r); last = std::max(last, r);
      g[steps[r].stream] = std::max(g[steps[r].stream], r);
    }
    startAt[first].push_back((int)b);
    endAt[last].push_back((int)b);
    guardOf[b] = std::move(g);
  }

  struct Block { std::size_t off, words; std::vector<int> guard; };
  std::vector<Block> freeList;                       // sorted by offset; adjacent blocks are kept apart unless their guards agree
  std::vector<std::vector<int>> vc(n, std::vector<int>(S, -1));   // vc[i][s]: last step of stream s that happens-before-or-is step i
  std::vector<int> prevOnStream(S, -1);
  auto merge = [&](std::vector<int> &into, const std::vector<int> &from) { for (int s = 0; s < S; s++) into[s] = std::max(into[s], from[s]); };
  auto missing = [&](const std::vector<int> &clock, const std::vector<int> &guard) {
    int m = 0;
    for (int s = 0; s < S; s++) if (guard[s] > clock[s]) m++;
    return m;
  };

  for (int i = 0; i < n; i++) {
    std::vector<int> &clock = vc[i];
    const int si = steps[i].stream;
    if (prevOnStream[si] >= 0) clock = vc[prevOnStream[si]];
    for (int w : steps[i].waits) merge(clock, vc[w]);
    clock[si] = i;
    prevOnStream[si] = i;

    std::vector<int> &mine = startAt[i];
    std::stable_sort(mine.begin(), mine.end(), [&](int a, int b) { return bufs[a].words > bufs[b].words; });
    for (int b : mine) {
      const std::size_t need = bufs[b].words;
      // best run of adjacent free blocks; the baseline is fresh words at the top (no wait, grows by `need`)
      auto key = [](std::size_t grow, int waits, std::size_t waste) { return std::make_tuple(grow > 0, waits, grow, waste); };
      int bestA = -1, bestB = -1;
      std::size_t bestGrow = need, bestWaste = 0;
      auto bestKey = key(need, 0, 0);
      for (int a = 0; a < (int)freeList.size(); a++) {
        std::vector<int> g(S, -1);
        std::size_t total = 0;
        for (int e = a; e < (int)freeList.size(); e++) {
          if (e > a && freeList[e].off != freeList[e - 1].off + freeList[e - 1].words) break;
          merge(g, freeList[e].guard);
          total += freeList[e].words;
          const bool atTop = freeList[e].off + freeList[e].words == top;
          if (total < need && !atTop) continue;
          const std::size_t grow = total < need ? need - total : 0;
          const std::size_t waste = total > need ? total - need : 0;
          const auto k = key(grow, missing(clock, g), waste);
          if (k < bestKey) { bestKey = k; bestA = a; bestB = e; bestGrow = grow; bestWaste = waste; }
          break;
        }
      }
      if (bestA < 0) {   // fresh words at the top
        res.offsets[b] = top;
        top += need;
        continue;
      }
      std::vector<int> g(S, -1);
      for (int e = bestA; e <= bestB; e++) merge(g, freeList[e].guard);
      res.offsets[b] = freeList[bestA].off;
      Block rest{0, 0, {}};
      if (bestWaste) { const Block &last = freeList[bestB]; rest = Block{res.offsets[b] + need, bestWaste, last.guard}; }
      freeList.erase(freeList.begin() + bestA, freeList.begin() + bestB + 1);
      if (bestWaste) freeList.insert(freeList.begin() + bestA, std::move(rest));
      top += bestGrow;
      for (int s = 0; s < S; s++)   // write-after-read across streams: wait for the last access of every stream not yet ordered
        if (g[s] > clock[s]) {
          res.waits.emplace_back(i, g[s]);
          merge(clock, vc[g[s]]);
        }
    }
    for (int b : endAt[i]) {   // free after the last access
      Block blk{res.offsets[b], bufs[b].words, guardOf[b]};
      auto it = std::lower_bound(freeList.begin(), freeList.end(), blk.off, [](const Block &x, std::size_t off) { return x.off < off; });
      it = freeList.insert(it, std::move(blk));
      if (it + 1 != freeList.end() && it->off + it->words == (it + 1)->off && it->guard == (it + 1)->guard) {
        it->words += (it + 1)->words;
        freeList.erase(it + 1);
      }
      if (it != freeList.begin() && (it - 1)->off + (it - 1)->words == it->off && (it - 1)->guard == it->guard) {
        (it - 1)->words += it->words;
        freeList.erase(it);
      }
    }
  }
  res.peak = top;
  return res;
}

}  // namespace evab
