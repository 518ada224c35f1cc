// rcvd_plan.h -- the block-Cholesky plan of one problem: elimination order, level schedule, multi-GPU distribution, block numbering
// and the task lists of every factorisation and substitution kernel.  Pure host code (no CUDA runtime call), computed once per
// problem structure by build_structure (rcvd_api.cu), which uploads it; rcvd_debug_factor_plan exposes it to the CPU tests.
#pragma once
#include <algorithm>
#include <map>
#include <set>
#include <tuple>
#include <vector>

#include "rcvd_linalg.cuh"
#include "rcvd_update.cuh"

namespace rcvd {

// frame_off: every frame of the level (substitution); own_off: the frames this rank factors; upd: the late update passes (main stream);
// upd2[0], upd2[1]: the deferred passes applied at this level (side stream), two launches in this order: [0] the passes into the
// columns of level + 2, which the next level's late passes need, [1] the rest; it / it2: the k_update_tma items of upd / upd2;
// join[s]: the first level whose late passes (U1) must wait for launch s -- one of its targets is in a column of level join[s] + 1
struct UpdPass { int dst; int first; int count; int flags; };   // products upd_pairs[first, first + count) into L block dst; flags bit0: symmetric target (tiles above the diagonal are never read), bit1: first pass into a fill block (the target is written, not read)

struct Level { int frame_off, nframes; int trsm_off, ntrsm; int upd_off, nupd; int upd2_off[2], nupd2[2]; int fwd_off, nfwd; int it_off, nit, it2_off[2], nit2[2]; int own_off, nown; int join[2]; };

// Deferred update passes group the wide levels (below the narrow tail) in aligned windows of kUpdWindow source levels when a frame block
// has at most kUpdWindowMaxNf unknowns; otherwise, and in the tail, one pass per source level.  A pass's read-modify-write of its target
// is amortised over its products; at nf = 775 the products are long enough that batching them saves nothing, and piling them onto fewer
// levels delays the main stream, as it would in the tail, whose side work must finish within the next level's potrf (DESIGN.md section 4).
constexpr int kUpdWindow = 2, kUpdWindowMaxNf = 256;

// DMMA work of an update item (m8n8 units x 4 k4 steps per source pair; a symmetric diagonal tile skips its upper warp tile)
inline long upd_item_cost(const UpdItem& a) { return (long)a.count * (a.mrows / 8) * (a.ncols / 8) * ((a.flags & kUpdSymDiag) ? 3 : 4); }

// Locality order of one update launch of `ctas` resident CTAs.  `in`: the launch's items, pass after pass, each pass's tiles adjacent.
// Every item streams an 80-row strip of X_rk and one of X_ck for each of its source pairs: ~10 flop per operand byte at K = 200, so the
// strips have to come from L2, and the factor (hundreds of MB) is far larger than L2.  A strip is reused only by the items that run at
// about the same time, i.e. in the same wave of `ctas` consecutive items.  So: the source frames k, heaviest first, each followed by the
// not yet emitted passes that read X_.k (all the tiles of a target stay adjacent; the d (d + 1) / 2 targets of a column k of d blocks
// share its d blocks).  Then, within each wave, the items go to the CTA slots so that the CTAs' summed work stays balanced (heaviest
// item to the least loaded CTA, from the last, partial wave backwards): the persistent CTAs take their items statically, so a
// cost-sorted list was what kept them even.  Returns false if two items of the launch write the same target tile (they run concurrently).
inline bool order_update_items(const std::vector<UpdItem>& in, const std::vector<int2>& pairs, const std::vector<int>& lcol, int ctas,
                               UpdItem* out) {
  struct Pass { size_t b, e; long cost; };
  std::vector<Pass> passes; std::set<std::tuple<int, int, int>> tiles;
  for (size_t i = 0; i < in.size(); ++i) {
    if (!tiles.insert(std::make_tuple(in[i].dst, (int)in[i].m0, (int)in[i].n0)).second) return false;
    if (i == 0 || in[i].dst != in[i - 1].dst || in[i].first != in[i - 1].first) passes.push_back({i, i, 0});
    passes.back().e = i + 1; passes.back().cost += upd_item_cost(in[i]);
  }
  std::map<int, std::vector<int>> readers; std::map<int, long> weight;   // source frame -> passes reading it (pass order), their work
  for (size_t q = 0; q < passes.size(); ++q) {
    const UpdItem& it = in[passes[q].b];
    std::set<int> ks; for (int p = it.first; p < it.first + it.count; ++p) ks.insert(lcol[pairs[p].x]);
    for (int k : ks) { readers[k].push_back((int)q); weight[k] += passes[q].cost; }
  }
  std::vector<int> ks; for (auto& kv : weight) ks.push_back(kv.first);
  std::stable_sort(ks.begin(), ks.end(), [&](int a, int b) { return weight[a] > weight[b]; });
  std::vector<UpdItem> seq; seq.reserve(in.size()); std::vector<uint8_t> done(passes.size(), 0);
  for (int k : ks) for (int q : readers[k]) if (!done[q]) { done[q] = 1; seq.insert(seq.end(), in.begin() + passes[q].b, in.begin() + passes[q].e); }
  const size_t n = seq.size(), G = (size_t)std::max(ctas, 1);
  std::vector<long> load(G, 0); std::vector<int> slot(G), idx;
  for (size_t w = (n + G - 1) / G; w-- > 0;) {
    const size_t b = w * G, m = std::min(G, n - b);
    idx.resize(m); for (size_t i = 0; i < m; ++i) idx[i] = (int)i;
    std::stable_sort(idx.begin(), idx.end(), [&](int x, int y) { return upd_item_cost(seq[b + x]) > upd_item_cost(seq[b + y]); });
    slot.resize(m); for (size_t s = 0; s < m; ++s) slot[s] = (int)s;
    std::stable_sort(slot.begin(), slot.end(), [&](int x, int y) { return load[x] < load[y]; });
    for (size_t i = 0; i < m; ++i) { out[b + slot[i]] = seq[b + idx[i]]; load[slot[i]] += upd_item_cost(seq[b + idx[i]]); }
  }
  return true;
}

// Every frame id below is internal: frames are numbered owner-major (uperm / iperm map to and from the caller's ids).
struct FactorPlan {
  std::vector<int> elim_order;                 // frames in elimination order
  std::vector<int> level, owner;               // per frame: elimination level, owning rank (0 without distribution)
  std::vector<Level> levels;
  // multi-GPU distribution (DESIGN.md section 5): levels < LB are phase A (owner computes), levels >= LB phase B (replicated)
  bool dist = false; int LB = 0;
  std::vector<int> uperm, iperm;               // internal frame -> caller's frame, and back
  std::vector<int> fa_off, fa_cnt, fb_off, fb_cnt, tseg, bseg, hseg;   // *_off/_cnt: per-owner frame ranges (phase A / B); segs: (first, count) pairs
  // blocks: L = N diagonal blocks, then nLoff off-diagonal factor blocks (T); H = N diagonal blocks, then one per coupled frame pair
  int nLoff = 0;
  std::vector<HBlock> hblocks, lblocks;        // lblocks: every L block with its H source (or -1: fill)
  std::vector<int32_t> blk_of;                 // N x N frame pair -> 2 * H block + (pair's first frame is the row side), or -1
  std::vector<int> own_lblocks, own_hblocks;   // blocks this rank loads into the factor / multiplies in the model term (all without distribution)
  std::vector<int> load_lblocks; int nload = 0;  // k_load_factor's list: own_lblocks with an H source or diagonal (nload), then the fill blocks
  // task lists of the level schedule
  std::vector<int> lvl_frames, lvl_own;
  std::vector<TrsmTask> trsm_tasks; std::vector<UpdPass> upd_tasks; std::vector<int2> upd_pairs; std::vector<SolveTask> fwd_tasks;
  // upd_items: k_update_tma's work items in locality order (order_update_items); upd_items_cost: the same items of every launch sorted
  // by cost, heaviest first (the A/B reference, rcvd_debug_set_update_order).  Both have the launches at the same offsets.
  std::vector<UpdItem> upd_items, upd_items_cost; int upd_rb = 0, upd_neff = 0;
  int upd_targets = 0;      // (source level, target block) pairs of the elimination structure this rank updates
  int upd_window = 1;       // source levels per window of the deferred update passes
  int TB = 0;               // tail boundary: levels >= TB are the trailing run of levels with fewer than 3 frames (= LB when distributed)
  double upd_flops = 0.0;   // algorithmic flops of the update GEMMs of one factorisation (2 nf^3 per product, nf^2 (nf+1) on symmetric targets)
  std::vector<SubTask> sub_tasks; std::vector<int> sub_need; int sub_first_level = 0;   // k_substitution: levels >= sub_first_level
};

// Fills P for the frame graph of `pairs` (frame pairs, flattened) and `trip_centers` under cfg.  Returns nullptr, or the message of the
// input error that makes the plan impossible.
inline const char* make_factor_plan(FactorPlan& P, const rcvd_config& cfg, const std::vector<int32_t>& pairs, const std::vector<int32_t>& trip_centers,
                                    int order_slack, int nranks, int rank, bool dist_enabled, int num_sms) {
  P = FactorPlan();
  Layout L;
  if (!make_layout(cfg, L) || cfg.num_frames <= 0) return "unsupported transform configuration";
  const int N = cfg.num_frames, npad = L.npad;
  // frame graph
  std::vector<std::set<int>> adj(N);
  auto addEdge = [&](int a, int b) { if (a != b) { adj[a].insert(b); adj[b].insert(a); } };
  for (size_t i = 0; i + 1 < pairs.size(); i += 2) {
    const int a = pairs[i], b = pairs[i + 1];
    if (a < 0 || a >= N || b < 0 || b >= N) return "pair frame index out of range";
    addEdge(a, b);
    if (cfg.intr_opt == RCVD_INTR_SHARED) { addEdge(a, 0); addEdge(b, 0); }
  }
  if (cfg.position_reg > 0.0) for (int f = 0; f + 2 < N; ++f) { addEdge(f, f + 1); addEdge(f, f + 2); addEdge(f + 1, f + 2); }
  for (size_t t = 0; t < trip_centers.size(); ++t) {
    const int f = trip_centers[t];
    if (f < 1 || f + 1 >= N) return "triplet centre frame out of range";
    addEdge(f - 1, f); addEdge(f - 1, f + 1); addEdge(f, f + 1);
    if (cfg.intr_opt == RCVD_INTR_SHARED) { addEdge(f - 1, 0); addEdge(f, 0); addEdge(f + 1, 0); }
  }
  std::vector<std::set<int>> orig = adj;
  // Multiple minimum-degree elimination: each round eliminates a maximal independent set of frames whose current degree is
  // within `slack` of the minimum (ties -> lowest frame id).  slack = 0 is plain greedy minimum degree one frame at a time
  // semantics-wise; a small slack trades a few % more fill for a shallower elimination tree (fewer sequential levels).
  std::vector<int> order, pos(N, -1); std::vector<std::vector<int>> cs(N);
  {
    std::vector<uint8_t> done(N, 0);
    const int slack = order_slack;
    while ((int)order.size() < N) {
      size_t md = (size_t)-1;
      for (int f = 0; f < N; ++f) if (!done[f]) md = std::min(md, adj[f].size());
      std::vector<int> cand;
      const size_t lim = md + (size_t)(slack > 0 ? slack : 0);
      for (int f = 0; f < N; ++f) if (!done[f] && adj[f].size() <= lim) cand.push_back(f);
      std::stable_sort(cand.begin(), cand.end(), [&](int a, int b) { return adj[a].size() < adj[b].size(); });
      std::vector<uint8_t> blocked(N, 0); std::vector<int> chosen;
      for (int f : cand) { if (blocked[f]) continue; chosen.push_back(f); blocked[f] = 1; for (int a : adj[f]) blocked[a] = 1; if (slack < 0) break; }
      for (int best : chosen) {
        done[best] = 1; pos[best] = (int)order.size(); order.push_back(best);
        std::vector<int> nb(adj[best].begin(), adj[best].end());
        cs[best] = nb;
        for (int a : nb) adj[a].erase(best);
        for (size_t i = 0; i < nb.size(); ++i) for (size_t j = i + 1; j < nb.size(); ++j) { adj[nb[i]].insert(nb[j]); adj[nb[j]].insert(nb[i]); }
      }
    }
    for (int f = 0; f < N; ++f) std::sort(cs[f].begin(), cs[f].end(), [&](int a, int b) { return pos[a] < pos[b]; });
  }
  // levels
  std::vector<int> lvl(N, 0); int nl = 0;
  for (int k : order) { for (int a : cs[k]) lvl[a] = std::max(lvl[a], lvl[k] + 1); nl = std::max(nl, lvl[k] + 1); }
  std::vector<std::vector<int>> lf(nl);
  for (int k : order) lf[lvl[k]].push_back(k);

  // ---- multi-GPU distribution of the factorisation (DESIGN.md section 5) ----
  // Phase A = the wide early levels (throughput-bound: thousands of block products): every frame (= block column of the factor) has an
  // owner rank that factors it (potrf, trsm) and computes every update INTO its column; after the trsm of a level the new off-diagonal
  // factor blocks X_rk are broadcast from their owners (they are the operands of everybody's updates and of the replicated
  // substitution).  Phase B = the tail of narrow levels (< 3 frames per level: a latency chain that does not shard) is replicated:
  // at the boundary every owner broadcasts its trailing blocks.  H is reduced to the owners only (no all-reduce of the matrix).
  const int R = nranks;
  bool dist = R > 1 && dist_enabled && cfg.intr_opt != RCVD_INTR_SHARED && !(cfg.position_reg > 0.0) && trip_centers.empty();
  int TB = nl; while (TB > 0 && (int)lf[TB - 1].size() < 3) --TB;
  int LB = 0;
  if (dist) { LB = TB; if (LB == 0) dist = false; }
  P.dist = dist; P.LB = LB; P.TB = TB;
  std::vector<int> own(N, 0);
  if (dist) {
    // incoming update work of every column over the phase-A levels (block products; symmetric targets count half)
    std::vector<double> tot_in(N, 0.0);
    for (int l = 0; l < LB; ++l) for (int k : lf[l]) { const auto& m = cs[k]; for (size_t a = 0; a < m.size(); ++a) for (size_t b = 0; b <= a; ++b) tot_in[m[b]] += (a == b) ? 0.5 : 1.0; }
    std::vector<double> load(R, 0.0);
    for (int l = 0; l < nl; ++l) {
      std::vector<int> fr = lf[l];
      auto w = [&](int k) { return tot_in[k] + (l < LB ? 0.6 * cs[k].size() + 0.3 : 0.0); };   // + its own trsm / potrf
      std::stable_sort(fr.begin(), fr.end(), [&](int a, int b) { return w(a) > w(b); });
      for (int k : fr) { int q = 0; for (int t = 1; t < R; ++t) if (load[t] < load[q]) q = t; own[k] = q; load[q] += w(k); }
    }
  }
  // internal frame numbering: owner-major, phase-A frames first -- every per-frame array an owner broadcasts / reduces is one contiguous range
  std::vector<int>& uperm = P.uperm; std::vector<int>& iperm = P.iperm;
  iperm.assign(N, -1);
  P.fa_off.assign(R, 0); P.fa_cnt.assign(R, 0); P.fb_off.assign(R, 0); P.fb_cnt.assign(R, 0);
  for (int q = 0; q < R; ++q) for (int ph = 0; ph < 2; ++ph) {
    (ph ? P.fb_off : P.fa_off)[q] = (int)uperm.size();
    for (int f = 0; f < N; ++f) if (own[f] == q && ((lvl[f] >= LB) == (ph == 1))) uperm.push_back(f);
    (ph ? P.fb_cnt : P.fa_cnt)[q] = (int)uperm.size() - (ph ? P.fb_off : P.fa_off)[q];
  }
  for (int i = 0; i < N; ++i) iperm[uperm[i]] = i;
  bool identity_perm = true; for (int i = 0; i < N; ++i) if (uperm[i] != i) identity_perm = false;
  if (!identity_perm) {
    auto I = [&](int f) { return iperm[f]; };
    std::vector<int> order2(N), pos2(N), lvl2(N), own2(N); std::vector<std::vector<int>> cs2(N); std::vector<std::set<int>> orig2(N);
    for (int i = 0; i < N; ++i) order2[i] = I(order[i]);
    for (int f = 0; f < N; ++f) { pos2[I(f)] = pos[f]; lvl2[I(f)] = lvl[f]; own2[I(f)] = own[f]; for (int a : cs[f]) cs2[I(f)].push_back(I(a)); for (int a : orig[f]) orig2[I(f)].insert(I(a)); }
    for (auto& v : lf) for (int& k : v) k = I(k);
    order.swap(order2); pos.swap(pos2); lvl.swap(lvl2); own.swap(own2); cs.swap(cs2); orig.swap(orig2);
  }
  // L off-diagonal blocks (r later than c).  Phase A: level-major, owner-major inside a level (what a rank produces in one level is one
  // contiguous range of T); phase B: owner-major (what a rank owns of the trailing matrix is one contiguous range of L).
  std::map<std::pair<int, int>, int> lid; int nLoff = 0;
  std::vector<int> lcol;   // column (earlier-eliminated) frame of each off-diagonal factor block
  auto number_col = [&](int k) { for (int r : cs[k]) { lid[{r, k}] = N + nLoff++; lcol.push_back(k); } };
  P.tseg.assign((size_t)std::max(LB, 0) * R * 2, 0); P.bseg.assign((size_t)R * 2, 0);
  for (int l = 0; l < LB; ++l) for (int q = 0; q < R; ++q) {
    const int first = nLoff;
    for (int k : lf[l]) if (own[k] == q) number_col(k);
    P.tseg[((size_t)l * R + q) * 2] = first; P.tseg[((size_t)l * R + q) * 2 + 1] = nLoff - first;
  }
  for (int q = 0; q < R; ++q) {
    const int first = nLoff;
    for (int l = LB; l < nl; ++l) for (int k : lf[l]) if (own[k] == q) number_col(k);
    P.bseg[(size_t)q * 2] = first; P.bseg[(size_t)q * 2 + 1] = nLoff - first;
  }
  P.nLoff = nLoff;
  // H blocks: diagonal first (internal frame order = owner-major), then original off-diagonals oriented (later, earlier), owner-major
  std::vector<HBlock>& hblocks = P.hblocks;
  P.blk_of.assign((size_t)N * N, -1);
  for (int f = 0; f < N; ++f) hblocks.push_back({f, f, f});
  P.hseg.assign((size_t)R * 2, 0);
  for (int q = 0; q < R; ++q) {
    P.hseg[(size_t)q * 2] = (int)hblocks.size();
    for (int a = 0; a < N; ++a) for (int b : orig[a]) if (a < b) {
      const int r = pos[a] > pos[b] ? a : b, c = pos[a] > pos[b] ? b : a;
      if (own[c] != q) continue;
      const int hid = (int)hblocks.size();
      hblocks.push_back({lid[{r, c}], r, c});
      P.blk_of[(size_t)r * N + c] = hid * 2 + 1;   // (fa = r) is the row side
      P.blk_of[(size_t)c * N + r] = hid * 2 + 0;
    }
    P.hseg[(size_t)q * 2 + 1] = (int)hblocks.size() - P.hseg[(size_t)q * 2];
  }
  const int nHblocks = (int)hblocks.size();
  // all L blocks with their H source (or -1)
  P.lblocks.resize(N + nLoff);
  for (int f = 0; f < N; ++f) P.lblocks[f] = {f, f, f};
  for (auto& kv : lid) P.lblocks[kv.second] = {-1, kv.first.first, kv.first.second};
  for (int h = N; h < nHblocks; ++h) P.lblocks[hblocks[h].lblk].lblk = h;
  P.elim_order = order; P.level = lvl; P.owner = own;
  for (int b = 0; b < N + nLoff; ++b) { const int c = b < N ? b : lcol[b - N]; if (!dist || own[c] == rank) P.own_lblocks.push_back(b); }
  for (int h = 0; h < nHblocks; ++h) if (!dist || own[hblocks[h].c] == rank) P.own_hblocks.push_back(h);
  for (int b : P.own_lblocks) if (P.lblocks[b].lblk >= 0) P.load_lblocks.push_back(b);
  P.nload = (int)P.load_lblocks.size();
  for (int b : P.own_lblocks) if (P.lblocks[b].lblk < 0) P.load_lblocks.push_back(b);
  // tile cut of the update targets: kUpdMaxTile-row tiles over the unknowns (rounded to 8)
  const int upd_neff = std::min(npad, (L.nf + 7) / 8 * 8);
  const int upd_nt = (upd_neff + kUpdMaxTile - 1) / kUpdMaxTile;
  const int upd_tile = std::min(kUpdMaxTile, upd_neff);          // 80-row tiles (balanced 5 x 5 units per warp), the remainder last
  P.upd_rb = upd_tile; P.upd_neff = upd_neff;
  // The block products (source frame k, target (r, c)) of every target, in source-level order.  c is eliminated before r: the target
  // lives in column c, and a rank updates only the columns it owns in phase A.
  auto col_of = [&](int target) { return target < N ? target : lcol[target - N]; };
  std::map<int, std::vector<std::pair<int, int2>>> prod;   // target L block id -> (source level, source pair)
  std::map<int, int> first_level;                           // target L block id -> earliest source level of any rank's products into it
  for (int l = 0; l < nl; ++l) {
    const bool shared_level = !dist || l >= LB;   // replicated work: every rank does all of it
    std::set<int> targets;
    for (int k : lf[l]) for (size_t a = 0; a < cs[k].size(); ++a) for (size_t b = 0; b <= a; ++b) {
      const int r = cs[k][a], c = cs[k][b];
      const int target = (r == c) ? r : lid[{r, c}];
      first_level.emplace(target, l);
      if (!shared_level && own[c] != rank) continue;
      prod[target].push_back({l, make_int2(lid[{r, k}] - N, lid[{c, k}] - N)});
      targets.insert(target);
    }
    P.upd_targets += (int)targets.size();
  }
  // Update passes.  The products from level Lc - 1 (Lc: the level of the target's column) are the late pass: it runs on the main stream
  // at Lc - 1, on the critical path.  The earlier products are deferred to the side stream, grouped in level windows (wide levels only,
  // see kUpdWindow), each window one pass applied at the level of its latest source: every pass reads and writes the whole target, so
  // fewer, longer passes move less of it through memory.  Within a level the passes are in target order.
  // The first pass into a fill block (an L block without an H source; k_load_factor leaves its interior alone) writes the target without
  // reading it.  Passes into one target run in launch order (the side stream is in order, and a late pass waits for its target's
  // deferred passes), so the first one enqueued is the first one executed.  Distributed, a rank's first pass is the block's first only if
  // it holds the block's earliest product: the phase-A passes into a phase-B column run on its owner alone, and the other ranks receive
  // the block with the broadcast at the phase boundary.
  const int W = P.upd_window = L.nf <= kUpdWindowMaxNf ? kUpdWindow : 1;
  auto window = [&](int l) { return l < TB ? l / W : nl + l; };
  std::vector<std::vector<std::pair<int, std::vector<int2>>>> late(nl), deferred(nl);   // per apply level: (target, source pairs)
  for (auto& kv : prod) {
    const int Lc = lvl[col_of(kv.first)];
    const auto& v = kv.second;
    for (size_t i = 0, j; i < v.size(); i = j) {
      const bool is_late = v[i].first == Lc - 1;
      for (j = i + 1; j < v.size() && (v[j].first == Lc - 1) == is_late && (is_late || window(v[j].first) == window(v[i].first)); ++j) {}
      auto& pass = (is_late ? late : deferred)[v[j - 1].first];
      pass.push_back({kv.first, {}});
      for (size_t q = i; q < j; ++q) pass.back().second.push_back(v[q].second);
    }
  }
  std::vector<uint8_t> updated(N + nLoff, 0);   // per L block: a pass into it is enqueued already
  for (int l = 0; l < nl; ++l) {
    Level lv; lv.frame_off = (int)P.lvl_frames.size(); lv.nframes = (int)lf[l].size(); lv.own_off = (int)P.lvl_own.size();
    lv.trsm_off = (int)P.trsm_tasks.size(); lv.upd_off = (int)P.upd_tasks.size(); lv.fwd_off = (int)P.fwd_tasks.size();
    const bool shared_level = !dist || l >= LB;
    for (int k : lf[l]) {
      P.lvl_frames.push_back(k);
      const bool mine = shared_level || own[k] == rank;
      if (mine) P.lvl_own.push_back(k);
      for (int r : cs[k]) {
        const int id = lid[{r, k}];
        if (mine) P.trsm_tasks.push_back({id - N, id, k});
        P.fwd_tasks.push_back({id - N, r, k});
      }
    }
    lv.nown = (int)P.lvl_own.size() - lv.own_off;
    // the deferred passes of a batched level are two launches, so that the next level's late passes wait only for the first
    lv.join[0] = lv.join[1] = nl;
    const bool split = W > 1 && l < TB;
    for (int pass = 0; pass < 3; ++pass) {
      if (pass > 0) lv.upd2_off[pass - 1] = (int)P.upd_tasks.size();
      for (auto& tp : (pass ? deferred : late)[l]) {
        const int Lc = lvl[col_of(tp.first)];
        if (pass > 0 && (!split || Lc == l + 2) != (pass == 1)) continue;
        if (pass > 0) lv.join[pass - 1] = std::min(lv.join[pass - 1], Lc - 1);
        const bool first_fill = P.lblocks[tp.first].lblk < 0 && !updated[tp.first] && prod[tp.first][0].first == first_level[tp.first];
        updated[tp.first] = 1;
        P.upd_tasks.push_back({tp.first, (int)P.upd_pairs.size(), (int)tp.second.size(), (tp.first < N ? 1 : 0) | (first_fill ? 2 : 0)});
        { const double n = (double)L.nf; P.upd_flops += (double)tp.second.size() * (tp.first < N ? n * n * (n + 1.0) : 2.0 * n * n * n); }
        P.upd_pairs.insert(P.upd_pairs.end(), tp.second.begin(), tp.second.end());
      }
    }
    lv.ntrsm = (int)P.trsm_tasks.size() - lv.trsm_off; lv.nupd = lv.upd2_off[0] - lv.upd_off; lv.nfwd = (int)P.fwd_tasks.size() - lv.fwd_off;
    lv.nupd2[0] = lv.upd2_off[1] - lv.upd2_off[0]; lv.nupd2[1] = (int)P.upd_tasks.size() - lv.upd2_off[1];
    // work items of the persistent update kernel: one per (target tile, source-pair list), per launch in cost order and in locality
    // order; a launch of the two-team shape is a single wave and keeps the cost order in both
    std::vector<UpdItem>& items = P.upd_items_cost;
    for (int pass = 0; pass < 3; ++pass) {
      const int t0 = pass ? lv.upd2_off[pass - 1] : lv.upd_off, tn = pass ? lv.nupd2[pass - 1] : lv.nupd;
      const size_t i0 = items.size();
      for (int q = t0; q < t0 + tn; ++q) {
        const UpdPass& tk = P.upd_tasks[q];
        for (int ti = 0; ti < upd_nt; ++ti) for (int tj = 0; tj < ((tk.flags & 1) ? ti + 1 : upd_nt); ++tj) {
          UpdItem it; it.dst = tk.dst; it.first = tk.first; it.count = tk.count; it.m0 = (short)(ti * upd_tile); it.n0 = (short)(tj * upd_tile);
          it.mrows = (short)std::min(upd_tile, upd_neff - ti * upd_tile); it.ncols = (short)std::min(upd_tile, upd_neff - tj * upd_tile);
          it.flags = (((tk.flags & 1) && ti == tj) ? kUpdSymDiag : 0) | ((tk.flags & 2) ? kUpdFirstFill : 0);
          items.push_back(it);
        }
      }
      P.upd_items.resize(items.size());
      const std::vector<UpdItem> built(items.begin() + i0, items.end());
      std::stable_sort(items.begin() + i0, items.end(), [](const UpdItem& a, const UpdItem& b) { return upd_item_cost(a) > upd_item_cost(b); });
      const int n = (int)built.size();
      if (!order_update_items(built, P.upd_pairs, lcol, upd_ctas(n, num_sms), P.upd_items.data() + i0))
        return "internal error: two update items of one launch write the same target tile";
      if (n <= num_sms) std::copy(items.begin() + i0, items.end(), P.upd_items.begin() + i0);
      if (pass) { lv.it2_off[pass - 1] = (int)i0; lv.nit2[pass - 1] = (int)(items.size() - i0); } else { lv.it_off = (int)i0; lv.nit = (int)(items.size() - i0); }
    }
    P.levels.push_back(lv);
  }
  // task list of the fused substitution kernel (k_substitution): forward levels ascending, backward levels descending, every GEMV cut
  // into kSubChunk-row / -column chunks; a task depends only on tasks before it
  P.sub_need.assign(2 * (size_t)N, 0);
  {
    const int nch = (npad + kSubChunk - 1) / kSubChunk;
    // The wide levels at the bottom of the tree stay level-scheduled launches (thousands of independent GEMVs: a launch spreads them
    // over the machine at once, a persistent CTA works through them one memory latency at a time); the narrow levels above them -- a
    // latency chain of four tiny launches per level -- run as ONE dataflow kernel: forward narrow, backward narrow in a single launch.
    const int limit = 4 * num_sms;
    int LS = (int)P.levels.size();
    while (LS > 0 && (P.levels[LS - 1].nframes + P.levels[LS - 1].nfwd) * nch <= limit) --LS;
    P.sub_first_level = LS;
    for (size_t l = LS; l < P.levels.size(); ++l) {
      const Level& lv = P.levels[l];
      for (int i = 0; i < lv.nframes; ++i) for (int c = 0; c < nch; ++c) P.sub_tasks.push_back({0, -1, -1, P.lvl_frames[lv.frame_off + i], c});
      for (int q = 0; q < lv.nfwd; ++q) { const SolveTask& t = P.fwd_tasks[lv.fwd_off + q]; for (int c = 0; c < nch; ++c) P.sub_tasks.push_back({1, t.blk, t.r, t.k, c}); P.sub_need[t.r] += nch; P.sub_need[N + t.k] += nch; }
    }
    for (int l = (int)P.levels.size() - 1; l >= LS; --l) {
      const Level& lv = P.levels[l];
      for (int q = 0; q < lv.nfwd; ++q) { const SolveTask& t = P.fwd_tasks[lv.fwd_off + q]; for (int c = 0; c < nch; ++c) P.sub_tasks.push_back({2, t.blk, t.r, t.k, c}); }
      for (int i = 0; i < lv.nframes; ++i) for (int c = 0; c < nch; ++c) P.sub_tasks.push_back({3, -1, -1, P.lvl_frames[lv.frame_off + i], c});
    }
  }
  return nullptr;
}

}  // namespace rcvd
