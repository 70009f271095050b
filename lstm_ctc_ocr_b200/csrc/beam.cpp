// CTC prefix beam search, host side (SURVEY §8(f)4).
//
// Replaces tf.nn.ctc_beam_search_decoder(logits, seq_len, merge_repeated=True) at lib/networks/network.py:656 and
// lib/lstm/test.py:30 (beam_width 100, top_paths 1, blank = C-1) + sparse_tensor_to_dense(default 0) at network.py:657.
// The reference's op is a CPU-only TensorFlow kernel that runs at validation / evaluation time only; so is this one: it
// takes HOST logits (the caller copies the [T,N,C] logits back once) and spreads the utterances over host threads.  The hot
// path's decoder is the greedy kernel in ctc.cu; this entry point exists for exact reproduction of the reference's decode on
// outputs that are not peaked.
//
// Algorithm [upstream-memory: tensorflow/core/util/ctc/ctc_beam_search.h, CTCBeamSearchDecoder::Step / TopPaths]: a prefix
// tree whose entries carry log P(prefix, ending in blank) and log P(prefix, ending in its last label) for the previous and the
// current frame; per frame (1) every entry of the beam is re-scored in place, (2) entries are expanded in descending order of
// their previous total against the running bottom of a beam_width-bounded list, a full list evicting its bottom.  The result is
// the label sequence of the best entry, with consecutive equal labels collapsed when merge_repeated is set (TF applies that to
// the decoded sequence, so "a, blank, a" also comes out as one "a").  crnn_ctc_beam_search_topk returns TopPaths' n best: the
// listed entries by total, highest first, exact ties in insertion order.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <limits>
#include <memory>
#include <thread>
#include <vector>

#include "../../include/crnn_ctc.h"

int crnn_fail(int status, const char* fmt, ...);

namespace {

constexpr double kLogZero = -std::numeric_limits<double>::infinity();

inline double log_add(double a, double b) {
  if (a == kLogZero) return b;
  if (b == kLogZero) return a;
  const double m = a > b ? a : b;
  return m + std::log1p(std::exp(-std::fabs(a - b)));
}

struct Prob {
  double total = kLogZero, blank = kLogZero, label = kLogZero;
  void reset() { total = blank = label = kLogZero; }
};

// One prefix of the tree.  Children are created on demand (only a child that enters the beam needs storage: an inactive child
// carries no state), `kids` is a per-entry table label -> arena index that appears with the first child.
struct Entry {
  Entry* parent = nullptr;
  int label = -1;
  int kids = -1;              // offset of this entry's (C-1)-slot child table in the table pool, -1 = no child yet
  int64_t leaf_seq = -1;      // insertion number while the entry is in the leaf list, -1 = not in it
  int evicted_kid_frame = -1; // last frame in which one of this entry's children was evicted from the list
  Prob oldp, newp;
  bool active() const { return newp.total != kLogZero; }
};

// The beam: entries in insertion order (what the next frame's stable sort and the final arg-max walk), plus a min-heap on
// (total, insertion number) so that the bottom -- the FIRST of the smallest totals in insertion order, the entry a full list
// evicts -- costs O(log width) instead of a scan per candidate.  Totals of listed entries do not change while candidates are
// being inserted (re-scoring happens before), so the heap keys stay valid for the whole frame.
struct Leaves {
  struct Item { double total; int64_t seq; Entry* e; };
  static bool above(const Item& a, const Item& b) { return a.total > b.total || (a.total == b.total && a.seq > b.seq); }   // min-heap order
  std::vector<Item> heap;
  std::vector<std::pair<Entry*, int64_t>> order;
  int64_t next_seq = 0;
  size_t size() const { return heap.size(); }
  double bottom_total() const { return heap.front().total; }
  void push(Entry* e) {
    e->leaf_seq = next_seq;
    order.emplace_back(e, next_seq);
    heap.push_back(Item{e->newp.total, next_seq, e});
    std::push_heap(heap.begin(), heap.end(), above);
    ++next_seq;
  }
  // evicts the bottom and lists `e` in its place: one sift-down instead of a pop and a push
  Entry* replace_bottom(Entry* e) {
    Entry* ev = heap.front().e;
    ev->leaf_seq = -1;
    e->leaf_seq = next_seq;
    order.emplace_back(e, next_seq);
    const Item it{e->newp.total, next_seq++, e};
    const size_t n = heap.size();
    size_t i = 0;
    for (;;) {
      size_t l = 2 * i + 1, r = l + 1, m = l;
      if (l >= n) break;
      if (r < n && above(heap[l], heap[r])) m = r;       // the smaller child
      if (!above(it, heap[m])) break;
      heap[i] = heap[m];
      i = m;
    }
    heap[i] = it;
    return ev;
  }
  // listed entries in insertion order; clears the list
  void drain(std::vector<Entry*>& out) {
    out.clear();
    for (auto& pr : order) if (pr.first->leaf_seq == pr.second) { out.push_back(pr.first); pr.first->leaf_seq = -1; }
    order.clear(); heap.clear(); next_seq = 0;
  }
};

// Per-thread working memory, reused from utterance to utterance: entries live in fixed chunks (stable addresses, no
// allocation per entry), child tables in one growing pool.
struct Scratch {
  static constexpr int kChunkBits = 10;
  std::vector<std::unique_ptr<Entry[]>> chunks;
  int used = 0;
  std::vector<int> kid_pool;                     // child tables, (C-1) slots each: entry index or -1
  Leaves leaves;
  std::vector<Entry*> branches;
  std::vector<double> lp, lp_desc;
  std::vector<int> by_lp;
  Entry* at(int i) { return &chunks[i >> kChunkBits][i & ((1 << kChunkBits) - 1)]; }
  int alloc() {
    if ((size_t)(used >> kChunkBits) == chunks.size()) chunks.emplace_back(new Entry[1 << kChunkBits]);
    Entry* e = at(used);
    *e = Entry();
    return used++;
  }
  void reset(int C) {
    used = 0; kid_pool.clear();
    leaves.order.clear(); leaves.heap.clear(); leaves.next_seq = 0;
    lp.assign(C, 0.0); lp_desc.assign(C - 1, 0.0); by_lp.assign(C - 1, 0);
  }
};

// out [top_paths, max_out], out_len / score [top_paths]; `score` gets newp.total (negated when `negate`), `num_paths` the count
// of real paths
void decode_one(Scratch& S, const float* logits, int stride_t, int len, int C, int beam_width, int top_paths, int merge_repeated,
                int strip, int* out, int max_out, int* out_len, float* score, int negate, int* num_paths) {
  const int blank = C - 1, nlab = C - 1;
  S.reset(C);
  std::vector<int>& kid_pool = S.kid_pool;
  Entry* root = S.at(S.alloc());
  root->newp.total = 0.0; root->newp.blank = 0.0; root->newp.label = kLogZero;
  Leaves& leaves = S.leaves;
  leaves.push(root);
  std::vector<Entry*>& branches = S.branches;
  std::vector<double>&lp = S.lp, &lp_desc = S.lp_desc;
  std::vector<int>& by_lp = S.by_lp;
  constexpr int kFewClasses = 16;
  for (int t = 0; t < len; ++t) {
    const float* row = logits + (size_t)t * stride_t;
    double mx = kLogZero;
    for (int c = 0; c < C; ++c) if (row[c] == row[c]) mx = std::max<double>(mx, row[c]);      // a NaN logit counts as -inf
    double se = 0.0;
    for (int c = 0; c < C; ++c) if (row[c] == row[c]) se += std::exp((double)row[c] - mx);
    const double norm = mx + std::log(se);
    for (int c = 0; c < C; ++c) lp[c] = (row[c] == row[c]) ? (double)row[c] - norm : kLogZero;
    if (!(norm == norm)) for (int c = 0; c < C; ++c) lp[c] = kLogZero;                      // an all -inf / NaN row: nothing survives it

    leaves.drain(branches);
    std::stable_sort(branches.begin(), branches.end(), [](const Entry* a, const Entry* b) { return a->newp.total > b->newp.total; });
    for (Entry* b : branches) b->oldp = b->newp;
    for (Entry* b : branches) {
      if (b->parent != nullptr) {
        if (b->parent->active()) {
          const double prev = (b->label == b->parent->label) ? b->parent->oldp.blank : b->parent->oldp.total;
          b->newp.label = log_add(b->newp.label, prev);
        }
        b->newp.label += lp[b->label];
      }
      b->newp.blank = b->oldp.total + lp[blank];
      b->newp.total = log_add(b->newp.blank, b->newp.label);
      leaves.push(b);
    }
    // classes in descending order of lp: once the list is full, only a class with lp[c] > bottom - total(b) can enter it from
    // branch b, and with peaked frames that is one or two classes instead of C-1
    for (int c = 0; c < nlab; ++c) by_lp[c] = c;
    std::sort(by_lp.begin(), by_lp.end(), [&](int a, int b) { return lp[a] > lp[b]; });
    for (int c = 0; c < nlab; ++c) lp_desc[c] = lp[by_lp[c]];

    const size_t width = (size_t)beam_width;
    for (Entry* b : branches) {
      const double btotal = b->oldp.total;
      const bool full = leaves.size() >= width;
      if (!(btotal > kLogZero && (!full || btotal > leaves.bottom_total()))) continue;
      int few[kFewClasses];
      int k = -1, pos = 0;                 // k >= 0: pruned visit of few[0..k), pos = index of the class being visited
      // TF's per-class step, unchanged: an active child was re-scored above; otherwise the child (label c appended to b) is a
      // candidate with lp[c] + P(b, not ending in c) and enters the list if it beats the bottom, evicting it when the list is full.
      // A rejected child that exists is wiped -- which matters when it is a branch of THIS frame that an earlier insertion
      // evicted: wiping its oldp is what stops the branch loop from expanding it later in the frame.
      auto try_class = [&](int c) {
        Entry* ch = (b->kids >= 0 && kid_pool[b->kids + c] >= 0) ? S.at(kid_pool[b->kids + c]) : nullptr;
        if (ch != nullptr && ch->active()) return;
        const double total = lp[c] + ((c == b->label) ? b->oldp.blank : btotal);
        if (!(total > kLogZero && (leaves.size() < width || total > leaves.bottom_total()))) {
          if (ch != nullptr) { ch->oldp.reset(); ch->newp.reset(); }
          return;
        }
        if (ch == nullptr) {
          if (b->kids < 0) {
            b->kids = (int)kid_pool.size();
            kid_pool.resize(kid_pool.size() + nlab, -1);
          }
          const int idx = S.alloc();
          kid_pool[b->kids + c] = idx;
          ch = S.at(idx);
          ch->parent = b;
          ch->label = c;
        }
        ch->newp.blank = kLogZero;
        ch->newp.label = total;
        ch->newp.total = total;
        if (leaves.size() == width) {
          Entry* ev = leaves.replace_bottom(ch);
          ev->newp.reset();
          if (ev->parent != nullptr) ev->parent->evicted_kid_frame = t;
          if (k >= 0 && ev->parent == b && ev->label > c) {
            // pruned visit: the full visit would still reach this child of b; if its class is not among the ones left to visit it
            // can only be rejected there (it is outside the superset), i.e. wiped
            bool later = false;
            for (int i = pos + 1; i < k; ++i) later |= (few[i] == ev->label);
            if (!later) ev->oldp.reset();
          }
        } else {
          leaves.push(ch);
        }
      };
      if (full && b->evicted_kid_frame != t) {
        // superset of the classes that can still enter: the bottom only rises while this branch is expanded, and the repeated
        // label uses oldp.blank <= oldp.total; the slack keeps the subtraction's rounding on the safe side (exact test in try_class).
        // Not used when a child of b was evicted earlier in this frame: the full visit has to reach (and wipe or re-admit) it.
        const double bt = leaves.bottom_total();
        const double thr = (bt - btotal) - 1e-9 * (1.0 + std::fabs(bt) + std::fabs(btotal));
        // lp_desc is descending: the count of elements >= thr
        const int cnt = (int)(std::upper_bound(lp_desc.begin(), lp_desc.end(), thr, [](double v, double e) { return v > e; }) - lp_desc.begin());
        if (cnt <= kFewClasses) k = cnt;
      }
      if (k < 0) {
        for (int c = 0; c < nlab; ++c) try_class(c);
      } else {
        for (int i = 0; i < k; ++i) {                   // insertion sort into ascending class order: TF visits classes by index
          int v = by_lp[i], j = i;
          while (j > 0 && few[j - 1] > v) { few[j] = few[j - 1]; --j; }
          few[j] = v;
        }
        for (pos = 0; pos < k; ++pos) try_class(few[pos]);
      }
    }
  }
  // TopPaths: the listed entries by total, highest first, exact ties in insertion order (the order drain leaves them in)
  leaves.drain(branches);
  std::stable_sort(branches.begin(), branches.end(), [](const Entry* a, const Entry* b) { return a->newp.total > b->newp.total; });
  const int paths = (int)std::min<size_t>(branches.size(), (size_t)top_paths);
  std::vector<int> seq;
  for (int p = 0; p < top_paths; ++p) {
    int* o = out + (size_t)p * max_out;
    int n = 0;
    double total = kLogZero;
    if (p < paths) {
      total = branches[p]->newp.total;
      seq.clear();
      for (Entry* e = branches[p]; e->parent != nullptr; e = e->parent) seq.push_back(e->label);
      int prev = -1;
      for (auto it = seq.rbegin(); it != seq.rend(); ++it) {
        const int l = *it;
        const bool keep = !(merge_repeated && l == prev);
        prev = l;
        if (keep && l != strip && n < max_out) o[n++] = l;
      }
    }
    for (int i = n; i < max_out; ++i) o[i] = 0;
    out_len[p] = n;
    if (score) score[p] = (float)(negate ? -total : total);
  }
  if (num_paths) *num_paths = paths;
}

// both host entry points: out [N, top_paths, T], out_len / score [N, top_paths], num_paths [N]
int beam_search_host(const float* logits_host, const int* input_len_host, int T, int N, int C, int beam_width, int top_paths,
                     int merge_repeated, int strip, int* out_host, int* out_len_host, float* score_host, int negate,
                     int* num_paths_host, int num_threads) {
  if (!logits_host || !input_len_host || !out_host || !out_len_host) return crnn_fail(CRNN_INVALID_VALUE, "beam_search: null pointer");
  if (T <= 0 || N <= 0 || C < 2 || beam_width < 1) return crnn_fail(CRNN_INVALID_VALUE, "beam_search: bad shape");
  if (top_paths < 1 || top_paths > beam_width)
    return crnn_fail(CRNN_INVALID_VALUE, "beam_search: top_paths %d outside [1, beam_width = %d]", top_paths, beam_width);
  for (int n = 0; n < N; ++n)
    if (input_len_host[n] < 0 || input_len_host[n] > T) return crnn_fail(CRNN_INVALID_VALUE, "beam_search: input_len[%d] outside [0, T]", n);
  int nt = num_threads > 0 ? num_threads : (int)std::thread::hardware_concurrency();
  nt = std::max(1, std::min(nt, N));
  // utterances are handed out one at a time (ragged lengths: a static split leaves threads idle); nothing may throw across the ABI
  std::atomic<int> next{0};
  std::atomic<bool> failed{false};
  auto work = [&]() {
    try {
      Scratch S;
      for (int n = next.fetch_add(1); n < N && !failed.load(std::memory_order_relaxed); n = next.fetch_add(1)) {
        const size_t row = (size_t)n * top_paths;
        decode_one(S, logits_host + (size_t)n * C, N * C, input_len_host[n], C, beam_width, top_paths, merge_repeated, strip,
                   out_host + row * T, T, out_len_host + row, score_host ? score_host + row : nullptr, negate,
                   num_paths_host ? num_paths_host + n : nullptr);
      }
    } catch (...) {
      failed.store(true);
    }
  };
  if (nt == 1) {
    work();
  } else {
    std::vector<std::thread> th;
    try {
      for (int i = 0; i < nt - 1; ++i) th.emplace_back(work);
    } catch (...) {}                                   // fewer helper threads than asked for: the caller's thread still drains the queue
    work();
    for (auto& t : th) t.join();
  }
  if (failed.load()) return crnn_fail(CRNN_INVALID_VALUE, "beam_search: out of host memory");
  return CRNN_OK;
}

}  // namespace

extern "C" int crnn_ctc_beam_search(const float* logits_host, const int* input_len_host, int T, int N, int C, int beam_width,
                                    int merge_repeated, int strip, int* out_host, int* out_len_host, float* neg_log_prob_host,
                                    int num_threads) {
  return beam_search_host(logits_host, input_len_host, T, N, C, beam_width, 1, merge_repeated, strip, out_host, out_len_host,
                          neg_log_prob_host, 1, nullptr, num_threads);
}

extern "C" int crnn_ctc_beam_search_topk(const float* logits_host, const int* input_len_host, int T, int N, int C, int beam_width,
                                         int top_paths, int merge_repeated, int strip, int* out_host, int* out_len_host,
                                         float* log_prob_host, int* num_paths_host, int num_threads) {
  return beam_search_host(logits_host, input_len_host, T, N, C, beam_width, top_paths, merge_repeated, strip, out_host, out_len_host,
                          log_prob_host, 0, num_paths_host, num_threads);
}
