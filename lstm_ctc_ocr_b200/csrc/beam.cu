// CTC prefix beam search on the device (SURVEY §8(f)4): the algorithm of beam.cpp -- TensorFlow's CTCBeamSearchDecoder
// (network.py:656, test.py:30: width 100, top_paths 1, blank = C-1, merge_repeated; any top_paths up to the width through
// crnn_ctc_beam_search_topk_device) -- for logits that are already on the GPU, so that cfg.DECODER = "beam" needs no copy of
// the [T,N,C] logits and no host decode.
//
// One CTA of one warp per utterance.  Per frame the warp computes the log-softmax row (exp in parallel, the normaliser's sum
// sequentially in class order, as the host does: on exactly tied frames the decode depends on its last bit) and ranks the
// classes by log-probability; then lane 0 runs the frame's sequential part, which is beam.cpp's step rule for rule:
//   drain the listed entries in insertion order and stable-sort them by total (descending); oldp = newp; re-score them in
//   that order (a parent sorted earlier has already been re-scored: its newp decides whether it is active); re-push them;
//   expand them in that order, classes in ascending index, against the bottom of the width-bounded list -- the FIRST of the
//   smallest totals in insertion order, kept in a (total, insertion number) min-heap -- evicting the bottom when full.
// The beam (heap, branch list, lp row) lives in shared memory, the prefix tree in the workspace.  After the last frame the
// whole warp ranks the listed entries and writes the top_paths best, one lane per path (finish_paths).
//
// Prefix identity.  A prefix that is evicted and later re-admitted must be the entry its listed children point at, so
// entries live in a tree keyed by (parent, label).  Only listed entries, their ancestors and the entries of the current frame
// carry state that can be observed: an entry outside that set is inactive and none of its fields is read again, so it behaves
// exactly like an entry that was never created (the host decoder keeps such entries; so does this one until it needs the
// room).  When a frame's admissions could overflow the arena, the tree is compacted at the frame's start to the listed
// entries and their ancestors (order-preserving, so a parent keeps a smaller index than its children).  Listed entries at
// the start of frame t have depth <= t, so at most 1 + width*t entries survive, and a frame adds at most width*(C-1): an
// arena of 1 + width*(T+C) entries per utterance is bounded by the shapes alone and never overflows.  Each entry's children form a list sorted by label; children
// of b are only created while b is expanded, in ascending class order, so one cursor walks the list alongside the classes.
//
// The visit of a branch covers the classes whose candidate can still enter the list plus every existing child.  That equals
// TF's visit of all C-1 classes: the bottom of a full list only rises, so any other class is rejected, and a rejected class
// without an entry has nothing to wipe.  The superset is taken from the classes ranked by lp, against the bottom as of the
// start of the visit, with the same slack as beam.cpp; the exact test is made per class.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kThreads = 32;
constexpr int kMaxClasses = 64;
constexpr int kMaxWidth = 128;

#define BEAM_HD __host__ __device__ __forceinline__

BEAM_HD double neg_inf() { return -HUGE_VAL; }

BEAM_HD double log_add(double a, double b) {
  if (a == neg_inf()) return b;
  if (b == neg_inf()) return a;
  const double m = a > b ? a : b;
  return m + log1p(exp(-fabs(a - b)));
}

BEAM_HD int lowest_bit(uint64_t m) {
#ifdef __CUDA_ARCH__
  return __ffsll((long long)m) - 1;
#else
  return __builtin_ctzll(m);
#endif
}

// One prefix.  oldp.label is never read, so only oldp's total and blank are kept.
struct Node {
  double ot, ob;              // oldp: total, blank
  double nt, nb, nl;          // newp: total, blank, label
  int parent, label;          // root: -1, -1
  int first_child, next_sib;  // children sorted by label, -1 terminated
  int leaf_seq;               // insertion number while listed, -1 otherwise
  int aux;                    // compaction: live mark, then new index
};

struct Item {
  double total;               // newp.total when pushed (the heap key)
  int seq, node;
};

BEAM_HD bool item_less(const Item& a, const Item& b) { return a.total < b.total || (a.total == b.total && a.seq < b.seq); }

struct Decoder {
  Node* nd;
  int used;
  Item* heap;                 // min-heap on (total, seq): heap[0] is the bottom
  int hsize, next_seq;
  Item* br;                   // this frame's branches in sorted order
  int nbr;
  int width, nlab;
  int cap;                    // arena entries

  BEAM_HD void clear_probs(Node& e) { e.ot = e.ob = e.nt = e.nb = e.nl = neg_inf(); }

  BEAM_HD void init() {
    Node& r = nd[0];
    clear_probs(r);
    r.nt = 0.0; r.nb = 0.0;
    r.parent = r.label = -1;
    r.first_child = r.next_sib = -1;
    r.leaf_seq = -1;
    used = 1;
    hsize = next_seq = 0;
    push(0);
  }

  BEAM_HD void push(int e) {
    nd[e].leaf_seq = next_seq;
    const Item it{nd[e].nt, next_seq++, e};
    int i = hsize++;
    while (i > 0) {
      const int p = (i - 1) / 2;
      if (!item_less(it, heap[p])) break;
      heap[i] = heap[p];
      i = p;
    }
    heap[i] = it;
  }

  // lists `e` in place of the bottom and returns the evicted entry (possibly `e` itself, through a stale item)
  BEAM_HD int replace_bottom(int e) {
    const int ev = heap[0].node;
    nd[ev].leaf_seq = -1;
    nd[e].leaf_seq = next_seq;
    const Item it{nd[e].nt, next_seq++, e};
    int i = 0;
    for (;;) {
      const int l = 2 * i + 1, r = l + 1;
      if (l >= hsize) break;
      const int m = (r < hsize && item_less(heap[r], heap[l])) ? r : l;
      if (!item_less(heap[m], it)) break;
      heap[i] = heap[m];
      i = m;
    }
    heap[i] = it;
    return ev;
  }

  // listed entries -> br, sorted by (newp.total descending, insertion number): beam.cpp's drain + stable sort
  BEAM_HD void drain() {
    nbr = 0;
    for (int i = 0; i < hsize; ++i) {
      const Item& it = heap[i];
      if (nd[it.node].leaf_seq == it.seq) br[nbr++] = Item{nd[it.node].nt, it.seq, it.node};
    }
    for (int i = 0; i < nbr; ++i) nd[br[i].node].leaf_seq = -1;
    hsize = next_seq = 0;
    for (int i = 1; i < nbr; ++i) {
      const Item v = br[i];
      int j = i;
      while (j > 0 && (br[j - 1].total < v.total || (br[j - 1].total == v.total && br[j - 1].seq > v.seq))) {
        br[j] = br[j - 1];
        --j;
      }
      br[j] = v;
    }
  }

  // keeps the branches and their ancestors, renumbered in order; the heap is empty here
  BEAM_HD void compact() {
    for (int i = 0; i < used; ++i) nd[i].aux = 0;
    for (int k = 0; k < nbr; ++k)
      for (int e = br[k].node; e >= 0 && !nd[e].aux; e = nd[e].parent) nd[e].aux = 1;
    int live = 0;
    for (int i = 0; i < used; ++i) nd[i].aux = nd[i].aux ? live++ : -1;
    if (live == used) return;
    // links to the first live child / next live sibling (dead entries are only walked through, their links stay intact)
    for (int i = 0; i < used; ++i) {
      Node& e = nd[i];
      if (e.aux < 0) continue;
      int fc = e.first_child, ns = e.next_sib;
      while (fc >= 0 && nd[fc].aux < 0) fc = nd[fc].next_sib;
      while (ns >= 0 && nd[ns].aux < 0) ns = nd[ns].next_sib;
      e.first_child = fc >= 0 ? nd[fc].aux : -1;
      e.next_sib = ns >= 0 ? nd[ns].aux : -1;
      e.parent = e.parent >= 0 ? nd[e.parent].aux : -1;
    }
    for (int k = 0; k < nbr; ++k) br[k].node = nd[br[k].node].aux;
    for (int i = 0; i < used; ++i)
      if (nd[i].aux >= 0 && nd[i].aux != i) nd[nd[i].aux] = nd[i];
    used = live;
  }

  BEAM_HD void rescore(const double* lp) {
    const int blank = nlab;
    for (int k = 0; k < nbr; ++k) {
      Node& b = nd[br[k].node];
      b.ot = b.nt; b.ob = b.nb;
    }
    for (int k = 0; k < nbr; ++k) {
      const int bi = br[k].node;
      Node& b = nd[bi];
      if (b.parent >= 0) {
        const Node& p = nd[b.parent];
        if (p.nt != neg_inf()) b.nl = log_add(b.nl, b.label == p.label ? p.ob : p.ot);
        b.nl += lp[b.label];
      }
      b.nb = b.ot + lp[blank];
      b.nt = log_add(b.nb, b.nl);
      push(bi);
    }
  }

  // lp_desc / by_lp: the label classes (not the blank) by descending lp
  BEAM_HD void expand(const double* lp, const double* lp_desc, const int* by_lp) {
    const uint64_t all = nlab >= 64 ? ~0ull : ((1ull << nlab) - 1);
    for (int k = 0; k < nbr; ++k) {
      const int bi = br[k].node;
      const double btotal = nd[bi].ot;
      const bool full = hsize >= width;
      if (!(btotal > neg_inf() && (!full || btotal > heap[0].total))) continue;
      uint64_t mask = all;
      if (full) {
        const double bt = heap[0].total;
        const double thr = (bt - btotal) - 1e-9 * (1.0 + fabs(bt) + fabs(btotal));
        mask = 0;
        for (int i = 0; i < nlab && lp_desc[i] >= thr; ++i) mask |= 1ull << by_lp[i];
      }
      const int blabel = nd[bi].label;
      int* link = &nd[bi].first_child;        // the child list from the first label >= the class being visited
      for (;;) {
        const int kid = *link;
        const int ck = kid >= 0 ? nd[kid].label : kMaxClasses;
        const int cm = mask ? lowest_bit(mask) : kMaxClasses;
        const int c = ck < cm ? ck : cm;
        if (c == kMaxClasses) break;
        if (c == cm) mask &= mask - 1;
        int ch = ck == c ? kid : -1;
        if (ch < 0 || nd[ch].nt == neg_inf()) {          // an active child was re-scored above
          const double total = lp[c] + (c == blabel ? nd[bi].ob : btotal);
          if (!(total > neg_inf() && (hsize < width || total > heap[0].total))) {
            if (ch >= 0) clear_probs(nd[ch]);            // stops a branch evicted earlier in this frame from being expanded
          } else {
            if (ch < 0) {
              ch = used++;
              Node& e = nd[ch];
              clear_probs(e);
              e.parent = bi; e.label = c;
              e.first_child = -1; e.next_sib = kid;
              e.leaf_seq = -1;
              *link = ch;
            }
            Node& e = nd[ch];
            e.nb = neg_inf(); e.nl = total; e.nt = total;
            if (hsize == width) {
              Node& ev = nd[replace_bottom(ch)];
              ev.nt = ev.nb = ev.nl = neg_inf();
            } else {
              push(ch);
            }
          }
        }
        if (*link >= 0 && nd[*link].label == c) link = &nd[*link].next_sib;
      }
    }
  }

  BEAM_HD void step(const double* lp, const double* lp_desc, const int* by_lp) {
    drain();
    if (used + width * nlab > cap) compact();   // only when this frame's admissions could overflow the arena
    rescore(lp);
    expand(lp, lp_desc, by_lp);
  }
};

// entries one utterance can hold at once (see the header comment); 0 when it does not fit an int index
size_t beam_node_cap(int T, int C, int beam_width) {
  const size_t cap = 1 + (size_t)beam_width * ((size_t)T + (size_t)C);
  return cap > (size_t)0x7fffffff ? 0 : cap;
}

// The warp's end of one utterance: the listed entries (the valid items of the heap's first `hsize`) ranked by (newp.total
// descending, insertion number ascending) -- beam.cpp's drain + stable sort, so path 0 is the entry the single-best decode
// returns -- and path p written by lane p % 32: its labels (merged, `strip` dropped) zero-padded to T in out[p], its length,
// and newp.total as a float (negated when `negate`).  Paths past the listed entries: length 0 and a -inf total.  `key` is
// scratch for hsize items.
__device__ void finish_paths(const Node* nd, const Item* heap, int hsize, Item* key, int* path_node, int T, int top_paths,
                             int merge_repeated, int strip, int* out, int* out_len, float* score, int negate, int* num_paths) {
  const int lane = threadIdx.x;
  for (int i = lane; i < hsize; i += kThreads) {
    const Item it = heap[i];
    key[i] = Item{nd[it.node].nt, nd[it.node].leaf_seq == it.seq ? it.seq : -1, it.node};    // seq -1: a stale item
  }
  __syncwarp();
  int listed = 0;
  for (int i0 = 0; i0 < hsize; i0 += kThreads) {
    const int i = i0 + lane;
    const bool valid = i < hsize && key[i].seq >= 0;
    if (valid) {
      const Item v = key[i];
      int r = 0;
      for (int k = 0; k < hsize; ++k) {
        const Item o = key[k];
        r += o.seq >= 0 && (o.total > v.total || (o.total == v.total && o.seq < v.seq));
      }
      if (r < top_paths) path_node[r] = v.node;
    }
    listed += __popc(__ballot_sync(0xffffffffu, valid));
  }
  __syncwarp();
  const int paths = min(listed, top_paths);
  for (int p = lane; p < top_paths; p += kThreads) {
    int* o = out + (size_t)p * T;
    int n = 0;
    double total = neg_inf();
    if (p < paths) {
      const int e0 = path_node[p];
      total = nd[e0].nt;
      int depth = 0;
      for (int e = e0; nd[e].parent >= 0; e = nd[e].parent) ++depth;
      int i = depth;
      for (int e = e0; nd[e].parent >= 0; e = nd[e].parent) o[--i] = nd[e].label;
      int prev = -1;
      for (i = 0; i < depth; ++i) {
        const int l = o[i];
        const bool keep = !(merge_repeated && l == prev);
        prev = l;
        if (keep && l != strip) o[n++] = l;
      }
    }
    for (int i = n; i < T; ++i) o[i] = 0;
    out_len[p] = n;
    if (score) score[p] = (float)(negate ? -total : total);
  }
  if (num_paths && lane == 0) *num_paths = paths;
}

__global__ void __launch_bounds__(kThreads) ctc_beam_kernel(const float* __restrict__ logits, const int* __restrict__ input_len,
                                                            int T, int N, int C, int beam_width, int top_paths, int merge_repeated,
                                                            int strip, int* __restrict__ out, int* __restrict__ out_len,
                                                            float* __restrict__ score, int negate, int* __restrict__ num_paths,
                                                            Node* __restrict__ arena, size_t node_cap) {
  __shared__ Item s_heap[kMaxWidth], s_br[kMaxWidth];
  __shared__ double s_lp[kMaxClasses], s_lp_desc[kMaxClasses], s_ex[kMaxClasses];
  __shared__ int s_by_lp[kMaxClasses];
  __shared__ int s_path[kMaxWidth];
  __shared__ double s_norm;
  const int n = blockIdx.x, lane = threadIdx.x;
  const int nlab = C - 1;
  const int len = min(max(input_len[n], 0), T);
  Decoder D;
  if (lane == 0) {
    D.nd = arena + (size_t)n * node_cap;
    D.heap = s_heap;
    D.br = s_br;
    D.width = beam_width;
    D.nlab = nlab;
    D.cap = (int)node_cap;
    D.init();
  }
  for (int t = 0; t < len; ++t) {
    const float* row = logits + ((size_t)t * N + n) * C;
    float x[2];
    double mx = neg_inf();
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int c = lane + 32 * j;
      x[j] = c < C ? row[c] : __int_as_float(0x7fc00000);
      if (x[j] == x[j]) mx = fmax(mx, (double)x[j]);    // a NaN logit counts as -inf
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int c = lane + 32 * j;
      if (c < C) s_ex[c] = x[j] == x[j] ? exp((double)x[j] - mx) : 0.0;
    }
    __syncwarp();
    if (lane == 0) {
      double se = 0.0;
      for (int c = 0; c < C; ++c) se += s_ex[c];                 // sequential, in class order
      s_norm = mx + log(se);
    }
    __syncwarp();
    const double norm = s_norm;
    double lpv[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int c = lane + 32 * j;
      lpv[j] = (x[j] == x[j] && norm == norm) ? (double)x[j] - norm : neg_inf();   // a NaN normaliser: nothing survives the frame
      if (c < C) s_lp[c] = lpv[j];
    }
    __syncwarp();
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int c = lane + 32 * j;
      if (c < nlab) {
        int r = 0;
        for (int i = 0; i < nlab; ++i) r += (s_lp[i] > lpv[j]) || (s_lp[i] == lpv[j] && i < c);
        s_lp_desc[r] = lpv[j];
        s_by_lp[r] = c;
      }
    }
    __syncwarp();
    if (lane == 0) D.step(s_lp, s_lp_desc, s_by_lp);
    __syncwarp();
  }
  __syncwarp();                                                   // lane 0's init when len == 0
  const int hsize = __shfl_sync(0xffffffffu, lane == 0 ? D.hsize : 0, 0);
  const size_t row = (size_t)n * top_paths;
  finish_paths(arena + (size_t)n * node_cap, s_heap, hsize, s_br, s_path, T, top_paths, merge_repeated, strip, out + row * T,
               out_len + row, score ? score + row : nullptr, negate, num_paths ? num_paths + n : nullptr);
}

int beam_check_shape(int T, int N, int C, int beam_width, size_t* node_cap) {
  if (T <= 0 || N <= 0) return crnn_fail(CRNN_INVALID_VALUE, "beam_search_device: bad shape");
  if (C < 2 || C > kMaxClasses) return crnn_fail(CRNN_UNSUPPORTED, "beam_search_device: C must lie in [2, %d]", kMaxClasses);
  if (beam_width < 1 || beam_width > kMaxWidth)
    return crnn_fail(CRNN_UNSUPPORTED, "beam_search_device: beam_width must lie in [1, %d]", kMaxWidth);
  *node_cap = beam_node_cap(T, C, beam_width);
  if (*node_cap == 0 || *node_cap > SIZE_MAX / sizeof(Node) / (size_t)N)
    return crnn_fail(CRNN_UNSUPPORTED, "beam_search_device: T too large for the workspace");
  return CRNN_OK;
}

}  // namespace

extern "C" int crnn_ctc_beam_workspace_size(int T, int N, int C, int beam_width, size_t* bytes) {
  if (!bytes) return crnn_fail(CRNN_INVALID_VALUE, "beam_workspace_size: null pointer");
  size_t cap = 0;
  const int st = beam_check_shape(T, N, C, beam_width, &cap);
  if (st != CRNN_OK) return st;
  *bytes = (size_t)N * cap * sizeof(Node);
  return CRNN_OK;
}

namespace {

// both device entry points: the argument checks and the launch
int beam_search_device(const float* logits, const int* input_len, int T, int N, int C, int beam_width, int top_paths,
                       int merge_repeated, int strip, int* out, int* out_len, float* score, int negate, int* num_paths,
                       void* workspace, size_t workspace_bytes, crnn_stream_t stream) {
  if (!logits || !input_len || !out || !out_len) return crnn_fail(CRNN_INVALID_VALUE, "beam_search_device: null pointer");
  size_t cap = 0;
  const int st = beam_check_shape(T, N, C, beam_width, &cap);
  if (st != CRNN_OK) return st;
  if (top_paths < 1 || top_paths > beam_width)
    return crnn_fail(CRNN_INVALID_VALUE, "beam_search_device: top_paths %d outside [1, beam_width = %d]", top_paths, beam_width);
  if (workspace_bytes < (size_t)N * cap * sizeof(Node))
    return crnn_fail(CRNN_WORKSPACE_TOO_SMALL, "beam_search_device: workspace %zu bytes, needs %zu", workspace_bytes,
                     (size_t)N * cap * sizeof(Node));
  if (!workspace || reinterpret_cast<uintptr_t>(workspace) % 16 != 0)
    return crnn_fail(CRNN_INVALID_VALUE, "beam_search_device: workspace must be a 16-byte aligned device pointer");
  ctc_beam_kernel<<<N, kThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      logits, input_len, T, N, C, beam_width, top_paths, merge_repeated ? 1 : 0, strip, out, out_len, score, negate, num_paths,
      reinterpret_cast<Node*>(workspace), cap);
  CUDA_TRY(cudaGetLastError());
  return CRNN_OK;
}

}  // namespace

extern "C" int crnn_ctc_beam_search_device(const float* logits, const int* input_len, int T, int N, int C, int beam_width,
                                           int merge_repeated, int strip, int* out, int* out_len, float* neg_log_prob,
                                           void* workspace, size_t workspace_bytes, crnn_stream_t stream) {
  return beam_search_device(logits, input_len, T, N, C, beam_width, 1, merge_repeated, strip, out, out_len, neg_log_prob, 1, nullptr,
                            workspace, workspace_bytes, stream);
}

extern "C" int crnn_ctc_beam_search_topk_device(const float* logits, const int* input_len, int T, int N, int C, int beam_width,
                                                int top_paths, int merge_repeated, int strip, int* out, int* out_len, float* log_prob,
                                                int* num_paths, void* workspace, size_t workspace_bytes, crnn_stream_t stream) {
  return beam_search_device(logits, input_len, T, N, C, beam_width, top_paths, merge_repeated, strip, out, out_len, log_prob, 0,
                            num_paths, workspace, workspace_bytes, stream);
}
