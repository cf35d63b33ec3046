// Subgraph matching kernel (subgraph_matching.py, Kriege & Mutzel 2012), one warp per graph pair.
//
// For graphs x, y the weighted product graph has a vertex p = (a, b) for every a in x, b in y with cv = kv(La, Lb) != 0,
// and between p and q (p.a != q.a, p.b != q.b; h the one with the larger x vertex, l the other) the weight
//   ce = -1                      neither x-edge h.a -> l.a nor y-edge h.b -> l.b exists (a d-edge)
//   ce = 0                       exactly one of them exists (or p, q share a vertex)
//   ce = ke(Lex, Ley), 1 if None both exist (a c-edge when ce > 0)
// tv[s - 1] sums, over the vertex sets S of size s that are cliques of ce != 0 and connected by the ce > 0 edges,
// prod cv * prod_{pairs} |ce|; K = sum_s lambda_s tv_s, folded as one fma chain from 0 in size order.
//
// The product graph is never built: ce is read from per-graph out-edge bitsets and edge-label matrices, cv from the
// label ids and the weight tables.  The warp's lanes take the product vertices v = (a, b) (id a n_y + b) as roots, and
// each enumerates the sets whose smallest id is v depth first, ESU style: the extension set of S holds the vertices
// adjacent (ce != 0) to all of S; taking w from it, the child's extension set is what remains of it after w, kept
// where ce(., w) != 0, plus the c-neighbours u > v of w with ce(u, s) < 0 for every s in S (u is adjacent to S but
// not yet its c-neighbour).  Every connected clique is reached exactly once (ESU's argument: cliques are closed under
// subsets, so dropping non-adjacent candidates only removes branches whose sets are not cliques).  The extension
// sets of one lane live as a stack of segments in a global workspace, interleaved by lane.
//
// Integer-valued weights are summed exactly in 64-bit integers; a term or per-size sum of absolute terms reaching
// 2^53 (where the reference's fp64 sums stop being exact) sets bit 1 of `err`.  Real weights are summed in fp64 per
// lane, then over the warp in a fixed shuffle order, so runs repeat bit for bit.
#pragma once
#include "common.cuh"
#include "random_walk.cuh"

namespace gk {

constexpr int SM_THREADS = 256;
constexpr int SM_WARPS = SM_THREADS / 32;
constexpr int SM_KMAX = 32;            // largest clique size enumerated
constexpr int SM_TAB_MAX = 4096;       // entries of one weight table (64 x 64 labels)
constexpr int SM_WL_BINS = 64;         // sm_wl_pairs: (n_iter + 1) x sizes enumerated, at most
constexpr int SM_HC_BINS = 64;         // sm_mask_pairs: n_iter x sizes enumerated, at most
enum { SM_W_TABLE = 0, SM_W_NONE = 1, SM_W_DIRAC = 2 };

// Per-graph record (32-bit words) of n vertices, W = ceil(n / 32):
//   out[n][W] out-edge bitsets | und[n][W] out- or in-edge bitsets | lab[n] vertex label ids | el[n][n] edge label ids
// (the last only with edge labels).  Self-loops are left out.
__host__ __device__ __forceinline__ long long sm_record_words(int n, bool elab) {
  const long long W = (n + 31) / 32;
  return 2 * n * W + n + (elab ? (long long)n * n : 0);
}

struct SmParams {
  const int* graph_ptr;
  const long long* rec_off;  // word offset of each graph's record
  const unsigned* rec;
  const double* vtab; int n_vl;  // kv table [n_vl][n_vl] (SM_W_TABLE)
  const double* etab; int n_el;  // ke table [n_el][n_el] (SM_W_TABLE)
  int kv, ke;
  int kk;       // sizes enumerated: max(k, 1), at most SM_KMAX
  int n_tv;     // k + 1 entries of tv and of the lambdas
  const double* lam;
  int exact;    // integer-valued tables: exact 64-bit sums
  int pairs, ordered;
  long long n_pairs;
  int row_g0, rows, cols;
  double* out; long long ld;  // K rows of the request (RECT / TRIANGLE) or per-graph diagonal (DIAG)
  double* tv_out;             // or nullptr: tv of pair pi at tv_out[pi * n_tv]
  unsigned* stack; long long stack_cap;  // extension-set stack: stack_cap entries per lane
  int stage_words;            // shared-memory words per warp for the two records (0: read them from global memory)
  unsigned long long* next;   // pair counter
  unsigned* err;              // bit 1: exact sum reached 2^53, bit 2: stack overflow
  // sm_wl_pairs / sm_mask_pairs only: n_lv (WL levels 0 .. n_iter, HadamardCode levels 0 .. n_iter - 1) class ids
  // per packed vertex, vertex-major; tv_out then holds n_lv x n_tv values per pair
  const int* wl_cls; int n_lv;
};

struct SmGraph {
  const unsigned *out, *und;
  const int *lab, *el;
  int n, W;
};

__device__ __forceinline__ SmGraph sm_graph(const unsigned* r, int n, bool elab) {
  SmGraph g;
  g.n = n; g.W = (n + 31) >> 5;
  g.out = r;
  g.und = r + (size_t)n * g.W;
  g.lab = reinterpret_cast<const int*>(r + 2 * (size_t)n * g.W);
  g.el = elab ? g.lab + n : nullptr;
  return g;
}

__device__ __forceinline__ bool sm_bit(const unsigned* bits, int W, int u, int v) {
  return (bits[u * W + (v >> 5)] >> (v & 31)) & 1u;
}

__device__ __forceinline__ double sm_cv(const SmParams& P, const SmGraph& X, const SmGraph& Y, const double* vtab,
                                        int a, int b) {
  if (P.kv == SM_W_NONE) return 1.0;
  const int la = X.lab[a], lb = Y.lab[b];
  if (P.kv == SM_W_DIRAC) return la == lb ? 1.0 : 0.0;
  return vtab[la * P.n_vl + lb];
}

__device__ __forceinline__ double sm_ce(const SmParams& P, const SmGraph& X, const SmGraph& Y, const double* etab,
                                        int pa, int pb, int qa, int qb) {
  if (pa == qa || pb == qb) return 0.0;
  if (pa < qa) { int t = pa; pa = qa; qa = t; t = pb; pb = qb; qb = t; }  // the edge runs from the larger x vertex
  const bool ex = sm_bit(X.out, X.W, pa, qa), ey = sm_bit(Y.out, Y.W, pb, qb);
  if (!ex && !ey) return -1.0;
  if (ex != ey) return 0.0;
  if (P.ke == SM_W_NONE) return 1.0;
  const int la = X.el[pa * X.n + qa], lb = Y.el[pb * Y.n + qb];
  if (P.ke == SM_W_DIRAC) return la == lb ? 1.0 : 0.0;
  return etab[la * P.n_el + lb];
}

// One lane's per-size sums of sm_pairs: exact sums in cnt / cabs, real sums in sum
struct SmLaneAcc {
  static constexpr bool wl = false;
  static constexpr bool masked = false;
  long long* cnt;
  unsigned long long* cabs;
  double* sum;
  __device__ __forceinline__ void add(const SmParams& P, int s, double t) const {
    if (P.exact) {
      const double at = fabs(t);
      if (at >= 0x1p53) atomicOr(P.err, 1u);
      cnt[s] += (long long)t;
      cabs[s] += (unsigned long long)at;
    } else {
      sum[s] += t;
    }
  }
};

// The (depth, size) bins of sm_wl_pairs.  A product vertex (a, b) has depth D(a, b), the largest WL level h with
// c_h(a) == c_h(b) (WL refines its partition, so the levels 0 .. D all agree); a clique counts at the levels 0 .. the
// least depth of its vertices.  Exact sums go to the warp's bins in shared memory ([depth][size] signed sums, then
// [depth][size] absolute sums, 64-bit shared atomics: integer addition, so the order does not matter); real sums go to
// the lane's own bins ([level][size], stride SM_THREADS), added at every level 0 .. depth in the enumeration order, so
// each level's lane sum is the one the per-level enumeration forms.
struct SmWlAcc {
  static constexpr bool wl = true;
  static constexpr bool masked = false;
  const int *cx, *cy;         // n_lv class ids per vertex of x and of y
  int n_lv, kk;
  bool all_levels;            // kv = None: every product vertex exists at every level
  unsigned long long* wbin;   // exact: this warp's bins
  double* lbin;               // real: this lane's bins
  __device__ __forceinline__ int depth(int a, int b) const {
    if (all_levels) return n_lv - 1;
    const int* p = cx + (size_t)a * n_lv;
    const int* q = cy + (size_t)b * n_lv;
    int d = 0;
    while (d + 1 < n_lv && p[d + 1] == q[d + 1]) ++d;
    return d;
  }
  __device__ __forceinline__ void add(const SmParams& P, int s, double t, int d) const {
    if (P.exact) {
      const double at = fabs(t);
      if (at >= 0x1p53) atomicOr(P.err, 1u);
      atomicAdd(&wbin[d * kk + s], (unsigned long long)(long long)t);
      atomicAdd(&wbin[(n_lv + d) * kk + s], (unsigned long long)at);
    } else {
      for (int h = 0; h <= d; ++h) lbin[(size_t)(h * kk + s) * SM_THREADS] += t;
    }
  }
};

// The (level, size) bins of sm_mask_pairs.  A product vertex (a, b) has the level mask M(a, b), bit h set when
// c_h(a) == c_h(b): HadamardCode's levels do not refine each other, so the levels of a vertex need not be a prefix.
// The union product graph has the vertices with M != 0 (kv = None: every vertex, every mask full), and a clique counts
// at exactly the levels of the AND of its vertices' masks.  Exact sums go to the warp's bins in shared memory
// ([level][size] signed sums, then [level][size] absolute sums, 64-bit shared atomics); real sums go to the lane's own
// bins ([level][size], stride SM_THREADS), added at every level of the mask in the enumeration order.
struct SmMaskAcc {
  static constexpr bool wl = false;
  static constexpr bool masked = true;
  const int *cx, *cy;         // n_lv class ids per vertex of x and of y
  int n_lv, kk;
  bool all_levels;            // kv = None
  unsigned long long* wbin;   // exact: this warp's bins
  double* lbin;               // real: this lane's bins
  __device__ __forceinline__ unsigned long long level_mask(int a, int b) const {
    if (all_levels) return n_lv >= 64 ? ~0ull : (1ull << n_lv) - 1;
    const int* p = cx + (size_t)a * n_lv;
    const int* q = cy + (size_t)b * n_lv;
    unsigned long long m = 0;
    for (int h = 0; h < n_lv; ++h) m |= (unsigned long long)(p[h] == q[h]) << h;
    return m;
  }
  __device__ __forceinline__ void add(const SmParams& P, int s, double t, unsigned long long m) const {
    if (P.exact) {
      const double at = fabs(t);
      if (at >= 0x1p53) atomicOr(P.err, 1u);
      for (; m; m &= m - 1) {
        const int h = __ffsll((long long)m) - 1;
        atomicAdd(&wbin[h * kk + s], (unsigned long long)(long long)t);
        atomicAdd(&wbin[(n_lv + h) * kk + s], (unsigned long long)at);
      }
    } else {
      for (; m; m &= m - 1) lbin[(size_t)((__ffsll((long long)m) - 1) * kk + s) * SM_THREADS] += t;
    }
  }
};

// cv of a product vertex; under sm_mask_pairs 1 on the union product graph (kv = _dirac at some level, or kv = None)
template <class Acc>
__device__ __forceinline__ double sm_acc_cv(const Acc& acc, const SmParams& P, const SmGraph& X, const SmGraph& Y,
                                            const double* vtab, int a, int b) {
  if constexpr (Acc::masked) return acc.level_mask(a, b) ? 1.0 : 0.0;
  else return sm_cv(P, X, Y, vtab, a, b);
}

// tv of the pair (x, y) for this lane's roots, into `acc`
template <class Acc>
__device__ void sm_lane_pair(const SmParams& P, const SmGraph& X, const SmGraph& Y, const double* vtab,
                             const double* etab, unsigned* stk, const Acc& acc) {
  const int lane = threadIdx.x & 31;
  const int ny = Y.n, nv = X.n * Y.n, kk = P.kk;
  const long long cap = P.stack_cap;
  int Sa[SM_KMAX], Sb[SM_KMAX];
  double term[SM_KMAX];
  long long f_start[SM_KMAX + 1];
  int f_len[SM_KMAX + 1], f_pos[SM_KMAX + 1];
  unsigned char md[Acc::wl ? SM_KMAX : 1];  // least depth of S's first i + 1 vertices (sm_wl_pairs)
  unsigned long long mk[Acc::masked ? SM_KMAX : 1];  // AND of the level masks of S's first i + 1 vertices
  auto push = [&](long long& top, unsigned u) {
    if (top >= cap) { atomicOr(P.err, 2u); return; }
    stk[(size_t)top * 32] = u;
    ++top;
  };
  for (int v = lane; v < nv; v += 32) {
    const int va = v / ny, vb = v - va * ny;
    double c0;
    if constexpr (Acc::masked) {
      mk[0] = acc.level_mask(va, vb);
      c0 = mk[0] ? 1.0 : 0.0;
    } else {
      c0 = sm_cv(P, X, Y, vtab, va, vb);
    }
    if (c0 == 0.0) continue;
    if constexpr (Acc::masked) {
      acc.add(P, 0, c0, mk[0]);
    } else if constexpr (Acc::wl) {
      md[0] = (unsigned char)acc.depth(va, vb);
      acc.add(P, 0, c0, md[0]);
    } else {
      acc.add(P, 0, c0);
    }
    if (kk < 2) continue;
    Sa[0] = va; Sb[0] = vb; term[0] = c0;
    // extension set of {v}: its c-neighbours with a larger id
    long long top = 0;
    for (int wa = 0; wa < X.W; ++wa) {
      for (unsigned ma = X.und[va * X.W + wa]; ma; ma &= ma - 1) {
        const int a = wa * 32 + __ffs(ma) - 1;
        for (int wb = 0; wb < Y.W; ++wb) {
          for (unsigned mb = Y.und[vb * Y.W + wb]; mb; mb &= mb - 1) {
            const int b = wb * 32 + __ffs(mb) - 1;
            const int u = a * ny + b;
            if (u <= v || sm_acc_cv(acc, P, X, Y, vtab, a, b) == 0.0) continue;
            if (sm_ce(P, X, Y, etab, va, vb, a, b) > 0.0) push(top, (unsigned)u);
          }
        }
      }
    }
    int depth = 1;  // |S|
    f_start[1] = 0; f_len[1] = (int)top; f_pos[1] = 0;
    while (depth >= 1) {
      if (f_pos[depth] == f_len[depth]) {
        top = f_start[depth];
        --depth;
        continue;
      }
      const long long fs = f_start[depth];
      const int fl = f_len[depth];
      const unsigned w = stk[(size_t)(fs + f_pos[depth]++) * 32];
      const int wa = (int)(w / (unsigned)ny), wb = (int)(w - (unsigned)wa * ny);
      unsigned long long mw = 0;
      if constexpr (Acc::masked) {
        mw = mk[depth - 1] & acc.level_mask(wa, wb);
        if (mw == 0) continue;  // no level has S + w, nor any set of its subtree
      }
      double t = term[depth - 1];
      if constexpr (!Acc::masked) t *= sm_cv(P, X, Y, vtab, wa, wb);
      for (int i = 0; i < depth; ++i) t *= fabs(sm_ce(P, X, Y, etab, wa, wb, Sa[i], Sb[i]));
      if constexpr (Acc::masked) {
        acc.add(P, depth, t, mw);
        mk[depth] = mw;
      } else if constexpr (Acc::wl) {
        const int dw = min((int)md[depth - 1], acc.depth(wa, wb));
        acc.add(P, depth, t, dw);
        md[depth] = (unsigned char)dw;
      } else {
        acc.add(P, depth, t);
      }
      if (depth + 1 >= kk) continue;
      // the child's extension set, above this frame
      top = fs + fl;
      const long long cs = top;
      for (int j = f_pos[depth]; j < fl; ++j) {
        const unsigned x = stk[(size_t)(fs + j) * 32];
        const int xa = (int)(x / (unsigned)ny), xb = (int)(x - (unsigned)xa * ny);
        if (sm_ce(P, X, Y, etab, xa, xb, wa, wb) != 0.0) push(top, x);
      }
      for (int ka = 0; ka < X.W; ++ka) {
        for (unsigned ma = X.und[wa * X.W + ka]; ma; ma &= ma - 1) {
          const int a = ka * 32 + __ffs(ma) - 1;
          for (int kb = 0; kb < Y.W; ++kb) {
            for (unsigned mb = Y.und[wb * Y.W + kb]; mb; mb &= mb - 1) {
              const int b = kb * 32 + __ffs(mb) - 1;
              const int u = a * ny + b;
              if (u <= v || sm_acc_cv(acc, P, X, Y, vtab, a, b) == 0.0) continue;
              if (!(sm_ce(P, X, Y, etab, wa, wb, a, b) > 0.0)) continue;
              bool ok = true;
              for (int i = 0; i < depth && ok; ++i) ok = sm_ce(P, X, Y, etab, a, b, Sa[i], Sb[i]) < 0.0;
              if (ok) push(top, (unsigned)u);
            }
          }
        }
      }
      Sa[depth] = wa; Sb[depth] = wb; term[depth] = t;
      ++depth;
      f_start[depth] = cs; f_len[depth] = (int)(top - cs); f_pos[depth] = 0;
    }
  }
}

// Persistent grid, one warp per pair taken from P.next.  Dynamic shared memory: the weight tables, then
// SM_WARPS x stage_words words for the two records of each warp's pair.
// One CTA per SM is the occupancy floor the compiler plans for: it then keeps the search state of sm_lane_pair in
// 80 registers without spills (with the default bound it spills to stay at 64).
__global__ void __launch_bounds__(SM_THREADS, 1) sm_pairs(SmParams P) {
  extern __shared__ __align__(16) unsigned char sm_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool elab = P.ke != SM_W_NONE;
  double* vtab = reinterpret_cast<double*>(sm_smem);
  const int nvt = P.kv == SM_W_TABLE ? P.n_vl * P.n_vl : 0;
  const int net = P.ke == SM_W_TABLE ? P.n_el * P.n_el : 0;
  double* etab = vtab + nvt;
  for (int i = threadIdx.x; i < nvt; i += SM_THREADS) vtab[i] = P.vtab[i];
  for (int i = threadIdx.x; i < net; i += SM_THREADS) etab[i] = P.etab[i];
  __syncthreads();
  unsigned* stage = reinterpret_cast<unsigned*>(etab + net) + (size_t)warp * P.stage_words;
  const size_t gwarp = (size_t)blockIdx.x * SM_WARPS + warp;
  unsigned* stk = P.stack + gwarp * 32 * (size_t)P.stack_cap + lane;
  long long cnt[SM_KMAX];
  unsigned long long cabs[SM_KMAX];
  double sum[SM_KMAX];
  for (;;) {
    long long pi = 0;
    if (lane == 0) pi = (long long)atomicAdd(P.next, 1ull);
    pi = __shfl_sync(0xffffffffu, pi, 0);
    if (pi >= P.n_pairs) break;
    int r, c, gi, gj;
    rw_pair_of(P.pairs, P.cols, P.row_g0, P.ordered, pi, r, c, gi, gj);
    const int nx = P.graph_ptr[gi + 1] - P.graph_ptr[gi], ny = P.graph_ptr[gj + 1] - P.graph_ptr[gj];
    const long long rx = sm_record_words(nx, elab), ry = sm_record_words(ny, elab);
    const unsigned* ax = P.rec + P.rec_off[gi];
    const unsigned* ay = P.rec + P.rec_off[gj];
    if (rx + ry <= P.stage_words) {
      for (long long i = lane; i < rx; i += 32) stage[i] = ax[i];
      for (long long i = lane; i < ry; i += 32) stage[rx + i] = ay[i];
      __syncwarp();
      ax = stage; ay = stage + rx;
    }
    const SmGraph X = sm_graph(ax, nx, elab), Y = sm_graph(ay, ny, elab);
    for (int s = 0; s < P.kk; ++s) { cnt[s] = 0; cabs[s] = 0; sum[s] = 0.0; }
    sm_lane_pair(P, X, Y, vtab, etab, stk, SmLaneAcc{cnt, cabs, sum});
    // tv over the warp (fixed shuffle order), then the lambda fold on lane 0
    double acc = 0.0;
    for (int s = 0; s < P.n_tv; ++s) {
      double tv = 0.0;
      if (s < P.kk) {
        if (P.exact) {
          long long a = cnt[s];
          unsigned long long b = cabs[s];
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            a += __shfl_xor_sync(0xffffffffu, a, o);
            b += __shfl_xor_sync(0xffffffffu, b, o);
          }
          if (lane == 0 && b >= (1ull << 53)) atomicOr(P.err, 1u);
          tv = (double)a;
        } else {
          tv = rw_warp_sum(sum[s]);
        }
      }
      acc = __fma_rn(P.lam[s], tv, acc);
      if (lane == 0 && P.tv_out) P.tv_out[(size_t)pi * P.n_tv + s] = tv;
    }
    if (lane == 0 && P.out) {
      if (P.pairs == RW_PAIRS_DIAG) {
        P.out[r] = acc;
      } else {
        P.out[(size_t)r * P.ld + c] = acc;
        if (P.pairs == RW_PAIRS_TRIANGLE && c != r) P.out[(size_t)c * P.ld + r] = acc;
      }
    }
    __syncwarp();  // the next pair overwrites the staged records
  }
}

// WeisfeilerLehman over SubgraphMatching in one enumeration (DESIGN 4.23).  With kv = _dirac the level-h product graph
// is the level-0 one induced on the vertices of depth >= h, and ESU's extension sets at level h are the level-0 ones
// restricted to them, in the same order; so a clique's term is the same at every level that has it, and every
// level's lane sums see the terms in the order the per-level enumeration does.  Per pair: the (depth, size) bins,
// then in the epilogue each level's tv (suffix sums over the depths), its fma lambda fold, and the level sum
// ((K_0 + K_1) + K_2) ... -- no per-level matrix exists.  Dynamic shared memory: the weight tables, the bins
// (exact: SM_WARPS x 2 n_lv kk words, real: SM_THREADS x n_lv kk doubles), then the staged records as in sm_pairs.
__global__ void __launch_bounds__(SM_THREADS, 1) sm_wl_pairs(SmParams P) {
  extern __shared__ __align__(16) unsigned char sm_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool elab = P.ke != SM_W_NONE;
  double* vtab = reinterpret_cast<double*>(sm_smem);
  const int nvt = P.kv == SM_W_TABLE ? P.n_vl * P.n_vl : 0;
  const int net = P.ke == SM_W_TABLE ? P.n_el * P.n_el : 0;
  double* etab = vtab + nvt;
  for (int i = threadIdx.x; i < nvt; i += SM_THREADS) vtab[i] = P.vtab[i];
  for (int i = threadIdx.x; i < net; i += SM_THREADS) etab[i] = P.etab[i];
  const int n_lv = P.n_lv, kk = P.kk, nb = n_lv * kk;
  unsigned long long* bins = reinterpret_cast<unsigned long long*>(etab + net);
  const int bin_words = P.exact ? SM_WARPS * 2 * nb : SM_THREADS * nb;
  for (int i = threadIdx.x; i < bin_words; i += SM_THREADS) bins[i] = 0ull;
  __syncthreads();
  unsigned long long* wbin = bins + (size_t)warp * 2 * nb;
  double* lbin = reinterpret_cast<double*>(bins) + threadIdx.x;
  unsigned* stage = reinterpret_cast<unsigned*>(bins + bin_words) + (size_t)warp * P.stage_words;
  const size_t gwarp = (size_t)blockIdx.x * SM_WARPS + warp;
  unsigned* stk = P.stack + gwarp * 32 * (size_t)P.stack_cap + lane;
  for (;;) {
    long long pi = 0;
    if (lane == 0) pi = (long long)atomicAdd(P.next, 1ull);
    pi = __shfl_sync(0xffffffffu, pi, 0);
    if (pi >= P.n_pairs) break;
    int r, c, gi, gj;
    rw_pair_of(P.pairs, P.cols, P.row_g0, P.ordered, pi, r, c, gi, gj);
    const int x0 = P.graph_ptr[gi], y0 = P.graph_ptr[gj];
    const int nx = P.graph_ptr[gi + 1] - x0, ny = P.graph_ptr[gj + 1] - y0;
    const long long rx = sm_record_words(nx, elab), ry = sm_record_words(ny, elab);
    const unsigned* ax = P.rec + P.rec_off[gi];
    const unsigned* ay = P.rec + P.rec_off[gj];
    if (rx + ry <= P.stage_words) {
      for (long long i = lane; i < rx; i += 32) stage[i] = ax[i];
      for (long long i = lane; i < ry; i += 32) stage[rx + i] = ay[i];
      __syncwarp();
      ax = stage; ay = stage + rx;
    }
    const SmGraph X = sm_graph(ax, nx, elab), Y = sm_graph(ay, ny, elab);
    const SmWlAcc acc{P.wl_cls + (size_t)x0 * n_lv, P.wl_cls + (size_t)y0 * n_lv, n_lv, kk, P.kv == SM_W_NONE,
                      wbin, lbin};
    sm_lane_pair(P, X, Y, vtab, etab, stk, acc);
    __syncwarp();
    // level h's tv[s] sums the bins of depth >= h; K = ((K_0 + K_1) + K_2) ..., K_h the fma fold of lambdas x tv_h
    double total = 0.0;
    for (int h = 0; h < n_lv; ++h) {
      double kh = 0.0;
      for (int s = 0; s < P.n_tv; ++s) {
        double tv = 0.0;
        if (s < kk) {
          if (P.exact) {
            long long a = 0;
            unsigned long long b = 0;
            for (int d = h; d < n_lv; ++d) {
              a += (long long)wbin[d * kk + s];
              b += wbin[(n_lv + d) * kk + s];
            }
            if (lane == 0 && b >= (1ull << 53)) atomicOr(P.err, 1u);
            tv = (double)a;
          } else {
            tv = rw_warp_sum(lbin[(size_t)(h * kk + s) * SM_THREADS]);
          }
        }
        kh = __fma_rn(P.lam[s], tv, kh);
        if (lane == 0 && P.tv_out) P.tv_out[((size_t)pi * n_lv + h) * P.n_tv + s] = tv;
      }
      total = h == 0 ? kh : total + kh;
    }
    if (lane == 0 && P.out) {
      if (P.pairs == RW_PAIRS_DIAG) {
        P.out[r] = total;
      } else {
        P.out[(size_t)r * P.ld + c] = total;
        if (P.pairs == RW_PAIRS_TRIANGLE && c != r) P.out[(size_t)c * P.ld + r] = total;
      }
    }
    __syncwarp();  // every lane has read the bins; the next pair overwrites them and the staged records
    if (P.exact) {
      for (int i = lane; i < 2 * nb; i += 32) wbin[i] = 0ull;
    } else {
      for (int i = 0; i < nb; ++i) lbin[(size_t)i * SM_THREADS] = 0.0;
    }
    __syncwarp();
  }
}

// HadamardCode over SubgraphMatching in one enumeration (DESIGN 4.24).  With kv = _dirac the level-h product graph is
// the union product graph (the vertices whose classes agree at some level) induced on the vertices whose classes
// agree at h.  ESU's extension sets over any vertex subset are the union's restricted to it, in the same order (a
// child's set is the rest of its parent's, filtered by ce with the new vertex, plus candidates tested against S and
// the new vertex only), so every level's lane sums see that level's terms in its own enumeration order.  Per pair:
// the (level, size) bins, then each level's fma lambda fold and the level sum ((K_0 + K_1) + K_2) ...  Dynamic shared
// memory as in sm_wl_pairs.
__global__ void __launch_bounds__(SM_THREADS, 1) sm_mask_pairs(SmParams P) {
  extern __shared__ __align__(16) unsigned char sm_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool elab = P.ke != SM_W_NONE;
  double* etab = reinterpret_cast<double*>(sm_smem);
  const int net = P.ke == SM_W_TABLE ? P.n_el * P.n_el : 0;
  for (int i = threadIdx.x; i < net; i += SM_THREADS) etab[i] = P.etab[i];
  const int n_lv = P.n_lv, kk = P.kk, nb = n_lv * kk;
  unsigned long long* bins = reinterpret_cast<unsigned long long*>(etab + net);
  const int bin_words = P.exact ? SM_WARPS * 2 * nb : SM_THREADS * nb;
  for (int i = threadIdx.x; i < bin_words; i += SM_THREADS) bins[i] = 0ull;
  __syncthreads();
  unsigned long long* wbin = bins + (size_t)warp * 2 * nb;
  double* lbin = reinterpret_cast<double*>(bins) + threadIdx.x;
  unsigned* stage = reinterpret_cast<unsigned*>(bins + bin_words) + (size_t)warp * P.stage_words;
  const size_t gwarp = (size_t)blockIdx.x * SM_WARPS + warp;
  unsigned* stk = P.stack + gwarp * 32 * (size_t)P.stack_cap + lane;
  for (;;) {
    long long pi = 0;
    if (lane == 0) pi = (long long)atomicAdd(P.next, 1ull);
    pi = __shfl_sync(0xffffffffu, pi, 0);
    if (pi >= P.n_pairs) break;
    int r, c, gi, gj;
    rw_pair_of(P.pairs, P.cols, P.row_g0, P.ordered, pi, r, c, gi, gj);
    const int x0 = P.graph_ptr[gi], y0 = P.graph_ptr[gj];
    const int nx = P.graph_ptr[gi + 1] - x0, ny = P.graph_ptr[gj + 1] - y0;
    const long long rx = sm_record_words(nx, elab), ry = sm_record_words(ny, elab);
    const unsigned* ax = P.rec + P.rec_off[gi];
    const unsigned* ay = P.rec + P.rec_off[gj];
    if (rx + ry <= P.stage_words) {
      for (long long i = lane; i < rx; i += 32) stage[i] = ax[i];
      for (long long i = lane; i < ry; i += 32) stage[rx + i] = ay[i];
      __syncwarp();
      ax = stage; ay = stage + rx;
    }
    const SmGraph X = sm_graph(ax, nx, elab), Y = sm_graph(ay, ny, elab);
    const SmMaskAcc acc{P.wl_cls + (size_t)x0 * n_lv, P.wl_cls + (size_t)y0 * n_lv, n_lv, kk, P.kv == SM_W_NONE,
                        wbin, lbin};
    sm_lane_pair(P, X, Y, etab, etab, stk, acc);
    __syncwarp();
    // K = ((K_0 + K_1) + K_2) ..., K_h the fma fold of lambdas x the level's own bins
    double total = 0.0;
    for (int h = 0; h < n_lv; ++h) {
      double kh = 0.0;
      for (int s = 0; s < P.n_tv; ++s) {
        double tv = 0.0;
        if (s < kk) {
          if (P.exact) {
            if (lane == 0 && wbin[(n_lv + h) * kk + s] >= (1ull << 53)) atomicOr(P.err, 1u);
            tv = (double)(long long)wbin[h * kk + s];
          } else {
            tv = rw_warp_sum(lbin[(size_t)(h * kk + s) * SM_THREADS]);
          }
        }
        kh = __fma_rn(P.lam[s], tv, kh);
        if (lane == 0 && P.tv_out) P.tv_out[((size_t)pi * n_lv + h) * P.n_tv + s] = tv;
      }
      total = h == 0 ? kh : total + kh;
    }
    if (lane == 0 && P.out) {
      if (P.pairs == RW_PAIRS_DIAG) {
        P.out[r] = total;
      } else {
        P.out[(size_t)r * P.ld + c] = total;
        if (P.pairs == RW_PAIRS_TRIANGLE && c != r) P.out[(size_t)c * P.ld + r] = total;
      }
    }
    __syncwarp();  // every lane has read the bins; the next pair overwrites them and the staged records
    if (P.exact) {
      for (int i = lane; i < 2 * nb; i += 32) wbin[i] = 0ull;
    } else {
      for (int i = 0; i < nb; ++i) lbin[(size_t)i * SM_THREADS] = 0.0;
    }
    __syncwarp();
  }
}

// Records of every packed graph from the packed CSR (one CTA per graph): bitsets, label ids, edge label ids; and
// the largest number of distinct out- or in-neighbours of a vertex (atomicMax into *max_und), which bounds the
// extension sets
__global__ void sm_build_records(const int* graph_ptr, const int* row_ptr, const int* col_idx, const int* labels,
                                 const int* edge_label, const long long* rec_off, unsigned* rec, int n_graphs,
                                 int* max_und) {
  const bool elab = edge_label != nullptr;
  for (int g = blockIdx.x; g < n_graphs; g += gridDim.x) {
    const int v0 = graph_ptr[g], n = graph_ptr[g + 1] - v0, W = (n + 31) >> 5;
    unsigned* r = rec + rec_off[g];
    const long long words = sm_record_words(n, elab);
    for (long long i = threadIdx.x; i < words; i += blockDim.x) r[i] = 0u;
    __syncthreads();
    unsigned* out = r;
    unsigned* und = r + (size_t)n * W;
    int* lab = reinterpret_cast<int*>(r + 2 * (size_t)n * W);
    for (int u = threadIdx.x; u < n; u += blockDim.x) {
      lab[u] = labels ? labels[v0 + u] : 0;
      for (int e = row_ptr[v0 + u]; e < row_ptr[v0 + u + 1]; ++e) {
        const int v = col_idx[e] - v0;
        if (v == u) continue;
        atomicOr(&out[u * W + (v >> 5)], 1u << (v & 31));
        atomicOr(&und[u * W + (v >> 5)], 1u << (v & 31));
        atomicOr(&und[v * W + (u >> 5)], 1u << (u & 31));
        if (elab) lab[n + u * n + v] = edge_label[e];
      }
    }
    __syncthreads();
    for (int u = threadIdx.x; u < n; u += blockDim.x) {
      int d = 0;
      for (int w = 0; w < W; ++w) d += __popc(und[u * W + w]);
      atomicMax(max_und, d);
    }
    __syncthreads();
  }
}

}  // namespace gk
