// OddSth (odd_sth.py; Da San Martino et al. 2012): the ordered DAG decomposition of every graph and the exact
// subtree identities of its nodes, as (graph, identity) counts.
//
// Root v's DAG is the BFS from v over the out-neighbours, cut at depth h: edge u -> w when w sits at depth(u) + 1 and
// depth(u) < h.  Kahn's algorithm orders it, popping by (label rank, insertion sequence): the reference re-sorts its
// queue by label with a stable sort before every pop, which is the same priority.  A node's identity is
// str(label) + "(" + its children's identities, last popped first, + ")" (a leaf: str(label)).
//
// No identity string is built.  odd_dags gives every (root, node) pair a 64-bit hash of its identity, bottom-up inside
// the DAG (children first: they are popped after their parents), and writes the node's record: label id, its children
// as node slots in identity order.  odd_insert / odd_verify then intern the hashes into one table and check every node
// against its slot's representative node: same label id, same number of children, children pairwise in the same slot.
// Passing that check makes the hash classes the identity classes (by induction on the height: equal hashes with
// verified signatures are equal identities; equal identities hash equally).  A failed check is a collision: the host
// repeats the whole pass with another seed.
#pragma once
#include "common.cuh"

namespace gk {

constexpr int ODD_MAX_N = 4096;      // vertices per graph (one warp's DAG state lives in shared memory)
constexpr int ODD_SMEM_PER_V = 36;   // bytes of that state per vertex (see odd_dags)
constexpr int ODD_MAX_WARPS = 4;     // odd_dags: up to four warps per CTA, each walking its own roots

struct OddParams {
  int N;
  long long V;
  int n_levels;                  // label sets: one DAG pass per (level, root); 1 for OddSth itself
  long long S, T;                // node and child slots of one level (the last entries of node_base / edge_base)
  const int* graph_ptr;
  const int* row_ptr;
  const int* col_idx;
  const int* vgraph;
  const int* labels;             // [n_levels][V] label id: one per distinct str(label), disjoint across levels
  const int* rank;               // [n_levels][V] rank of the label's value among the values of its graph (ties share a rank)
  const long long* node_base;    // per graph: first node slot of its first root (sum of n^2 before it)
  const long long* edge_base;    // per graph: first child slot of its first root (sum of n m before it)
  int depth;                     // h, < 0 without a limit
  int n_pad;                     // per-warp state length: the largest graph, rounded up to 4
  int degenerate;                // tests only: hash (label, child count) alone, so that verification must fail
  unsigned long long seed;
  unsigned long long* key;       // [S] identity hash of the node in the slot
  int* lab;                      // [S] its label id, -1 for an unused slot
  int* gr;                       // [S] its graph
  int* cb;                       // [S] first child slot in ch
  int* nc;                       // [S] number of children
  int* ch;                       // [T] children as node slots, in identity order
};

__device__ __forceinline__ unsigned long long odd_mix(unsigned long long x) {
  x ^= x >> 33;
  x *= 0xff51afd7ed558ccdULL;
  x ^= x >> 33;
  x *= 0xc4ceb9fe1a85ec53ULL;
  x ^= x >> 33;
  return x;
}

__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long x) {
#pragma unroll
  for (int o = 16; o; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}

// One warp per root.  Shared state per warp, n_pad entries each: dep (BFS depth, -1 outside the DAG), indeg, pos (pop
// index), at (BFS list, then the vertex of each pop index), qv / qk (Kahn queue: vertex, (rank << 32 | sequence)),
// hs (identity hash).
__global__ void __launch_bounds__(ODD_MAX_WARPS * 32)
odd_dags(OddParams p) {
  extern __shared__ __align__(16) unsigned char odd_smem[];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpc = blockDim.x >> 5;
  const int n_pad = p.n_pad;
  unsigned char* base = odd_smem + (size_t)wib * n_pad * ODD_SMEM_PER_V;
  unsigned long long* hs = reinterpret_cast<unsigned long long*>(base);
  unsigned long long* qk = hs + n_pad;
  int* dep = reinterpret_cast<int*>(qk + n_pad);
  int* indeg = dep + n_pad;
  int* pos = indeg + n_pad;
  int* at = pos + n_pad;
  int* qv = at + n_pad;
  __shared__ int s_cnt[ODD_MAX_WARPS];
  const unsigned FULL = 0xffffffffu;

  for (long long lvv = (long long)blockIdx.x * wpc + wib; lvv < p.V * p.n_levels; lvv += (long long)gridDim.x * wpc) {
    // level-major: the nodes of level l take the slots [l S, (l + 1) S), their children [l T, (l + 1) T)
    const long long level = lvv / p.V, v = lvv - level * p.V;
    const int* labels = p.labels + level * p.V;
    const int* rank = p.rank + level * p.V;
    const int g = p.vgraph[v];
    const int g0 = p.graph_ptr[g], n = p.graph_ptr[g + 1] - g0;
    const int m = p.row_ptr[g0 + n] - p.row_ptr[g0];
    const int lv = (int)(v - g0);
    const long long nb = level * p.S + p.node_base[g] + (long long)lv * n;
    const long long eb = level * p.T + p.edge_base[g] + (long long)lv * m;
    const int* rp = p.row_ptr + g0;
    for (int i = lane; i < n; i += 32) { dep[i] = -1; indeg[i] = 0; }
    __syncwarp();
    // ---- BFS, one level at a time; the lanes share the frontier's adjacency entries
    if (lane == 0) { dep[lv] = 0; at[0] = lv; s_cnt[wib] = 1; }
    __syncwarp();
    int lo = 0, hi = 1, d = 0;
    while (lo < hi && (p.depth < 0 || d < p.depth)) {
      for (int k = lo; k < hi; ++k) {
        const int u = at[k];
        for (int j = rp[u] + lane; j < rp[u + 1]; j += 32) {
          const int w = p.col_idx[j] - g0;
          if (atomicCAS(&dep[w], -1, d + 1) == -1) at[atomicAdd(&s_cnt[wib], 1)] = w;
        }
      }
      __syncwarp();
      lo = hi;
      hi = s_cnt[wib];
      ++d;
      __syncwarp();
    }
    const int cnt = hi;
    auto expanded = [&](int u) { return p.depth < 0 || dep[u] < p.depth; };
    // ---- in-degrees of the DAG
    for (int k = 0; k < cnt; ++k) {
      const int u = at[k];
      if (!expanded(u)) continue;
      for (int j = rp[u] + lane; j < rp[u + 1]; j += 32) {
        const int w = p.col_idx[j] - g0;
        if (dep[w] == dep[u] + 1) atomicAdd(&indeg[w], 1);
      }
    }
    __syncwarp();
    // ---- Kahn: pop the least (rank, sequence); a child whose in-degree drops to 0 is queued in edge order
    if (lane == 0) { qv[0] = lv; qk[0] = (unsigned long long)(unsigned)rank[g0 + lv] << 32; }
    int qn = 1, seq = 1;
    __syncwarp();
    for (int i = 0; i < cnt; ++i) {
      unsigned long long best = ~0ULL;
      int bi = -1;
      for (int k = lane; k < qn; k += 32)
        if (qk[k] < best) { best = qk[k]; bi = k; }
#pragma unroll
      for (int o = 16; o; o >>= 1) {
        const unsigned long long ob = __shfl_xor_sync(FULL, best, o);
        const int oi = __shfl_xor_sync(FULL, bi, o);
        if (ob < best) { best = ob; bi = oi; }
      }
      const int u = qv[bi];
      __syncwarp();
      if (lane == 0) {
        pos[u] = i;
        at[i] = u;
        qv[bi] = qv[qn - 1];
        qk[bi] = qk[qn - 1];
      }
      --qn;
      __syncwarp();
      if (expanded(u)) {
        for (int j0 = rp[u]; j0 < rp[u + 1]; j0 += 32) {
          const int j = j0 + lane;
          bool ready = false;
          int w = 0;
          if (j < rp[u + 1]) {
            w = p.col_idx[j] - g0;
            if (dep[w] == dep[u] + 1) ready = atomicSub(&indeg[w], 1) == 1;
          }
          const unsigned b = __ballot_sync(FULL, ready);
          if (ready) {
            const int r = __popc(b & ((1u << lane) - 1u));
            qv[qn + r] = w;
            qk[qn + r] = ((unsigned long long)(unsigned)rank[g0 + w] << 32) | (unsigned)(seq + r);
          }
          qn += __popc(b);
          seq += __popc(b);
          __syncwarp();
        }
      }
    }
    // ---- identities, last pop first: a node's children (popped after it) already have their hashes.  The children
    // come in ascending `ordering` = descending pop index; each child's place in that order is its rank r, the number
    // of children popped after it.
    int e_off = 0;
    for (int i = cnt - 1; i >= 0; --i) {
      const int u = at[i];
      const int lab = labels[g0 + u];
      unsigned long long acc = 0;
      int nch = 0;
      if (expanded(u)) {
        for (int j = rp[u] + lane; j - lane < rp[u + 1]; j += 32) {
          const bool child = j < rp[u + 1] && dep[p.col_idx[j] - g0] == dep[u] + 1;
          if (child) {
            const int w = p.col_idx[j] - g0, pw = pos[w];
            int r = 0;
            for (int t = rp[u]; t < rp[u + 1]; ++t) {
              const int x = p.col_idx[t] - g0;
              r += (dep[x] == dep[u] + 1 && pos[x] > pw) ? 1 : 0;
            }
            if (!p.degenerate) acc += odd_mix(hs[w] + (unsigned long long)(r + 1) * 0x9e3779b97f4a7c15ULL + p.seed);
            p.ch[eb + e_off + r] = (int)(nb + pw);
          }
          nch += __popc(__ballot_sync(FULL, child));
        }
      }
      acc = warp_sum_u64(acc);
      unsigned long long hv = odd_mix(odd_mix(p.seed ^ ((unsigned long long)(unsigned)lab << 16) ^ (unsigned)nch) + acc);
      if (hv == EMPTY64) hv = EMPTY64 - 1;  // EMPTY64 marks a free slot of the interning table
      if (lane == 0) {
        hs[u] = hv;
        const long long s = nb + i;
        p.key[s] = hv;
        p.lab[s] = lab;
        p.gr[s] = g;
        p.cb[s] = (int)(eb + e_off);
        p.nc[s] = nch;
      }
      e_off += nch;
      __syncwarp();
    }
    for (int i = cnt + lane; i < n; i += 32) p.lab[nb + i] = -1;
    __syncwarp();
  }
}

// ---- interning: the node's hash finds (or claims) its slot, and the lowest node slot of the class represents it
__global__ void __launch_bounds__(256)
odd_insert(long long S, const unsigned long long* __restrict__ key, const int* __restrict__ lab,
           unsigned long long* tab, int* rep, unsigned long long mask, int* slot_of) {
  const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= S || lab[n] < 0) return;
  const unsigned long long k = key[n];
  unsigned long long s = k & mask;
  for (;;) {
    unsigned long long cur = tab[s];
    if (cur == EMPTY64) {
      cur = atomicCAS(&tab[s], EMPTY64, k);
      if (cur == EMPTY64) cur = k;
    }
    if (cur == k) break;
    s = (s + 1) & mask;
  }
  slot_of[n] = (int)s;
  atomicMin(&rep[s], (int)n);
}

// Every node against its class representative: same label id, same number of children, children pairwise in the
// same slot.  Any difference is a hash collision.
__global__ void __launch_bounds__(256)
odd_verify(long long S, const int* __restrict__ lab, const int* __restrict__ nc, const int* __restrict__ cb,
           const int* __restrict__ ch, const int* __restrict__ slot_of, const int* __restrict__ rep, unsigned* collision) {
  const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= S || lab[n] < 0) return;
  const int r = rep[slot_of[n]];
  if (r == n) return;
  bool bad = lab[r] != lab[n] || nc[r] != nc[n];
  for (int k = 0; !bad && k < nc[n]; ++k) bad = slot_of[ch[cb[n] + k]] != slot_of[ch[cb[r] + k]];
  if (bad) atomicOr(collision, 1u);
}

// Feature ids: the representative of a class numbers it.
__global__ void __launch_bounds__(256)
odd_number(long long S, const int* __restrict__ lab, const int* __restrict__ slot_of, const int* __restrict__ rep,
           int* colid, int* rep_of, unsigned long long* n_feat) {
  const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= S || lab[n] < 0) return;
  const int s = slot_of[n];
  if (rep[s] == n) {
    const int f = (int)atomicAdd(n_feat, 1ULL);
    colid[s] = f;
    rep_of[f] = (int)n;
  }
}

// fid of every node; C[f] = the feature's count in the first graph that has it (the graph of its representative, the
// lowest node slot); phi: (graph << 32 | fid) -> count.
__global__ void __launch_bounds__(256)
odd_count(long long S, const int* __restrict__ lab, const int* __restrict__ gr, const int* __restrict__ slot_of,
          const int* __restrict__ colid, const int* __restrict__ rep_of, int* fid, unsigned* Cf,
          unsigned long long* keys, unsigned* cnt, unsigned long long mask) {
  const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= S || lab[n] < 0) return;
  const int f = colid[slot_of[n]];
  fid[n] = f;
  const int g = gr[n];
  if (gr[rep_of[f]] == g) atomicAdd(&Cf[f], 1u);
  const unsigned long long k = ((unsigned long long)(unsigned)g << 32) | (unsigned)f;
  unsigned long long s = odd_mix(k) & mask;
  for (;;) {
    unsigned long long cur = keys[s];
    if (cur == EMPTY64) {
      cur = atomicCAS(&keys[s], EMPTY64, k);
      if (cur == EMPTY64) cur = k;
    }
    if (cur == k) { atomicAdd(&cnt[s], 1u); return; }
    s = (s + 1) & mask;
  }
}

// Self similarities sum_f C[f] phi[f, g]^2 (u64) and the entries of every bit plane of C.
__global__ void __launch_bounds__(256)
odd_phi_stats(size_t cap, const unsigned long long* __restrict__ keys, const unsigned* __restrict__ cnt,
              const unsigned* __restrict__ Cf, unsigned long long* diag, unsigned long long* plane_entries) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (size_t)gridDim.x * blockDim.x) {
    const unsigned long long k = keys[i];
    if (k == EMPTY64) continue;
    const unsigned c = cnt[i], C = Cf[(unsigned)k];
    atomicAdd(&diag[k >> 32], (unsigned long long)C * c * c);
    for (unsigned b = C; b; b &= b - 1) atomicAdd(&plane_entries[__ffs(b) - 1], 1ULL);
  }
}

// Columns of bit plane b: the features whose C has bit b.
__global__ void __launch_bounds__(256)
odd_plane_cols(int F, const unsigned* __restrict__ Cf, int b, int* colb, unsigned long long* n_cols) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  if ((Cf[f] >> b) & 1u) colb[f] = (int)atomicAdd(n_cols, 1ULL);
}

// Bit plane b's (graph, column) -> count table: the phi entries of its features (distinct keys: one insert each).
__global__ void __launch_bounds__(256)
odd_plane_fill(size_t cap_in, const unsigned long long* __restrict__ keys_in, const unsigned* __restrict__ cnt_in,
               const unsigned* __restrict__ Cf, int b, const int* __restrict__ colb, unsigned long long* keys,
               unsigned* cnt, unsigned long long mask) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap_in; i += (size_t)gridDim.x * blockDim.x) {
    const unsigned long long k0 = keys_in[i];
    if (k0 == EMPTY64) continue;
    const unsigned f = (unsigned)k0;
    if (!((Cf[f] >> b) & 1u)) continue;
    const unsigned long long k = (k0 & 0xffffffff00000000ULL) | (unsigned)colb[f];
    unsigned long long s = odd_mix(k) & mask;
    while (atomicCAS(&keys[s], EMPTY64, k) != EMPTY64) s = (s + 1) & mask;
    cnt[s] = cnt_in[i];
  }
}

// K += 2^b G_b: G_b an exact integer in fp64, the scaling exact, the sum exact below 2^53.
__global__ void odd_fold(int rows, int cols, const double* __restrict__ G, long long ldg, int b, double* out, long long ld) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)rows * cols) return;
  const int i = (int)(t / cols), j = (int)(t % cols);
  double* o = out + (long long)i * ld + j;
  *o = __dadd_rn(*o, ldexp(G[(long long)i * ldg + j], b));
}

__global__ void odd_diag_f64(int N, const unsigned long long* __restrict__ d, double* out) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < N) out[g] = (double)d[g];
}

}  // namespace gk
