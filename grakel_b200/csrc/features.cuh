// Sparse feature block -> column statistics -> (dense bf16 head panel, sparse tail).
//
// The feature block is the (graph, column) -> count hash table filled by the WL /
// SP feature kernels: it is the reference's per-level `csr_matrix` Phi_i
// (vertex_histogram.py:125-150) for all levels side by side, or the dense
// `phi_x` of ShortestPath (shortest_path.py:396-400).
//
// K = Phi Phi^T is split by column frequency m_c (number of graphs holding column c):
//   m_c = 1 (square) / column missing from X or from Y (rectangular):
//       contributes to self similarities only -- never contracted;
//       the rectangular rule is exactly the `Y[:, :X.shape[1]]` slice of
//       vertex_histogram.py:179 (unseen columns are dropped);
//   m_c >  T : "head" -- scattered into a dense bf16 panel, contracted on the tensor cores;
//   m_c <= T : "tail" -- m_c^2 exact atomic updates of K (config 2: 94 % of the shared
//       columns are in <= 64 of the 10 000 graphs; contracting them densely would be
//       18x the tensor work for 4.5 M updates).
// T is chosen on the device from a log2 histogram of m_c with a two-term cost model.
// Self similarities use ALL columns (vertex_histogram.py:186-219) and are exact integers.
#pragma once
#include "common.cuh"
#include "wl.cuh"

namespace gk {

// Decisions of one ASYNCHRONOUS pass, taken on the device (gram_choose) so that the host never waits between the
// feature kernels and the GEMM: the head/tail threshold and everything that follows from it.  `bad` != 0: the pass
// cannot be finished this way (see the bits) -- the remaining kernels then do no harm and the host repeats the pass
// through the synchronous route.
struct GramDyn {
  int T;             // head/tail threshold
  int Dc, Dc_pad;    // head columns, padded to the k-block
  int num_k_blocks;  // Dc_pad / (elements per k-block), or 1 when bad (the GEMM still runs, its result is discarded)
  int n_tail_cols, n_tail_ent;
  int bad;           // 1: a count the pass's panel type cannot hold (> 255 for u8, > 256 for bf16) or a self similarity
                     //    >= 2^24 (beyond exact fp32 output), 2: no head column,
                     // 4: panel stride too small, 8: tail buffers too small, 16: WL hash collision, 32: table overflow
  unsigned ticket;   // blocks of col_stats_fused that have finished (reset by the last one)
  unsigned long long tail_work;
  // what the host wants to know afterwards, gathered here so that ONE copy brings it back
  unsigned long long max_count, max_diag, n_entries;
  long long n_columns;              // level_base[L]
  long long level_dims[MAX_LEVELS];
  ColStats hist;
};

// rectangular (transform) case only: smallest / largest graph id per column.  In table
// (hash) order the running extrema converge after O(log m) updates per column, so the
// L2-read filter removes almost all atomics even for columns present in every graph.
__global__ void __launch_bounds__(256)
feat_minmax(size_t cap, const unsigned long long* __restrict__ keys, const int* __restrict__ row_map, int* colmin,
            int* colmax) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (size_t)gridDim.x * blockDim.x) {
    const unsigned long long k = keys[i];
    if (k == EMPTY64) continue;
    const int g = row_map ? row_map[(int)(k >> 32)] : (int)(k >> 32);
    const unsigned c = (unsigned)k;
    if (__ldcg(&colmin[c]) > g) atomicMin(&colmin[c], g);
    if (__ldcg(&colmax[c]) < g) atomicMax(&colmax[c], g);
  }
}

// Row map (gk_set_row_map): several packed graphs feed one row of K (CoreFramework: the k-core
// subgraphs of a graph).  Their feature columns are disjoint, so a row's self similarity is the sum
// of its packed graphs' self similarities.
__global__ void __launch_bounds__(256)
diag_remap(int n_packed, const int* __restrict__ row_map, const unsigned long long* __restrict__ diag,
           unsigned long long* diag_rows) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < n_packed && diag[g]) atomicAdd(&diag_rows[row_map[g]], diag[g]);
}

__global__ void __launch_bounds__(256)
diag_finish(int N, const unsigned long long* __restrict__ diag, double* __restrict__ diag_f64,
            int n_part, const unsigned* __restrict__ part_max, const unsigned* __restrict__ part_new,
            DevScalars* sc) {
  int g = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long d = 0;
  if (g < N) {
    d = diag[g];
    diag_f64[g] = (double)d;
  }
  // fold the per-CTA partials of the feature kernels (max count, created entries)
  unsigned mx = 0;
  unsigned long long nn = 0;
  for (int i = g; i < n_part; i += gridDim.x * blockDim.x) { mx = max(mx, part_max[i]); nn += part_new[i]; }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
    unsigned long long o = __shfl_xor_sync(0xffffffffu, d, s);
    d = d > o ? d : o;
    mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, s));
    nn += __shfl_xor_sync(0xffffffffu, nn, s);
  }
  if ((threadIdx.x & 31) == 0) {
    if (d) atomicMax(&sc->max_diag, d);
    if (mx) atomicMax(&sc->max_count, (unsigned long long)mx);
    if (nn) atomicAdd(&sc->n_entries, nn);
  }
}

// does a column contribute to an off-diagonal (square) / cross (rectangular) entry, and an
// upper bound of the pair updates it would cost in the tail
__device__ __forceinline__ bool col_contributes(unsigned m, int gmin, int gmax, int n_fit, bool square,
                                                unsigned long long* work) {
  *work = (unsigned long long)m * (m - 1);
  if (square) return m >= 2;
  return m >= 2 && gmin < n_fit && gmax >= n_fit;  // present on both sides
}

__device__ __forceinline__ int size_bucket(unsigned m) {
  if (m >= COL_CAP) return HIST_BUCKETS - 1;
  int b = 0;
  while ((1u << b) < m) ++b;
  return b < HIST_BUCKETS - 1 ? b : HIST_BUCKETS - 2;
}

// log2 histogram of contributing columns: count and pair work per size bucket
__global__ void __launch_bounds__(256)
col_hist(long long D, int square, int n_fit, const unsigned* __restrict__ colcnt, const int* __restrict__ colmin,
         const int* __restrict__ colmax, ColStats* cs) {
  __shared__ unsigned long long hc[HIST_BUCKETS], hw[HIST_BUCKETS], he[HIST_BUCKETS];
  if (threadIdx.x < HIST_BUCKETS) { hc[threadIdx.x] = 0; hw[threadIdx.x] = 0; he[threadIdx.x] = 0; }
  __syncthreads();
  long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c < D) {
    const unsigned m = colcnt[c];
    unsigned long long work;
    if (m && col_contributes(m, square ? 0 : colmin[c], square ? 0 : colmax[c], n_fit, square, &work)) {
      const int b = size_bucket(m);
      atomicAdd(&hc[b], 1ULL);
      atomicAdd(&hw[b], work);
      atomicAdd(&he[b], (unsigned long long)m);
    }
  }
  __syncthreads();
  if (threadIdx.x < HIST_BUCKETS && hc[threadIdx.x]) {
    atomicAdd(&cs->hist_cols[threadIdx.x], hc[threadIdx.x]);
    atomicAdd(&cs->hist_work[threadIdx.x], hw[threadIdx.x]);
    atomicAdd(&cs->hist_entries[threadIdx.x], he[threadIdx.x]);
  }
}

// Column statistics of the asynchronous pass in ONE launch: self similarities + per-CTA partials (diag_finish), the log2
// histogram of the contributing columns (col_hist, square case), and -- in the block that finishes last -- the
// host-side choice of gk_gram on the device: threshold T = 2^k minimising head_cols * flops_per_col / rate +
// tail_updates * t_atomic (one thread per candidate k), the bucket sums that follow from it, the exactness bounds,
// the capacity checks; everything the host reads afterwards is copied into `dyn`.  The first words of `cs` (the tail
// counters of col_classify) are cleared on the way out.
struct ColFusedParams {
  long long D; int N; int L;
  const unsigned* colcnt;
  const unsigned long long* diag; double* diag_f64;
  int n_part; const unsigned* part_max; const unsigned* part_new;
  ColStats* cs; DevScalars* sc; GramDyn* dyn;
  double flops_per_col, rate, t_atomic;  // rate: dense GEMM rate of the pass's panel type
  int force_T, stride_cap, bk;           // stride_cap: panel row pitch; bk: elements per k-block (both of that type)
  unsigned max_panel_count;              // largest count the panel type holds exactly (255 u8, 256 bf16)
  long long cap_tail_cols, cap_tail_ent;
};
__global__ void __launch_bounds__(256)
col_stats_fused(ColFusedParams q) {
  __shared__ unsigned long long hc[HIST_BUCKETS], hw[HIST_BUCKETS], he[HIST_BUCKETS];
  __shared__ double s_cost[HIST_BUCKETS];
  __shared__ bool s_last;
  const int tid = threadIdx.x;
  if (tid < HIST_BUCKETS) { hc[tid] = 0; hw[tid] = 0; he[tid] = 0; }
  __syncthreads();
  // ---- self similarities and partials (diag_finish); a few hundred fat blocks, grid-stride: every block costs one
  // ticket and a handful of same-address atomics at the end
  {
    const int g0 = blockIdx.x * blockDim.x + tid, gs = gridDim.x * blockDim.x;
    unsigned long long d = 0;
    for (int g = g0; g < q.N; g += gs) {
      const unsigned long long x = q.diag[g];
      q.diag_f64[g] = (double)x;
      d = d > x ? d : x;
    }
    unsigned mx = 0;
    unsigned long long nn = 0;
    for (int i = g0; i < q.n_part; i += gs) { mx = max(mx, q.part_max[i]); nn += q.part_new[i]; }
#pragma unroll
    for (int s2 = 16; s2 > 0; s2 >>= 1) {
      const unsigned long long o = __shfl_xor_sync(0xffffffffu, d, s2);
      d = d > o ? d : o;
      mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, s2));
      nn += __shfl_xor_sync(0xffffffffu, nn, s2);
    }
    if ((tid & 31) == 0) {
      if (d) atomicMax(&q.sc->max_diag, d);
      if (mx) atomicMax(&q.sc->max_count, (unsigned long long)mx);
      if (nn) atomicAdd(&q.sc->n_entries, nn);
    }
  }
  // ---- histogram of the contributing columns (col_hist, square)
  {
    for (long long c = (long long)blockIdx.x * blockDim.x + tid; c < q.D; c += (long long)gridDim.x * blockDim.x) {
      const unsigned m = q.colcnt[c];
      if (m >= 2) {
        const int b = size_bucket(m);
        atomicAdd(&hc[b], 1ULL);
        atomicAdd(&hw[b], (unsigned long long)m * (m - 1));
        atomicAdd(&he[b], (unsigned long long)m);
      }
    }
  }
  __syncthreads();
  if (tid < HIST_BUCKETS && hc[tid]) {
    atomicAdd(&q.cs->hist_cols[tid], hc[tid]);
    atomicAdd(&q.cs->hist_work[tid], hw[tid]);
    atomicAdd(&q.cs->hist_entries[tid], he[tid]);
  }
  // ---- the last block decides
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = atomicAdd(&q.dyn->ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  volatile ColStats* cs = q.cs;
  volatile DevScalars* sc = q.sc;
  GramDyn* dyn = q.dyn;
  if (tid < HIST_BUCKETS) {
    hc[tid] = cs->hist_cols[tid]; hw[tid] = cs->hist_work[tid]; he[tid] = cs->hist_entries[tid];
  }
  __syncthreads();
  if (tid < HIST_BUCKETS) {  // candidate k = tid
    double head_cols = 0, tail_upd = 0;
    for (int b = 0; b < HIST_BUCKETS; ++b) {
      if (b > tid) head_cols += (double)hc[b];
      else tail_upd += (double)hw[b];
    }
    s_cost[tid] = head_cols * q.flops_per_col / q.rate + tail_upd * q.t_atomic;
    dyn->hist.hist_cols[tid] = hc[tid]; dyn->hist.hist_work[tid] = hw[tid]; dyn->hist.hist_entries[tid] = he[tid];
  }
  for (int i = tid; i < MAX_LEVELS; i += blockDim.x) dyn->level_dims[i] = sc->level_dims[i];
  __syncthreads();
  if (tid == 0) {
    int T = 1;
    double best = -1.0;
    for (int k = 0; k <= HIST_BUCKETS - 2; ++k)
      if (best < 0 || s_cost[k] < best) { best = s_cost[k]; T = 1 << k; }
    if (q.force_T >= 1) T = q.force_T;
    long long Dc = 0, n_tail_cols = 0, n_tail_ent = 0;
    unsigned long long tail_work = 0;
    for (int b = 0; b < HIST_BUCKETS; ++b) {
      if (b < HIST_BUCKETS - 1 && (1LL << b) <= T) { n_tail_cols += (long long)hc[b]; n_tail_ent += (long long)he[b]; tail_work += hw[b]; }
      else Dc += (long long)hc[b];
    }
    const long long Dc_pad = (Dc + q.bk - 1) / q.bk * q.bk;
    const unsigned long long max_count = sc->max_count, max_diag = sc->max_diag;
    int bad = 0;
    if (max_count > (unsigned long long)q.max_panel_count || max_diag >= (1ULL << 24)) bad |= 1;
    if (Dc == 0) bad |= 2;
    if (Dc_pad > q.stride_cap) bad |= 4;
    if (n_tail_cols > q.cap_tail_cols || n_tail_ent > q.cap_tail_ent) bad |= 8;
    if (sc->collision) bad |= 16;
    if (sc->ft_overflow) bad |= 32;
    dyn->T = T;
    dyn->Dc = (int)Dc; dyn->Dc_pad = (int)Dc_pad;
    dyn->num_k_blocks = bad ? 1 : (int)(Dc_pad / q.bk);
    dyn->n_tail_cols = bad ? 0 : (int)n_tail_cols;
    dyn->n_tail_ent = (int)n_tail_ent;
    dyn->bad = bad;
    dyn->tail_work = tail_work;
    dyn->max_count = max_count; dyn->max_diag = max_diag; dyn->n_entries = sc->n_entries;
    dyn->n_columns = sc->level_base[q.L];
    dyn->hist.T = T;
    dyn->ticket = 0u;  // ready for the next pass
    // the tail counters of col_classify live in the first words of the histogram block
    unsigned* counters = reinterpret_cast<unsigned*>(q.cs);
    counters[0] = counters[1] = counters[2] = counters[3] = 0u;
  }
}

// zero the panel: `w16` 16-byte units of every row (row pitch `ld_bytes`); one warp per row, grid-stride
__global__ void __launch_bounds__(256)
panel_zero_rows(unsigned char* __restrict__ panel, long long n_rows, long long ld_bytes, int w16) {
  const int lane = threadIdx.x & 31;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  const uint4 z = make_uint4(0u, 0u, 0u, 0u);
  for (long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n_rows; r += n_warps) {
    uint4* row = reinterpret_cast<uint4*>(panel + r * ld_bytes);
    for (int c = lane; c < w16; c += 32) row[c] = z;
  }
}

// Classification + slot allocation in ONE pass over the columns (replaces a three-kernel
// flag / scan / assign pipeline: only ~1.5 % of the columns contribute, so warp-aggregated
// atomics on three counters are cheaper than scanning 1.6 M columns three times).
//   colslot[c] >= 0  : head column index in the dense panel
//   colslot[c] == -1 : column does not contribute to any off-diagonal entry
//   colslot[c] <= -2 : tail column t = -(colslot+2); tail_desc[t] = {first entry, m}
// Slot order depends on scheduling; K does not (exact integer arithmetic, see gram_tc.cuh).
// counters: [0] head columns, [1] tail columns, [2] tail entries (zeroed by the host).
__global__ void __launch_bounds__(256)
col_classify(long long D, int square, int n_fit, const unsigned* __restrict__ colcnt, const int* __restrict__ colmin,
             const int* __restrict__ colmax, int T, int* __restrict__ colslot, int2* __restrict__ tail_desc,
             unsigned* __restrict__ tail_cur, unsigned* counters, const GramDyn* __restrict__ dyn = nullptr) {
  const int lane = threadIdx.x & 31;
  bool off = false;
  if (dyn) { T = dyn->T; off = dyn->bad != 0; }  // asynchronous pass: the threshold was chosen on the device
  // grid-stride over whole warps (a launch may have one thread per column or a few hundred fat blocks)
  const long long D32 = (D + 31) / 32 * 32;
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < D32; c += (long long)gridDim.x * blockDim.x) {
  int kind = 0;
  unsigned m = 0;
  if (c < D && !off) {
    m = colcnt[c];
    unsigned long long work;
    if (m && col_contributes(m, square ? 0 : colmin[c], square ? 0 : colmax[c], n_fit, square, &work))
      kind = (m > (unsigned)T || m >= COL_CAP) ? 1 : 2;
  }
  const unsigned hm = __ballot_sync(0xffffffffu, kind == 1), tm = __ballot_sync(0xffffffffu, kind == 2);
  const unsigned below = (1u << lane) - 1u;
  int slot = -1;
  if (hm) {
    unsigned base = 0;
    if (lane == __ffs(hm) - 1) base = atomicAdd(&counters[0], (unsigned)__popc(hm));
    base = __shfl_sync(0xffffffffu, base, __ffs(hm) - 1);
    if (kind == 1) slot = (int)(base + __popc(hm & below));
  }
  if (tm) {
    // exclusive prefix of m over the tail lanes of the warp
    unsigned incl = kind == 2 ? m : 0u;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const unsigned y = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += y;
    }
    const unsigned total = __shfl_sync(0xffffffffu, incl, 31);
    unsigned tbase = 0, ebase = 0;
    if (lane == __ffs(tm) - 1) {
      tbase = atomicAdd(&counters[1], (unsigned)__popc(tm));
      ebase = atomicAdd(&counters[2], total);
    }
    tbase = __shfl_sync(0xffffffffu, tbase, __ffs(tm) - 1);
    ebase = __shfl_sync(0xffffffffu, ebase, __ffs(tm) - 1);
    if (kind == 2) {
      const int t = (int)(tbase + __popc(tm & below));
      tail_desc[t] = make_int2((int)(ebase + incl - m), (int)m);
      tail_cur[t] = 0u;
      slot = -(t + 2);
    }
  }
  if (c < D) colslot[c] = slot;
  }
}

// pass 2 over the table: head entries -> zeroed panel (u8 or bf16: PanelT, the host chose a type that holds every
// count exactly), tail entries -> per-column lists
template <typename PanelT>
__global__ void __launch_bounds__(256)
feat_scatter(size_t cap, const unsigned long long* __restrict__ keys, const unsigned* __restrict__ cnt,
             const int* __restrict__ colslot, const int* __restrict__ row_map, PanelT* __restrict__ panel,
             long long ld, unsigned* __restrict__ tail_cur, const int2* __restrict__ tail_desc,
             int2* __restrict__ tail_ent) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (size_t)gridDim.x * blockDim.x) {
    unsigned long long k = keys[i];
    if (k == EMPTY64) continue;
    const unsigned c = (unsigned)k;
    const int slot = colslot[c];
    if (slot == -1) continue;
    const int g = row_map ? row_map[(int)(k >> 32)] : (int)(k >> 32);
    if (slot >= 0) {
      if constexpr (sizeof(PanelT) == 1) panel[(long long)g * ld + slot] = (PanelT)cnt[i];
      else panel[(long long)g * ld + slot] = __float2bfloat16_rn((float)cnt[i]);
    } else {
      const int t = -(slot + 2);
      const unsigned pos = atomicAdd(&tail_cur[t], 1u);
      tail_ent[tail_desc[t].x + pos] = make_int2(g, (int)cnt[i]);
    }
  }
}

// same, into a u32 panel (exact CUDA-core Gram; no tail in that mode)
__global__ void __launch_bounds__(256)
feat_fill_panel_u32(size_t cap, const unsigned long long* __restrict__ keys, const unsigned* __restrict__ cnt,
                    const int* __restrict__ colslot, const int* __restrict__ row_map, unsigned* __restrict__ panel,
                    long long ld) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cap) return;
  unsigned long long k = keys[i];
  if (k == EMPTY64) return;
  const int dc = colslot[(unsigned)k];
  if (dc < 0) return;
  const int g = row_map ? row_map[(int)(k >> 32)] : (int)(k >> 32);
  panel[(long long)g * ld + dc] = cnt[i];
}

// Tail contraction: one warp per tail column, all ordered pairs of its entries.
//   square      : K[ga][gb] += ca*cb for a != b (the diagonal is written exactly elsewhere)
//   rectangular : rows are Y graphs (g >= n_fit), columns X graphs (g < n_fit)
// Values are integers < 2^24 (checked by the host), so float atomics are exact and
// order independent.
template <typename OutT>
__global__ void __launch_bounds__(256)
tail_pairs(long long n_tail_cols, const int2* __restrict__ tail_desc, const int2* __restrict__ tail_ent,
           int n_fit, int square, int row0, int row1, OutT* __restrict__ out, long long ld,
           const GramDyn* __restrict__ dyn = nullptr) {
  const int lane = threadIdx.x & 31;
  if (dyn) n_tail_cols = dyn->n_tail_cols;  // asynchronous pass: fixed grid, the column count lives on the device
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < n_tail_cols; w += n_warps) {
    const int2 d = tail_desc[w];
    const int2* ent = tail_ent + d.x;
    const int m = d.y;
    const int mm = m * m;
    for (int p = lane; p < mm; p += 32) {
      const int a = p / m, b = p - a * m;
      if (a == b) continue;
      const int2 ea = ent[a], eb = ent[b];
      int r, c;
      if (square) { r = ea.x; c = eb.x; }
      else {
        if (ea.x < n_fit || eb.x >= n_fit) continue;
        r = ea.x - n_fit; c = eb.x;
      }
      if (r < row0 || r >= row1) continue;
      atomicAdd(&out[(long long)(r - row0) * ld + c], (OutT)((float)ea.y * (float)eb.y));
    }
  }
}

// Tail fused into the GEMM epilogue (gram_tc.cuh, GramParams::tb_cnt): the ordered pairs of every tail column, bucketed by
// 32 x 32 block of K.  Entry = row | col << 5 | value << 10 in ONE word (counts are at most 255 on this path -- the
// asynchronous pass fills a u8 panel, or at most 256 when it fills a bf16 one -- so a product has at most 17 bits); a block's TB_CAP entries are one 128-byte line, the rest go to the overflow list {row, col, value} that
// tail_overflow_apply adds with global atomics after the GEMM.  Several columns may update the same element: the
// epilogue adds entries one by one (exact integer sums in fp32).  The host clears counters AND entry lines first: a
// fully written line is allocated in L2 without a fetch, so the 1.5 M scattered 4-byte stores below hit there instead of
// costing a DRAM sector read each (which is what made the separate tail kernel slow in the first place).
__global__ void __launch_bounds__(256)
tail_bucket(const int2* __restrict__ tail_desc, const int2* __restrict__ tail_ent, const GramDyn* __restrict__ dyn, int nb32, int cap, int stride, int sym,
            unsigned* __restrict__ tb_cnt, unsigned* __restrict__ tb_ent, int4* __restrict__ ovf, unsigned ovf_cap, unsigned* __restrict__ ovf_n) {
  const int lane = threadIdx.x & 31;
  const long long n_cols = dyn->n_tail_cols;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < n_cols; w += n_warps) {
    const int2 d = tail_desc[w];
    const int2* ent = tail_ent + d.x;
    const int m = d.y;
    const int mm = m * m;
    // a column of at most 32 graphs (the usual threshold): one entry per lane, pairs through shuffles -- no loads in the loop
    const bool in_regs = m <= 32;
    int2 mine = make_int2(0, 0);
    if (in_regs && lane < m) mine = ent[lane];
    for (int p0 = 0; p0 < mm; p0 += 32) {  // (whole warp iterates: the shuffles need every lane)
      const int p = p0 + lane;
      const int a = p < mm ? p / m : 0, b = p < mm ? p - a * m : 0;
      int2 ea, eb;
      if (in_regs) {
        ea.x = __shfl_sync(0xffffffffu, mine.x, a); ea.y = __shfl_sync(0xffffffffu, mine.y, a);
        eb.x = __shfl_sync(0xffffffffu, mine.x, b); eb.y = __shfl_sync(0xffffffffu, mine.y, b);
      } else {
        ea = ent[a]; eb = ent[b];
      }
      if (p >= mm || a == b) continue;
      const int r = ea.x, c = eb.x;
      if (sym && r > c) continue;  // symmetric lists: the pair (c, r) of this column files the update (half the atomics)
      const unsigned val = (unsigned)ea.y * (unsigned)eb.y;
      const long long blk = (long long)(r >> 5) * nb32 + (c >> 5);
      const unsigned pos = atomicAdd(&tb_cnt[blk], 1u);
      if (pos < (unsigned)cap && val < (1u << 22)) {
        tb_ent[blk * stride + pos] = (unsigned)(r & 31) | ((unsigned)(c & 31) << 5) | (val << 10);
      } else {
        const unsigned o = atomicAdd(ovf_n, 1u);
        if (o < ovf_cap) ovf[o] = make_int4(r, c, (int)__float_as_uint((float)val), 0);
      }
    }
  }
}
__global__ void __launch_bounds__(256)
tail_overflow_apply(const int4* __restrict__ ovf, const unsigned* __restrict__ ovf_n, unsigned ovf_cap, float* __restrict__ out, long long ld,
                    int sym) {
  const unsigned n = min(*ovf_n, ovf_cap);
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int4 e = ovf[i];
    atomicAdd(&out[(long long)e.x * ld + e.y], __uint_as_float((unsigned)e.z));
    if (sym) atomicAdd(&out[(long long)e.y * ld + e.x], __uint_as_float((unsigned)e.z));
  }
}

__global__ void __launch_bounds__(256) add_u64(int n, const unsigned long long* __restrict__ src, unsigned long long* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] += src[i];
}

// Upper triangle of an fp32 matrix of integers < 65 536 -> band-packed u16 (host_deliver.h tri_bands): band c holds
// rows [start[c], start[c+1]) x columns [start[c], n) contiguously at element offset off[c].  One CTA per (band, row).
__global__ void __launch_bounds__(256)
pack_tri_u16(const float* __restrict__ K, long long ld, long long n, const long long* __restrict__ start, const long long* __restrict__ off,
             int n_bands, unsigned short* __restrict__ out) {
  for (long long row = blockIdx.x; row < n; row += gridDim.x) {
    int c = 0;  // band of this row (bands are few: linear search from a proportional guess)
    {
      int lo = 0, hi = n_bands - 1;
      while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (start[mid] <= row) lo = mid; else hi = mid - 1; }
      c = lo;
    }
    const long long r0 = start[c], w = n - r0;
    const float* src = K + row * ld + r0;
    unsigned short* dst = out + off[c] + (row - r0) * w;
    for (long long j = threadIdx.x; j < w; j += blockDim.x) dst[j] = (unsigned short)src[j];
  }
}

// normalisation pass when a tail exists: K_ij / sqrt(d_i d_j)  (+ nan_to_num)
template <typename OutT>
__global__ void __launch_bounds__(256)
normalize_rows(long long rows, long long cols, OutT* __restrict__ out, long long ld,
               const double* __restrict__ diag_rows, const double* __restrict__ diag_cols, int nan_to_num) {
  const long long total = rows * cols;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols, c = i - r * cols;
    double v = (double)out[r * ld + c];
    v = v / sqrt(diag_rows[r] * diag_cols[c]);
    if (nan_to_num) {
      if (v != v) v = 0.0;
      else if (isinf(v)) v = v > 0 ? 1.7976931348623157e308 : -1.7976931348623157e308;
    }
    out[r * ld + c] = (OutT)v;
  }
}

// WL over a base kernel with per-level fp64 K: dst += src elementwise, one level at a time, so that the sum rounds as
// numpy's np.sum(levels, axis=0) does: ((K_0 + K_1) + K_2) ...
__global__ void __launch_bounds__(256)
add_f64(long long n, const double* __restrict__ src, double* __restrict__ dst) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    dst[i] = dst[i] + src[i];
}

// CoreFramework: sum[rows[j], cols[c]] += K[j, c] for one core level, the reference's K[idx_j, idx] += K_i[j, :].
// The maps hold no index twice, so every element of the sum has one writer.
__global__ void __launch_bounds__(256)
core_scatter_add_f64(long long k_rows, long long k_cols, const double* __restrict__ K, const int* __restrict__ rows,
                     const int* __restrict__ cols, double* __restrict__ sum, long long sum_ld) {
  const long long n = k_rows * k_cols;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long j = i / k_cols, c = i - j * k_cols;
    double* d = sum + (long long)rows[j] * sum_ld + cols[c];
    *d = *d + K[i];
  }
}

// out[i] = K[i ld + i]: the diagonal of a full square K
__global__ void __launch_bounds__(256)
diag_of_f64(long long n, const double* __restrict__ K, long long ld, double* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = K[i * ld + i];
}

}  // namespace gk
