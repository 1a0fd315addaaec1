// Marching cubes on the GPU: sign bits -> crossed-cell list -> classify -> prefix scans -> vertex emit -> face emit.
//
// Replaces MCSurfaceExtractor.run (Hunyuan3D-2/hy3dgen/shapegen/models/autoencoders/surface_extractors.py:67-76),
// which copies the grid to the host and runs scikit-image's single-threaded Lewiner marching cubes.
// The sequential algorithm appends vertices and faces in cell-traversal order (z, y, x with x = last array
// axis) and creates a shared edge vertex at the first cell that uses it.  Here the same order is produced
// without any sequential dependency:
//   * the first user of a grid edge is a pure function of the edge ("owner" cell, see owns_edge), so
//     vertex ids = exclusive prefix sum over cells of the number of owned vertices + rank inside the cell,
//   * face ids   = exclusive prefix sum over cells of the triangle count.
// HBM-bound integer/byte work, no tensor cores.  The float grid is streamed ONCE (mc_bits: one bit per point, min / max
// on the way).  Everything after that touches only what the surface crosses: mc_mark turns eight bit words into the
// 32-cell mask of a segment with a handful of logic operations, mc_compact writes the crossed cells out in traversal
// order, and the Lewiner tests, the scans and the two emit passes run one thread per CROSSED cell (dense warps; the
// eight corner values of those cells are re-read through L2).
// R3G_MC_DUAL (dual marching cubes, the 'dmc' extractor) shares the passes up to and including the Lewiner decisions and
// the scans; only its vertex pass (one vertex per connected patch of a cell's tiling) and face pass (one quad per
// interior sign-changing grid edge) differ, and their output order comes from the same scans.
#include <float.h>

#include "r3g_internal.h"

#define R3G_MC_TABLE_QUAL static __device__ const
#include "../../include/r3g_mc_tables.h"

namespace {

constexpr int kThreads = 256;

constexpr int kWarps = kThreads / 32;

struct McDims {
  int n0, n1, n2;   // grid points per axis (axis2 fastest)
  int c0, c1, c2;   // cells per axis
  int64_t ncells;
  int64_t npts;     // n0 * n1 * n2; the sign bits are indexed by the flat point index (z * n1 + y) * n2 + x
  unsigned segs;    // 32-cell segments per row of c2 cells
  unsigned nsegs;   // c0 * c1 * segs; segment s = (row, seg) in row-major order = the traversal order of the cells
};

struct Cell {
  int ci;       // cube index 0..255
  int til;      // tiling index
  int nt;       // triangles
  int nv;       // vertices this cell creates
};

__device__ __forceinline__ bool face_pos_connected(const double* cv, int face) {
  const unsigned char* fc = &r3g_mc_face_corner[4 * face];
  double A = cv[fc[0]], B = cv[fc[1]], C = cv[fc[2]], D = cv[fc[3]];
  // explicit roundings: no fma contraction, so the decision does not depend on the compiler's contraction choices
  double ac = __dmul_rn(A, C), bd = __dmul_rn(B, D);
  double pmn = (A > 0.0) ? __dsub_rn(ac, bd) : __dsub_rn(bd, ac);
  return pmn > -R3G_MC_EPS;
}

// Lewiner's test_interior (scikit-image: test_internal) for the sub-cases 4, 6.1, 7.4, 10.1, 12.1, 13.5: is the pair of
// same-sign corners on a body diagonal joined through the interior of the cell (then the tunnel tiling is used)?
// desc = r3g_mc_interior entry (mode, reference edge, sigma), see tools/gen_mc_tables.py.  Every product / sum is an
// explicitly rounded operation in source order (no fma contraction): the decision does not depend on the compiler.
__device__ __forceinline__ double lerp_rn(double a, double b, double t) {
  return __dadd_rn(a, __dmul_rn(__dsub_rn(b, a), t));
}
__device__ __noinline__ bool interior_joined(const double* cv, int desc) {
  const int mode = desc & 3, edge = (desc >> 2) & 15, sigma = (desc >> 6) & 1;
  double At, Bt, Ct, Dt;
  if (mode == 1) {
    const double d40 = __dsub_rn(cv[4], cv[0]), d62 = __dsub_rn(cv[6], cv[2]);
    const double d73 = __dsub_rn(cv[7], cv[3]), d51 = __dsub_rn(cv[5], cv[1]);
    const double a = __dsub_rn(__dmul_rn(d40, d62), __dmul_rn(d73, d51));
    const double b = __dsub_rn(__dsub_rn(__dadd_rn(__dmul_rn(cv[2], d40), __dmul_rn(cv[0], d62)), __dmul_rn(cv[1], d73)),
                               __dmul_rn(cv[3], d51));
    const double t = __ddiv_rn(-b, __dmul_rn(2.0, a));
    if (t < 0.0 || t > 1.0) return sigma == 0;
    At = lerp_rn(cv[0], cv[4], t);
    Bt = lerp_rn(cv[3], cv[7], t);
    Ct = lerp_rn(cv[2], cv[6], t);
    Dt = lerp_rn(cv[1], cv[5], t);
  } else {
    const int u = r3g_mc_edge_corner[2 * edge], w = r3g_mc_edge_corner[2 * edge + 1];
    const unsigned char* sl = &r3g_mc_slice[6 * edge];
    const double t = __ddiv_rn(cv[u], __dsub_rn(cv[u], cv[w]));
    At = 0.0;
    Bt = lerp_rn(cv[sl[0]], cv[sl[1]], t);
    Ct = lerp_rn(cv[sl[2]], cv[sl[3]], t);
    Dt = lerp_rn(cv[sl[4]], cv[sl[5]], t);
  }
  const int test = (At >= 0.0 ? 1 : 0) + (Bt >= 0.0 ? 2 : 0) + (Ct >= 0.0 ? 4 : 0) + (Dt >= 0.0 ? 8 : 0);
  const double acbd = __dsub_rn(__dmul_rn(At, Ct), __dmul_rn(Bt, Dt));
  bool pos_joined;
  switch (test) {
    case 7: case 11: case 13: case 14: case 15: pos_joined = true; break;
    case 5: pos_joined = !(acbd < R3G_MC_EPS); break;
    case 10: pos_joined = !(acbd >= R3G_MC_EPS); break;
    default: pos_joined = false; break;
  }
  return sigma ? pos_joined : !pos_joined;
}

// Does cell (x,y,z) create the vertex on its edge e?  (first cell in traversal order sharing the edge)
__device__ __forceinline__ bool owns_edge(int e, int x, int y, int z) {
  int info = r3g_mc_edge_info[e];
  int ox = info & 1, oy = (info >> 1) & 1, oz = (info >> 2) & 1, axis = info >> 3;
  bool okx = (axis == 0) || ox || x == 0;
  bool oky = (axis == 1) || oy || y == 0;
  bool okz = (axis == 2) || oz || z == 0;
  return okx && oky && okz;
}

__device__ __forceinline__ void load_cell(const float* __restrict__ g, const McDims& d, int x, int y, int z,
                                          float* raw) {
  const float* p = g + ((int64_t)z * d.n1 + y) * d.n2 + x;
  const int64_t sy = d.n2, sz = (int64_t)d.n1 * d.n2;
  raw[0] = __ldg(p);            raw[1] = __ldg(p + 1);
  raw[3] = __ldg(p + sy);       raw[2] = __ldg(p + sy + 1);
  raw[4] = __ldg(p + sz);       raw[5] = __ldg(p + sz + 1);
  raw[7] = __ldg(p + sz + sy);  raw[6] = __ldg(p + sz + sy + 1);
}

// (double)v - (double)level > 0  <=>  v > level for floats (the difference is exact in double), so the cube index
// is computed in float and the double-precision work below only runs for the few cells the surface crosses.
__device__ __forceinline__ int cube_index(const float* raw, float level) {
  int ci = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) ci |= (raw[i] > level) ? (1 << i) : 0;
  return ci;
}

// The Lewiner tiling of a crossed cell (cube index ci, neither 0 nor 255): face tests, then the interior test where it
// applies.  Fills cv with the corner values minus the level.  Both extractors take their decisions from here.
__device__ __forceinline__ int cell_tiling(int ci, const float* raw, float level, double* cv) {
#pragma unroll
  for (int i = 0; i < 8; ++i) cv[i] = (double)raw[i] - (double)level;
  int sub = 0, j = 0;
  unsigned amb = r3g_mc_amb_faces[ci];
  for (int f = 0; f < 6; ++f)
    if (amb & (1u << f)) {
      if (face_pos_connected(cv, f)) sub |= 1 << j;
      ++j;
    }
  int til = r3g_mc_tiling_offset[ci] + sub;
  const int idesc = r3g_mc_interior[til];
  if (idesc && interior_joined(cv, idesc)) til = r3g_mc_tunnel[til];
  return til;
}

__device__ __forceinline__ Cell eval_cell(int ci, const float* raw, float level, double* cv, int x, int y, int z) {
  Cell c;
  c.ci = ci;
  c.til = 0; c.nt = 0; c.nv = 0;
  if (c.ci == 0 || c.ci == 255) return c;
  c.til = cell_tiling(c.ci, raw, level, cv);
  int t0 = r3g_mc_tiling_start[c.til], t1 = r3g_mc_tiling_start[c.til + 1];
  c.nt = (t1 - t0) / 3;
  unsigned seen = 0;
  for (int t = t0; t < t1; ++t) {
    int e = r3g_mc_tri[t];
    unsigned bit = 1u << e;
    if (seen & bit) continue;
    seen |= bit;
    if (e == 12 || owns_edge(e, x, y, z)) c.nv++;
  }
  return c;
}

__device__ __forceinline__ unsigned f2ord(float f) {
  unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float ord2f(unsigned u) {
  unsigned v = (u & 0x80000000u) ? (u & 0x7FFFFFFFu) : ~u;
#ifdef __CUDA_ARCH__
  return __uint_as_float(v);
#else
  float f;
  memcpy(&f, &v, 4);
  return f;
#endif
}

// Block-wide exclusive scan in thread order (one or two counters); returns the block totals.
template <int N>
__device__ __forceinline__ void block_scan(const unsigned (&v)[N], unsigned (&excl)[N], unsigned (&total)[N]) {
  __shared__ unsigned ws[N][kWarps];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  unsigned inc[N];
#pragma unroll
  for (int k = 0; k < N; ++k) inc[k] = v[k];
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
#pragma unroll
    for (int k = 0; k < N; ++k) {
      unsigned n = __shfl_up_sync(0xffffffffu, inc[k], o);
      if (lane >= o) inc[k] += n;
    }
  }
  if (lane == 31) {
#pragma unroll
    for (int k = 0; k < N; ++k) ws[k][w] = inc[k];
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < N; ++k) {
    unsigned off = 0, sum = 0;
#pragma unroll
    for (int i = 0; i < kWarps; ++i) {
      const unsigned t = ws[k][i];
      if (i < w) off += t;
      sum += t;
    }
    excl[k] = off + inc[k] - v[k];
    total[k] = sum;
  }
  __syncthreads();
}

__device__ __forceinline__ bool cell_coords(const McDims& d, int64_t cell, int& x, int& y, int& z) {
  if (cell >= d.ncells) return false;
  x = (int)(cell % d.c2);
  int64_t r = cell / d.c2;
  y = (int)(r % d.c1);
  z = (int)(r / d.c1);
  return true;
}

// A crossed cell is named by its slot = segment * 32 + lane: segment s = (row, seg) with row = z * c1 + y, cell x = 32 seg +
// lane.  Slots increase in traversal order.
__device__ __forceinline__ void slot_coords(const McDims& d, unsigned slot, int& x, int& y, int& z) {
  const unsigned s = slot >> 5;
  const unsigned row = s / d.segs;
  x = (int)((s - row * d.segs) * 32u + (slot & 31u));
  z = (int)(row / (unsigned)d.c1);
  y = (int)(row - (unsigned)z * (unsigned)d.c1);
}

// info word of a crossed cell: tiling (10 bits) | number of vertices the cell creates (4 bits)
__device__ __forceinline__ unsigned short pack_info(int til, int nv) { return (unsigned short)(til | (nv << 10)); }

// Pass 0: the only pass over the float grid, as a flat stream.  One bit per point (value > level, the comparison of
// cube_index), bit p of the bit volume = point p = (z * n1 + y) * n2 + x, and the min / max of the volume (for skimage's
// level check) per block.  A warp takes 128 consecutive points per trip (one 16-byte load per lane, four trips in
// flight); the eight lanes of a group assemble their nibbles into one word with three shuffles.
template <bool kVec>
__global__ void __launch_bounds__(kThreads) mc_bits_kernel(const float* __restrict__ g, int64_t npts, float level,
                                                           unsigned* __restrict__ bits,
                                                           unsigned* __restrict__ block_minmax) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t gw = (int64_t)blockIdx.x * kWarps + warp, nw = (int64_t)gridDim.x * kWarps;
  const int64_t ngroups = npts / 128;
  float lo = INFINITY, hi = -INFINITY;      // fminf / fmaxf skip NaNs (FlashVDM grids carry them)
  for (int64_t grp = gw; grp < ngroups; grp += 4 * nw) {
    float4 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int64_t gg = grp + u * nw;
      if (gg < ngroups) {
        if (kVec) {
          v[u] = __ldg(reinterpret_cast<const float4*>(g) + gg * 32 + lane);
        } else {
          const float* q = g + gg * 128 + 4 * lane;
          v[u] = make_float4(__ldg(q), __ldg(q + 1), __ldg(q + 2), __ldg(q + 3));
        }
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int64_t gg = grp + u * nw;
      if (gg < ngroups) {       // warp-uniform
        const unsigned nib = (v[u].x > level ? 1u : 0u) | (v[u].y > level ? 2u : 0u) | (v[u].z > level ? 4u : 0u) |
                             (v[u].w > level ? 8u : 0u);
        unsigned word = nib << (4 * (lane & 7));
        word |= __shfl_xor_sync(0xffffffffu, word, 1);
        word |= __shfl_xor_sync(0xffffffffu, word, 2);
        word |= __shfl_xor_sync(0xffffffffu, word, 4);
        lo = fminf(fminf(lo, v[u].x), fminf(fminf(v[u].y, v[u].z), v[u].w));
        hi = fmaxf(fmaxf(hi, v[u].x), fmaxf(fmaxf(v[u].y, v[u].z), v[u].w));
        if ((lane & 7) == 0) bits[gg * 4 + (lane >> 3)] = word;
      }
    }
  }
  if (gw == 0) {      // the last npts % 128 points (up to four words) and two words of padding (mc_mark reads one past)
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      const int64_t q = ngroups * 128 + 32 * j + lane;
      const bool has = q < npts;
      const float t = has ? __ldg(g + q) : level;
      const unsigned b = __ballot_sync(0xffffffffu, t > level);
      if (has) { lo = fminf(lo, t); hi = fmaxf(hi, t); }
      if (lane == 0) bits[ngroups * 4 + j] = b;
    }
  }
  __shared__ unsigned slo[kWarps], shi[kWarps];
  unsigned ulo = __reduce_min_sync(0xffffffffu, f2ord(lo)), uhi = __reduce_max_sync(0xffffffffu, f2ord(hi));
  if (lane == 0) { slo[warp] = ulo; shi[warp] = uhi; }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int i = 1; i < kWarps; ++i) { ulo = min(ulo, slo[i]); uhi = max(uhi, shi[i]); }
    block_minmax[2 * blockIdx.x] = ulo;       // no same-address atomics: mc_scan1 reduces these
    block_minmax[2 * blockIdx.x + 1] = uhi;
  }
}

// 33 sign bits starting at point p: the 32 own points of a segment's cells and, shifted by one, their x + 1 neighbours
__device__ __forceinline__ void sign_words(const unsigned* __restrict__ bits, int64_t p, unsigned& own, unsigned& next) {
  const int64_t w = p >> 5;
  const unsigned sh = (unsigned)p & 31u;
  const unsigned w0 = __ldg(bits + w), w1 = __ldg(bits + w + 1);
  own = __funnelshift_r(w0, w1, sh);
  next = __funnelshift_r(own, (w1 >> sh) & 1u, 1);
}

// Pass 1: one thread per segment.  The cube index of a cell is 0 or 255 exactly when its eight sign bits agree, so the
// mask of crossed cells of a segment is (OR of the eight shifted words) & ~(AND of them).
__global__ void __launch_bounds__(kThreads) mc_mark_kernel(const unsigned* __restrict__ bits, McDims d,
                                                           unsigned* __restrict__ act, unsigned* __restrict__ block_sum) {
  const unsigned s = blockIdx.x * kThreads + threadIdx.x;
  unsigned m = 0;
  if (s < d.nsegs) {
    const unsigned row = s / d.segs, seg = s - row * d.segs;
    const unsigned z = row / (unsigned)d.c1, y = row - z * (unsigned)d.c1;
    const int64_t sy = d.n2, sz = (int64_t)d.n1 * d.n2;
    const int64_t p = ((int64_t)z * d.n1 + y) * d.n2 + seg * 32u;     // point (32 seg, y, z)
    unsigned a, a1, b, b1, c, c1, e, e1;
    sign_words(bits, p, a, a1);
    sign_words(bits, p + sy, b, b1);
    sign_words(bits, p + sz, c, c1);
    sign_words(bits, p + sz + sy, e, e1);
    const unsigned any = a | a1 | b | b1 | c | c1 | e | e1, all = a & a1 & b & b1 & c & c1 & e & e1;
    const unsigned rem = (unsigned)d.c2 - seg * 32u;      // cells of this segment that exist (bits past them: masked)
    m = any & ~all & (rem >= 32u ? 0xffffffffu : ((1u << rem) - 1u));
    act[s] = m;
  }
  unsigned cnt = __reduce_add_sync(0xffffffffu, (unsigned)__popc(m));
  __shared__ unsigned sw[kWarps];
  if ((threadIdx.x & 31) == 0) sw[threadIdx.x >> 5] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int i = 1; i < kWarps; ++i) cnt += sw[i];
    block_sum[blockIdx.x] = cnt;
  }
}

// Single-block exclusive scans (32 warps; warp w owns a contiguous range of entries and walks it 32 at a time, twice:
// totals, then offsets).  mc_scan1: the per-block crossed-cell counts of mc_mark (+ the min / max reduction);
// mc_scan2: the per-block (vertex, triangle) counts of mc_eval, whose number of entries lives on the device.
__device__ __forceinline__ void scan_range(int n, int& begin, int& end) {
  const int w = threadIdx.x >> 5;
  const int per = (((n + 31) / 32) + 31) & ~31;      // entries per warp, a multiple of 32
  begin = (int)min((long long)n, (long long)w * per);
  end = (int)min((long long)n, (long long)begin + per);
}

__global__ void __launch_bounds__(1024) mc_scan1_kernel(const unsigned* __restrict__ sums, unsigned* __restrict__ offsets,
                                                        int n, const uint2* __restrict__ block_minmax, int nminmax,
                                                        int64_t* __restrict__ totals) {
  __shared__ unsigned long long sv[32];
  __shared__ unsigned slo[32], shi[32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int begin, end;
  scan_range(n, begin, end);
  unsigned long long av = 0;
  for (int i = begin + lane; i < end; i += 32) av += sums[i];
  unsigned lo = 0xffffffffu, hi = 0u;
  for (int i = threadIdx.x; i < nminmax; i += 1024) {
    const uint2 m = block_minmax[i];
    lo = min(lo, m.x); hi = max(hi, m.y);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) av += __shfl_xor_sync(0xffffffffu, av, o);
  lo = __reduce_min_sync(0xffffffffu, lo);
  hi = __reduce_max_sync(0xffffffffu, hi);
  if (lane == 0) { sv[w] = av; slo[w] = lo; shi[w] = hi; }
  __syncthreads();
  unsigned long long run = 0, all = 0;
  for (int k = 0; k < 32; ++k) {
    if (k < w) run += sv[k];
    all += sv[k];
    lo = min(lo, slo[k]); hi = max(hi, shi[k]);
  }
  for (int base = begin; base < end; base += 32) {
    const int i = base + lane;
    const unsigned c = i < end ? sums[i] : 0u;
    unsigned inc = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += t;
    }
    if (i < end) offsets[i] = (unsigned)(run + inc - c);
    run += __shfl_sync(0xffffffffu, inc, 31);
  }
  if (threadIdx.x == 0) {
    totals[2] = (int64_t)lo;
    totals[3] = (int64_t)hi;
    totals[4] = (int64_t)all;       // crossed cells; read by the later kernels on the device
  }
}

__global__ void __launch_bounds__(1024) mc_scan2_kernel(const uint2* __restrict__ counts, uint2* __restrict__ offsets,
                                                        int64_t* __restrict__ totals) {
  __shared__ unsigned long long sv[32], st[32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int n = (int)((totals[4] + kThreads - 1) / kThreads);
  int begin, end;
  scan_range(n, begin, end);
  unsigned long long av = 0, at = 0;
  for (int i = begin + lane; i < end; i += 32) {
    const uint2 c = counts[i];
    av += c.x; at += c.y;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    av += __shfl_xor_sync(0xffffffffu, av, o);
    at += __shfl_xor_sync(0xffffffffu, at, o);
  }
  if (lane == 0) { sv[w] = av; st[w] = at; }
  __syncthreads();
  unsigned long long run_v = 0, run_t = 0, all_v = 0, all_t = 0;
  for (int k = 0; k < 32; ++k) {
    if (k < w) { run_v += sv[k]; run_t += st[k]; }
    all_v += sv[k]; all_t += st[k];
  }
  for (int base = begin; base < end; base += 32) {
    const int i = base + lane;
    const uint2 c = i < end ? counts[i] : make_uint2(0u, 0u);
    unsigned iv = c.x, it = c.y;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned nv = __shfl_up_sync(0xffffffffu, iv, o), nt = __shfl_up_sync(0xffffffffu, it, o);
      if (lane >= o) { iv += nv; it += nt; }
    }
    if (i < end) offsets[i] = make_uint2((unsigned)(run_v + iv - c.x), (unsigned)(run_t + it - c.y));
    run_v += __shfl_sync(0xffffffffu, iv, 31);
    run_t += __shfl_sync(0xffffffffu, it, 31);
  }
  if (threadIdx.x == 0) {
    totals[0] = (int64_t)all_v;
    totals[1] = (int64_t)all_t;
  }
}

// Pass 2: the crossed cells, in traversal order, as a list of slots.
__global__ void __launch_bounds__(kThreads) mc_compact_kernel(const unsigned* __restrict__ act, McDims d,
                                                              const unsigned* __restrict__ block_off,
                                                              unsigned* __restrict__ list) {
  const unsigned s = blockIdx.x * kThreads + threadIdx.x;
  unsigned m = s < d.nsegs ? act[s] : 0u;
  const unsigned cnt[1] = {(unsigned)__popc(m)};
  unsigned excl[1], tot[1];
  block_scan<1>(cnt, excl, tot);
  int64_t k = (int64_t)block_off[blockIdx.x] + excl[0];
  while (m) {
    const unsigned i = (unsigned)__ffs((int)m) - 1u;
    list[k++] = s * 32u + i;
    m &= m - 1u;
  }
}

// Dual marching cubes: the grid edges a cell owns, as a mask over the array axes (bit a: the edge along axis a).  A
// sign-changing grid edge whose four incident cells all lie in the grid gives one quad; its owner is the first of the
// four in traversal order, the one whose maximum corner (corner 6) the edge touches: local edge 10 (axis 0, corners
// 2-6), 5 (axis 1, corners 5-6) or 6 (axis 2, corners 7-6).
__device__ __forceinline__ unsigned dual_owned(int ci, const McDims& d, int x, int y, int z) {
  const int up = (ci >> 6) & 1;
  unsigned m = 0;
  if (x + 1 < d.c2 && y + 1 < d.c1 && up != ((ci >> 2) & 1)) m |= 1u;
  if (x + 1 < d.c2 && z + 1 < d.c0 && up != ((ci >> 5) & 1)) m |= 2u;
  if (y + 1 < d.c1 && z + 1 < d.c0 && up != ((ci >> 7) & 1)) m |= 4u;
  return m;
}

// Pass 3: the Lewiner tests, one thread per crossed cell: the info word of the cell and, per block of 256 list entries,
// the (vertex, triangle) counts.  kDual: the cell's vertices are its patches (r3g_mc_dual_npatch) and its triangles two
// per owned quad.
template <bool kDual>
__global__ void __launch_bounds__(kThreads) mc_eval_kernel(const float* __restrict__ g, McDims d, float level,
                                                           const unsigned* __restrict__ list,
                                                           const int64_t* __restrict__ totals,
                                                           unsigned short* __restrict__ info,
                                                           uint2* __restrict__ block_counts) {
  const int64_t nactive = totals[4];
  const int64_t nblocks = (nactive + kThreads - 1) / kThreads;
  for (int64_t kb = blockIdx.x; kb < nblocks; kb += gridDim.x) {
    const int64_t k = kb * kThreads + threadIdx.x;
    unsigned cnt[2] = {0, 0};
    if (k < nactive) {
      int x, y, z;
      slot_coords(d, list[k], x, y, z);
      float raw[8];
      load_cell(g, d, x, y, z, raw);
      double cv[8];
      const int ci = cube_index(raw, level);
      if (kDual) {
        const int til = cell_tiling(ci, raw, level, cv);      // a listed cell is crossed: ci is neither 0 nor 255
        const int np = r3g_mc_dual_npatch[til];
        info[k] = pack_info(til, np);
        cnt[0] = np; cnt[1] = 2u * __popc(dual_owned(ci, d, x, y, z));
      } else {
        const Cell c = eval_cell(ci, raw, level, cv, x, y, z);
        info[k] = pack_info(c.til, c.nv);
        cnt[0] = c.nv; cnt[1] = c.nt;
      }
    }
    unsigned excl[2], tot[2];
    block_scan<2>(cnt, excl, tot);
    if (threadIdx.x == 0) block_counts[kb] = make_uint2(tot[0], tot[1]);
  }
}

__device__ __forceinline__ int64_t edge_slot(const McDims& d, int e, int x, int y, int z) {
  if (e == 12) return 4 * (((int64_t)z * d.n1 + y) * d.n2 + x) + 3;
  int info = r3g_mc_edge_info[e];
  int gx = x + (info & 1), gy = y + ((info >> 1) & 1), gz = z + ((info >> 2) & 1);
  return 4 * (((int64_t)gz * d.n1 + gy) * d.n2 + gx) + (info >> 3);
}

struct Rescale {
  int enabled;
  double lo[3], size[3], n[3];
};

// Pass 4: every crossed cell writes the vertices it owns, in first-use order of its tiling, and publishes their ids.
__global__ void __launch_bounds__(kThreads) mc_vertex_kernel(const float* __restrict__ g, McDims d, float level,
                                                             const unsigned* __restrict__ list,
                                                             const int64_t* __restrict__ totals,
                                                             const unsigned short* __restrict__ info,
                                                             const uint2* __restrict__ block_offsets,
                                                             int32_t* __restrict__ vid, float* __restrict__ verts,
                                                             Rescale rs) {
  const int64_t nactive = totals[4];
  const int64_t nblocks = (nactive + kThreads - 1) / kThreads;
  for (int64_t kb = blockIdx.x; kb < nblocks; kb += gridDim.x) {
    const int64_t k = kb * kThreads + threadIdx.x;
    const unsigned word = k < nactive ? info[k] : 0u;
    const unsigned nv[1] = {word >> 10};
    unsigned excl[1], tot[1];
    block_scan<1>(nv, excl, tot);
    if (nv[0] == 0) continue;
    int x, y, z;
    slot_coords(d, list[k], x, y, z);
    const int til = word & 1023;
    double cv[8];
    {
      float raw[8];
      load_cell(g, d, x, y, z, raw);
#pragma unroll
      for (int i = 0; i < 8; ++i) cv[i] = (double)raw[i] - (double)level;
    }
    unsigned id = block_offsets[kb].x + excl[0];
    const int t0 = r3g_mc_tiling_start[til], t1 = r3g_mc_tiling_start[til + 1];
    // the edges this cell owns, in first-use order of its tiling (4 bits each; at most 13): integer work only, so that the
    // float64 part below runs max-over-the-warp(nv) times, not once per tiling position at which some lane owns an edge
    unsigned long long owned = 0;
    unsigned seen = 0;
    int n = 0;
    for (int t = t0; t < t1; ++t) {
      const int e = r3g_mc_tri[t];
      const unsigned bit = 1u << e;
      if (seen & bit) continue;
      seen |= bit;
      if (e == 12 || owns_edge(e, x, y, z)) { owned |= (unsigned long long)e << (4 * n); ++n; }
    }
    for (int k = 0; k < n; ++k) {
      const int e = (int)((owned >> (4 * k)) & 15ull);
      double fx = 0, fy = 0, fz = 0, ff = 0;
      if (e == 12) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const unsigned char* o = &r3g_mc_corner_xyz[3 * i];
          double w = 1.0 / (R3G_MC_EPS + fabs(cv[i]));
          fx += o[0] * w; fy += o[1] * w; fz += o[2] * w; ff += w;
        }
      } else {
        const int a = r3g_mc_edge_corner[2 * e], b = r3g_mc_edge_corner[2 * e + 1];
        const unsigned char *oa = &r3g_mc_corner_xyz[3 * a], *ob = &r3g_mc_corner_xyz[3 * b];
        double wa = 1.0 / (R3G_MC_EPS + fabs(cv[a]));
        double wb = 1.0 / (R3G_MC_EPS + fabs(cv[b]));
        fx = oa[0] * wa + ob[0] * wb;   // offsets are 0/1: products exact, fma-safe
        fy = oa[1] * wa + ob[1] * wb;
        fz = oa[2] * wa + ob[2] * wb;
        ff = wa + wb;
      }
      float p[3];
      p[0] = (float)((double)z + fz / ff);
      p[1] = (float)((double)y + fy / ff);
      p[2] = (float)((double)x + fx / ff);
      if (rs.enabled) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          double q = __dadd_rn(__dmul_rn(__ddiv_rn((double)p[a], rs.n[a]), rs.size[a]), rs.lo[a]);
          p[a] = (float)q;
        }
      }
      verts[3 * (int64_t)id + 0] = p[0];
      verts[3 * (int64_t)id + 1] = p[1];
      verts[3 * (int64_t)id + 2] = p[2];
      vid[edge_slot(d, e, x, y, z)] = (int32_t)id;
      ++id;
    }
  }
}

// Pass 5: faces, in cell order then tiling order, looking vertex ids up by grid edge.  Reads no grid values.
__global__ void __launch_bounds__(kThreads) mc_face_kernel(McDims d, const unsigned* __restrict__ list,
                                                           const int64_t* __restrict__ totals,
                                                           const unsigned short* __restrict__ info,
                                                           const uint2* __restrict__ block_offsets,
                                                           const int32_t* __restrict__ vid,
                                                           int32_t* __restrict__ faces) {
  const int64_t nactive = totals[4];
  const int64_t nblocks = (nactive + kThreads - 1) / kThreads;
  for (int64_t kb = blockIdx.x; kb < nblocks; kb += gridDim.x) {
    const int64_t k = kb * kThreads + threadIdx.x;
    const int til = k < nactive ? (info[k] & 1023) : 0;
    const int t0 = r3g_mc_tiling_start[til], t1 = r3g_mc_tiling_start[til + 1];
    const unsigned nt[1] = {(unsigned)(t1 - t0) / 3u};
    unsigned excl[1], tot[1];
    block_scan<1>(nt, excl, tot);
    if (nt[0] == 0) continue;
    int x, y, z;
    slot_coords(d, list[k], x, y, z);
    int64_t fo = 3 * (int64_t)(block_offsets[kb].y + excl[0]);
    for (int t = t0; t < t1; ++t) faces[fo++] = vid[edge_slot(d, r3g_mc_tri[t], x, y, z)];
  }
}

// Dual marching cubes keeps, per crossed cell, (first vertex id, tiling | cube index << 16) in the first 8 of the 16
// vertex-id bytes of the cell's origin point: the face pass finds the vertex of a neighbour's patch from it.
__device__ __forceinline__ int2* dual_cell(int32_t* vid, const McDims& d, int x, int y, int z) {
  return reinterpret_cast<int2*>(vid + 4 * (((int64_t)z * d.n1 + y) * d.n2 + x));
}

// crossing of the cell edge a -> b along one array axis: p_a + t (p_b - p_a), corners at integer positions
__device__ __forceinline__ double dual_cross(int pa, int pb, double t) {
  return __dadd_rn((double)pa, __dmul_rn(t, __dsub_rn((double)pb, (double)pa)));
}

// Dual pass 4: every crossed cell writes one vertex per patch, in patch order (patches are numbered by their smallest
// cube edge): the mean of the patch's edge crossings, t = v_a / (v_a - v_b), summed in increasing edge order, divided by
// the edge count and by (n_axis - 1), every float64 operation explicitly rounded; stored float32 in array-axis order.
__global__ void __launch_bounds__(kThreads) mc_dual_vertex_kernel(const float* __restrict__ g, McDims d, float level,
                                                                  const unsigned* __restrict__ list,
                                                                  const int64_t* __restrict__ totals,
                                                                  const unsigned short* __restrict__ info,
                                                                  const uint2* __restrict__ block_offsets,
                                                                  int32_t* __restrict__ vid, float* __restrict__ verts) {
  const int64_t nactive = totals[4];
  const int64_t nblocks = (nactive + kThreads - 1) / kThreads;
  for (int64_t kb = blockIdx.x; kb < nblocks; kb += gridDim.x) {
    const int64_t k = kb * kThreads + threadIdx.x;
    const unsigned word = k < nactive ? info[k] : 0u;
    const unsigned np[1] = {word >> 10};
    unsigned excl[1], tot[1];
    block_scan<1>(np, excl, tot);
    if (np[0] == 0) continue;
    int x, y, z;
    slot_coords(d, list[k], x, y, z);
    const int til = word & 1023;
    float raw[8];
    load_cell(g, d, x, y, z, raw);
    double cv[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) cv[i] = (double)raw[i] - (double)level;
    const unsigned id = block_offsets[kb].x + excl[0];
    *dual_cell(vid, d, x, y, z) = make_int2((int)id, til | (cube_index(raw, level) << 16));
    const unsigned char* patch = &r3g_mc_dual_patch[12 * til];
    for (unsigned p = 0; p < np[0]; ++p) {
      double s0 = 0.0, s1 = 0.0, s2 = 0.0;
      int n = 0;
      for (int e = 0; e < 12; ++e) {
        if (patch[e] != p) continue;
        const int a = r3g_mc_edge_corner[2 * e], b = r3g_mc_edge_corner[2 * e + 1];
        const unsigned char *oa = &r3g_mc_corner_xyz[3 * a], *ob = &r3g_mc_corner_xyz[3 * b];
        const double t = __ddiv_rn(cv[a], __dsub_rn(cv[a], cv[b]));
        s0 = __dadd_rn(s0, dual_cross(z + oa[2], z + ob[2], t));
        s1 = __dadd_rn(s1, dual_cross(y + oa[1], y + ob[1], t));
        s2 = __dadd_rn(s2, dual_cross(x + oa[0], x + ob[0], t));
        ++n;
      }
      float* out = verts + 3 * (int64_t)(id + p);
      out[0] = (float)__ddiv_rn(__ddiv_rn(s0, (double)n), (double)d.c0);
      out[1] = (float)__ddiv_rn(__ddiv_rn(s1, (double)n), (double)d.c1);
      out[2] = (float)__ddiv_rn(__ddiv_rn(s2, (double)n), (double)d.c2);
    }
  }
}

// The quad of the grid edge an owner cell holds along array axis a: the four cells around the edge as offsets
// (dx, dy, dz) from the owner, and the cube edge the grid edge is in each of them, counter-clockwise seen from the
// edge's upper end (q0 = the owner).
__device__ const unsigned char kDualQuad[3][4][4] = {
    {{0, 0, 0, 10}, {0, 1, 0, 9}, {1, 1, 0, 8}, {1, 0, 0, 11}},   // axis 0 (z): cells in the (y, x) plane
    {{0, 0, 0, 5}, {1, 0, 0, 7}, {1, 0, 1, 3}, {0, 0, 1, 1}},     // axis 1 (y): cells in the (x, z) plane
    {{0, 0, 0, 6}, {0, 0, 1, 2}, {0, 1, 1, 0}, {0, 1, 0, 4}},     // axis 2 (x): cells in the (z, y) plane
};

__device__ __forceinline__ double dual_dist2(const float* __restrict__ verts, int i, int j) {
  const float *p = verts + 3 * (int64_t)i, *q = verts + 3 * (int64_t)j;
  const double d0 = __dsub_rn((double)p[0], (double)q[0]), d1 = __dsub_rn((double)p[1], (double)q[1]);
  const double d2 = __dsub_rn((double)p[2], (double)q[2]);
  return __dadd_rn(__dadd_rn(__dmul_rn(d0, d0), __dmul_rn(d1, d1)), __dmul_rn(d2, d2));
}

// Dual pass 5: every crossed cell writes the two triangles of each quad it owns, axes 0, 1, 2 in turn.  The quad is
// wound so that its normal points towards increasing values (the edge's upper end above the level: counter-clockwise
// from there) and split along its shorter diagonal (squared float64 lengths of the float32 vertices; a tie takes 0-2).
__global__ void __launch_bounds__(kThreads) mc_dual_face_kernel(McDims d, const unsigned* __restrict__ list,
                                                                const int64_t* __restrict__ totals,
                                                                const uint2* __restrict__ block_offsets,
                                                                int32_t* __restrict__ vid,
                                                                const float* __restrict__ verts,
                                                                int32_t* __restrict__ faces) {
  const int64_t nactive = totals[4];
  const int64_t nblocks = (nactive + kThreads - 1) / kThreads;
  for (int64_t kb = blockIdx.x; kb < nblocks; kb += gridDim.x) {
    const int64_t k = kb * kThreads + threadIdx.x;
    int x = 0, y = 0, z = 0;
    int2 own_cell = make_int2(0, 0);
    unsigned own = 0;
    if (k < nactive) {
      slot_coords(d, list[k], x, y, z);
      own_cell = *dual_cell(vid, d, x, y, z);
      own = dual_owned(own_cell.y >> 16, d, x, y, z);
    }
    const unsigned nt[1] = {2u * __popc(own)};
    unsigned excl[1], tot[1];
    block_scan<1>(nt, excl, tot);
    if (own == 0) continue;
    const bool up = (own_cell.y >> 22) & 1;      // corner 6, the upper end of every owned edge, is above the level
    int64_t fo = 3 * (int64_t)(block_offsets[kb].y + excl[0]);
    for (int a = 0; a < 3; ++a) {
      if (!((own >> a) & 1u)) continue;
      int q[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const unsigned char* c = kDualQuad[a][j];
        const int2 cell = j == 0 ? own_cell : *dual_cell(vid, d, x + c[0], y + c[1], z + c[2]);
        q[j] = cell.x + r3g_mc_dual_patch[12 * (cell.y & 0xffff) + c[3]];
      }
      if (!up) { const int t = q[1]; q[1] = q[3]; q[3] = t; }
      const bool d13 = dual_dist2(verts, q[1], q[3]) < dual_dist2(verts, q[0], q[2]);
      const int t0[3] = {q[0], q[1], d13 ? q[3] : q[2]};
      const int t1[3] = {d13 ? q[1] : q[0], q[2], q[3]};
#pragma unroll
      for (int i = 0; i < 3; ++i) faces[fo + i] = t0[i];
#pragma unroll
      for (int i = 0; i < 3; ++i) faces[fo + 3 + i] = t1[i];
      fo += 6;
    }
  }
}

__global__ void __launch_bounds__(kThreads) mc_case_kernel(const float* __restrict__ g, McDims d, float level,
                                                           unsigned char* __restrict__ out) {
  const int64_t cell = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  int x, y, z;
  if (!cell_coords(d, cell, x, y, z)) return;
  float raw[8];
  load_cell(g, d, x, y, z, raw);
  out[cell] = r3g_mc_case[cube_index(raw, level)];
}

struct McWorkspace {
  int32_t* vid;           // 4 per grid point: the vertex id on the x / y / z edge starting there, and of the cell centre
  unsigned* bits;         // one bit per point (+ padding)
  unsigned* act;          // nsegs: mask of crossed cells
  unsigned* list;         // ncells (worst case): slots of the crossed cells in traversal order
  unsigned short* info;   // ncells (worst case)
  unsigned* seg_sum;      // per block of 256 segments: crossed cells
  unsigned* seg_off;
  uint2* cell_counts;     // per block of 256 crossed cells: (vertices, triangles)
  uint2* cell_off;
  unsigned* minmax;       // per block of mc_bits
  int64_t* totals;        // vertices, triangles, min, max (ordered uints), crossed cells
  int seg_blocks, cell_blocks_max, bits_grid;
};

int make_dims(r3g_ctx* ctx, int n0, int n1, int n2, McDims& d) {
  if (n0 < 2 || n1 < 2 || n2 < 2) return r3g_fail(ctx, R3G_E_INVALID, "mc: grid must be at least 2x2x2");
  d.n0 = n0; d.n1 = n1; d.n2 = n2;
  d.c0 = n0 - 1; d.c1 = n1 - 1; d.c2 = n2 - 1;
  d.ncells = (int64_t)d.c0 * d.c1 * d.c2;
  d.npts = (int64_t)n0 * n1 * n2;
  d.segs = (unsigned)((d.c2 + 31) / 32);
  const int64_t nsegs = (int64_t)d.c0 * d.c1 * d.segs;
  // slots (segment * 32 + lane) are 32-bit
  if (nsegs >= (1LL << 27)) return r3g_fail(ctx, R3G_E_INVALID, "mc: grid too large");
  d.nsegs = (unsigned)nsegs;
  return R3G_OK;
}

constexpr int kBitsGridMax = 148 * 8 * 2;     // upper bound used for the workspace (the launch uses num_sms * 8)

// points w's buffers into `base` (null: only measures) and returns the bytes they take
size_t carve_sizes(int n0, int n1, int n2, McWorkspace& w, char* base) {
  const int64_t npts = (int64_t)n0 * n1 * n2;
  const int64_t ncells = (int64_t)(n0 - 1) * (n1 - 1) * (n2 - 1);
  const int64_t nwords = (npts / 128) * 4 + 6;      // whole 128-point groups + the tail's words + padding
  const int64_t nsegs = (int64_t)(n0 - 1) * (n1 - 1) * ((n2 - 1 + 31) / 32);
  const size_t seg_blocks = (size_t)((nsegs + kThreads - 1) / kThreads);
  const size_t cell_blocks = (size_t)((ncells + kThreads - 1) / kThreads);
  r3g_carver c{base};
  w.vid = c.take<int32_t>(4 * (size_t)npts);
  w.bits = c.take<unsigned>((size_t)nwords);
  w.act = c.take<unsigned>((size_t)nsegs);
  w.list = c.take<unsigned>((size_t)ncells);
  w.info = c.take<unsigned short>((size_t)ncells);
  w.seg_sum = c.take<unsigned>(seg_blocks);
  w.seg_off = c.take<unsigned>(seg_blocks);
  w.cell_counts = c.take<uint2>(cell_blocks);
  w.cell_off = c.take<uint2>(cell_blocks);
  w.minmax = c.take<unsigned>(2 * kBitsGridMax);
  w.totals = c.take<int64_t>(5);
  w.seg_blocks = (int)seg_blocks;
  w.cell_blocks_max = (int)cell_blocks;
  return c.off;
}

int carve(r3g_ctx* ctx, const McDims& d, void* ws, size_t ws_bytes, McWorkspace& w) {
  const size_t need = carve_sizes(d.n0, d.n1, d.n2, w, (char*)ws);
  if (need > ws_bytes || !ws) return r3g_fail(ctx, R3G_E_WORKSPACE, "mc: workspace %zu < required %zu", ws_bytes, need);
  const int groups_per_block = kWarps * 4;
  const int64_t want = (d.npts / 128 + groups_per_block - 1) / groups_per_block + 1;
  const int full = ctx->num_sms * 8 < kBitsGridMax ? ctx->num_sms * 8 : kBitsGridMax;
  w.bits_grid = (int)(want < full ? want : full);
  return R3G_OK;
}

// resident blocks of 256 threads per SM x SMs: the grid of the kernels that walk the crossed-cell list
int list_grid(const r3g_ctx* ctx, int per_sm) { return ctx->num_sms * per_sm; }

}  // namespace

extern "C" size_t r3g_mc_workspace_bytes(int n0, int n1, int n2) {
  if (n0 < 2 || n1 < 2 || n2 < 2) return 0;
  McWorkspace w;
  return carve_sizes(n0, n1, n2, w, nullptr);
}

extern "C" int r3g_mc_count(r3g_ctx* ctx, const float* grid, int n0, int n1, int n2, float level, int method,
                            void* workspace, size_t workspace_bytes, int64_t* nv_host, int64_t* nf_host, void* stream) {
  R3G_ENTRY(ctx, "mc_count");
  if (!grid || !nv_host || !nf_host) return r3g_fail(ctx, R3G_E_INVALID, "mc_count: null argument");
  if (method != R3G_MC_LEWINER && method != R3G_MC_DUAL)
    return r3g_fail(ctx, R3G_E_INVALID, "mc_count: unknown method %d", method);
  const bool dual = method == R3G_MC_DUAL;
  cudaStream_t s = (cudaStream_t)stream;
  McDims d;
  McWorkspace w;
  int rc = make_dims(ctx, n0, n1, n2, d);
  if (rc) return rc;
  rc = carve(ctx, d, workspace, workspace_bytes, w);
  if (rc) return rc;
  if (r3g_aligned16(grid))   // 16-byte loads when the grid's base allows them
    mc_bits_kernel<true><<<w.bits_grid, kThreads, 0, s>>>(grid, d.npts, level, w.bits, w.minmax);
  else
    mc_bits_kernel<false><<<w.bits_grid, kThreads, 0, s>>>(grid, d.npts, level, w.bits, w.minmax);
  R3G_LAUNCH_OK(ctx);
  mc_mark_kernel<<<w.seg_blocks, kThreads, 0, s>>>(w.bits, d, w.act, w.seg_sum);
  R3G_LAUNCH_OK(ctx);
  mc_scan1_kernel<<<1, 1024, 0, s>>>(w.seg_sum, w.seg_off, w.seg_blocks, (const uint2*)w.minmax, w.bits_grid, w.totals);
  R3G_LAUNCH_OK(ctx);
  mc_compact_kernel<<<w.seg_blocks, kThreads, 0, s>>>(w.act, d, w.seg_off, w.list);
  R3G_LAUNCH_OK(ctx);
  // from here on the number of crossed cells stays on the device (totals[4]): machine-sized grids walk the list
  if (dual)
    mc_eval_kernel<true><<<list_grid(ctx, 4), kThreads, 0, s>>>(grid, d, level, w.list, w.totals, w.info,
                                                                w.cell_counts);
  else
    mc_eval_kernel<false><<<list_grid(ctx, 4), kThreads, 0, s>>>(grid, d, level, w.list, w.totals, w.info,
                                                                 w.cell_counts);
  R3G_LAUNCH_OK(ctx);
  mc_scan2_kernel<<<1, 1024, 0, s>>>(w.cell_counts, w.cell_off, w.totals);
  R3G_LAUNCH_OK(ctx);
  R3G_CUDA_OK(ctx, cudaMemcpyAsync(ctx->pinned, w.totals, 4 * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  R3G_CUDA_OK(ctx, cudaStreamSynchronize(s));
  *nv_host = ctx->pinned[0];
  *nf_host = ctx->pinned[1];
  const float vmin = ord2f((unsigned)ctx->pinned[2]), vmax = ord2f((unsigned)ctx->pinned[3]);
  if (!dual && !(level >= vmin && level <= vmax)) {
    *nv_host = *nf_host = 0;
    return r3g_fail(ctx, R3G_E_LEVEL, "Surface level must be within volume data range. (level %g, range [%g, %g])",
                    level, vmin, vmax);
  }
  if (*nv_host == 0) return r3g_fail(ctx, R3G_E_NOSURFACE, "No surface found at the given iso value.");
  return R3G_OK;
}

extern "C" int r3g_mc_extract(r3g_ctx* ctx, const float* grid, int n0, int n1, int n2, float level, int method,
                              const double* bounds_host, void* workspace, size_t workspace_bytes, float* verts,
                              int32_t* faces, void* stream) {
  R3G_ENTRY(ctx, "mc_extract");
  if (!grid || !verts || !faces) return r3g_fail(ctx, R3G_E_INVALID, "mc_extract: null argument");
  if (method != R3G_MC_LEWINER && method != R3G_MC_DUAL)
    return r3g_fail(ctx, R3G_E_INVALID, "mc_extract: unknown method %d", method);
  if (method == R3G_MC_DUAL && bounds_host)
    return r3g_fail(ctx, R3G_E_INVALID, "mc_extract: the dual method takes no bounds (its vertices are in [0, 1])");
  cudaStream_t s = (cudaStream_t)stream;
  McDims d;
  McWorkspace w;
  int rc = make_dims(ctx, n0, n1, n2, d);
  if (rc) return rc;
  rc = carve(ctx, d, workspace, workspace_bytes, w);
  if (rc) return rc;
  if (method == R3G_MC_DUAL) {
    mc_dual_vertex_kernel<<<list_grid(ctx, 4), kThreads, 0, s>>>(grid, d, level, w.list, w.totals, w.info, w.cell_off,
                                                                 w.vid, verts);
    R3G_LAUNCH_OK(ctx);
    mc_dual_face_kernel<<<list_grid(ctx, 8), kThreads, 0, s>>>(d, w.list, w.totals, w.cell_off, w.vid, verts, faces);
    R3G_LAUNCH_OK(ctx);
    return R3G_OK;
  }
  Rescale rs;
  rs.enabled = bounds_host != nullptr;
  const int nax[3] = {n0, n1, n2};
  for (int a = 0; a < 3; ++a) {
    rs.lo[a] = bounds_host ? bounds_host[a] : 0.0;
    rs.size[a] = bounds_host ? bounds_host[3 + a] - bounds_host[a] : 1.0;
    rs.n[a] = (double)nax[a];
  }
  mc_vertex_kernel<<<list_grid(ctx, 4), kThreads, 0, s>>>(grid, d, level, w.list, w.totals, w.info, w.cell_off, w.vid,
                                                          verts, rs);
  R3G_LAUNCH_OK(ctx);
  mc_face_kernel<<<list_grid(ctx, 8), kThreads, 0, s>>>(d, w.list, w.totals, w.info, w.cell_off, w.vid, faces);
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}

extern "C" int r3g_mc_classify(r3g_ctx* ctx, const float* grid, int n0, int n1, int n2, float level,
                               unsigned char* case_out, void* stream) {
  R3G_ENTRY(ctx, "mc_classify");
  if (!grid || !case_out) return r3g_fail(ctx, R3G_E_INVALID, "mc_classify: null argument");
  McDims d;
  int rc = make_dims(ctx, n0, n1, n2, d);
  if (rc) return rc;
  if ((d.ncells + kThreads - 1) / kThreads > 0x7fffffffLL) return r3g_fail(ctx, R3G_E_INVALID, "mc: grid too large");
  const int nblocks = (int)((d.ncells + kThreads - 1) / kThreads);
  mc_case_kernel<<<nblocks, kThreads, 0, (cudaStream_t)stream>>>(grid, d, level, case_out);
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}
