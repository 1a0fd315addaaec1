// Quadric edge-collapse decimation on the device (include/r3g.h describes the algorithm): the face reduction of
// stage 3 (src/2d_to_3d_models/run.py:95).  Each round rebuilds the adjacency from the face array (half-edges sorted by
// vertex pair, a vertex -> face CSR), prices every edge, selects an independent set by two rounds of 64-bit atomicMin
// and applies it in place.  Every float64 operation is an explicit _rn intrinsic, so the numpy mirror
// the tests compare against, performing the same operations in the same order agrees bit for bit; integer atomics only
// count or take minima, so nothing depends on thread order.
#include <cub/cub.cuh>

#include "r3g_internal.h"

namespace {

typedef unsigned long long u64;
constexpr u64 NO_KEY = ~0ull;
constexpr int V_BOUNDARY = 1, V_FROZEN = 2;
constexpr int MIN_COMPONENT = 4;      // vertices a component keeps
// device counters
enum { C_NLIVE, C_NSEL, C_REMOVED, C_BAD, C_COUNT };

struct d3 { double x, y, z; };
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ d3 sub3(d3 a, d3 b) { return {dsub(a.x, b.x), dsub(a.y, b.y), dsub(a.z, b.z)}; }
__device__ __forceinline__ double dot3(d3 u, d3 v) { return dadd(dadd(dmul(u.x, v.x), dmul(u.y, v.y)), dmul(u.z, v.z)); }
__device__ __forceinline__ d3 cross3(d3 u, d3 v) {
  return {dsub(dmul(u.y, v.z), dmul(u.z, v.y)), dsub(dmul(u.z, v.x), dmul(u.x, v.z)), dsub(dmul(u.x, v.y), dmul(u.y, v.x))};
}
__device__ __forceinline__ d3 ld3(const double* p, int v) { return {p[3 * v], p[3 * v + 1], p[3 * v + 2]}; }

// Q += s u u^T for the plane u = (n, d); Q = (a2 ab ac ad b2 bc bd c2 cd d2)
__device__ __forceinline__ void add_plane(double* q, d3 n, double d, double s) {
  const double u[4] = {n.x, n.y, n.z, d};
  int k = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = i; j < 4; ++j, ++k) q[k] = dadd(q[k], dmul(dmul(u[i], u[j]), s));
}

// v^T Q v with v = (p, 1)
__device__ __forceinline__ double quadric_err(const double* q, d3 p) {
  const double r0 = dadd(dadd(dadd(dmul(q[0], p.x), dmul(q[1], p.y)), dmul(q[2], p.z)), q[3]);
  const double r1 = dadd(dadd(dadd(dmul(q[1], p.x), dmul(q[4], p.y)), dmul(q[5], p.z)), q[6]);
  const double r2 = dadd(dadd(dadd(dmul(q[2], p.x), dmul(q[5], p.y)), dmul(q[7], p.z)), q[8]);
  const double r3 = dadd(dadd(dadd(dmul(q[3], p.x), dmul(q[6], p.y)), dmul(q[8], p.z)), q[9]);
  return dadd(dadd(dadd(dmul(r0, p.x), dmul(r1, p.y)), dmul(r2, p.z)), r3);
}

// the minimiser of v^T Q v by the adjugate, or the cheapest of a, b and the midpoint when Q's 3x3 block is ill-conditioned
__device__ __forceinline__ d3 placement(const double* q, d3 a, d3 b) {
  const double c00 = dsub(dmul(q[4], q[7]), dmul(q[5], q[5]));
  const double c01 = dsub(dmul(q[2], q[5]), dmul(q[1], q[7]));
  const double c02 = dsub(dmul(q[1], q[5]), dmul(q[2], q[4]));
  const double c11 = dsub(dmul(q[0], q[7]), dmul(q[2], q[2]));
  const double c12 = dsub(dmul(q[1], q[2]), dmul(q[0], q[5]));
  const double c22 = dsub(dmul(q[0], q[4]), dmul(q[1], q[1]));
  const double det = dadd(dadd(dmul(q[0], c00), dmul(q[1], c01)), dmul(q[2], c02));
  const double tr = dadd(dadd(q[0], q[4]), q[7]);
  const double thr = dmul(dmul(dmul(1e-6, tr), tr), tr);
  if (fabs(det) > thr) {
    return {__ddiv_rn(-dadd(dadd(dmul(c00, q[3]), dmul(c01, q[6])), dmul(c02, q[8])), det),
            __ddiv_rn(-dadd(dadd(dmul(c01, q[3]), dmul(c11, q[6])), dmul(c12, q[8])), det),
            __ddiv_rn(-dadd(dadd(dmul(c02, q[3]), dmul(c12, q[6])), dmul(c22, q[8])), det)};
  }
  const d3 mid = {dmul(dadd(a.x, b.x), 0.5), dmul(dadd(a.y, b.y), 0.5), dmul(dadd(a.z, b.z), 0.5)};
  d3 best = a;
  double eb = quadric_err(q, a);
  const double e1 = quadric_err(q, b);
  if (e1 < eb) { best = b; eb = e1; }
  if (quadric_err(q, mid) < eb) best = mid;
  return best;
}

__device__ __forceinline__ bool face_has(const int* f, int x) { return f[0] == x || f[1] == x || f[2] == x; }

// ---- set-up -------------------------------------------------------------------------------------------------------
__global__ void init_faces_kernel(const int32_t* __restrict__ in, int64_t nf, int64_t nv, int* __restrict__ out,
                                  int* __restrict__ cnt) {
  const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  const int a = in[3 * f], b = in[3 * f + 1], c = in[3 * f + 2];
  if (a < 0 || b < 0 || c < 0 || a >= nv || b >= nv || c >= nv) {
    atomicExch(&cnt[C_BAD], 1);
    return;
  }
  const bool live = a != b && b != c && a != c;        // a repeated index: dropped (autoclean)
  out[3 * f] = live ? a : -1;
  out[3 * f + 1] = live ? b : -1;
  out[3 * f + 2] = live ? c : -1;
  if (live) atomicAdd(&cnt[C_NLIVE], 1);
}

__global__ void init_verts_kernel(const float* __restrict__ v, int64_t nv, double* __restrict__ pos,
                                  int* __restrict__ remap) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nv) return;
  pos[3 * i] = v[3 * i];
  pos[3 * i + 1] = v[3 * i + 1];
  pos[3 * i + 2] = v[3 * i + 2];
  remap[i] = (int)i;
}

// ---- adjacency of one round ---------------------------------------------------------------------------------------
// half-edge 3f + j runs from corner j to corner j + 1; key (min vertex << 32 | max vertex), dead faces sort last
__global__ void halfedge_kernel(const int* __restrict__ faces, int n_he, u64* __restrict__ key, int* __restrict__ val) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_he) return;
  const int f = i / 3, j = i - 3 * f;
  const int u = faces[3 * f + j], w = faces[3 * f + (j == 2 ? 0 : j + 1)];
  key[i] = u < 0 ? NO_KEY : ((u64)min(u, w) << 32) | (u64)max(u, w);
  val[i] = i;
}

__global__ void head_kernel(const u64* __restrict__ key, int n_he, int* __restrict__ head) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n_he) return;
  head[i] = i < n_he && key[i] != NO_KEY && (i == 0 || key[i] != key[i - 1]);
}

// eidx = exclusive scan of head (eidx[n_he] = number of edges); estart[e] = first sorted half-edge of edge e,
// estart[E] = number of live half-edges; he_edge[half-edge] = its edge
__global__ void edge_kernel(const u64* __restrict__ key, const int* __restrict__ val, const int* __restrict__ head,
                            const int* __restrict__ eidx, int n_he, int* __restrict__ estart, int* __restrict__ he_edge) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_he || key[i] == NO_KEY) return;
  const int e = eidx[i] + head[i] - 1;        // the heads up to and including i, less one
  he_edge[val[i]] = e;
  if (head[i]) estart[e] = i;
  if (i + 1 == n_he || key[i + 1] == NO_KEY) estart[e + 1] = i + 1;
}

__global__ void vertex_flag_kernel(const u64* __restrict__ key, const int* __restrict__ estart,
                                   const int* __restrict__ n_edges, int cap, int* __restrict__ vflag) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= cap || e >= *n_edges) return;
  const int cnt = estart[e + 1] - estart[e];
  if (cnt == 2) return;
  const u64 k = key[estart[e]];
  const int bit = cnt == 1 ? V_BOUNDARY : V_FROZEN;
  atomicOr(&vflag[(int)(k >> 32)], bit);
  atomicOr(&vflag[(int)(k & 0xffffffffu)], bit);
}

__global__ void vf_count_kernel(const int* __restrict__ faces, int nf, int* __restrict__ vf_cnt) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf || faces[3 * f] < 0) return;
  for (int c = 0; c < 3; ++c) atomicAdd(&vf_cnt[faces[3 * f + c]], 1);
}

__global__ void vf_fill_kernel(const int* __restrict__ faces, int nf, const int* __restrict__ vf_off,
                               int* __restrict__ vf_cur, int* __restrict__ vf_list) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf || faces[3 * f] < 0) return;
  for (int c = 0; c < 3; ++c) {
    const int v = faces[3 * f + c];
    vf_list[vf_off[v] + atomicAdd(&vf_cur[v], 1)] = f;
  }
}

// each vertex's faces in ascending order (the fill above is in arrival order)
__global__ void vf_sort_kernel(const int* __restrict__ vf_off, int nv, int* __restrict__ vf_list) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nv) return;
  int* l = vf_list + vf_off[v];
  const int n = vf_off[v + 1] - vf_off[v];
  for (int i = 1; i < n; ++i) {
    const int x = l[i];
    int j = i - 1;
    while (j >= 0 && l[j] > x) { l[j + 1] = l[j]; --j; }
    l[j + 1] = x;
  }
}

// ---- round 0: quadrics and component sizes ------------------------------------------------------------------------
__global__ void quadric_kernel(const int* __restrict__ faces, const double* __restrict__ pos,
                               const int* __restrict__ vf_off, const int* __restrict__ vf_list,
                               const int* __restrict__ estart, const int* __restrict__ he_edge, int nv,
                               double* __restrict__ Q) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nv) return;
  double q[10];
#pragma unroll
  for (int k = 0; k < 10; ++k) q[k] = 0.0;
  for (int i = vf_off[v]; i < vf_off[v + 1]; ++i) {
    const int f = vf_list[i];
    const int* fc = faces + 3 * f;
    const d3 p[3] = {ld3(pos, fc[0]), ld3(pos, fc[1]), ld3(pos, fc[2])};
    const d3 n = cross3(sub3(p[1], p[0]), sub3(p[2], p[0]));
    const double nn = dot3(n, n);
    if (!(nn > 0.0)) continue;
    add_plane(q, n, -dot3(n, p[0]), __ddiv_rn(1.0, __dsqrt_rn(nn)));
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const int j1 = j == 2 ? 0 : j + 1;
      if (fc[j] != v && fc[j1] != v) continue;
      const int e = he_edge[3 * f + j];
      if (estart[e + 1] - estart[e] != 1) continue;
      const d3 ed = sub3(p[j1], p[j]);
      const d3 m = cross3(ed, n);
      const double mm = dot3(m, m);
      if (!(mm > 0.0)) continue;
      add_plane(q, m, -dot3(m, p[j]), __ddiv_rn(dmul(3.0, dot3(ed, ed)), mm));
    }
  }
#pragma unroll
  for (int k = 0; k < 10; ++k) Q[10 * (int64_t)v + k] = q[k];
}

__global__ void component_size_kernel(const int* __restrict__ vf_off, const int* __restrict__ label, int nv,
                                      int* __restrict__ comp_nv) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nv || vf_off[v + 1] == vf_off[v]) return;
  atomicAdd(&comp_nv[label[v]], 1);
}

// ---- pricing and selection ----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256, 2) cost_kernel(
    const u64* __restrict__ hkey, const int* __restrict__ estart, const int* __restrict__ n_edges, int cap,
    const int* __restrict__ faces, const int* __restrict__ vf_off, const int* __restrict__ vf_list,
    const int* __restrict__ vflag, const int* __restrict__ label, const int* __restrict__ comp_nv,
    const double* __restrict__ pos, const double* __restrict__ Q, u64* __restrict__ ekey, double* __restrict__ ep,
    u64* __restrict__ m) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= cap || e >= *n_edges) return;
  ekey[e] = NO_KEY;
  const int cnt = estart[e + 1] - estart[e];
  const u64 k = hkey[estart[e]];
  const int a = (int)(k >> 32), b = (int)(k & 0xffffffffu);
  const int fa = vflag[a], fb = vflag[b];
  if (cnt > 2 || ((fa | fb) & V_FROZEN)) return;
  if (cnt == 2 && (fa & V_BOUNDARY) && (fb & V_BOUNDARY)) return;
  if (comp_nv[label[a]] <= MIN_COMPONENT) return;
  const int a0 = vf_off[a], a1 = vf_off[a + 1], b0 = vf_off[b], b1 = vf_off[b + 1];
  // link condition: the distinct common neighbours of a and b are as many as the edge's faces
  int common = 0;
  for (int i = a0; i < a1; ++i) {
    const int* fc = faces + 3 * vf_list[i];
    for (int c = 0; c < 3; ++c) {
      const int x = fc[c];
      if (x == a || x == b) continue;
      bool seen = false;
      for (int i2 = a0; i2 < i && !seen; ++i2) seen = face_has(faces + 3 * vf_list[i2], x);
      if (seen) continue;
      for (int j = b0; j < b1; ++j)
        if (face_has(faces + 3 * vf_list[j], x)) { ++common; break; }
    }
  }
  if (common != cnt) return;
  double q[10];
#pragma unroll
  for (int i = 0; i < 10; ++i) q[i] = dadd(Q[10 * (int64_t)a + i], Q[10 * (int64_t)b + i]);
  const d3 pa = ld3(pos, a), pb = ld3(pos, b);
  const d3 p = placement(q, pa, pb);
  // the faces that survive around a, then b, with the endpoint moved to p: no flip, lowest quality
  double qmin = 1.0;
  for (int side = 0; side < 2; ++side) {
    const int s = side ? b : a, o = side ? a : b;
    for (int i = side ? b0 : a0, end = side ? b1 : a1; i < end; ++i) {
      const int* fc = faces + 3 * vf_list[i];
      if (face_has(fc, o)) continue;
      const d3 x0 = ld3(pos, fc[0]), x1 = ld3(pos, fc[1]), x2 = ld3(pos, fc[2]);
      const d3 y0 = fc[0] == s ? p : x0, y1 = fc[1] == s ? p : x1, y2 = fc[2] == s ? p : x2;
      const d3 n0 = cross3(sub3(x1, x0), sub3(x2, x0));
      const d3 e01 = sub3(y1, y0), e12 = sub3(y2, y1), e20 = sub3(y0, y2);
      const d3 n1 = cross3(e01, sub3(y2, y0));
      if (dot3(n0, n0) > 0.0 && !(dot3(n0, n1) > 0.0)) return;     // a zero-area face has no side to flip
      const double l2 = dadd(dadd(dot3(e01, e01), dot3(e12, e12)), dot3(e20, e20));
      const double qual = l2 > 0.0 ? __ddiv_rn(dmul(__dsqrt_rn(dot3(n1, n1)), 3.4641016151377544), l2) : 0.0;
      qmin = qual < qmin ? qual : qmin;
    }
  }
  qmin = qmin < 1e-3 ? 1e-3 : qmin;
  double err = quadric_err(q, p);
  err = err > 0.0 ? err : 0.0;
  const d3 ab = sub3(pb, pa);
  const double l2 = dot3(ab, ab);
  const double cost = __ddiv_rn(dadd(err, dmul(1e-4, dmul(l2, l2))), qmin);
  const u64 key = ((u64)__float_as_uint(__double2float_ru(cost)) << 32) | (u64)e;
  ekey[e] = key;
  ep[3 * (int64_t)e] = p.x;
  ep[3 * (int64_t)e + 1] = p.y;
  ep[3 * (int64_t)e + 2] = p.z;
  atomicMin(&m[a], key);
  atomicMin(&m[b], key);
}

// M(v) = min of m over v's closed 1-ring (M starts as a copy of m)
__global__ void ring_kernel(const u64* __restrict__ hkey, const int* __restrict__ estart, const int* __restrict__ n_edges,
                            int cap, const u64* __restrict__ m, u64* __restrict__ M) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= cap || e >= *n_edges) return;
  const u64 k = hkey[estart[e]];
  const int a = (int)(k >> 32), b = (int)(k & 0xffffffffu);
  atomicMin(&M[a], m[b]);
  atomicMin(&M[b], m[a]);
}

__global__ void select_kernel(const u64* __restrict__ hkey, const int* __restrict__ estart,
                              const int* __restrict__ n_edges, int cap, const u64* __restrict__ ekey,
                              const u64* __restrict__ M, const int* __restrict__ label, int* __restrict__ esel,
                              int* __restrict__ comp_sel, u64* __restrict__ comp_min) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= cap || e >= *n_edges) return;
  const u64 k = hkey[estart[e]];
  const int a = (int)(k >> 32), b = (int)(k & 0xffffffffu);
  const u64 key = ekey[e];
  const bool sel = key != NO_KEY && key == M[a] && key == M[b];
  esel[e] = sel;
  if (sel) {
    atomicAdd(&comp_sel[label[a]], 1);
    atomicMin(&comp_min[label[a]], key);
  }
}

// a component that would fall under MIN_COMPONENT vertices keeps only its cheapest selected edge; skey = the keys of
// the edges that stay selected (NO_KEY elsewhere, up to cap) for the last round's cut
__global__ void component_trim_kernel(const u64* __restrict__ hkey, const int* __restrict__ estart,
                                      const int* __restrict__ n_edges, int cap, const u64* __restrict__ ekey,
                                      const int* __restrict__ label, const int* __restrict__ comp_nv,
                                      const int* __restrict__ comp_sel, const u64* __restrict__ comp_min,
                                      int* __restrict__ esel, u64* __restrict__ skey, int* __restrict__ cnt) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= cap) return;
  if (e >= *n_edges || !esel[e]) {
    skey[e] = NO_KEY;
    return;
  }
  const int c = label[(int)(hkey[estart[e]] >> 32)];
  const u64 key = ekey[e];
  if (comp_nv[c] - comp_sel[c] < MIN_COMPONENT && key != comp_min[c]) {
    esel[e] = 0;
    skey[e] = NO_KEY;
    return;
  }
  skey[e] = key;
  atomicAdd(&cnt[C_NSEL], 1);
}

// keep only the selected edges whose key is at most the k-th smallest (sorted[k - 1])
__global__ void cut_kernel(const int* __restrict__ n_edges, int cap, const u64* __restrict__ ekey,
                           const u64* __restrict__ sorted, int k, int* __restrict__ esel) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= cap || e >= *n_edges) return;
  if (esel[e] && ekey[e] > sorted[k - 1]) esel[e] = 0;
}

__global__ void apply_kernel(const u64* __restrict__ hkey, const int* __restrict__ hval, const int* __restrict__ estart,
                             const int* __restrict__ n_edges, int cap, const int* __restrict__ esel,
                             const double* __restrict__ ep, const int* __restrict__ label, double* __restrict__ pos,
                             double* __restrict__ Q, int* __restrict__ remap, int* __restrict__ faces,
                             int* __restrict__ comp_nv, int* __restrict__ cnt) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= cap || e >= *n_edges || !esel[e]) return;
  const int s = estart[e], t = estart[e + 1];
  const u64 k = hkey[s];
  const int a = (int)(k >> 32), b = (int)(k & 0xffffffffu);
  for (int i = 0; i < 3; ++i) pos[3 * (int64_t)a + i] = ep[3 * (int64_t)e + i];
  for (int i = 0; i < 10; ++i) Q[10 * (int64_t)a + i] = dadd(Q[10 * (int64_t)a + i], Q[10 * (int64_t)b + i]);
  remap[b] = a;
  for (int h = s; h < t; ++h) {
    const int f = hval[h] / 3;
    faces[3 * f] = faces[3 * f + 1] = faces[3 * f + 2] = -1;
  }
  atomicAdd(&cnt[C_REMOVED], t - s);
  atomicSub(&comp_nv[label[a]], 1);
}

__global__ void rewrite_kernel(int* __restrict__ faces, int nf, const int* __restrict__ remap) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf || faces[3 * f] < 0) return;
  for (int c = 0; c < 3; ++c) faces[3 * f + c] = remap[faces[3 * f + c]];
}

// ---- output -------------------------------------------------------------------------------------------------------
__global__ void mark_kernel(const int* __restrict__ faces, int nf, int* __restrict__ vref, int* __restrict__ fkeep) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > nf) return;
  const bool live = f < nf && faces[3 * f] >= 0;
  fkeep[f] = live;
  if (live)
    for (int c = 0; c < 3; ++c) vref[faces[3 * f + c]] = 1;
}

__global__ void out_verts_kernel(const double* __restrict__ pos, const int* __restrict__ vref,
                                 const int* __restrict__ vnew, int nv, float* __restrict__ out) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nv || !vref[v]) return;
  const int o = vnew[v];
  for (int i = 0; i < 3; ++i) out[3 * (int64_t)o + i] = __double2float_rn(pos[3 * (int64_t)v + i]);
}

__global__ void out_faces_kernel(const int* __restrict__ faces, const int* __restrict__ fkeep,
                                 const int* __restrict__ fnew, const int* __restrict__ vnew, int nf,
                                 int32_t* __restrict__ out) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf || !fkeep[f]) return;
  const int o = fnew[f];
  for (int c = 0; c < 3; ++c) out[3 * (int64_t)o + c] = vnew[faces[3 * f + c]];
}

// ---- workspace ----------------------------------------------------------------------------------------------------
struct Workspace {
  // per vertex
  double *pos, *Q;      // position (3), quadric (10)
  int *remap, *label, *comp_nv, *comp_sel, *vflag, *vf_cnt, *vf_off, *vf_cur, *vref, *vnew;
  u64 *comp_min, *m, *M;
  // per half-edge (3 per face)
  int *faces, *vf_list, *hval_in, *hval, *head, *eidx, *estart, *he_edge, *esel;
  u64 *hkey_in, *hkey, *ekey, *skey, *skey_sorted;
  double* ep;
  // per face, and the C_* counters
  int *fkeep, *fnew, *cnt;
};

bool sizes_ok(int64_t nv, int64_t nf) { return nv >= 0 && nf >= 0 && nv <= 0x7ffffffeLL && 3 * nf <= 0x7ffffffeLL; }

// points w's buffers into `base` (null: only measures) and returns the bytes they take
size_t carve(Workspace& w, char* base, int64_t nv, int64_t nf) {
  const size_t V = (size_t)nv, F = (size_t)nf, H = 3 * F;
  r3g_carver c{base};
  w.pos = c.take<double>(V * 3);
  w.Q = c.take<double>(V * 10);
  w.remap = c.take<int>(V);
  w.label = c.take<int>(V);
  w.comp_nv = c.take<int>(V);
  w.comp_sel = c.take<int>(V);
  w.comp_min = c.take<u64>(V);
  w.vflag = c.take<int>(V);
  w.m = c.take<u64>(V);
  w.M = c.take<u64>(V);
  w.vf_cnt = c.take<int>(V + 1);
  w.vf_off = c.take<int>(V + 1);
  w.vf_cur = c.take<int>(V);
  w.vref = c.take<int>(V + 1);
  w.vnew = c.take<int>(V + 1);
  w.faces = c.take<int>(H);
  w.vf_list = c.take<int>(H);
  w.hkey_in = c.take<u64>(H);
  w.hkey = c.take<u64>(H);
  w.hval_in = c.take<int>(H);
  w.hval = c.take<int>(H);
  w.head = c.take<int>(H + 1);
  w.eidx = c.take<int>(H + 1);
  w.estart = c.take<int>(H + 1);
  w.he_edge = c.take<int>(H);
  w.ekey = c.take<u64>(H);
  w.ep = c.take<double>(H * 3);
  w.esel = c.take<int>(H);
  w.skey = c.take<u64>(H);
  w.skey_sorted = c.take<u64>(H);
  w.fkeep = c.take<int>(F + 1);
  w.fnew = c.take<int>(F + 1);
  w.cnt = c.take<int>(C_COUNT);
  return c.off;
}

inline unsigned blocks(int64_t n) { return (unsigned)((n + 255) / 256); }

// CUB's temporary storage for the whole call, returned to the stream-ordered pool on every exit path
struct CubTemp {
  void* p = nullptr;
  size_t bytes = 0;
  cudaStream_t s = nullptr;
  ~CubTemp() {
    if (p) cudaFreeAsync(p, s);
  }
};

}  // namespace

extern "C" size_t r3g_decimate_workspace_bytes(int64_t nv, int64_t nf) {
  Workspace w;
  return sizes_ok(nv, nf) ? carve(w, nullptr, nv, nf) : 0;
}

extern "C" int r3g_mesh_decimate(r3g_ctx* ctx, const float* verts, int64_t nv, const int32_t* faces, int64_t nf,
                                 int64_t target, void* workspace, size_t workspace_bytes, float* verts_out,
                                 int32_t* faces_out, int64_t* nv_out_host, int64_t* nf_out_host, int64_t* rounds_host,
                                 void* stream) {
  R3G_ENTRY(ctx, "mesh_decimate");
  if (!sizes_ok(nv, nf) || target < 0 || !nv_out_host || !nf_out_host || (nv > 0 && (!verts || !verts_out)) ||
      (nf > 0 && (!faces || !faces_out)))
    return r3g_fail(ctx, R3G_E_INVALID, "mesh_decimate: bad arguments (nv %lld, nf %lld, target %lld)", (long long)nv,
                    (long long)nf, (long long)target);
  Workspace w;
  const size_t need = carve(w, (char*)workspace, nv, nf);
  if (!workspace || workspace_bytes < need)
    return r3g_fail(ctx, R3G_E_WORKSPACE, "mesh_decimate: workspace of %zu bytes, %zu needed", workspace_bytes, need);
  *nv_out_host = *nf_out_host = 0;
  if (rounds_host) *rounds_host = 0;
  if (nv == 0 || nf == 0) return R3G_OK;
  cudaStream_t s = (cudaStream_t)stream;
  int* host = reinterpret_cast<int*>(ctx->pinned);
  const int NV = (int)nv, NF = (int)nf, NH = 3 * NF;
  const int* n_edges = w.eidx + NH;

  CubTemp tmp;
  tmp.s = s;
  {
    size_t b = 0;
    R3G_CUDA_OK(ctx, cub::DeviceRadixSort::SortPairs(nullptr, b, w.hkey_in, w.hkey, w.hval_in, w.hval, NH, 0, 64, s));
    tmp.bytes = b;
    R3G_CUDA_OK(ctx, cub::DeviceRadixSort::SortKeys(nullptr, b, w.skey, w.skey_sorted, NH, 0, 64, s));
    tmp.bytes = b > tmp.bytes ? b : tmp.bytes;
    R3G_CUDA_OK(ctx, cub::DeviceScan::ExclusiveSum(nullptr, b, w.head, w.eidx, NH + 1, s));
    tmp.bytes = b > tmp.bytes ? b : tmp.bytes;
    R3G_CUDA_OK(ctx, cub::DeviceScan::ExclusiveSum(nullptr, b, w.vf_cnt, w.vf_off, NV + 1, s));
    tmp.bytes = b > tmp.bytes ? b : tmp.bytes;
    R3G_CUDA_OK(ctx, cub::DeviceScan::ExclusiveSum(nullptr, b, w.fkeep, w.fnew, NF + 1, s));
    tmp.bytes = b > tmp.bytes ? b : tmp.bytes;
    R3G_CUDA_OK(ctx, cudaMallocAsync(&tmp.p, tmp.bytes, s));
  }

  R3G_CUDA_OK(ctx, cudaMemsetAsync(w.cnt, 0, C_COUNT * sizeof(int), s));
  init_faces_kernel<<<blocks(NF), 256, 0, s>>>(faces, nf, nv, w.faces, w.cnt);
  R3G_LAUNCH_OK(ctx);
  init_verts_kernel<<<blocks(NV), 256, 0, s>>>(verts, nv, w.pos, w.remap);
  R3G_LAUNCH_OK(ctx);
  R3G_CUDA_OK(ctx, cudaMemcpyAsync(host, w.cnt, C_COUNT * sizeof(int), cudaMemcpyDeviceToHost, s));
  R3G_CUDA_OK(ctx, cudaStreamSynchronize(s));
  if (host[C_BAD]) return r3g_fail(ctx, R3G_E_INVALID, "mesh_decimate: a face index is outside [0, nv)");
  int64_t live = host[C_NLIVE];

  // the adjacency of the current face array: sorted half-edges, edges, boundary / frozen flags, vertex -> face CSR
  auto adjacency = [&]() -> int {
    halfedge_kernel<<<blocks(NH), 256, 0, s>>>(w.faces, NH, w.hkey_in, w.hval_in);
    R3G_LAUNCH_OK(ctx);
    R3G_CUDA_OK(ctx, cub::DeviceRadixSort::SortPairs(tmp.p, tmp.bytes, w.hkey_in, w.hkey, w.hval_in, w.hval, NH, 0, 64,
                                                     s));
    head_kernel<<<blocks(NH + 1), 256, 0, s>>>(w.hkey, NH, w.head);
    R3G_LAUNCH_OK(ctx);
    R3G_CUDA_OK(ctx, cub::DeviceScan::ExclusiveSum(tmp.p, tmp.bytes, w.head, w.eidx, NH + 1, s));
    edge_kernel<<<blocks(NH), 256, 0, s>>>(w.hkey, w.hval, w.head, w.eidx, NH, w.estart, w.he_edge);
    R3G_LAUNCH_OK(ctx);
    R3G_CUDA_OK(ctx, cudaMemsetAsync(w.vflag, 0, nv * sizeof(int), s));
    vertex_flag_kernel<<<blocks(NH), 256, 0, s>>>(w.hkey, w.estart, n_edges, NH, w.vflag);
    R3G_LAUNCH_OK(ctx);
    R3G_CUDA_OK(ctx, cudaMemsetAsync(w.vf_cnt, 0, (nv + 1) * sizeof(int), s));
    R3G_CUDA_OK(ctx, cudaMemsetAsync(w.vf_cur, 0, nv * sizeof(int), s));
    vf_count_kernel<<<blocks(NF), 256, 0, s>>>(w.faces, NF, w.vf_cnt);
    R3G_LAUNCH_OK(ctx);
    R3G_CUDA_OK(ctx, cub::DeviceScan::ExclusiveSum(tmp.p, tmp.bytes, w.vf_cnt, w.vf_off, NV + 1, s));
    vf_fill_kernel<<<blocks(NF), 256, 0, s>>>(w.faces, NF, w.vf_off, w.vf_cur, w.vf_list);
    R3G_LAUNCH_OK(ctx);
    vf_sort_kernel<<<blocks(NV), 256, 0, s>>>(w.vf_off, NV, w.vf_list);
    R3G_LAUNCH_OK(ctx);
    return R3G_OK;
  };

  int64_t rounds = 0;
  if (live > target) {
    if (int rc = adjacency()) return rc;
    quadric_kernel<<<blocks(NV), 256, 0, s>>>(w.faces, w.pos, w.vf_off, w.vf_list, w.estart, w.he_edge, NV, w.Q);
    R3G_LAUNCH_OK(ctx);
    if (int rc = r3g_launch_components(ctx, w.faces, nf, nv, w.label, w.cnt + C_BAD, true, s)) return rc;
    R3G_CUDA_OK(ctx, cudaMemsetAsync(w.comp_nv, 0, nv * sizeof(int), s));
    component_size_kernel<<<blocks(NV), 256, 0, s>>>(w.vf_off, w.label, NV, w.comp_nv);
    R3G_LAUNCH_OK(ctx);
    while (live > target) {
      if (rounds > 0)
        if (int rc = adjacency()) return rc;
      R3G_CUDA_OK(ctx, cudaMemsetAsync(w.m, 0xff, nv * sizeof(u64), s));
      cost_kernel<<<blocks(NH), 256, 0, s>>>(w.hkey, w.estart, n_edges, NH, w.faces, w.vf_off, w.vf_list, w.vflag,
                                             w.label, w.comp_nv, w.pos, w.Q, w.ekey, w.ep, w.m);
      R3G_LAUNCH_OK(ctx);
      R3G_CUDA_OK(ctx, cudaMemcpyAsync(w.M, w.m, nv * sizeof(u64), cudaMemcpyDeviceToDevice, s));
      ring_kernel<<<blocks(NH), 256, 0, s>>>(w.hkey, w.estart, n_edges, NH, w.m, w.M);
      R3G_LAUNCH_OK(ctx);
      R3G_CUDA_OK(ctx, cudaMemsetAsync(w.comp_sel, 0, nv * sizeof(int), s));
      R3G_CUDA_OK(ctx, cudaMemsetAsync(w.comp_min, 0xff, nv * sizeof(u64), s));
      select_kernel<<<blocks(NH), 256, 0, s>>>(w.hkey, w.estart, n_edges, NH, w.ekey, w.M, w.label, w.esel, w.comp_sel,
                                               w.comp_min);
      R3G_LAUNCH_OK(ctx);
      R3G_CUDA_OK(ctx, cudaMemsetAsync(w.cnt + C_NSEL, 0, 2 * sizeof(int), s));
      component_trim_kernel<<<blocks(NH), 256, 0, s>>>(w.hkey, w.estart, n_edges, NH, w.ekey, w.label, w.comp_nv,
                                                       w.comp_sel, w.comp_min, w.esel, w.skey, w.cnt);
      R3G_LAUNCH_OK(ctx);
      R3G_CUDA_OK(ctx, cudaMemcpyAsync(host, w.cnt, C_COUNT * sizeof(int), cudaMemcpyDeviceToHost, s));
      R3G_CUDA_OK(ctx, cudaStreamSynchronize(s));
      const int nsel = host[C_NSEL];
      if (nsel == 0) break;
      const int64_t k = (live - target + 1) / 2;
      if (nsel > k) {      // the last round: only the k cheapest, so the count lands on target or target - 1
        R3G_CUDA_OK(ctx, cub::DeviceRadixSort::SortKeys(tmp.p, tmp.bytes, w.skey, w.skey_sorted, NH, 0, 64, s));
        cut_kernel<<<blocks(NH), 256, 0, s>>>(n_edges, NH, w.ekey, w.skey_sorted, (int)k, w.esel);
        R3G_LAUNCH_OK(ctx);
      }
      apply_kernel<<<blocks(NH), 256, 0, s>>>(w.hkey, w.hval, w.estart, n_edges, NH, w.esel, w.ep, w.label, w.pos, w.Q,
                                              w.remap, w.faces, w.comp_nv, w.cnt);
      R3G_LAUNCH_OK(ctx);
      rewrite_kernel<<<blocks(NF), 256, 0, s>>>(w.faces, NF, w.remap);
      R3G_LAUNCH_OK(ctx);
      R3G_CUDA_OK(ctx, cudaMemcpyAsync(host, w.cnt, C_COUNT * sizeof(int), cudaMemcpyDeviceToHost, s));
      R3G_CUDA_OK(ctx, cudaStreamSynchronize(s));
      live -= host[C_REMOVED];
      ++rounds;
    }
  }

  // stable compaction of the surviving faces and the vertices they reference
  R3G_CUDA_OK(ctx, cudaMemsetAsync(w.vref, 0, (nv + 1) * sizeof(int), s));
  mark_kernel<<<blocks(NF + 1), 256, 0, s>>>(w.faces, NF, w.vref, w.fkeep);
  R3G_LAUNCH_OK(ctx);
  R3G_CUDA_OK(ctx, cub::DeviceScan::ExclusiveSum(tmp.p, tmp.bytes, w.vref, w.vnew, NV + 1, s));
  R3G_CUDA_OK(ctx, cub::DeviceScan::ExclusiveSum(tmp.p, tmp.bytes, w.fkeep, w.fnew, NF + 1, s));
  out_verts_kernel<<<blocks(NV), 256, 0, s>>>(w.pos, w.vref, w.vnew, NV, verts_out);
  R3G_LAUNCH_OK(ctx);
  out_faces_kernel<<<blocks(NF), 256, 0, s>>>(w.faces, w.fkeep, w.fnew, w.vnew, NF, faces_out);
  R3G_LAUNCH_OK(ctx);
  R3G_CUDA_OK(ctx, cudaMemcpyAsync(host, w.vnew + nv, sizeof(int), cudaMemcpyDeviceToHost, s));
  R3G_CUDA_OK(ctx, cudaMemcpyAsync(host + 1, w.fnew + nf, sizeof(int), cudaMemcpyDeviceToHost, s));
  R3G_CUDA_OK(ctx, cudaStreamSynchronize(s));
  *nv_out_host = host[0];
  *nf_out_host = host[1];
  if (rounds_host) *rounds_host = rounds;
  return R3G_OK;
}
