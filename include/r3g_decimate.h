/* r3g decimation -- quadric edge-collapse mesh reduction on the device, the face reduction of stage 3
 * (src/2d_to_3d_models/run.py:95: FaceReducer, Hunyuan3D-2/hy3dgen/shapegen/postprocessors.py:37-51,118-128, pymeshlab
 * meshing_decimation_quadric_edge_collapse to 40 000 faces with qualitythr 1, preserveboundary, boundaryweight 3,
 * preservenormal, preservetopology, autoclean).  The algorithm below is r3g's own, not MeshLab's collapse order; it is
 * deterministic and pinned bit for bit by the numpy mirror oracle/decimate.py.  Same conventions as r3g.h (device
 * pointers unless the name ends in _host, 0 = OK, negative = R3G_E_*, r3g_last_error for the message); this header is
 * compiled into the same libr3g.so.
 *
 * Algorithm: rounds of independent edge collapses.
 *   Quadrics (float64, computed once from the input): every non-degenerate face adds u u^T / |n| with n = (p1-p0) x (p2-p0),
 *     u = (n, -n.p0) -- the plane quadric weighted by twice the face area; every boundary edge (one face) from corner j to
 *     j+1 adds 3 (e.e) m m^T / (m.m) with e = p_{j+1} - p_j, m = e x n, the plane (m, -m.p_j) through the edge
 *     perpendicular to its face.  A vertex sums the terms of its faces in ascending face order, each face's own plane
 *     before its boundary edges in corner order.  A collapse gives the kept vertex Q_a + Q_b.
 *   Placement: p minimises v^T Q v (v = (p, 1)) by the adjugate of Q's 3x3 block when |det| > 1e-6 trace^3; otherwise the
 *     cheapest of a, b and (a + b) / 2 (ties to the earlier).  err = max(v^T Q v, 0).
 *   Cost: (err + 1e-4 |a-b|^4) / clamp(min quality, 1e-3, 1), over the faces around a or b that survive with the endpoint
 *     moved to p; quality = 2 sqrt(3) |n| / (sum of squared edge lengths) (1 for an equilateral triangle).  Rounded up to
 *     float32; key = (float32 bits << 32) | edge index, edges numbered in ascending (min vertex, max vertex) order.
 *   Validity (an invalid edge waits for a later round): at most two faces on the edge and neither endpoint on an edge of
 *     more (frozen); not an interior edge between two boundary vertices; link condition (a and b have exactly as many
 *     common neighbours as the edge has faces); the component keeps at least 4 vertices; no surviving face around a or b
 *     with a non-zero normal flips (old normal . new normal <= 0 rejects; a zero-area face, such as marching cubes
 *     leaves where the field is 0 at a grid point, constrains nothing and so can be collapsed away).
 *   Selection: m(v) = min key of the valid edges at v, M(v) = min of m over v's closed 1-ring; an edge is collapsed iff
 *     key == M(a) == M(b).  Selected edges share no faces and no adjacent endpoints, so the tests above stay true while
 *     they are applied together, in any thread order.  A component that would fall under 4 vertices keeps only its
 *     cheapest selected edge.  When more than ceil((nf - target) / 2) edges remain selected, only that many of the
 *     cheapest are applied, so the face count ends at target or target - 1.
 *   Apply: the smaller endpoint index survives at p, the edge's faces die, the other faces keep their winding.
 *   The rounds stop when nf <= target or no edge is selectable (then the result is the smallest mesh the rules allow).
 *   Output: surviving vertices and faces compacted in their original relative order, positions rounded to float32; faces
 *     with a repeated index and unreferenced vertices are dropped.
 */
#ifndef R3G_DECIMATE_H
#define R3G_DECIMATE_H
#include "r3g.h"
#ifdef __cplusplus
extern "C" {
#endif

/* Device workspace r3g_mesh_decimate needs for a mesh of nv vertices and nf faces (pure arithmetic, no device): about
 * 170 bytes per vertex and 310 per face (0.1 GB at 222 000 faces); 0 for sizes r3g_mesh_decimate refuses. */
size_t r3g_decimate_workspace_bytes(int64_t nv, int64_t nf);

/* verts float32 [nv][3], faces int32 [nf][3] -> verts_out float32 [*nv_out_host][3], faces_out int32 [*nf_out_host][3]
 * (capacities nv and nf); target >= 0.  *rounds_host (if not NULL) receives the number of collapse rounds.
 * SYNCHRONISES `stream` (the host loop reads the face count every round).  An index outside [0, nv), nv > 2^31 - 1 or
 * 3 nf > 2^31 - 1 returns R3G_E_INVALID; a workspace under r3g_decimate_workspace_bytes(nv, nf), R3G_E_WORKSPACE. */
int r3g_mesh_decimate(r3g_ctx* ctx, const float* verts, int64_t nv, const int32_t* faces, int64_t nf, int64_t target,
                      void* workspace, size_t workspace_bytes, float* verts_out, int32_t* faces_out,
                      int64_t* nv_out_host, int64_t* nf_out_host, int64_t* rounds_host, void* stream);

#ifdef __cplusplus
}
#endif
#endif
