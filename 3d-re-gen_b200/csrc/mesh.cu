// Mesh clean-up on the device: connected components of a triangle mesh (lock-free union-find over the vertices,
// hooked by the faces) -- the computation behind FloaterRemover
// (Hunyuan3D-2/hy3dgen/shapegen/postprocessors.py:58-63,118-129: pymeshlab's
// compute_selection_by_small_disconnected_components_per_face + remove), which src/2d_to_3d_models/run.py:93 applies to
// every generated mesh.  The marching-cubes output never leaves the GPU for it.  Integer work, HBM / atomics bound.
#include "r3g_internal.h"

namespace {

// find with path halving; concurrent writers only ever replace a parent by one of its ancestors
__device__ __forceinline__ int uf_find(int* parent, int x) {
  volatile int* vp = parent;     // L1 is not coherent across SMs: hooks (CAS at L2) must be seen by the retry loops
  while (true) {
    const int p = vp[x];
    if (p == x) return x;
    const int g = vp[p];
    if (g != p) vp[x] = g;
    x = p;
  }
}

// the larger root is hooked under the smaller one, so a component's final root is its smallest vertex index
__device__ __forceinline__ void uf_union(int* parent, int a, int b) {
  while (true) {
    a = uf_find(parent, a);
    b = uf_find(parent, b);
    if (a == b) return;
    if (a < b) { const int t = a; a = b; b = t; }
    if (atomicCAS(&parent[a], a, b) == a) return;
  }
}

__global__ void uf_init_kernel(int* __restrict__ parent, int64_t nv) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nv) parent[i] = (int)i;
}

__global__ void uf_hook_kernel(int* parent, const int32_t* __restrict__ faces, int64_t nf, int64_t nv,
                               int* __restrict__ bad) {
  const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nf) return;
  const int a = faces[3 * f], b = faces[3 * f + 1], c = faces[3 * f + 2];
  if (a < 0 || b < 0 || c < 0 || a >= nv || b >= nv || c >= nv) {
    atomicExch(bad, 1);
    return;
  }
  uf_union(parent, a, b);
  uf_union(parent, b, c);
}

// labels alias the parent array: the only writes in this pass are label[i] = root(i), each a valid (and final) parent of
// i.  The walk must NOT compress here -- a halving store from a thread passing through i could land after i's own final
// store and leave a non-root ancestor in label[i].
__global__ void uf_flatten_kernel(int* parent, int64_t nv) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nv) return;
  int x = (int)i;
  while (true) {
    const int p = *reinterpret_cast<volatile int*>(parent + x);
    if (p == x) break;
    x = p;
  }
  parent[i] = x;
}

}  // namespace

extern "C" int r3g_mesh_components(r3g_ctx* ctx, const int32_t* faces, int64_t nf, int64_t nv, int32_t* labels,
                                   void* stream) {
  R3G_ENTRY(ctx, "mesh_components");
  if (!labels || (nf > 0 && !faces) || nv < 0 || nf < 0 || nv > 0x7fffffffLL)
    return r3g_fail(ctx, R3G_E_INVALID, "mesh_components: bad arguments");
  if (nv == 0) return R3G_OK;
  cudaStream_t s = (cudaStream_t)stream;
  // labels doubles as the parent array (int32 [nv]); the flag lives in the context's pinned scratch
  int* parent = reinterpret_cast<int*>(labels);
  int* bad_dev = nullptr;
  R3G_CUDA_OK(ctx, cudaMallocAsync((void**)&bad_dev, sizeof(int), s));
  R3G_CUDA_OK(ctx, cudaMemsetAsync(bad_dev, 0, sizeof(int), s));
  uf_init_kernel<<<(unsigned)((nv + 255) / 256), 256, 0, s>>>(parent, nv);
  R3G_LAUNCH_OK(ctx);
  if (nf > 0) {
    uf_hook_kernel<<<(unsigned)((nf + 255) / 256), 256, 0, s>>>(parent, faces, nf, nv, bad_dev);
    R3G_LAUNCH_OK(ctx);
  }
  uf_flatten_kernel<<<(unsigned)((nv + 255) / 256), 256, 0, s>>>(parent, nv);
  R3G_LAUNCH_OK(ctx);
  int* bad_host = reinterpret_cast<int*>(ctx->pinned);
  R3G_CUDA_OK(ctx, cudaMemcpyAsync(bad_host, bad_dev, sizeof(int), cudaMemcpyDeviceToHost, s));
  R3G_CUDA_OK(ctx, cudaFreeAsync(bad_dev, s));
  R3G_CUDA_OK(ctx, cudaStreamSynchronize(s));
  if (*bad_host) return r3g_fail(ctx, R3G_E_INVALID, "mesh_components: a face index is outside [0, nv)");
  return R3G_OK;
}
