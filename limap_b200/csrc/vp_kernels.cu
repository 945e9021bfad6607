// vp_kernels.cu — J-Linkage vanishing-point clustering, one CTA per image (persistent over images).
//
// Replaces the external library call of JLinkage::ComputeVPLabels
// (vplib/JLinkage/JLinkage.cc:40-46: VPSample::run(&pts, 5000, 2, 0, 3); VPCluster::run(..., inlier_threshold, 2))
// from B1ueber2y/JLinkage@75dadd5, which is not part of /root/reference: the published algorithm is restated
// (Toldo-Fusiello J-Linkage, Tardif's VP consistency measure; float arithmetic like the library) with a
// counter-based RNG so that results are reproducible. The specification (sampling, consensus test, merge
// order, label numbering) is written out in DESIGN.md "J-Linkage"; every float operation below is an explicit
// round-to-nearest intrinsic so that no FMA contraction changes a consensus decision.
//
//   stage 1  models: 5000 VPs from pairs of segments (splitmix64 counters) -> shared memory
//   stage 2  preference sets: bit matrix [n][ceil(M/32)] in a per-CTA global slab (L2 resident)
//   stage 3  agglomerative clustering on a cached (intersection, union) matrix; each round picks the pair
//            with the largest |A&B|/|A|B| (integer cross-multiplication, ties: smallest a then b)
#include "vp_kernels.cuh"

namespace lm {

LM_D uint64_t splitmix64(uint64_t seed, uint64_t counter) {
  uint64_t z = seed + 0x9E3779B97F4A7C15ull * (counter + 1);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

LM_D float3 cross_rn(float3 a, float3 b) {
  float3 c;
  c.x = __fsub_rn(__fmul_rn(a.y, b.z), __fmul_rn(a.z, b.y));
  c.y = __fsub_rn(__fmul_rn(a.z, b.x), __fmul_rn(a.x, b.z));
  c.z = __fsub_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x));
  return c;
}
LM_D float3 line_coords_rn(float4 p) { // (x1,y1,1) x (x2,y2,1)
  float3 l;
  l.x = __fsub_rn(p.y, p.w);
  l.y = __fsub_rn(p.z, p.x);
  l.z = __fsub_rn(__fmul_rn(p.x, p.w), __fmul_rn(p.z, p.y));
  return l;
}
// Tardif's consistency: distance of an endpoint to the line through the segment midpoint and the VP
LM_D bool consensus_rn(float4 p, float3 vp, float th) {
  float3 m;
  m.x = __fmul_rn(__fadd_rn(p.x, p.z), 0.5f);
  m.y = __fmul_rn(__fadd_rn(p.y, p.w), 0.5f);
  m.z = 1.0f;
  const float3 l = cross_rn(m, vp);
  const float den = __fsqrt_rn(__fadd_rn(__fmul_rn(l.x, l.x), __fmul_rn(l.y, l.y)));
  const float num = fabsf(__fadd_rn(__fadd_rn(__fmul_rn(l.x, p.x), __fmul_rn(l.y, p.y)), l.z));
  return __fdiv_rn(num, den) < th;
}

struct Best {
  uint32_t in, un; // intersection / union sizes (un == 0: no candidate)
  uint32_t a, b;
};
LM_D bool better(const Best &x, const Best &y) { // x strictly preferred over y
  if (x.un == 0) return false;
  if (y.un == 0) return true;
  const uint64_t l = (uint64_t)x.in * y.un, r = (uint64_t)y.in * x.un;
  if (l != r) return l > r;
  if (x.a != y.a) return x.a < y.a;
  return x.b < y.b;
}

__global__ void __launch_bounds__(256) jlinkage_kernel(const __grid_constant__ VPParams p) {
  extern __shared__ __align__(16) unsigned char smem[];
  float3 *models = reinterpret_cast<float3 *>(smem);                 // [M]
  uint16_t *rep = reinterpret_cast<uint16_t *>(models + p.n_models);  // [max_n]
  uint8_t *active = reinterpret_cast<uint8_t *>(rep + p.max_n);       // [max_n]
  __shared__ Best s_best[8];
  __shared__ Best s_pick;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarp = blockDim.x >> 5;
  const int W = (p.n_models + 31) >> 5;
  uint32_t *ps = p.ps_slab + (size_t)blockIdx.x * p.max_n * W;          // preference bits [n][W]
  uint32_t *mat = p.mat_slab + (size_t)blockIdx.x * p.max_n * p.max_n;   // (in << 16 | un) for a < b

  for (int im = blockIdx.x; im < p.n_images; im += gridDim.x) {
    const int64_t o = p.valid_off[im];
    const int n = (int)(p.valid_off[im + 1] - o);
    const float4 *pts = p.pts + o;
    int32_t *labels = p.labels + o;
    if (n < p.min_lines) { // JLinkage.cc:37-38
      for (int i = tid; i < n; i += blockDim.x) labels[i] = -1;
      if (tid == 0) p.n_clusters[im] = 0;
      continue;
    }
    // stage 1: models
    const uint64_t gim = p.image_index ? (uint64_t)p.image_index[im] : (uint64_t)im;
    for (int m = tid; m < p.n_models; m += blockDim.x) {
      const uint64_t z = splitmix64(p.seed, gim * (uint64_t)p.n_models + (uint64_t)m);
      int i = (int)((uint32_t)(z & 0xffffffffu) % (uint32_t)n);
      int j = (int)((uint32_t)(z >> 32) % (uint32_t)(n - 1));
      if (j >= i) ++j;
      float3 vp = cross_rn(line_coords_rn(pts[i]), line_coords_rn(pts[j]));
      const float nr = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(vp.x, vp.x), __fmul_rn(vp.y, vp.y)), __fmul_rn(vp.z, vp.z)));
      if (nr > 0.0f) { vp.x = __fdiv_rn(vp.x, nr); vp.y = __fdiv_rn(vp.y, nr); vp.z = __fdiv_rn(vp.z, nr); }
      models[m] = vp;
    }
    for (int i = tid; i < n; i += blockDim.x) { rep[i] = (uint16_t)i; active[i] = 1; }
    __syncthreads();
    // stage 2: preference bit matrix, one 32-model word per thread step
    for (int idx = tid; idx < n * W; idx += blockDim.x) {
      const int pl = idx / W, w = idx - pl * W;
      const float4 q = pts[pl];
      uint32_t bits = 0;
      const int m0 = w << 5, m1 = min(m0 + 32, p.n_models);
      for (int m = m0; m < m1; ++m)
        if (consensus_rn(q, models[m], p.inlier_threshold)) bits |= 1u << (m - m0);
      ps[idx] = bits;
    }
    __syncthreads();
    // stage 3a: initial (intersection, union) matrix, one warp per pair row segment
    for (int a = warp; a < n; a += nwarp)
      for (int b = a + 1; b < n; ++b) {
        uint32_t in = 0, un = 0;
        for (int w = lane; w < W; w += 32) {
          const uint32_t x = ps[(size_t)a * W + w], y = ps[(size_t)b * W + w];
          in += __popc(x & y);
          un += __popc(x | y);
        }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) { in += __shfl_xor_sync(0xffffffffu, in, d); un += __shfl_xor_sync(0xffffffffu, un, d); }
        if (lane == 0) mat[(size_t)a * p.max_n + b] = (in << 16) | un;
      }
    __syncthreads();
    // stage 3b: merge loop
    while (true) {
      Best best;
      best.in = 0; best.un = 0; best.a = 0xffffffffu; best.b = 0xffffffffu;
      for (int a = warp; a < n; a += nwarp) {
        if (!active[a]) continue;
        for (int b = a + 1 + lane; b < n; b += 32) {
          if (!active[b]) continue;
          const uint32_t v = mat[(size_t)a * p.max_n + b];
          Best c;
          c.in = v >> 16; c.un = v & 0xffffu; c.a = (uint32_t)a; c.b = (uint32_t)b;
          if (c.in == 0) continue;
          if (better(c, best)) best = c;
        }
      }
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) {
        Best o;
        o.in = __shfl_xor_sync(0xffffffffu, best.in, d); o.un = __shfl_xor_sync(0xffffffffu, best.un, d);
        o.a = __shfl_xor_sync(0xffffffffu, best.a, d); o.b = __shfl_xor_sync(0xffffffffu, best.b, d);
        if (better(o, best)) best = o;
      }
      if (lane == 0) s_best[warp] = best;
      __syncthreads();
      if (tid == 0) {
        Best b0 = s_best[0];
        for (int w = 1; w < nwarp; ++w) if (better(s_best[w], b0)) b0 = s_best[w];
        s_pick = b0;
      }
      __syncthreads();
      const Best pick = s_pick;
      if (pick.un == 0) break;
      const int a = (int)pick.a, b = (int)pick.b;
      // PS_a &= PS_b ; b leaves
      for (int w = tid; w < W; w += blockDim.x) ps[(size_t)a * W + w] &= ps[(size_t)b * W + w];
      for (int i = tid; i < n; i += blockDim.x) if (rep[i] == (uint16_t)b) rep[i] = (uint16_t)a;
      if (tid == 0) active[b] = 0;
      __syncthreads();
      // refresh row / column a of the matrix
      for (int k = warp; k < n; k += nwarp) {
        if (k == a || !active[k]) continue;
        uint32_t in = 0, un = 0;
        for (int w = lane; w < W; w += 32) {
          const uint32_t x = ps[(size_t)a * W + w], y = ps[(size_t)k * W + w];
          in += __popc(x & y);
          un += __popc(x | y);
        }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) { in += __shfl_xor_sync(0xffffffffu, in, d); un += __shfl_xor_sync(0xffffffffu, un, d); }
        if (lane == 0) {
          const int lo = min(a, k), hi = max(a, k);
          mat[(size_t)lo * p.max_n + hi] = (in << 16) | un;
        }
      }
      __syncthreads();
    }
    // labels: clusters numbered by their smallest member (= representative), ascending
    if (tid == 0) {
      int nc = 0;
      for (int i = 0; i < n; ++i)
        if (active[i]) { mat[i] = (uint32_t)nc; ++nc; } // reuse the first matrix row as the id table
      p.n_clusters[im] = nc;
    }
    __syncthreads();
    for (int i = tid; i < n; i += blockDim.x) labels[i] = (int32_t)mat[rep[i]];
    __syncthreads();
  }
}

size_t vp_smem_bytes(int n_models, int max_n) { return (size_t)n_models * sizeof(float3) + (size_t)max_n * 3 + 16; }

cudaError_t vp_static_smem_bytes(size_t *out) {
  cudaFuncAttributes fa;
  const cudaError_t e = cudaFuncGetAttributes(&fa, jlinkage_kernel);
  *out = e == cudaSuccess ? fa.sharedSizeBytes : 0;
  return e;
}

cudaError_t launch_jlinkage(const VPParams &p, int grid, size_t static_smem, cudaStream_t s) {
  const size_t smem = vp_smem_bytes(p.n_models, p.max_n);
  // the default limit of 48 KB bounds static plus dynamic shared memory; the attribute is per device, so it is set on
  // every launch above that limit
  if (smem + static_smem > 48 * 1024) {
    const cudaError_t e = cudaFuncSetAttribute(jlinkage_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  jlinkage_kernel<<<grid, 256, smem, s>>>(p);
  return cudaGetLastError();
}

} // namespace lm
