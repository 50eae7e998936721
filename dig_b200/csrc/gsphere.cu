// G-SphereNet generation step (reference dig/ggraph3D/method/G_SphereNet/model/sphgen.py:82-204) and the parts of its
// SphereNet copy (model/spherenet.py) that the threedgraph SphereNet does not have.  The dense layers run on the
// existing linear primitives; everything element-wise, segmented or index-shuffling of a step lives here.
//
// Generation state is padded per molecule: z[G, ld] (int64), pos[G, ld, 3], focus[G, ld] (int64); every active molecule
// holds the same number of atoms n at a given step, so molecule g's atoms are rows g*n .. g*n + n - 1 of the flattened
// node arrays.
#include <math.h>

#include "common.cuh"
#include "gsphere_att.cuh"

using namespace dig3d;

namespace {

constexpr int kThreads = 256;

// ---- SphereNet copy: masked re-scatters -----------------------------------------------------------------------------
// flag[e] = 1 for every edge that appears in cat(idx_ji, idx_kj) (spherenet.py:170): an edge with triplets of its own,
// or the k->j edge of some triplet.  Only ones are written (no read-modify-write): the caller zeroes flag.
__global__ void edge_flags_kernel(const int32_t* __restrict__ trip_ptr, const int64_t* __restrict__ idx_kj,
                                  int64_t n_edges, int64_t n_triplets, int32_t* __restrict__ flag) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n_edges && trip_ptr[t + 1] > trip_ptr[t]) flag[t] = 1;
  if (t < n_triplets) flag[idx_kj[t]] = 1;
}

// x[r] = fb[r] + (x[r] - fb[r]) for kept rows (the mean of identical messages, spherenet.py:171-172,205,297),
// fb[r] for the others; fb = fallback[idx ? idx[r] : r] or 0.  A row is kept when flag[r] != 0 or, without flag,
// when its CSR segment ptr[r] .. ptr[r+1] is not empty.
__global__ void keep_rows_kernel(const int32_t* __restrict__ flag, const int32_t* __restrict__ ptr,
                                 float* __restrict__ x, const float* __restrict__ fallback,
                                 const int64_t* __restrict__ fb_idx, int64_t rows, int width) {
  const int64_t n = rows * width;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = k / width;
    const int c = (int)(k - r * width);
    const bool keep = flag ? flag[r] != 0 : ptr[r + 1] > ptr[r];
    float fb = 0.f;
    if (fallback) fb = fallback[(fb_idx ? fb_idx[r] : r) * width + c];
    x[k] = keep ? (fallback ? __fadd_rn(fb, __fsub_rn(x[k], fb)) : x[k]) : fb;
  }
}

// ---- attention pooling (att.py:18-35) -------------------------------------------------------------------------------
// One CTA per query, one warp per head, lane = channel of the head (d_k = 32).  Keys / values of query g are the rows
// g*n_keys .. g*n_keys + n_keys - 1 of kv ([rows, ld_kv], keys at column k_off, values at v_off).  Softmax with the
// segment maximum subtracted and 1e-16 added to the sum (torch_geometric.utils.softmax).
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void attention_kernel(const float* __restrict__ q, const float* __restrict__ kv, int ld_kv, int k_off,
                                 int v_off, int n_keys, int n_heads, float* __restrict__ out) {
  const int g = blockIdx.x;
  const int h = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (h >= n_heads) return;
  const int width = n_heads * 32;
  const int c = h * 32 + lane;
  const float qv = q[(int64_t)g * width + c];
  const float scale = sqrtf(32.f);
  const float* base = kv + (int64_t)g * n_keys * ld_kv;
  float m = -INFINITY;
  for (int k = 0; k < n_keys; ++k) {
    const float s = __fdiv_rn(warp_sum(qv * base[(int64_t)k * ld_kv + k_off + c]), scale);
    m = fmaxf(m, s);
  }
  float sum = 0.f;
  for (int k = 0; k < n_keys; ++k) {
    const float s = __fdiv_rn(warp_sum(qv * base[(int64_t)k * ld_kv + k_off + c]), scale);
    sum += expf(s - m);
  }
  const float denom = sum + 1e-16f;
  float acc = 0.f;
  for (int k = 0; k < n_keys; ++k) {
    const float s = __fdiv_rn(warp_sum(qv * base[(int64_t)k * ld_kv + k_off + c]), scale);
    acc = fmaf(base[(int64_t)k * ld_kv + v_off + c], __fdiv_rn(expf(s - m), denom), acc);
  }
  out[(int64_t)g * width + c] = acc;
}

// ---- attention pooling, any head width d_k (lane mapping: gsphere_att.cuh) --------------------------------------------
// attention_kernel's op sequence with the scores summed over a head's slices; the weighted value sum runs per slice.
__global__ void attention_dk_kernel(const float* __restrict__ q, const float* __restrict__ kv, int ld_kv, int k_off,
                                    int v_off, int n_keys, int n_heads, int d_k, int seg, float scale,
                                    float* __restrict__ out) {
  const int64_t g = blockIdx.x;
  const int warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5, per_warp = 32 / seg;
  const float* base = kv + g * n_keys * ld_kv;
  for (int h0 = warp * per_warp; h0 < n_heads; h0 += n_warps * per_warp) {      // uniform across the warp
    const HeadLanes l = head_lanes(h0, n_heads, d_k, seg);
    const int64_t hc = (int64_t)l.h * d_k;
    const float* qh = q + g * l.width + hc;
    auto score = [&](int k) { return __fdiv_rn(l.dot(qh, base + (int64_t)k * ld_kv + k_off + hc), scale); };
    float m = -INFINITY;
    for (int k = 0; k < n_keys; ++k) m = fmaxf(m, score(k));
    float sum = 0.f;
    for (int k = 0; k < n_keys; ++k) sum += expf(score(k) - m);
    const float denom = sum + 1e-16f;
    for (int i = 0; i < l.slices; ++i) {
      const bool own = l.owns(i);
      const int64_t c = l.col(i);
      float acc = 0.f;
      for (int k = 0; k < n_keys; ++k)
        acc = fmaf(own ? base[(int64_t)k * ld_kv + v_off + c] : 0.f, __fdiv_rn(expf(score(k) - m), denom), acc);
      if (own) out[g * l.width + c] = acc;
    }
  }
}

// ---- flow reverse (net_utils.py:28-37,75-80) ------------------------------------------------------------------------
__global__ void tanh_kernel(const float* __restrict__ x, int64_t n, float* __restrict__ y) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x)
    y[k] = tanhf(x[k]);
}

// st[g, l, :] = linear2 output of flow layer l ([s | t], 2*dim wide; all layers from one block-diagonal GEMM); layers
// applied last to first: s = exp(exp(w_l) * tanh(s)), latent = latent / s - t.
__global__ void flow_reverse_kernel(const float* __restrict__ st, const float* __restrict__ rescale, int64_t rows,
                                    int dim, int n_layers, float* __restrict__ latent) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= rows * dim) return;
  const int64_t g = k / dim;
  const int d = (int)(k - g * dim);
  float x = latent[k];
  for (int l = n_layers - 1; l >= 0; --l) {
    const float* row = st + (g * n_layers + l) * 2 * dim;
    const float s = expf(__fmul_rn(expf(rescale[l]), tanhf(row[d])));
    x = __fsub_rn(__fdiv_rn(x, s), row[dim + d]);
  }
  latent[k] = x;
}

// ---- focus decision and compaction (sphgen.py:116-142) --------------------------------------------------------------
// Single CTA.  score = sigmoid(logit); an atom can be the focus when score < focus_th and z > 0; a molecule without
// one is complete (emitted when `emit`), one with a NaN / inf score is dropped, the others continue.  Continuing and
// emitted molecules keep their order: cont_src / emit_src list their rows, can_focus[k, :] is the row of the k-th
// continuing molecule, counts = (continuing, emitted).
__global__ void __launch_bounds__(1024) focus_select_kernel(const float* __restrict__ logit,
                                                            const int64_t* __restrict__ z, int64_t n_mols, int n,
                                                            int ld, float focus_th, int emit,
                                                            float* __restrict__ score, float* __restrict__ can_focus,
                                                            int32_t* __restrict__ cont_src,
                                                            int32_t* __restrict__ emit_src, int32_t* __restrict__ counts) {
  __shared__ int s_c[1024], s_e[1024];
  __shared__ int base_c, base_e;
  if (threadIdx.x == 0) base_c = base_e = 0;
  __syncthreads();
  for (int64_t start = 0; start < n_mols; start += blockDim.x) {
    const int64_t g = start + threadIdx.x;
    int cont = 0, em = 0;
    if (g < n_mols) {
      bool any = false, dirty = false;
      for (int a = 0; a < n; ++a) {
        const float s = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-logit[g * n + a])));
        score[g * n + a] = s;
        any |= (s < focus_th) && (z[g * ld + a] > 0);
        dirty |= isnan(s) || isinf(s);
      }
      cont = any && !dirty;
      em = (!any) && emit;
    }
    s_c[threadIdx.x] = cont;
    s_e[threadIdx.x] = em;
    __syncthreads();
    for (int o = 1; o < (int)blockDim.x; o <<= 1) {       // inclusive Hillis-Steele scan of both flags
      int vc = 0, ve = 0;
      if ((int)threadIdx.x >= o) vc = s_c[threadIdx.x - o], ve = s_e[threadIdx.x - o];
      __syncthreads();
      s_c[threadIdx.x] += vc;
      s_e[threadIdx.x] += ve;
      __syncthreads();
    }
    if (cont) {
      const int k = base_c + s_c[threadIdx.x] - 1;
      cont_src[k] = (int32_t)g;
      for (int a = 0; a < n; ++a)
        can_focus[(int64_t)k * n + a] = (score[g * n + a] < focus_th && z[g * ld + a] > 0) ? 1.f : 0.f;
    }
    if (em) emit_src[base_e + s_e[threadIdx.x] - 1] = (int32_t)g;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) base_c += s_c[threadIdx.x], base_e += s_e[threadIdx.x];
    __syncthreads();
  }
  if (threadIdx.x == 0) counts[0] = base_c, counts[1] = base_e;
}

// out rows k = in rows src[k]: the first n_atoms columns of z / pos and the first n_atoms - 1 of focus.
__global__ void compact_kernel(const int32_t* __restrict__ src, int64_t rows, int n_atoms, int ld_in, int ld_out,
                               const int64_t* __restrict__ z, const float* __restrict__ pos,
                               const int64_t* __restrict__ focus, int64_t* __restrict__ z_out,
                               float* __restrict__ pos_out, int64_t* __restrict__ focus_out) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= rows * n_atoms) return;
  const int64_t r = k / n_atoms;
  const int a = (int)(k - r * n_atoms);
  const int64_t s = src[r];
  z_out[r * ld_out + a] = z[s * ld_in + a];
#pragma unroll
  for (int c = 0; c < 3; ++c) pos_out[(r * ld_out + a) * 3 + c] = pos[(s * ld_in + a) * 3 + c];
  if (a + 1 < n_atoms) focus_out[r * ld_out + a] = focus[s * ld_in + a];
}

// ---- placement (sphgen.py:151-202, geometric_computing.py:107-122) --------------------------------------------------
__device__ __forceinline__ f3 ld_pos(const float* __restrict__ pos, int64_t g, int ld, int64_t a) {
  const float* p = pos + ((g * ld) + a) * 3;
  return {p[0], p[1], p[2]};
}

__device__ __forceinline__ float sqdist(const f3 a, const f3 b) {
  const f3 d = sub3(a, b);
  return sum3_aten(mul3(d, d));
}

// c1 = the atom nearest to the focus (first minimum over the other atoms in index order, which is what argmin over the
// masked rows plus the index shift of sphgen.py:165-169 selects); c2 = the atom nearest to c1 among the rest
// (sphgen.py:185-189).
__global__ void neighbors_kernel(const float* __restrict__ pos, int ld, int64_t n_mols, int n,
                                 const int64_t* __restrict__ focus_id, int64_t* __restrict__ c1_out,
                                 int64_t* __restrict__ c2_out) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_mols) return;
  const int64_t f = focus_id[g];
  const f3 pf = ld_pos(pos, g, ld, f);
  int64_t c1 = -1;
  float best = 0.f;
  for (int a = 0; a < n; ++a) {
    if (a == f) continue;
    const float d = sqdist(ld_pos(pos, g, ld, a), pf);
    if (c1 < 0 || d < best || (isnan(d) && !isnan(best))) best = d, c1 = a;
  }
  c1_out[g] = c1;
  if (!c2_out) return;
  const f3 p1 = ld_pos(pos, g, ld, c1);
  int64_t c2 = -1;
  for (int a = 0; a < n; ++a) {
    if (a == f || a == c1) continue;
    const float d = sqdist(ld_pos(pos, g, ld, a), p1);
    if (c2 < 0 || d < best || (isnan(d) && !isnan(best))) best = d, c2 = a;
  }
  c2_out[g] = c2;
}

__device__ __forceinline__ f3 scale3(const f3 a, float s) {
  return {__fmul_rn(a.x, s), __fmul_rn(a.y, s), __fmul_rn(a.z, s)};
}
__device__ __forceinline__ f3 div3(const f3 a, float s) {
  return {__fdiv_rn(a.x, s), __fdiv_rn(a.y, s), __fdiv_rn(a.z, s)};
}
__device__ __forceinline__ f3 add3(const f3 a, const f3 b) {
  return {__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z)};
}

// The new atom of every molecule: type, position (step 0 on the x axis, step 1 in the xy plane, dattoxyz after that)
// and focus, written to column n of z / pos and column n - 1 of focus.
__global__ void place_kernel(int64_t n_mols, int n, int ld, const int64_t* __restrict__ focus_id,
                             const int64_t* __restrict__ c1_id, const int64_t* __restrict__ c2_id,
                             const float* __restrict__ dist, const float* __restrict__ angle,
                             const float* __restrict__ torsion, const int64_t* __restrict__ type_id,
                             int64_t* __restrict__ z, float* __restrict__ pos, int64_t* __restrict__ focus) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_mols) return;
  const int64_t fi = focus_id[g];
  const float d = dist[g];
  f3 p;
  if (n == 1) {
    p = {d, 0.f, 0.f};
  } else if (n == 2) {
    const f3 f = ld_pos(pos, g, ld, fi), c1 = ld_pos(pos, g, ld, c1_id[g]);
    const float x = __fsub_rn(c1.x, f.x);
    const float sg = x > 0.f ? 1.f : (x < 0.f ? -1.f : (isnan(x) ? x : 0.f));
    const float a = angle[g];
    p = {__fadd_rn(__fmul_rn(__fmul_rn(cosf(a), sg), d), f.x), __fadd_rn(__fmul_rn(__fmul_rn(sinf(a), sg), d), f.y),
         __fadd_rn(0.f, f.z)};
  } else {
    const f3 f = ld_pos(pos, g, ld, fi), c1 = ld_pos(pos, g, ld, c1_id[g]), c2 = ld_pos(pos, g, ld, c2_id[g]);
    const float a = angle[g], t = torsion[g];
    const f3 c1c2 = sub3(c2, c1), c1f = sub3(f, c1);
    const f3 c1c3 = div3(scale3(c1f, sum3_aten(mul3(c1c2, c1f))), sum3_aten(mul3(c1f, c1f)));
    const f3 c3 = add3(c1c3, c1);
    const f3 c3c2 = sub3(c2, c3);
    const float nf = norm3_aten(c1f);
    const f3 c3c4 = add3(scale3(c3c2, cosf(t)), scale3(div3(cross_aten(c3c2, c1f), nf), sinf(t)));
    const float n34 = norm3_aten(c3c4);
    const f3 neg = {-c1f.x, -c1f.y, -c1f.z};
    p = scale3(scale3(div3(neg, nf), d), cosf(a));
    p = add3(p, scale3(scale3(div3(c3c4, n34), d), sinf(a)));
    p = add3(p, f);
  }
  float* out = pos + (g * ld + n) * 3;
  out[0] = p.x, out[1] = p.y, out[2] = p.z;
  z[g * ld + n] = type_id[g];
  focus[g * ld + n - 1] = fi;
}

// out[g, j*H .. j*H + H) = feat[g*n + ids_j[g]] for the (up to three) id vectors given: the local query features
// (sphgen.py:145,156,172,192).
__global__ void gather_local_kernel(const float* __restrict__ feat, int64_t n_mols, int n, int width,
                                    const int64_t* __restrict__ id0, const int64_t* __restrict__ id1,
                                    const int64_t* __restrict__ id2, int n_ids, float* __restrict__ out) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t per = (int64_t)n_ids * width;
  if (k >= n_mols * per) return;
  const int64_t g = k / per;
  const int j = (int)((k - g * per) / width), c = (int)(k - g * per - (int64_t)j * width);
  const int64_t* ids = j == 0 ? id0 : (j == 1 ? id1 : id2);
  out[k] = feat[(g * n + ids[g]) * width + c];
}

// type[g] = argmax latent[g, :] (first maximum, NaN wins as in torch.argmax); out = feat * emb[type[g]] broadcast over
// the molecule's atoms (sphgen.py:151-153).
__global__ void type_scale_kernel(const float* __restrict__ latent, int dim, const float* __restrict__ emb,
                                  const float* __restrict__ feat, int64_t n_mols, int n, int width,
                                  int64_t* __restrict__ type_out, float* __restrict__ out) {
  const int64_t total = n_mols * n * width;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t g = k / ((int64_t)n * width);
    const int c = (int)(k % width);
    const float* row = latent + g * dim;
    int best = 0;
    float bv = row[0];
    for (int d = 1; d < dim; ++d) {
      const float v = row[d];
      if (!isnan(bv) && (v > bv || isnan(v))) bv = v, best = d;
    }
    out[k] = __fmul_rn(feat[k], emb[(int64_t)best * width + c]);
    if (type_out && k == g * n * width) type_out[g] = best;
  }
}

int grid_for(int64_t n) {
  const int64_t b = (n + kThreads - 1) / kThreads;
  return (int)(b < 4096 ? (b > 0 ? b : 1) : 4096);
}

}  // namespace

extern "C" {

int dig3d_gsphere_edge_flags(const int32_t* trip_ptr, const int64_t* idx_kj, int64_t n_edges, int64_t n_triplets,
                             int32_t* flag, void* stream) {
  DIG3D_REQUIRE(flag && (n_edges == 0 || trip_ptr) && (n_triplets == 0 || idx_kj), "gsphere_edge_flags: null pointer");
  const int64_t n = n_edges > n_triplets ? n_edges : n_triplets;
  if (n == 0) return DIG3D_OK;
  edge_flags_kernel<<<ceil_div(n, kThreads), kThreads, 0, (cudaStream_t)stream>>>(trip_ptr, idx_kj, n_edges,
                                                                                  n_triplets, flag);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_gsphere_keep_rows(const int32_t* flag, const int32_t* ptr, float* x, const float* fallback,
                            const int64_t* fallback_idx, int64_t rows, int32_t width, void* stream) {
  DIG3D_REQUIRE(x && (flag || ptr) && width > 0 && (!fallback_idx || fallback), "gsphere_keep_rows: bad arguments");
  if (rows == 0) return DIG3D_OK;
  keep_rows_kernel<<<grid_for(rows * width), kThreads, 0, (cudaStream_t)stream>>>(flag, ptr, x, fallback,
                                                                                  fallback_idx, rows, width);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_gsphere_attention(const float* q, const float* kv, int32_t ld_kv, int32_t k_off, int32_t v_off,
                            int64_t n_queries, int32_t n_keys, int32_t n_heads, float* out, void* stream) {
  DIG3D_REQUIRE(q && kv && out && n_keys > 0 && n_heads >= 1 && n_heads <= 32 && n_queries < (1LL << 31),
                "gsphere_attention: bad arguments (d_k is 32, at most 32 heads)");
  if (n_queries == 0) return DIG3D_OK;
  attention_kernel<<<(unsigned)n_queries, 32 * n_heads, 0, (cudaStream_t)stream>>>(q, kv, ld_kv, k_off, v_off, n_keys,
                                                                                  n_heads, out);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_gsphere_attention_dk(const float* q, const float* kv, int32_t ld_kv, int32_t k_off, int32_t v_off,
                               int64_t n_queries, int32_t n_keys, int32_t n_heads, int32_t d_k, float* out,
                               void* stream) {
  DIG3D_REQUIRE(q && kv && out && n_keys > 0 && n_heads >= 1 && d_k >= 1 && n_queries >= 0 &&
                    n_queries < (1LL << 31) && (int64_t)n_heads * d_k <= ld_kv,
                "gsphere_attention_dk: bad arguments");
  if (n_queries == 0) return DIG3D_OK;
  const AttShape sh = att_shape(n_heads, d_k);
  attention_dk_kernel<<<(unsigned)n_queries, sh.threads, 0, (cudaStream_t)stream>>>(
      q, kv, ld_kv, k_off, v_off, n_keys, n_heads, d_k, sh.seg, sh.scale, out);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_gsphere_tanh(const float* x, int64_t n, float* y, void* stream) {
  DIG3D_REQUIRE(x && y, "gsphere_tanh: null pointer");
  if (n == 0) return DIG3D_OK;
  tanh_kernel<<<grid_for(n), kThreads, 0, (cudaStream_t)stream>>>(x, n, y);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_gsphere_flow_reverse(const float* st, const float* rescale, int64_t rows, int32_t dim, int32_t n_layers,
                               float* latent, void* stream) {
  DIG3D_REQUIRE(st && rescale && latent && dim > 0 && n_layers > 0, "gsphere_flow_reverse: bad arguments");
  if (rows == 0) return DIG3D_OK;
  flow_reverse_kernel<<<ceil_div(rows * dim, kThreads), kThreads, 0, (cudaStream_t)stream>>>(st, rescale, rows, dim,
                                                                                            n_layers, latent);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_gsphere_focus_select(const float* logit, const int64_t* z, int64_t n_mols, int32_t n_atoms, int32_t ld,
                               double focus_th, int32_t emit, float* score, float* can_focus, int32_t* cont_src,
                               int32_t* emit_src, int32_t* counts, void* stream) {
  DIG3D_REQUIRE(logit && z && score && can_focus && cont_src && emit_src && counts && n_atoms > 0 && ld >= n_atoms,
                "gsphere_focus_select: bad arguments");
  focus_select_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(logit, z, n_mols, n_atoms, ld, (float)focus_th, emit, score,
                                                            can_focus, cont_src, emit_src, counts);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_gsphere_compact(const int32_t* src, int64_t rows, int32_t n_atoms, int32_t ld_in, int32_t ld_out,
                          const int64_t* z, const float* pos, const int64_t* focus, int64_t* z_out, float* pos_out,
                          int64_t* focus_out, void* stream) {
  DIG3D_REQUIRE(src && z && pos && focus && z_out && pos_out && focus_out && n_atoms > 0 && ld_in >= n_atoms &&
                    ld_out >= n_atoms,
                "gsphere_compact: bad arguments");
  if (rows == 0) return DIG3D_OK;
  compact_kernel<<<ceil_div(rows * n_atoms, kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      src, rows, n_atoms, ld_in, ld_out, z, pos, focus, z_out, pos_out, focus_out);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_gsphere_neighbors(const float* pos, int32_t ld, int64_t n_mols, int32_t n_atoms, const int64_t* focus_id,
                            int64_t* c1, int64_t* c2, void* stream) {
  DIG3D_REQUIRE(pos && focus_id && c1 && n_atoms >= 2 && (!c2 || n_atoms >= 3) && ld >= n_atoms,
                "gsphere_neighbors: bad arguments");
  if (n_mols == 0) return DIG3D_OK;
  neighbors_kernel<<<ceil_div(n_mols, 128), 128, 0, (cudaStream_t)stream>>>(pos, ld, n_mols, n_atoms, focus_id, c1,
                                                                             c2);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_gsphere_place(int64_t n_mols, int32_t n_atoms, int32_t ld, const int64_t* focus_id, const int64_t* c1,
                        const int64_t* c2, const float* dist, const float* angle, const float* torsion,
                        const int64_t* type_id, int64_t* z, float* pos, int64_t* focus, void* stream) {
  DIG3D_REQUIRE(focus_id && dist && type_id && z && pos && focus && n_atoms >= 1 && ld > n_atoms &&
                    (n_atoms < 2 || (c1 && angle)) && (n_atoms < 3 || (c2 && torsion)),
                "gsphere_place: bad arguments");
  if (n_mols == 0) return DIG3D_OK;
  place_kernel<<<ceil_div(n_mols, 128), 128, 0, (cudaStream_t)stream>>>(n_mols, n_atoms, ld, focus_id, c1, c2, dist,
                                                                         angle, torsion, type_id, z, pos, focus);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_gsphere_gather_local(const float* feat, int64_t n_mols, int32_t n_atoms, int32_t width, const int64_t* id0,
                               const int64_t* id1, const int64_t* id2, int32_t n_ids, float* out, void* stream) {
  DIG3D_REQUIRE(feat && out && id0 && n_ids >= 1 && n_ids <= 3 && (n_ids < 2 || id1) && (n_ids < 3 || id2) &&
                    width > 0,
                "gsphere_gather_local: bad arguments");
  if (n_mols == 0) return DIG3D_OK;
  gather_local_kernel<<<ceil_div(n_mols * n_ids * width, kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      feat, n_mols, n_atoms, width, id0, id1, id2, n_ids, out);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

int dig3d_gsphere_type_scale(const float* latent, int32_t dim, const float* emb, const float* feat, int64_t n_mols,
                             int32_t n_atoms, int32_t width, int64_t* type_out, float* out, void* stream) {
  DIG3D_REQUIRE(latent && emb && feat && out && dim > 0 && n_atoms > 0 && width > 0, "gsphere_type_scale: bad arguments");
  if (n_mols == 0) return DIG3D_OK;
  type_scale_kernel<<<grid_for(n_mols * n_atoms * width), kThreads, 0, (cudaStream_t)stream>>>(
      latent, dim, emb, feat, n_mols, n_atoms, width, type_out, out);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

}  // extern "C"
