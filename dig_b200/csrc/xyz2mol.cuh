// Bond orders and validity of one generated geometry (reference dig/ggraph3D/utils/eval_validity_utils.py, xyz2mol with
// use_graph=True), as __host__ __device__ code: csrc/xyz2mol.cu runs it with one thread per molecule, and the CPU tests
// compile this header alone with a host compiler to check it against networkx without a device.
//
//   1. distances  d_ij = sqrt((dx*dx + dy*dy) + dz*dz) in fp64, each op correctly rounded (scipy's distance_matrix)
//   2. AC         i = 1..n-1, j = 0..i-1: bond when (min z, max z) has a threshold, d_ij <= threshold and j's running
//                 degree is below its valence (only j is capped)                                        (get_AC :32-69)
//   3. valid      0 when AC is disconnected, an atom's degree exceeds its valence or its element has none (AC2BO)
//   4. BO         BO = AC; while the maximum matching of the AC graph on the unsaturated atoms is not empty, add it
//                 (get_UA / get_UA_pairs / get_BO :114-174); with a single valence combination AC2BO returns this BO
//
// The matching is a port of networkx.max_weight_matching (Galil's O(n^3) blossom algorithm after J. van Rantwijk,
// integer duals, maxcardinality=False, all weights 1) that keeps networkx's iteration orders, because a graph with
// several maximum matchings gets networkx's one only that way: nodes in order of first appearance in the reference's
// bond list, each node's neighbours in edge insertion order (ascending atom index here), the S-vertex queue popped
// from the back, blossoms in creation order in the dual updates, strict `<` in every least-slack search, and the
// leaf order of networkx's Blossom.leaves().  Recursion (augmentBlossom, expandBlossom) is unrolled on explicit stacks.
//
// Limits: n <= 64 atoms (AC rows are uint64 masks).  A blossom's children and edges live in fixed arrays; their
// bounds follow from the laminar blossom family (at most 31 blossoms, 63 children each, for 64 vertices).  A bound
// that is ever exceeded makes xyz2mol_one return kInternalError instead of writing past an array.
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define X2M_HD __host__ __device__
#else
#define X2M_HD
#endif

namespace x2m {

constexpr int kMaxAtoms = 64;
constexpr int kMaxBlossoms = 32;                     // ids kMaxAtoms .. kMaxAtoms + kMaxBlossoms - 1
constexpr int kIds = kMaxAtoms + kMaxBlossoms;
constexpr int kInternalError = -1;

X2M_HD inline int popc64(uint64_t x) {
#ifdef __CUDA_ARCH__
  return __popcll(x);
#else
  return __builtin_popcountll(x);
#endif
}

X2M_HD inline int ctz64(uint64_t x) {
#ifdef __CUDA_ARCH__
  return __ffsll((long long)x) - 1;
#else
  return __builtin_ctzll(x);
#endif
}

// d = sqrt((dx*dx + dy*dy) + dz*dz), every operation rounded once (no contraction into FMAs)
X2M_HD inline double distance(const double* a, const double* b) {
#ifdef __CUDA_ARCH__
  const double dx = __dsub_rn(a[0], b[0]), dy = __dsub_rn(a[1], b[1]), dz = __dsub_rn(a[2], b[2]);
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
#else
  volatile double dx = a[0] - b[0], dy = a[1] - b[1], dz = a[2] - b[2];
  volatile double xx = dx * dx, yy = dy * dy, zz = dz * dz;
  volatile double s = xx + yy;
  volatile double t = s + zz;
  return sqrt(t);
#endif
}

// element code: H, C, N, O, F -> 0..4; every other atomic number has no valence and no bond (-1)
X2M_HD inline int element(int64_t z) {
  switch (z) {
    case 1: return 0;
    case 6: return 1;
    case 7: return 2;
    case 8: return 3;
    case 9: return 4;
    default: return -1;
  }
}

X2M_HD inline int valence(int e) {          // atomic_valence, e >= 0
  return e == 0 ? 1 : e == 1 ? 4 : e == 2 ? 3 : e == 3 ? 2 : 1;
}

// atomic_valid_bond[(min z, max z)], or a negative value for a pair without a bond type
X2M_HD inline double threshold(int ea, int eb) {
  const int lo = ea < eb ? ea : eb, hi = ea < eb ? eb : ea;
  if (lo == 0) return hi == 1 ? 1.1284 : hi == 2 ? 1.0478 : hi == 3 ? 1.0187 : -1.0;
  if (lo == 1) return hi == 1 ? 1.7721 : hi == 2 ? 1.7876 : hi == 3 ? 1.5731 : 1.3620;
  if (lo == 2) return hi == 2 ? 1.4208 : hi == 3 ? 1.7692 : -1.0;
  return -1.0;
}

// networkx.max_weight_matching on a graph of at most kMaxAtoms vertices with unit weights.  Vertices are local indices
// 0..nv-1 in node order; ids >= kMaxAtoms are non-trivial blossoms.  -1 stands for Python's None / NoNode.
struct Matcher {
  int nv;
  int err;
  uint64_t nbr[kMaxAtoms];        // neighbours of a local vertex as a mask over atom indices (iterated ascending)
  int8_t local[kMaxAtoms];        // atom index -> local vertex
  uint64_t allow[kMaxAtoms];      // allowedge, symmetric, over local indices
  int8_t mate[kMaxAtoms];
  int8_t inblossom[kMaxAtoms];
  int32_t dual[kMaxAtoms];        // 2 u(v)
  int8_t label[kIds];             // 0 None, 1 S, 2 T, 5 S with breadcrumb
  int8_t le_v[kIds], le_w[kIds];  // labeledge
  int8_t be_v[kIds], be_w[kIds];  // bestedge
  int8_t parent[kIds];            // blossomparent
  int8_t base[kIds];              // blossombase
  int32_t bdual[kMaxBlossoms];
  int8_t nchild[kMaxBlossoms];
  int8_t childs[kMaxBlossoms][kMaxAtoms];
  int8_t ed_v[kMaxBlossoms][kMaxAtoms], ed_w[kMaxBlossoms][kMaxAtoms];
  int8_t nbest[kMaxBlossoms];     // length of mybestedges, -1 for None
  int8_t mb_v[kMaxBlossoms][kMaxAtoms], mb_w[kMaxBlossoms][kMaxAtoms];
  int8_t order[kMaxBlossoms];     // live blossoms in creation order (the key order of blossomparent / blossomdual)
  int norder;
  int8_t freeid[kMaxBlossoms];
  int nfree;
  int8_t queue[2 * kMaxAtoms];
  int nq;

  X2M_HD static bool is_blossom(int t) { return t >= kMaxAtoms; }
  X2M_HD int slack(int v, int w) const { return dual[v] + dual[w] - 2; }

  X2M_HD void push(int v) {
    if (nq < 2 * kMaxAtoms) queue[nq++] = (int8_t)v;
    else err = 1;
  }

  // Blossom.leaves(): a stack seeded with the children, popped from the back, blossoms replaced by their children
  X2M_HD int leaves(int b, int8_t* out) {
    int8_t st[kIds];
    int ns = 0, n = 0;
    const int s0 = b - kMaxAtoms;
    for (int k = 0; k < nchild[s0]; ++k) st[ns++] = childs[s0][k];
    while (ns) {
      const int t = st[--ns];
      if (is_blossom(t)) {
        const int s = t - kMaxAtoms;
        if (ns + nchild[s] > kIds) { err = 1; return n; }
        for (int k = 0; k < nchild[s]; ++k) st[ns++] = childs[s][k];
      } else {
        out[n++] = (int8_t)t;
      }
    }
    return n;
  }

  X2M_HD void assign_label(int w, int t, int v) {
    for (;;) {
      const int b = inblossom[w];
      label[w] = label[b] = (int8_t)t;
      le_v[w] = le_v[b] = (int8_t)v;
      le_w[w] = le_w[b] = (int8_t)w;
      be_v[w] = be_v[b] = -1;
      if (t == 1) {
        if (is_blossom(b)) {
          int8_t lv[kMaxAtoms];
          const int nl = leaves(b, lv);
          for (int k = 0; k < nl; ++k) push(lv[k]);
        } else {
          push(b);
        }
        return;
      }
      const int bs = base[b];                   // T: label the mate of the base S
      w = mate[bs];
      t = 1;
      v = bs;
    }
  }

  X2M_HD int scan_blossom(int v, int w) {
    int8_t path[kIds];
    int np = 0, found = -1;
    while (v != -1) {
      int b = inblossom[v];
      if (label[b] & 4) { found = base[b]; break; }
      path[np++] = (int8_t)b;
      label[b] = 5;
      if (le_v[b] == -1) {
        v = -1;
      } else {
        v = le_v[b];
        b = inblossom[v];
        v = le_v[b];
      }
      if (w != -1) { const int x = v; v = w; w = x; }
    }
    for (int k = 0; k < np; ++k) label[path[k]] = 1;
    return found;
  }

  X2M_HD void consider(int i, int j, int k_v, int k_w, int b, int8_t* bt_v, int8_t* bt_w, int8_t* keys, int& nkeys) {
    if (inblossom[j] == b) { const int x = i; i = j; j = x; }
    const int bj = inblossom[j];
    if (bj != b && label[bj] == 1 && (bt_v[bj] == -1 || slack(i, j) < slack(bt_v[bj], bt_w[bj]))) {
      if (bt_v[bj] == -1) keys[nkeys++] = (int8_t)bj;
      bt_v[bj] = (int8_t)k_v;
      bt_w[bj] = (int8_t)k_w;
    }
  }

  X2M_HD void add_blossom(int bse, int v, int w) {
    const int bb = inblossom[bse];
    int bv = inblossom[v], bw = inblossom[w];
    if (nfree == 0) { err = 1; return; }
    const int b = freeid[--nfree], s = b - kMaxAtoms;
    order[norder++] = (int8_t)b;
    base[b] = (int8_t)bse;
    parent[b] = -1;
    parent[bb] = (int8_t)b;
    int nc = 0;
    int8_t* ch = childs[s];
    int8_t* ev = ed_v[s];
    int8_t* ew = ed_w[s];
    ev[0] = (int8_t)v;
    ew[0] = (int8_t)w;
    int ne = 1;
    while (bv != bb) {
      if (nc >= kMaxAtoms - 1 || ne >= kMaxAtoms) { err = 1; return; }
      parent[bv] = (int8_t)b;
      ch[nc++] = (int8_t)bv;
      ev[ne] = le_v[bv];
      ew[ne++] = le_w[bv];
      v = le_v[bv];
      bv = inblossom[v];
    }
    ch[nc++] = (int8_t)bb;
    for (int a = 0, z = nc - 1; a < z; ++a, --z) { const int8_t x = ch[a]; ch[a] = ch[z]; ch[z] = x; }
    for (int a = 0, z = ne - 1; a < z; ++a, --z) {
      int8_t x = ev[a]; ev[a] = ev[z]; ev[z] = x;
      x = ew[a]; ew[a] = ew[z]; ew[z] = x;
    }
    while (bw != bb) {
      if (nc >= kMaxAtoms || ne >= kMaxAtoms) { err = 1; return; }
      parent[bw] = (int8_t)b;
      ch[nc++] = (int8_t)bw;
      ev[ne] = le_w[bw];
      ew[ne++] = le_v[bw];
      w = le_v[bw];
      bw = inblossom[w];
    }
    nchild[s] = (int8_t)nc;
    label[b] = 1;
    le_v[b] = le_v[bb];
    le_w[b] = le_w[bb];
    bdual[s] = 0;
    {
      int8_t lv[kMaxAtoms];
      const int nl = leaves(b, lv);
      for (int k = 0; k < nl; ++k) {
        if (label[inblossom[lv[k]]] == 2) push(lv[k]);
        inblossom[lv[k]] = (int8_t)b;
      }
    }
    // b.mybestedges: the least-slack edge to each neighbouring top-level S-blossom, keyed in order of first insertion
    int8_t bt_v[kIds], bt_w[kIds], keys[kIds];
    int nkeys = 0;
    for (int k = 0; k < kIds; ++k) bt_v[k] = -1;
    for (int c = 0; c < nc; ++c) {
      const int sb = ch[c];
      if (is_blossom(sb) && nbest[sb - kMaxAtoms] >= 0) {
        const int q = sb - kMaxAtoms;
        for (int k = 0; k < nbest[q]; ++k) consider(mb_v[q][k], mb_w[q][k], mb_v[q][k], mb_w[q][k], b, bt_v, bt_w, keys,
                                                    nkeys);
        nbest[q] = -1;
      } else if (is_blossom(sb)) {
        int8_t lv[kMaxAtoms];
        const int nl = leaves(sb, lv);
        for (int k = 0; k < nl; ++k)
          for (uint64_t m = nbr[lv[k]]; m; m &= m - 1) {
            const int x = local[ctz64(m)];
            consider(lv[k], x, lv[k], x, b, bt_v, bt_w, keys, nkeys);
          }
      } else {
        for (uint64_t m = nbr[sb]; m; m &= m - 1) {
          const int x = local[ctz64(m)];
          consider(sb, x, sb, x, b, bt_v, bt_w, keys, nkeys);
        }
      }
      be_v[sb] = -1;
    }
    if (nkeys > kMaxAtoms) { err = 1; return; }
    nbest[s] = (int8_t)nkeys;
    int best_v = -1, best_w = -1, best_slack = 0;
    for (int k = 0; k < nkeys; ++k) {
      mb_v[s][k] = bt_v[keys[k]];
      mb_w[s][k] = bt_w[keys[k]];
      const int ks = slack(mb_v[s][k], mb_w[s][k]);
      if (best_v == -1 || ks < best_slack) { best_v = mb_v[s][k]; best_w = mb_w[s][k]; best_slack = ks; }
    }
    be_v[b] = (int8_t)best_v;
    be_w[b] = (int8_t)best_w;
  }

  X2M_HD static int wrap(int j, int n) { return j < 0 ? j + n : j; }

  X2M_HD int child_index(int b, int t) const {
    const int s = b - kMaxAtoms;
    for (int k = 0; k < nchild[s]; ++k)
      if (childs[s][k] == t) return k;
    return 0;
  }

  X2M_HD void remove_blossom(int b) {
    label[b] = 0;
    le_v[b] = -1;
    be_v[b] = -1;
    parent[b] = -1;
    int k = 0;
    while (k < norder && order[k] != b) ++k;
    for (; k + 1 < norder; ++k) order[k] = order[k + 1];
    --norder;
    freeid[nfree++] = (int8_t)b;
  }

  // the relabelling of expandBlossom when a T-blossom is expanded during a stage (label.get(b) == 2, not endstage)
  X2M_HD void relabel_expanded_t(int b) {
    const int s = b - kMaxAtoms, len = nchild[s];
    const int8_t* ch = childs[s];
    const int8_t* ev = ed_v[s];
    const int8_t* ew = ed_w[s];
    const int entry = inblossom[le_w[b]];
    int j = child_index(b, entry), jstep;
    if (j & 1) { j -= len; jstep = 1; }
    else jstep = -1;
    int v = le_v[b], w = le_w[b];
    while (j != 0) {
      int p, q;
      if (jstep == 1) { p = ev[wrap(j, len)]; q = ew[wrap(j, len)]; }
      else { q = ev[wrap(j - 1, len)]; p = ew[wrap(j - 1, len)]; }
      label[w] = 0;
      label[q] = 0;
      assign_label(w, 2, v);
      allow[p] |= 1ull << q;
      allow[q] |= 1ull << p;
      j += jstep;
      if (jstep == 1) { v = ev[wrap(j, len)]; w = ew[wrap(j, len)]; }
      else { w = ev[wrap(j - 1, len)]; v = ew[wrap(j - 1, len)]; }
      allow[v] |= 1ull << w;
      allow[w] |= 1ull << v;
      j += jstep;
    }
    const int bw = ch[wrap(j, len)];
    label[w] = label[bw] = 2;
    le_v[w] = le_v[bw] = (int8_t)v;
    le_w[w] = le_w[bw] = (int8_t)w;
    be_v[bw] = -1;
    j += jstep;
    while (ch[wrap(j, len)] != entry) {
      const int bv = ch[wrap(j, len)];
      if (label[bv] == 1) { j += jstep; continue; }
      int x = bv;
      if (is_blossom(bv)) {
        int8_t lv[kMaxAtoms];
        const int nl = leaves(bv, lv);
        for (int k = 0; k < nl; ++k) {
          x = lv[k];
          if (label[x]) break;
        }
      }
      if (label[x]) {
        label[x] = 0;
        label[mate[base[bv]]] = 0;
        assign_label(x, 2, le_v[x]);
      }
      j += jstep;
    }
  }

  X2M_HD void expand_blossom(int b0, bool endstage) {
    int8_t fb[kMaxBlossoms], fi[kMaxBlossoms];
    int depth = 0;
    fb[depth] = (int8_t)b0;
    fi[depth++] = 0;
    while (depth) {
      const int b = fb[depth - 1], i = fi[depth - 1], s = b - kMaxAtoms;
      if (i < nchild[s]) {
        const int c = childs[s][i];
        fi[depth - 1] = (int8_t)(i + 1);
        parent[c] = -1;
        if (is_blossom(c)) {
          if (endstage && bdual[c - kMaxAtoms] == 0) {
            if (depth >= kMaxBlossoms) { err = 1; return; }
            fb[depth] = (int8_t)c;
            fi[depth++] = 0;
          } else {
            int8_t lv[kMaxAtoms];
            const int nl = leaves(c, lv);
            for (int k = 0; k < nl; ++k) inblossom[lv[k]] = (int8_t)c;
          }
        } else {
          inblossom[c] = (int8_t)c;
        }
        continue;
      }
      if (!endstage && label[b] == 2) relabel_expanded_t(b);
      remove_blossom(b);
      --depth;
    }
  }

  X2M_HD void augment_blossom(int b0, int v0) {
    // frame: blossom, entry vertex, i, j, jstep, pending edge (w, x), resume point
    int8_t fb[kMaxBlossoms], fv[kMaxBlossoms], fw[kMaxBlossoms], fx[kMaxBlossoms], fph[kMaxBlossoms];
    int16_t fi[kMaxBlossoms], fj[kMaxBlossoms], fs[kMaxBlossoms];
    int depth = 0;
    fb[0] = (int8_t)b0;
    fv[0] = (int8_t)v0;
    fph[0] = 0;
    depth = 1;
    while (depth) {
      const int d = depth - 1, b = fb[d], s = b - kMaxAtoms, len = nchild[s];
      if (fph[d] == 0) {
        int t = fv[d];
        while (parent[t] != b) t = parent[t];
        const int i = child_index(b, t);
        fi[d] = (int16_t)i;
        if (i & 1) { fj[d] = (int16_t)(i - len); fs[d] = 1; }
        else { fj[d] = (int16_t)i; fs[d] = -1; }
        fph[d] = 1;
        if (is_blossom(t)) {
          if (depth >= kMaxBlossoms) { err = 1; return; }
          fb[depth] = (int8_t)t; fv[depth] = fv[d]; fph[depth] = 0; ++depth;
        }
        continue;
      }
      if (fph[d] == 1) {
        if (fj[d] == 0) {                       // rotate the children to put the new base at the front
          const int i = fi[d];
          int8_t tc[kMaxAtoms], tv[kMaxAtoms], tw[kMaxAtoms];
          for (int k = 0; k < len; ++k) {
            tc[k] = childs[s][(i + k) % len];
            tv[k] = ed_v[s][(i + k) % len];
            tw[k] = ed_w[s][(i + k) % len];
          }
          for (int k = 0; k < len; ++k) { childs[s][k] = tc[k]; ed_v[s][k] = tv[k]; ed_w[s][k] = tw[k]; }
          base[b] = base[childs[s][0]];
          --depth;
          continue;
        }
        int j = fj[d] + fs[d];
        const int t = childs[s][wrap(j, len)];
        if (fs[d] == 1) { fw[d] = ed_v[s][wrap(j, len)]; fx[d] = ed_w[s][wrap(j, len)]; }
        else { fx[d] = ed_v[s][wrap(j - 1, len)]; fw[d] = ed_w[s][wrap(j - 1, len)]; }
        fj[d] = (int16_t)j;
        fph[d] = 2;
        if (is_blossom(t)) {
          if (depth >= kMaxBlossoms) { err = 1; return; }
          fb[depth] = (int8_t)t; fv[depth] = fw[d]; fph[depth] = 0; ++depth;
        }
        continue;
      }
      if (fph[d] == 2) {
        const int j = fj[d] + fs[d];
        const int t = childs[s][wrap(j, len)];
        fj[d] = (int16_t)j;
        fph[d] = 3;
        if (is_blossom(t)) {
          if (depth >= kMaxBlossoms) { err = 1; return; }
          fb[depth] = (int8_t)t; fv[depth] = fx[d]; fph[depth] = 0; ++depth;
        }
        continue;
      }
      mate[fw[d]] = fx[d];                     // fph == 3: match the edge connecting the two sub-blossoms
      mate[fx[d]] = fw[d];
      fph[d] = 1;
    }
  }

  X2M_HD void augment_matching(int v, int w) {
    for (int pass = 0; pass < 2; ++pass) {
      int s = pass == 0 ? v : w, j = pass == 0 ? w : v;
      for (;;) {
        const int bs = inblossom[s];
        if (is_blossom(bs)) augment_blossom(bs, s);
        mate[s] = (int8_t)j;
        if (le_v[bs] == -1) break;
        const int t = le_v[bs], bt = inblossom[t];
        s = le_v[bt];
        j = le_w[bt];
        if (is_blossom(bt)) augment_blossom(bt, j);
        mate[j] = (int8_t)s;
      }
    }
  }

  // Runs the matching on the graph already described by nv / nbr / local; leaves mate[].
  X2M_HD void solve() {
    err = 0;
    for (int v = 0; v < nv; ++v) {
      mate[v] = -1;
      inblossom[v] = (int8_t)v;
      dual[v] = 1;                              // maxweight
      parent[v] = -1;
      base[v] = (int8_t)v;
    }
    norder = 0;
    nfree = kMaxBlossoms;
    for (int k = 0; k < kMaxBlossoms; ++k) freeid[k] = (int8_t)(kIds - 1 - k);
    if (nv == 0) return;
    for (;;) {                                  // stages
      for (int k = 0; k < kIds; ++k) { label[k] = 0; le_v[k] = -1; be_v[k] = -1; }
      for (int k = 0; k < norder; ++k) nbest[order[k] - kMaxAtoms] = -1;
      for (int v = 0; v < nv; ++v) allow[v] = 0;
      nq = 0;
      for (int v = 0; v < nv; ++v)
        if (mate[v] == -1 && label[inblossom[v]] == 0) assign_label(v, 1, -1);
      bool augmented = false;
      for (;;) {                                // substages
        while (nq && !augmented) {
          if (err) return;
          const int v = queue[--nq];
          for (uint64_t m = nbr[v]; m; m &= m - 1) {
            const int w = local[ctz64(m)];
            const int bv = inblossom[v], bw = inblossom[w];
            if (bv == bw) continue;
            int kslack = 0;
            if (!((allow[v] >> w) & 1)) {
              kslack = slack(v, w);
              if (kslack <= 0) { allow[v] |= 1ull << w; allow[w] |= 1ull << v; }
            }
            if ((allow[v] >> w) & 1) {
              if (label[bw] == 0) {
                assign_label(w, 2, v);
              } else if (label[bw] == 1) {
                const int bse = scan_blossom(v, w);
                if (bse != -1) {
                  add_blossom(bse, v, w);
                  if (err) return;
                } else {
                  augment_matching(v, w);
                  augmented = true;
                  break;
                }
              } else if (label[w] == 0) {
                label[w] = 2;
                le_v[w] = (int8_t)v;
                le_w[w] = (int8_t)w;
              }
            } else if (label[bw] == 1) {
              if (be_v[bv] == -1 || kslack < slack(be_v[bv], be_w[bv])) { be_v[bv] = (int8_t)v; be_w[bv] = (int8_t)w; }
            } else if (label[w] == 0) {
              if (be_v[w] == -1 || kslack < slack(be_v[w], be_w[w])) { be_v[w] = (int8_t)v; be_w[w] = (int8_t)w; }
            }
          }
        }
        if (err) return;
        if (augmented) break;
        int dtype = 1, delta = dual[0], dv = -1, dw = -1, dblossom = -1;
        for (int v = 1; v < nv; ++v)
          if (dual[v] < delta) delta = dual[v];
        for (int v = 0; v < nv; ++v)
          if (label[inblossom[v]] == 0 && be_v[v] != -1) {
            const int d = slack(be_v[v], be_w[v]);
            if (d < delta) { delta = d; dtype = 2; dv = be_v[v]; dw = be_w[v]; }
          }
        for (int k = 0; k < nv + norder; ++k) {
          const int b = k < nv ? k : order[k - nv];
          if (parent[b] == -1 && label[b] == 1 && be_v[b] != -1) {
            const int d = slack(be_v[b], be_w[b]) / 2;
            if (d < delta) { delta = d; dtype = 3; dv = be_v[b]; dw = be_w[b]; }
          }
        }
        for (int k = 0; k < norder; ++k) {
          const int b = order[k];
          if (parent[b] == -1 && label[b] == 2 && bdual[b - kMaxAtoms] < delta) {
            delta = bdual[b - kMaxAtoms];
            dtype = 4;
            dblossom = b;
          }
        }
        for (int v = 0; v < nv; ++v) {
          const int l = label[inblossom[v]];
          if (l == 1) dual[v] -= delta;
          else if (l == 2) dual[v] += delta;
        }
        for (int k = 0; k < norder; ++k) {
          const int b = order[k];
          if (parent[b] == -1) {
            if (label[b] == 1) bdual[b - kMaxAtoms] += delta;
            else if (label[b] == 2) bdual[b - kMaxAtoms] -= delta;
          }
        }
        if (dtype == 1) break;
        if (dtype == 2 || dtype == 3) {
          allow[dv] |= 1ull << dw;
          allow[dw] |= 1ull << dv;
          push(dv);
        } else {
          expand_blossom(dblossom, false);
        }
        if (err) return;
      }
      if (!augmented) return;
      int8_t snap[kMaxBlossoms];
      const int ns = norder;
      for (int k = 0; k < ns; ++k) snap[k] = order[k];
      for (int k = 0; k < ns; ++k) {
        const int b = snap[k];
        bool live = false;
        for (int q = 0; q < norder; ++q) live = live || order[q] == b;
        if (live && parent[b] == -1 && label[b] == 1 && bdual[b - kMaxAtoms] == 0) expand_blossom(b, true);
        if (err) return;
      }
    }
  }
};

// xyz2mol(z, pos) for one molecule of n atoms (1 <= n <= kMaxAtoms).  bo: the molecule's n x n slice of the output,
// written with AC and then the matching increments.  Returns the validity flag (0 / 1), or kInternalError.
X2M_HD inline int xyz2mol_one(int n, const int64_t* z, const double* pos, int8_t* bo, Matcher& m) {
  uint64_t ac[kMaxAtoms];
  int8_t el[kMaxAtoms];
  for (int i = 0; i < n; ++i) {
    el[i] = (int8_t)element(z[i]);
    ac[i] = 0;
  }
  for (int i = 1; i < n; ++i) {
    if (el[i] < 0) continue;
    for (int j = 0; j < i; ++j) {
      if (el[j] < 0) continue;
      const double thr = threshold(el[i], el[j]);
      if (thr < 0.0) continue;
      if (distance(pos + 3 * i, pos + 3 * j) <= thr && popc64(ac[j]) < valence(el[j])) {
        ac[i] |= 1ull << j;
        ac[j] |= 1ull << i;
      }
    }
  }
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < n; ++j) bo[(int64_t)i * n + j] = (int8_t)((ac[i] >> j) & 1);
  // check_connected: breadth-first closure from atom 0
  const uint64_t all = n == 64 ? ~0ull : (1ull << n) - 1;
  uint64_t seen = 1, frontier = 1;
  while (frontier) {
    uint64_t next = 0;
    for (uint64_t f = frontier; f; f &= f - 1) next |= ac[ctz64(f)];
    frontier = next & ~seen;
    seen |= next;
  }
  if (seen != all) return 0;
  int val[kMaxAtoms];                           // BO row sums
  uint64_t ua = 0;
  for (int i = 0; i < n; ++i) {
    val[i] = popc64(ac[i]);
    if (el[i] < 0 || val[i] > valence(el[i])) return 0;
    if (val[i] < valence(el[i])) ua |= 1ull << i;
  }
  while (ua) {
    // the matching graph: AC bonds among unsaturated atoms, nodes in order of first appearance in get_bonds' list
    m.nv = 0;
    for (uint64_t r = ua; r; r &= r - 1) m.local[ctz64(r)] = -1;
    for (uint64_t r = ua; r; r &= r - 1) {
      const int i = ctz64(r);
      const uint64_t up = ac[i] & ua & ~((2ull << i) - 1);
      if (!up) continue;
      if (m.local[i] < 0) m.local[i] = (int8_t)m.nv++;
      for (uint64_t u = up; u; u &= u - 1) {
        const int j = ctz64(u);
        if (m.local[j] < 0) m.local[j] = (int8_t)m.nv++;
      }
    }
    if (m.nv == 0) break;
    for (uint64_t r = ua; r; r &= r - 1) {
      const int i = ctz64(r);
      if (m.local[i] >= 0) m.nbr[m.local[i]] = ac[i] & ua;
    }
    m.solve();
    if (m.err) return kInternalError;
    bool added = false;
    for (uint64_t r = ua; r; r &= r - 1) {
      const int i = ctz64(r), li = m.local[i];
      if (li < 0 || m.mate[li] < 0) continue;
      const uint64_t nb = m.nbr[li];
      for (uint64_t u = nb; u; u &= u - 1) {    // the atom of the mate (a neighbour of i)
        const int j = ctz64(u);
        if (m.local[j] == m.mate[li]) {
          bo[(int64_t)i * n + j] += 1;
          ++val[i];
          added = true;
          break;
        }
      }
    }
    if (!added) break;
    ua = 0;
    for (int i = 0; i < n; ++i)
      if (val[i] < valence(el[i])) ua |= 1ull << i;
  }
  return 1;
}

}  // namespace x2m
