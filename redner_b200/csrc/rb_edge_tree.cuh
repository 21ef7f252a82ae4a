// Secondary-edge trees (reference: EdgeTree::EdgeTree, src/edge_tree.cpp:724-882): the steps that decide the trees, written once.
// host_build_edge_tree (rb_scene_host.hpp) runs them in serial loops, rb_edge_tree.cu runs them in kernels; both give the same records
// bit for bit because only the orchestration differs between them (sorts, reductions, the order in which the bottom-up passes visit
// the nodes, how the subset areas of a treelet are filled):
//   ETNode / ETOps        node of the reference-shaped tree and its algebra: box union, SAH area, refresh, cost propagation,
//                         treelet formation and re-wiring                                        :391-445, :546-684
//   et_leaf               edge -> leaf (position box, Hough box of the two face planes, length x exterior angle) :23-66, :749-756
//   et_morton             Morton code of a leaf centre inside its tree's bounds                 :166-266
//   et_karras_split       children of an inner node of the Karras radix tree                    :282-376
//   et_best_partition     optimal partition of one subset of a treelet's leaves (Karras & Aila 2013, Algorithm 2) :502-544
//   et_record             the 128-byte EdgeNode of an inner node that rb_secondary.cuh walks (both children's bounds)
// Everything that decides the shape of the tree is computed in double like the reference (areas, costs, Morton quantisation).
#pragma once
#include <cstring>

#include "rb_edge.cuh"

RB_HD int et_popc(unsigned x) {
#ifdef __CUDA_ARCH__
    return __popc(x);
#else
    return __builtin_popcount(x);
#endif
}
RB_HD int et_ffs(unsigned x) {
#ifdef __CUDA_ARCH__
    return __ffs((int)x);
#else
    return __builtin_ffs((int)x);
#endif
}
RB_HD int et_clz64(unsigned long long x) {
#ifdef __CUDA_ARCH__
    return __clzll((long long)x);
#else
    return x == 0 ? 64 : __builtin_clzll(x);
#endif
}
// std::min / std::max semantics: the FIRST argument wins ties -- fmin / fmax order -0 below +0, and the Hough bounds are full of
// signed zeros (axis-aligned faces); the records must equal the host builder's bit for bit
RB_HD double et_min(double a, double b) { return b < a ? b : a; }
RB_HD double et_max(double a, double b) { return a < b ? b : a; }

struct ETNode { // node of the reference-shaped tree (double precision like the reference's Real); 128 bytes
    double pmin[3], pmax[3], dmin[3], dmax[3];
    double wlen, cost;
    int parent, child[2], edge_id;
};
RB_HD ETNode et_blank_node() { // an inner node before the bottom-up passes: empty box, no links
    ETNode x;
    for (int k = 0; k < 3; k++) {
        x.pmin[k] = x.dmin[k] = INFINITY;
        x.pmax[k] = x.dmax[k] = -INFINITY;
    }
    x.wlen = 0;
    x.cost = 0;
    x.parent = -1;
    x.child[0] = x.child[1] = -1;
    x.edge_id = -1;
    return x;
}

// Node algebra on a node array.  Its members are ordinary (not force-inlined) functions: k_et_optimize calls them from a warp's lane 0.
struct ETOps {
    ETNode* n;
    int six; // the 6-D tree: areas include the Hough box
    __host__ __device__ static void merge_into(ETNode& o, const ETNode& a, const ETNode& b) {
        for (int k = 0; k < 3; k++) {
            o.pmin[k] = et_min(a.pmin[k], b.pmin[k]);
            o.pmax[k] = et_max(a.pmax[k], b.pmax[k]);
            o.dmin[k] = et_min(a.dmin[k], b.dmin[k]);
            o.dmax[k] = et_max(a.dmax[k], b.dmax[k]);
        }
    }
    __host__ __device__ double area(const ETNode& a) const {
        double dx = a.pmax[0] - a.pmin[0], dy = a.pmax[1] - a.pmin[1], dz = a.pmax[2] - a.pmin[2];
        double s = dx * dy + dx * dz + dy * dz;
        if (six) {
            double ex = a.dmax[0] - a.dmin[0], ey = a.dmax[1] - a.dmin[1], ez = a.dmax[2] - a.dmin[2];
            s += ex * ey + ex * ez + ey * ez;
        }
        return 2 * s;
    }
    __host__ __device__ void refresh(int i) { // bounds, weighted length and SAH cost of an inner node from its children
        ETNode o = n[i];
        const ETNode a = n[o.child[0]], b = n[o.child[1]];
        merge_into(o, a, b);
        o.wlen = a.wlen + b.wlen;
        o.cost = area(o) + a.cost + b.cost;
        n[i] = o;
    }
    __host__ __device__ void propagate_cost(int root, const int* lv, int cnt) { // src/edge_tree.cpp:546-579
        for (int i = 0; i < cnt; i++) {
            int cur = lv[i];
            while (cur != root) {
                if (n[cur].cost < 0) {
                    if (n[n[cur].child[0]].cost >= 0 && n[n[cur].child[1]].cost >= 0) refresh(cur);
                    else break;
                }
                cur = n[cur].parent;
            }
        }
        refresh(root);
    }
    __host__ __device__ void restruct(int parent, int child_index, const int* lv, const int* inner, unsigned char partition, const unsigned char* optimal,
                                      int& index, int cnt) { // src/edge_tree.cpp:586-626
        unsigned char st_part[8], st_child[8];
        int st_parent[8];
        int sp = 0;
        st_part[sp] = partition;
        st_child[sp] = (unsigned char)child_index;
        st_parent[sp] = parent;
        sp++;
        while (sp > 0) {
            sp--;
            unsigned char part = st_part[sp], ch = st_child[sp];
            int par = st_parent[sp];
            if (et_popc(part) == 1) {
                int leaf = lv[et_ffs(part) - 1];
                n[par].child[ch] = leaf;
                n[leaf].parent = par;
            } else {
                int node = inner[index++];
                n[node].cost = -1;
                n[par].child[ch] = node;
                n[node].parent = par;
                unsigned char lp = optimal[part];
                unsigned char rp = (unsigned char)((~lp) & part);
                st_part[sp] = lp;
                st_child[sp] = 0;
                st_parent[sp] = node;
                sp++;
                st_part[sp] = rp;
                st_child[sp] = 1;
                st_parent[sp] = node;
                sp++;
            }
        }
        propagate_cost(parent, lv, cnt);
    }
    // Treelet of inner node `root` (src/edge_tree.cpp:627-684): starting from its two children, open the inner node of largest area
    // until there are 7 treelet leaves or none is left to open.  Returns the number of treelet leaves (lv), inner gets the opened nodes.
    __host__ __device__ int treelet_form(int root, int* lv, int* inner) const {
        int cnt = 0, icnt = 0;
        lv[cnt++] = n[root].child[0];
        lv[cnt++] = n[root].child[1];
        int max_idx = 0;
        while (cnt < 7 && max_idx != -1) {
            max_idx = -1;
            double max_area = -1;
            for (int i = 0; i < cnt; i++)
                if (n[lv[i]].edge_id == -1) {
                    double ar = area(n[lv[i]]);
                    if (ar > max_area) {
                        max_area = ar;
                        max_idx = i;
                    }
                }
            if (max_idx != -1) {
                int tmp = lv[max_idx];
                inner[icnt++] = tmp;
                lv[max_idx] = lv[cnt - 1];
                lv[cnt - 1] = n[tmp].child[0];
                lv[cnt] = n[tmp].child[1];
                cnt++;
            }
        }
        return cnt;
    }
    // Re-wires the treelet of `root` by the optimal partitions of its leaf subsets (src/edge_tree.cpp:672-684).
    __host__ __device__ void treelet_rewire(int root, const int* lv, const int* inner, const unsigned char* optimal, int cnt) {
        unsigned char mask = (unsigned char)((1u << cnt) - 1);
        int index = 0;
        unsigned char left = optimal[mask];
        restruct(root, 0, lv, inner, left, optimal, index, cnt);
        unsigned char right = (unsigned char)((~left) & mask);
        restruct(root, 1, lv, inner, right, optimal, index, cnt);
        refresh(root);
    }
};

// Optimal partition of subset s (two or more leaves) of a treelet's leaves, Karras & Aila 2013 Algorithm 2 (src/edge_tree.cpp:502-544):
// needs c_opt of every smaller subset and a[s], the area of the subset's union -- which in the reference always starts from leaf 0, also
// for subsets that do not contain it (:491-500).  The partitions are tried in the reference's order, the first of equal costs wins.
RB_HD void et_best_partition(unsigned s, const double* a, double* c_opt, unsigned char* optimal) {
    double c_s = INFINITY;
    unsigned p_s = 0;
    unsigned d = (s - 1u) & s;
    unsigned p = (0u - d) & s;
    do {
        double c = c_opt[p] + c_opt[s ^ p];
        if (c < c_s) {
            c_s = c;
            p_s = p;
        }
        p = (p - d) & s;
    } while (p != 0);
    c_opt[s] = a[s] + c_s;
    optimal[s] = (unsigned char)p_s;
}

inline __host__ __device__ V3 et_edge_normal(const rb_shape* shapes, const Edge& e, int which) { // unit normal of face f0 / f1, or 0
    V3 v0 = edge_v0(shapes, e), v1 = edge_v1(shapes, e);
    V3 n;
    if (which == 0) {
        V3 o = edge_opposite0(shapes, e);
        n = cross(v0 - o, v1 - o);
    } else {
        V3 o = edge_opposite1(shapes, e);
        n = cross(v1 - o, v0 - o);
    }
    Real l2 = length_sq(n);
    if (l2 < Real(1e-20)) return zero3();
    return n / sqrt(l2);
}
// Leaf of edge `id` (src/edge_tree.cpp:23-66): box of the end points, box of the Hough transforms of the two face planes seen from the
// camera origin co, and length x exterior dihedral angle.  Returns whether the edge is a camera silhouette, i.e. belongs to the 3-D tree
// (:749-756).
RB_HD bool et_leaf(const rb_shape* shapes, const Edge& e, int id, const double co[3], ETNode& n) {
    V3 v0 = edge_v0(shapes, e), v1 = edge_v1(shapes, e);
    V3 n0 = et_edge_normal(shapes, e, 0);
    V3 n1 = e.f1 == -1 ? -n0 : et_edge_normal(shapes, e, 1);
    double p[3], p0d = 0, p1d = 0;
    for (int k = 0; k < 3; k++) p[k] = 0.5 * ((double)v0[k] + (double)v1[k]) - co[k];
    for (int k = 0; k < 3; k++) {
        p0d += p[k] * (double)n0[k];
        p1d += p[k] * (double)n1[k];
    }
    for (int k = 0; k < 3; k++) {
        double h0 = (double)n0[k] * p0d, h1 = (double)n1[k] * p1d;
        n.pmin[k] = et_min((double)v0[k], (double)v1[k]);
        n.pmax[k] = et_max((double)v0[k], (double)v1[k]);
        n.dmin[k] = et_min(h0, h1);
        n.dmax[k] = et_max(h0, h1);
    }
    double ext = M_PI;
    if (e.f1 != -1) ext = acos(et_min(1.0, et_max(-1.0, (double)dot(n0, n1))));
    n.wlen = (double)length(v1 - v0) * ext;
    n.parent = -1;
    n.child[0] = n.child[1] = -1;
    n.edge_id = id;
    n.cost = 0;
    return edge_is_silhouette(shapes, mk3((Real)co[0], (Real)co[1], (Real)co[2]), e);
}

RB_HD unsigned long long expand21(unsigned long long x) { // 2 zeros before each bit of a 21-bit integer
    x &= 0x1fffffULL;
    x = (x | x << 32) & 0x1f00000000ffffULL;
    x = (x | x << 16) & 0x1f0000ff0000ffULL;
    x = (x | x << 8) & 0x100f00f00f00f00fULL;
    x = (x | x << 4) & 0x10c30c30c30c30c3ULL;
    x = (x | x << 2) & 0x1249249249249249ULL;
    return x;
}
RB_HD unsigned long long expand10(unsigned long long x) { // 5 zeros before each bit of a 10-bit integer
    unsigned long long r = 0;
    for (int b = 0; b < 10; b++) r |= ((x >> b) & 1ULL) << (5 * b);
    return r;
}
// Morton code of the centre of leaf n inside its tree's bounds lo / hi (position axes, then Hough axes): 63 bits over the position
// for the 3-D tree, 60 bits over all six axes for the 6-D tree (src/edge_tree.cpp:166-266).
RB_HD unsigned long long et_morton(const ETNode& n, const double lo[6], const double hi[6], bool six) {
    double q[6];
    for (int k = 0; k < 3; k++) {
        double cp = 0.5 * (n.pmin[k] + n.pmax[k]), cd = 0.5 * (n.dmin[k] + n.dmax[k]);
        q[k] = hi[k] - lo[k] <= 0 ? 0.5 : (cp - lo[k]) / (hi[k] - lo[k]);
        q[3 + k] = hi[3 + k] - lo[3 + k] <= 0 ? 0.5 : (cd - lo[3 + k]) / (hi[3 + k] - lo[3 + k]);
    }
    if (!six) {
        double sc = (1 << 21) - 1;
        return (expand21((unsigned long long)(q[0] * sc)) << 2) | (expand21((unsigned long long)(q[1] * sc)) << 1) | expand21((unsigned long long)(q[2] * sc));
    }
    unsigned long long c = 0;
    for (int k = 0; k < 6; k++) c |= expand10((unsigned long long)(q[k] * 1023)) << (5 - k);
    return c;
}

// Common-prefix length of two sorted leaves with codes a, b and edge ids ida, idb: equal codes are told apart by their edge ids, which is
// the reference's tie break.
RB_HD int et_prefix(unsigned long long a, unsigned long long b, int ida, int idb) {
    if (a == b) return et_clz64(a ^ b) + et_clz64((unsigned long long)ida ^ (unsigned long long)idb);
    return et_clz64(a ^ b);
}
// Children c0, c1 of inner node i of the Karras radix tree over L >= 2 sorted leaves (src/edge_tree.cpp:282-376), numbered like the
// node array: inner nodes 0 .. L-2, then sorted leaf j at L-1+j.  prefix(i, j) is et_prefix of sorted leaves i and j (both in range).
template <typename Prefix>
RB_HD void et_karras_split(int i, int L, const Prefix& prefix, int& c0, int& c1) {
    auto lcp = [&](int j) { return j < 0 || j >= L ? -1 : prefix(i, j); };
    int d = (lcp(i + 1) - lcp(i - 1)) >= 0 ? 1 : -1;
    int dmin = lcp(i - d);
    int lmax = 2;
    while (lcp(i + lmax * d) > dmin) lmax *= 2;
    int l = 0;
    for (int t = lmax / 2; t >= 1; t /= 2)
        if (lcp(i + (l + t) * d) > dmin) l += t;
    int j = i + l * d;
    int dnode = lcp(j);
    int s = 0, div = 2;
    for (int t = (l + (div - 1)) / div; t >= 1;) {
        if (lcp(i + (s + t) * d) > dnode) s += t;
        if (t == 1) break;
        div *= 2;
        t = (l + (div - 1)) / div;
    }
    int gamma = i + s * d + (d < 0 ? d : 0);
    int lo = i < j ? i : j, hi = i < j ? j : i;
    c0 = lo == gamma ? L - 1 + gamma : gamma;
    c1 = hi == gamma + 1 ? L - 1 + gamma + 1 : gamma + 1;
}

// Record of inner node `node`: both children's bounds and weighted lengths, and their references -- ~edge id for a leaf, the record
// number (number[child]) for an inner node.
RB_HD EdgeNode et_record(const ETNode* n, int node, const int* number) {
    EdgeNode en;
    memset(&en, 0, sizeof(en));
    for (int c = 0; c < 2; c++) {
        const int ci = n[node].child[c];
        const ETNode& h = n[ci];
        for (int k = 0; k < 3; k++) {
            en.c[c].pmin[k] = (float)h.pmin[k];
            en.c[c].pmax[k] = (float)h.pmax[k];
            en.c[c].dmin[k] = (float)h.dmin[k];
            en.c[c].dmax[k] = (float)h.dmax[k];
        }
        en.c[c].wlen = (float)h.wlen;
        en.c[c].ref = h.edge_id != -1 ? ~h.edge_id : number[ci];
    }
    return en;
}
