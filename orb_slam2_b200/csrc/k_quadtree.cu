// Quadtree keypoint distribution: one CTA per (image, level).
//
// Replaces ORBextractor::DistributeOctTree + ExtractorNode::DivideNode (reference
// src/ORBextractor.cc:539-763, :481-537).  The reference walks a std::list with push_front/erase and
// sorts (size, node address) pairs; here the list is an ARRAY IN LIST ORDER (index 0 = front) and
// every pass is data-parallel.  One pass of the list:
//   1. processing order: phase 1 = list order; phase 2 = (size desc, later-created first), every node ranked by
//      counting the nodes ahead of it — "later-created first" == smaller list index, the canonical tie-break of SURVEY §7;
//   2. prefix sums give the cut (first divide that reaches N), every child's creation rank and the
//      new list  = reversed(created children) ++ undivided nodes in old order, written through a
//      (node, quadrant) -> new index table;
//   3. every point moves to its new node through that table and votes its quadrant there (smem atomics), which is
//      what the next pass divides by.
// A point carries its slot 4 * node + quadrant, so step 3 is one table lookup and one box lookup per point.
// The winner per node is max response, ties to the earliest candidate in the reference's emission
// order (cell row, cell col, y, x) — one 64-bit atomicMax per point (ORBextractor.cc:744-760).
// Node membership is decided by the same comparison chain as the reference (root = trunc(x/hX), then
// x<midX / y<midY), never by box containment: roots' integer boxes do not contain all their points.
//
// Bound: latency (a few hundred nodes, a few thousand points); the batch supplies the parallelism.  A level's candidates
// are read once into registers (QT_PPT per thread) and their slots live there too, so a pass costs no global memory
// traffic; a level with more than QT_ONCHIP candidates keeps its slots in `pnode` instead, through the same code.
// Point loops keep shared-memory loads and atomics in separate loops: a load cannot be moved above an atomic on the same
// (dynamic) shared memory, so a loop that mixes them waits out every point's load chain in turn.
#include "borb_internal.h"

namespace borb {

namespace {

constexpr int QT_THREADS = 256;
constexpr int QT_PPT = 20;                       // candidates per thread held in registers
constexpr int QT_ONCHIP = QT_THREADS * QT_PPT;   // 5120; KITTI-shaped frames at 2000 features have < 4000 per level

// Shared memory of one CTA for a node capacity C (list arrays indexed by list position).
struct QtView {
    int* cc[2];       // [b][4k+q]: points of node k of list b in quadrant q; after the last pass the spare one holds the winners
    short4* box[2];   // [b][k]: node box (x0, x1, y0, y1)
    int* cnt[2];      // [b][k]: points in the node; zero from the list's end to the next multiple of 4
    int* tbl;         // [4k+q]: new list index of the points of node k in quadrant q (all four alike if k is not divided)
    int* order;       // phase 2: processing position -> node
    int* rank;        // phase 2: node -> processing position (E if the node is not expandable)
    int* pre;         // phase 2: pre[r] = sum over the first r processed nodes of (children - 1)
    int* misc;        // [0..32] scan scratch, [33] cut, [34] new nodes with more than one point
};

__device__ inline QtView carve(unsigned char* base, int C) {
    QtView v;
    int* ip = reinterpret_cast<int*>(base);
    v.cc[0] = ip; ip += 4 * C;
    v.cc[1] = ip; ip += 4 * C;
    short4* bp = reinterpret_cast<short4*>(ip);
    v.box[0] = bp; bp += C;
    v.box[1] = bp; bp += C;
    ip = reinterpret_cast<int*>(bp);
    v.cnt[0] = ip; ip += C;
    v.cnt[1] = ip; ip += C;
    v.tbl = ip; ip += 4 * C;
    v.order = ip; ip += C;
    v.rank = ip; ip += C;
    v.pre = ip; ip += C + 1;
    v.misc = ip;
    return v;
}

// Exclusive scan over i in [0, m) by the whole CTA: val(i) is the input, use(i, prefix, total) then runs on the thread that
// owns i (threads own contiguous runs).  Returns the total.  Starts with the inputs readable by every thread and wsum[0..32]
// free; ends without a barrier, so what use() writes needs one before other threads read it.
template <class V, class U>
__device__ __forceinline__ int block_exscan(int m, int* wsum, V val, U use) {
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5, nw = QT_THREADS >> 5;
    const int per = (m + QT_THREADS - 1) / QT_THREADS;
    const int beg = min(tid * per, m), end = min(beg + per, m);
    int s = 0;
    for (int i = beg; i < end; i++) s += val(i);
    int incl = s;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        int t = __shfl_up_sync(0xFFFFFFFFu, incl, off);
        if (lane >= off) incl += t;
    }
    if (lane == 31) wsum[w] = incl;
    __syncthreads();
    if (w == 0) {
        int x = lane < nw ? wsum[lane] : 0;
        int inc2 = x;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            int t = __shfl_up_sync(0xFFFFFFFFu, inc2, off);
            if (lane >= off) inc2 += t;
        }
        wsum[lane] = inc2 - x;
        if (lane == 31) wsum[32] = inc2;
    }
    __syncthreads();
    int base = wsum[w] + incl - s;
    const int total = wsum[32];
    for (int i = beg; i < end; i++) {
        const int t = val(i);
        use(i, base, total);
        base += t;
    }
    return total;
}

__device__ __forceinline__ int quadrant(uint32_t e, short4 b) {
    const int x = xys_x(e) - MIN_BORDER, y = xys_y(e) - MIN_BORDER;
    const int mx = b.x + ((b.y - b.x + 1) >> 1);   // UL.x + ceil((UR.x-UL.x)/2.f)   (ORBextractor.cc:483)
    const int my = b.z + ((b.w - b.z + 1) >> 1);
    return (x < mx) ? ((y < my) ? 0 : 2) : ((y < my) ? 1 : 3);
}

// f(e, s) for every candidate e of the level, s = its stored root index / slot / node (READ: s holds the stored value;
// WRITE: f's change to s is kept).  On chip, candidate i of a thread is e[i] and its value the 16-bit half i&1 of nd[i/2]
// (slots < 4 * node_cap < 2^16, see build_geometry).
template <bool READ, bool WRITE, class F>
__device__ __forceinline__ void for_points(bool onchip, int P, const uint32_t (&e)[QT_PPT], uint32_t (&nd)[QT_PPT / 2],
                                           const uint32_t* __restrict__ pts, int* __restrict__ pn, F f) {
    if (onchip) {
#pragma unroll
        for (int i = 0; i < QT_PPT; i++)
            if (threadIdx.x + i * QT_THREADS < P) {
                const int sh = 16 * (i & 1);
                int s = (nd[i / 2] >> sh) & 0xFFFF;
                f(e[i], s);
                if (WRITE) nd[i / 2] = (nd[i / 2] & ~(0xFFFFu << sh)) | ((uint32_t)s << sh);
            }
    } else {
        for (int p = threadIdx.x; p < P; p += QT_THREADS) {
            int s = READ ? pn[p] : 0;
            f(pts[p], s);
            if (WRITE) pn[p] = s;
        }
    }
}

}  // namespace

size_t quadtree_smem_bytes(int node_cap) {
    const size_t C = (size_t)node_cap;
    return C * (2 * 4 * 4 + 2 * 8 + 2 * 4 + 4 * 4 + 3 * 4) + 4 + 35 * 4;   // == carve(): 84 B per node
}

__global__ void __launch_bounds__(QT_THREADS, 4) quadtree_kernel(const __grid_constant__ Geometry g, const uint32_t* __restrict__ cand,
                                                                 const int* __restrict__ cand_cnt, int* __restrict__ pnode,
                                                                 uint32_t* __restrict__ sel, int* __restrict__ sel_cnt) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int img = blockIdx.y, l = blockIdx.x;
    const LevelGeom& L = g.lv[l];
    const int tid = threadIdx.x, T = QT_THREADS;
    QtView v = carve(smem_raw, L.node_cap);
    const int P = min(cand_cnt[img * g.nlevels + l], L.cand_cap);
    const int N = L.quota;
    const uint32_t* pts = cand + (size_t)img * g.cand_image_stride + L.cand_off;
    int* pn = pnode + (size_t)img * g.cand_image_stride + L.cand_off;
    uint32_t* out = sel + (size_t)img * g.sel_image_stride + L.sel_off;
    if (P == 0) {
        if (tid == 0) sel_cnt[img * g.nlevels + l] = 0;
        return;
    }
    const bool onchip = P <= QT_ONCHIP;
    uint32_t e[QT_PPT], nd[QT_PPT / 2] = {};
    if (onchip) {
#pragma unroll
        for (int i = 0; i < QT_PPT; i++) e[i] = tid + i * T < P ? pts[tid + i * T] : 0u;
    }
    // ---- roots (ORBextractor.cc:543-585); their point counts go to cc[1], free until the first pass
    const int nIni = L.nIni;
    const float hX = L.hX;
    int* rc = v.cc[1];
    for (int i = tid; i < nIni; i += T) rc[i] = 0;
    __syncthreads();
    for_points<false, true>(onchip, P, e, nd, pts, pn, [&](uint32_t x, int& s) {
        const int r = (int)__fdiv_rn((float)(xys_x(x) - MIN_BORDER), hX);
        s = min(max(r, 0), nIni - 1);
        atomicAdd(&rc[s], 1);
    });
    __syncthreads();
    int n = block_exscan(nIni, v.misc, [&](int i) { return rc[i] > 0; }, [&](int i, int j, int) {
        if (rc[i] > 0) {
            v.box[0][j] = make_short4((short)(int)__fmul_rn(hX, (float)i), (short)(int)__fmul_rn(hX, (float)(i + 1)), 0,
                                      (short)(L.h - 2 * MIN_BORDER));
            v.cnt[0][j] = rc[i];
            v.tbl[i] = j;
        }
    });
    for (int j = n + tid; j < ((n + 3) & ~3); j += T) v.cnt[0][j] = 0;
    for (int j = tid; j < 4 * n; j += T) v.cc[0][j] = 0;
    __syncthreads();
    // the current list (B, CN, CC) and the one a pass builds (NB, NCN, NCC)
    short4 *B = v.box[0], *NB = v.box[1];
    int *CN = v.cnt[0], *NCN = v.cnt[1], *CC = v.cc[0], *NCC = v.cc[1];
    // every point moves through tbl to its node k of list (bx, cc) and votes its quadrant there; the votes of a node that
    // is not expandable are never read
    auto move_and_vote = [&](const short4* bx, int* cc) {
        for_points<true, true>(onchip, P, e, nd, pts, pn, [&](uint32_t x, int& s) {
            const int k = v.tbl[s];
            s = 4 * k + quadrant(x, bx[k]);
        });
        for_points<true, false>(onchip, P, e, nd, pts, pn, [&](uint32_t, int& s) { atomicAdd(&cc[s], 1); });
    };
    move_and_vote(B, CC);
    __syncthreads();

    int E = 0, nn;   // E: expandable nodes in the list (phase 2 only); nn: size of the list a pass builds
    bool phase2 = false;
    for (;;) {
        auto children = [&](int k) { return (CC[4 * k] > 0) + (CC[4 * k + 1] > 0) + (CC[4 * k + 2] > 0) + (CC[4 * k + 3] > 0); };
        // DivideNode (ORBextractor.cc:481-537): the non-empty quadrants of node k become nodes j0, j0-1, ...
        int big = 0;
        auto divide = [&](int k, int j) {
            const short4 b = B[k];
            const short mx = (short)(b.x + ((b.y - b.x + 1) >> 1)), my = (short)(b.z + ((b.w - b.z + 1) >> 1));
#pragma unroll
            for (int q = 0; q < 4; q++) {
                const int cq = CC[4 * k + q];
                if (cq > 0) {
                    v.tbl[4 * k + q] = j;
                    NB[j] = make_short4((q & 1) ? mx : b.x, (q & 1) ? b.y : mx, (q & 2) ? my : b.z, (q & 2) ? b.w : my);
                    NCN[j] = cq;
                    big += cq > 1;
                    j--;
                }
            }
        };
        auto keep = [&](int k, int j) {
            v.tbl[4 * k] = v.tbl[4 * k + 1] = v.tbl[4 * k + 2] = v.tbl[4 * k + 3] = j;
            NB[j] = B[k];
            NCN[j] = CN[k];
        };
        if (tid == 0) v.misc[34] = 0;
        int created;
        if (!phase2) {
            // every expandable node is divided, in list order: one scan of (children << 16 | undivided); a list holds
            // fewer than 2^14 nodes (build_geometry's shared-memory bound), so neither half overflows
            const int tot = block_exscan(n, v.misc, [&](int k) { return CN[k] > 1 ? children(k) << 16 : 1; }, [&](int k, int pre, int total) {
                if (CN[k] > 1) divide(k, (total >> 16) - 1 - (pre >> 16));
                else keep(k, (total >> 16) + (pre & 0xFFFF));
            });
            created = tot >> 16;
            nn = created + (tot & 0xFFFF);
        } else {
            // largest first (ORBextractor.cc:684-720): rank = expandable nodes that are larger, or as large and earlier
            const int4* CN4 = reinterpret_cast<const int4*>(CN);
            for (int k = tid; k < n; k += T) {
                const int s = CN[k];
                if (s > 1) {
                    int r = 0;
                    for (int j = 0; j < n; j += 4) {
                        const int4 c = CN4[j >> 2];
                        r += (c.x + (j < k) > s) + (c.y + (j + 1 < k) > s) + (c.z + (j + 2 < k) > s) + (c.w + (j + 3 < k) > s);
                    }
                    v.order[r] = k;
                    v.rank[k] = r;
                } else
                    v.rank[k] = E;
            }
            if (tid == 0) { v.misc[33] = E; v.pre[0] = 0; }   // cut r* (first divide reaching N), default: none
            __syncthreads();
            block_exscan(E, v.misc, [&](int r) { return children(v.order[r]) - 1; }, [&](int r, int pre, int) {
                const int d = children(v.order[r]) - 1;
                v.pre[r + 1] = pre + d;
                if (n + pre + d >= N) atomicMin(&v.misc[33], r);
            });
            __syncthreads();
            const int Dn = min(v.misc[33] + 1, E);
            created = v.pre[Dn] + Dn;
            for (int r = tid; r < Dn; r += T) divide(v.order[r], created - 1 - v.pre[r] - r);
            nn = created + block_exscan(n, v.misc, [&](int k) { return v.rank[k] >= Dn; }, [&](int k, int pre, int) {
                if (v.rank[k] >= Dn) keep(k, created + pre);
            });
        }
        if (big) atomicAdd(&v.misc[34], big);
        // termination (ORBextractor.cc:669-673, :734-735)
        const bool last = nn >= N || nn == n;
        // the new list's votes, or after the last pass its winners (nn u64)
        for (int j = tid; j < 4 * nn; j += T) NCC[j] = 0;
        for (int j = nn + tid; j < ((nn + 3) & ~3); j += T) NCN[j] = 0;
        __syncthreads();
        if (last) break;
        const int nToExpand = v.misc[34];
        move_and_vote(NB, NCC);
        __syncthreads();
        if (!phase2 && nn + 3 * nToExpand > N) phase2 = true;
        n = nn;
        E = nToExpand;   // a pass that does not finish divides every expandable node, so only new children can be
                         // expandable: the reference's vSizeAndPointerToNode
        short4* tb = B; B = NB; NB = tb;
        int* tc = CN; CN = NCN; NCN = tc;
        tc = CC; CC = NCC; NCC = tc;
    }
    // ---- best point per node (ORBextractor.cc:744-760), output in list order
    typedef unsigned long long u64;
    const u64 ORD_MASK = (1ull << 40) - 1;
    u64* best = reinterpret_cast<u64*>(NCC);
    for_points<true, false>(onchip, P, e, nd, pts, pn, [&](uint32_t x, int& s) {
        const int xx = xys_x(x), yy = xys_y(x);
        const u64 ord = ((u64)((yy - EDGE) / L.hCell) << 32) | ((u64)((xx - EDGE) / L.wCell) << 24) | ((u64)yy << 12) | (u64)xx;
        atomicMax(&best[v.tbl[s]], ((u64)xys_s(x) << 40) | (ORD_MASK - ord));
    });
    __syncthreads();
    for (int k = tid; k < nn; k += T) {
        const u64 key = best[k];
        const u64 ord = ORD_MASK - (key & ORD_MASK);
        out[k] = pack_xys((int)(ord & 0xFFF), (int)((ord >> 12) & 0xFFF), (int)(key >> 40));
    }
    if (tid == 0) sel_cnt[img * g.nlevels + l] = nn;
}

int launch_quadtree(const Geometry& g, const Workspace& ws, int n_images, cudaStream_t s) {
    int maxC = 0;
    for (int l = 0; l < g.nlevels; l++) maxC = g.lv[l].node_cap > maxC ? g.lv[l].node_cap : maxC;
    const size_t smem = quadtree_smem_bytes(maxC);
    allow_max_smem((const void*)quadtree_kernel);      // once per device; never lowered (handles on other threads share it)
    dim3 grid(g.nlevels, n_images);
    quadtree_kernel<<<grid, QT_THREADS, smem, s>>>(g, ws.cand, ws.cand_cnt, ws.pnode, ws.sel, ws.sel_cnt);
    return 1;
}

}  // namespace borb
