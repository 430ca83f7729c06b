// text_regions.cu -- the segmentation demo's second image (Examples/demo_segmentation.py:17-25, 40-45, draw_bounding_box):
// every outer text contour whose cv2.contourArea exceeds a threshold, its cv2.convexHull filled by cv2.drawContours in RGB
// (50, 128, 30) on the page's to_pil_image bytes.  Contour tracing is sequential; this computes the same image from the
// parallel formulation of DESIGN 4.14 (F1-F5), eleven launches, no host synchronisation:
//   1. exterior: 4-connected union-find of the background (rows as runs, unions at run overlaps, path halving), then the
//      roots of every border pixel's component are flagged: the background 4-connected to the ring of zeros findContours pads;
//   2. regions: 8-connected union-find of the other pixels; a region's label is its first pixel in raster order (its root);
//   3. statistics per root: A2 = 2 Q4 + Q3 over the 2x2 windows of the zero-padded (h + 1) x (w + 1) grid (contourArea =
//      A2 / 2) and the last row, with warp-aggregated atomics;
//   4. selection (A2 * 0.5 > threshold in double) and, per selected region, one slot per row it spans (at most one region per
//      pixel, so the slots fit in n * h * w), holding the row's leftmost and rightmost pixel (atomicMin / atomicMax); the same
//      pass writes the page bytes of the output;
//   5. the hull per region: monotone chains of the row extents (left and right boundary, collinear points dropped);
//   6. per (region, row) the span cv2.fillPoly (LINE_8) paints there: the Bresenham pixels of the hull edges on the row and
//      the 16-bit fixed-point scanline fill, one contiguous span (F5), painted by the region's warp.
// Painting is idempotent (overlapping hulls write the same colour), so the output does not depend on the order of the atomics.
#include "pil_data.cuh"

#include <algorithm>
#include <climits>
#include <cmath>

#define ST static_cast<cudaStream_t>(stream)
#define PCB_API extern "C" __attribute__((visibility("default")))

namespace {

constexpr int LT = 256;                        // threads per block
constexpr int RW = LT / 32;                    // rows per block of the run kernel (one warp per row)
constexpr unsigned NONE = 0xffffffffu;         // aux of a root that is not selected
constexpr unsigned FULL = 0xffffffffu;
constexpr unsigned char C0 = 50, C1 = 128, C2 = 30;

struct Region {                                // one selected region
    long long off;                             // first row slot
    int page, ymin, height;
    int nl, nr;                                // vertices of the left and right hull chains
    int pad;
};

struct Counters {
    unsigned long long slots;
    unsigned int regions;
};

struct Ws {
    int *lab;                                  // [n][h * w] page-local parent / root index, -1 = not in the set being labelled
    unsigned *aux;                             // per root: exterior flag (pass 1), A2 (statistics), region index (selection)
    int *ymax;                                 // per root: last row
    int2 *ext;                                 // per slot: (leftmost, rightmost) x of the region's row
    int *lchain, *rchain;                      // per slot: row indices of the left / right hull chain vertices
    Region *regions;
    Counters *cnt;
};

size_t align256(size_t v) { return (v + 255) / 256 * 256; }

// at most one region per 2 x 2 block of a page: two regions are never 8-adjacent
long long max_regions(int n, int h, int w) { return static_cast<long long>(n) * ((h + 1) / 2) * ((w + 1) / 2); }

size_t ws_bytes(int n, int h, int w, Ws *ws, char *base) {
    const size_t px = static_cast<size_t>(n) * h * w;
    const size_t sizes[7] = {align256(px * 4), align256(px * 4), align256(px * 4), align256(px * 8), align256(px * 4),
                             align256(px * 4), align256(static_cast<size_t>(max_regions(n, h, w)) * sizeof(Region))};
    size_t o[8] = {0};
    for (int i = 0; i < 7; ++i) o[i + 1] = o[i] + sizes[i];
    if (ws) {
        ws->lab = reinterpret_cast<int *>(base + o[0]);
        ws->aux = reinterpret_cast<unsigned *>(base + o[1]);
        ws->ymax = reinterpret_cast<int *>(base + o[2]);
        ws->ext = reinterpret_cast<int2 *>(base + o[3]);
        ws->lchain = reinterpret_cast<int *>(base + o[4]);
        ws->rchain = reinterpret_cast<int *>(base + o[5]);
        ws->regions = reinterpret_cast<Region *>(base + o[6]);
        ws->cnt = reinterpret_cast<Counters *>(base + o[7]);
    }
    return o[7] + 256;
}

// ------------------------------------------------------------------------------------------------ union-find
// Parents only ever point to smaller indices (runs start at their first pixel, unions link the larger root under the smaller,
// path halving skips to a grandparent), so every component ends with its first pixel in raster order as the root.  Reads go
// through L2 (__ldcg): a stale parent is still an ancestor, and atomicMin on a root that has meanwhile been linked returns
// the new parent, which the loop follows.
__device__ __forceinline__ int find(int *L, int x) {
    for (;;) {
        const int p = __ldcg(L + x);
        if (p == x) return x;
        const int g = __ldcg(L + p);
        if (g != p) L[x] = g;
        x = p;
    }
}

// The root without writes, for the compress passes: there each pixel's thread stores its final root, and a halving store of
// another thread's find, read before that store, could overwrite it with an ancestor that is not the root.
__device__ __forceinline__ int find_root(const int *L, int x) {
    for (;;) {
        const int p = __ldcg(L + x);
        if (p == x) return x;
        x = p;
    }
}

__device__ __forceinline__ void unite(int *L, int a, int b) {
    for (;;) {
        a = find(L, a);
        b = find(L, b);
        if (a == b) return;
        if (a > b) {
            const int t = a;
            a = b;
            b = t;
        }
        const int old = atomicMin(L + b, a);
        if (old == b) return;
        b = old;
    }
}

// One warp per page row: each pixel of the set starts parented to the first pixel of its horizontal run (ballots of the
// breaks), others get -1.  PASS 0, the background: mask == 0; it also clears the exterior flags and the counters.  PASS 1, the
// regions: text, or background whose pass-0 root is not flagged exterior (each lane reads and rewrites its own lab entry).
template <int PASS>
__global__ void __launch_bounds__(LT) runs_kernel(const uint8_t *__restrict__ mask, int n, int h, int w, Ws ws) {
    const int lane = threadIdx.x & 31;
    const long long row = static_cast<long long>(blockIdx.x) * RW + (threadIdx.x >> 5);
    if (PASS == 0 && blockIdx.x == 0 && threadIdx.x == 0) {
        ws.cnt->slots = 0;
        ws.cnt->regions = 0;
    }
    if (row >= static_cast<long long>(n) * h) return;                 // whole warps leave together
    const int b = static_cast<int>(row / h), y = static_cast<int>(row % h);
    const size_t base = static_cast<size_t>(b) * h * w, rbase = base + static_cast<size_t>(y) * w;
    int carry = 0;
    for (int x0 = 0; x0 < w; x0 += 32) {
        const int x = x0 + lane;
        bool e = false;
        if (x < w) {
            const size_t p = rbase + x;
            const bool fg = __ldg(mask + p) != 0;
            if (PASS == 0) {
                e = !fg;
                ws.aux[p] = 0;
            } else {
                e = fg || __ldcg(ws.aux + base + ws.lab[p]) == 0;
            }
        }
        const unsigned brk = __ballot_sync(FULL, !e);
        const unsigned upto = brk & (FULL >> (31 - lane));
        const int start = upto ? x0 + 32 - __clz(upto) : carry;
        if (x < w) ws.lab[rbase + x] = e ? y * w + start : -1;
        if (brk) carry = x0 + 32 - __clz(brk);
    }
}

// One thread per pixel: the unions with the row above, only where a run overlap begins.  4-connected: the pixel above.
// 8-connected: the three above from the first pixel of a run, further along a run only a run above that starts up-right.
template <bool CONN8>
__global__ void __launch_bounds__(LT) merge_kernel(int n, int h, int w, Ws ws) {
    const long long i = static_cast<long long>(blockIdx.x) * LT + threadIdx.x;
    const long long hw = static_cast<long long>(h) * w;
    if (i >= n * hw) return;
    const int b = static_cast<int>(i / hw), p = static_cast<int>(i % hw), y = p / w, x = p - y * w;
    int *L = ws.lab + static_cast<size_t>(b) * hw;
    if (y == 0 || L[p] < 0) return;
    const int q = p - w;
    const bool left = x > 0 && L[p - 1] >= 0;
    if (!CONN8) {
        if (L[q] >= 0 && (!left || L[q - 1] < 0)) unite(L, p, q);
        return;
    }
    if (!left) {
        if (x > 0 && L[q - 1] >= 0) unite(L, p, q - 1);
        if (L[q] >= 0) unite(L, p, q);
        if (x + 1 < w && L[q + 1] >= 0) unite(L, p, q + 1);
    } else if (x + 1 < w && L[q + 1] >= 0 && L[q] < 0) {
        unite(L, p, q + 1);
    }
}

// One thread per pixel: lab = root.  PASS 0 flags the roots of border pixels as exterior; PASS 1 clears the statistics.
template <int PASS>
__global__ void __launch_bounds__(LT) compress_kernel(int n, int h, int w, Ws ws) {
    const long long i = static_cast<long long>(blockIdx.x) * LT + threadIdx.x;
    const long long hw = static_cast<long long>(h) * w;
    if (i >= n * hw) return;
    const int b = static_cast<int>(i / hw), p = static_cast<int>(i % hw);
    const size_t base = static_cast<size_t>(b) * hw;
    int *L = ws.lab + base;
    if (PASS == 1) {
        ws.aux[i] = 0;
        ws.ymax[i] = 0;
    }
    if (L[p] < 0) return;
    const int r = find_root(L, p);
    L[p] = r;
    if (PASS == 0) {
        const int y = p / w, x = p - y * w;
        if (y == 0 || y == h - 1 || x == 0 || x == w - 1) ws.aux[base + r] = 1;
    }
}

// Block 32 x 8 over the windows of the zero-padded grid: window (wy, wx) holds pixels (wy - 1 .. wy, wx - 1 .. wx).  The
// labelled pixels of a window belong to one region (regions are never 8-adjacent).  A warp is 32 windows of one row: lanes
// with the same root add their windows' 2 [s == 4] + [s == 3] in one atomic, and the pixel (wy, wx) raises its root's last row.
__global__ void __launch_bounds__(LT) stats_kernel(int h, int w, Ws ws) {
    const int b = blockIdx.z, wy = blockIdx.y * 8 + threadIdx.y, wx = blockIdx.x * 32 + threadIdx.x;
    const size_t base = static_cast<size_t>(b) * h * w;
    const int *L = ws.lab + base;
    int s = 0, r = -1, own = -1;
    if (wy <= h && wx <= w) {
#pragma unroll
        for (int dy = -1; dy <= 0; ++dy)
#pragma unroll
            for (int dx = -1; dx <= 0; ++dx) {
                const int y = wy + dy, x = wx + dx;
                if (y >= 0 && y < h && x >= 0 && x < w) {
                    const int l = L[y * w + x];
                    if (l >= 0) {
                        ++s;
                        r = l;
                        if (dy == 0 && dx == 0) own = l;
                    }
                }
            }
    }
    const int lane = threadIdx.x;
    const int k4 = s == 4 ? r : -1, k3 = s == 3 ? r : -1;
    const unsigned m4 = __match_any_sync(FULL, k4), m3 = __match_any_sync(FULL, k3), my = __match_any_sync(FULL, own);
    if (k4 >= 0 && lane == __ffs(m4) - 1) atomicAdd(ws.aux + base + k4, 2u * __popc(m4));
    if (k3 >= 0 && lane == __ffs(m3) - 1) atomicAdd(ws.aux + base + k3, static_cast<unsigned>(__popc(m3)));
    if (own >= 0 && lane == __ffs(my) - 1) atomicMax(ws.ymax + base + own, wy);
}

// One thread per pixel; roots only: select on A2 * 0.5 > threshold, take a region index and one slot per row, clear the slots.
__global__ void __launch_bounds__(LT) select_kernel(int n, int h, int w, double threshold, Ws ws) {
    const long long i = static_cast<long long>(blockIdx.x) * LT + threadIdx.x;
    const long long hw = static_cast<long long>(h) * w;
    if (i >= n * hw) return;
    const int b = static_cast<int>(i / hw), p = static_cast<int>(i % hw);
    if (ws.lab[i] != p) return;
    const unsigned a2 = ws.aux[i];
    if (!(static_cast<double>(a2) * 0.5 > threshold)) {
        ws.aux[i] = NONE;
        return;
    }
    const int ymin = p / w, height = ws.ymax[i] - ymin + 1;
    const unsigned k = atomicAdd(&ws.cnt->regions, 1u);
    const long long off = static_cast<long long>(atomicAdd(&ws.cnt->slots, static_cast<unsigned long long>(height)));
    ws.regions[k] = Region{off, b, ymin, height, 0, 0, 0};
    ws.aux[i] = k;
    for (int r = 0; r < height; ++r) ws.ext[off + r] = make_int2(INT_MAX, INT_MIN);
}

// Block 32 x 8 over the page: every pixel's output bytes (to_pil_image of the page), and the row extents of selected regions
// (a warp is 32 consecutive pixels of a row: the lowest lane of a root holds its least x, the highest its greatest).
__global__ void __launch_bounds__(LT) extents_kernel(const float *__restrict__ page, int h, int w, Ws ws, uint8_t *__restrict__ out) {
    const int b = blockIdx.z, y = blockIdx.y * 8 + threadIdx.y, x = blockIdx.x * 32 + threadIdx.x;
    const size_t plane = static_cast<size_t>(h) * w, base = static_cast<size_t>(b) * plane;
    int key = -1;
    unsigned k = NONE;
    if (y < h && x < w) {
        const size_t pix = static_cast<size_t>(y) * w + x;
        const float *pg = page + base * 3 + pix;
        uint8_t *o = out + (base + pix) * 3;
        o[0] = static_cast<uint8_t>(pil::page_byte(__ldg(pg)));
        o[1] = static_cast<uint8_t>(pil::page_byte(__ldg(pg + plane)));
        o[2] = static_cast<uint8_t>(pil::page_byte(__ldg(pg + 2 * plane)));
        const int l = ws.lab[base + pix];
        if (l >= 0) {
            k = __ldg(ws.aux + base + l);
            if (k != NONE) key = l;
        }
    }
    const unsigned m = __match_any_sync(FULL, key);
    if (key < 0) return;
    const int lane = threadIdx.x;
    const bool first = lane == __ffs(m) - 1, last = lane == 31 - __clz(m);
    if (!first && !last) return;
    const Region rg = ws.regions[k];
    int2 *e = ws.ext + rg.off + (y - rg.ymin);
    if (first) atomicMin(&e->x, x);
    if (last) atomicMax(&e->y, x);
}

// One thread per region: the left chain (x convex in y: pop while the middle point is not strictly left of the chord) and
// the right chain (pop while not strictly right) over the rows' extents, as row indices into the region's slots.
__global__ void __launch_bounds__(LT) hull_kernel(Ws ws) {
    const unsigned nreg = ws.cnt->regions;
    for (unsigned k = blockIdx.x * LT + threadIdx.x; k < nreg; k += gridDim.x * LT) {
        Region &rg = ws.regions[k];
        const int2 *e = ws.ext + rg.off;
        int *lc = ws.lchain + rg.off, *rc = ws.rchain + rg.off;
        int nl = 0, nr = 0;
        for (int i = 0; i < rg.height; ++i) {
            const int2 xi = e[i];
            while (nl >= 2) {
                const int a = lc[nl - 2], m = lc[nl - 1];
                const long long cross = static_cast<long long>(e[m].x - e[a].x) * (i - a) - static_cast<long long>(m - a) * (xi.x - e[a].x);
                if (cross < 0) break;
                --nl;
            }
            lc[nl++] = i;
            while (nr >= 2) {
                const int a = rc[nr - 2], m = rc[nr - 1];
                const long long cross = static_cast<long long>(e[m].y - e[a].y) * (i - a) - static_cast<long long>(m - a) * (xi.y - e[a].y);
                if (cross > 0) break;
                --nr;
            }
            rc[nr++] = i;
        }
        rg.nl = nl;
        rg.nr = nr;
    }
}

// floor(a / b) for b > 0 and |a| < 2^50, without the 64-bit division subroutine (whose call spills): the double quotient is
// within one of the result, and one integer step corrects it
__device__ __forceinline__ long long floor_div(long long a, long long b) {
    long long q = static_cast<long long>(floor(__ddiv_rn(static_cast<double>(a), static_cast<double>(b))));
    if (q * b > a) --q;
    else if ((q + 1) * b <= a) ++q;
    return q;
}
__device__ __forceinline__ long long ceil_div(long long a, long long b) { return -floor_div(-a, b); }

// The pixels cv2.line (LINE_8, LineIterator from the left end) sets on row y of the segment p0-p1, widened into [lo, hi]:
// along the major axis every pixel, the minor coordinate after k steps being ceil((2 minor k - major) / (2 major)).
__device__ __forceinline__ void line_row(int x0, int y0, int x1, int y1, int y, int &lo, int &hi) {
    if (x1 < x0) {
        int t = x0; x0 = x1; x1 = t;
        t = y0; y0 = y1; y1 = t;
    }
    const long long DX = x1 - x0, DY = y1 > y0 ? y1 - y0 : y0 - y1;
    const long long m = y1 < y0 ? y0 - y : y - y0;
    if (m < 0 || m > DY) return;
    long long a, z;
    if (DY > DX) {
        a = z = x0 + floor_div(2 * DX * m + DY - 1, 2 * DY);
    } else if (DY == 0) {
        a = x0;
        z = x1;
    } else {
        const long long k0 = ceil_div(2 * DX * m - DX + 1, 2 * DY), k1 = ceil_div(2 * DX * (m + 1) - DX + 1, 2 * DY) - 1;
        a = x0 + (k0 > 0 ? k0 : 0);
        z = x0 + (k1 < DX ? k1 : DX);
    }
    lo = min(lo, static_cast<int>(a));
    hi = max(hi, static_cast<int>(z));
}

// the last chain vertex at or above row i (chain row indices ascend from 0 to height - 1)
__device__ __forceinline__ int chain_at(const int *c, int nc, int i) {
    int lo = 0, hi = nc - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (c[mid] <= i) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// fillPoly's x of edge (xa, ya)-(xb, yb), ya < yb, at row y: 16-bit fixed point from xa << 16, by a truncated step per row
__device__ __forceinline__ long long edge_x(int xa, int ya, int xb, int yb, int y) {
    const long long num = static_cast<long long>(xb - xa) * 65536;
    const long long dx = num >= 0 ? floor_div(num, yb - ya) : -floor_div(-num, yb - ya);     // C division: truncated
    return static_cast<long long>(xa) * 65536 + static_cast<long long>(y - ya) * dx;
}

// The lines of a chain's edges through row i (k: the chain's last vertex at or above the row); RIGHT reads the row extents'
// rightmost x.
template <bool RIGHT>
__device__ __forceinline__ void chain_lines(const int2 *e, const int *c, int nc, int k, int i, int &lo, int &hi) {
    const int xk = RIGHT ? e[c[k]].y : e[c[k]].x;
    if (k + 1 < nc) line_row(xk, c[k], RIGHT ? e[c[k + 1]].y : e[c[k + 1]].x, c[k + 1], i, lo, hi);
    if (k > 0 && c[k] == i) line_row(RIGHT ? e[c[k - 1]].y : e[c[k - 1]].x, c[k - 1], xk, c[k], i, lo, hi);
}

// Region row i's painted span: the lines of the chain edges through it (and of the top / bottom edge on the first / last row),
// and unless it is the last row the fill between the left and right chain's edges, the lower x rounded up, the higher down.
__device__ __forceinline__ int2 row_span(const Region &rg, const int2 *e, const int *lc, const int *rc, int i) {
    int lo = INT_MAX, hi = INT_MIN;
    const int ka = chain_at(lc, rg.nl, i), kb = chain_at(rc, rg.nr, i);
    chain_lines<false>(e, lc, rg.nl, ka, i, lo, hi);
    chain_lines<true>(e, rc, rg.nr, kb, i, lo, hi);
    const int last = rg.height - 1;
    if (i == 0) line_row(e[0].x, 0, e[0].y, 0, 0, lo, hi);
    if (i == last) line_row(e[last].x, last, e[last].y, last, last, lo, hi);
    if (i < last) {
        const long long xl = edge_x(e[lc[ka]].x, lc[ka], e[lc[ka + 1]].x, lc[ka + 1], i);
        const long long xr = edge_x(e[rc[kb]].y, rc[kb], e[rc[kb + 1]].y, rc[kb + 1], i);
        const int x1 = static_cast<int>((min(xl, xr) + 65535) >> 16), x2 = static_cast<int>(max(xl, xr) >> 16);
        if (x1 <= x2) {
            lo = min(lo, x1);
            hi = max(hi, x2);
        }
    }
    return make_int2(lo, hi);
}

// One warp per region: 32 rows' spans at a time, one per lane, then each span painted by the whole warp.
__global__ void __launch_bounds__(LT) paint_kernel(int h, int w, Ws ws, uint8_t *__restrict__ out) {
    const unsigned nreg = ws.cnt->regions;
    const int lane = threadIdx.x & 31;
    const unsigned warps = gridDim.x * (LT / 32);
    for (unsigned k = blockIdx.x * (LT / 32) + (threadIdx.x >> 5); k < nreg; k += warps) {
        const Region rg = ws.regions[k];
        const int2 *e = ws.ext + rg.off;
        const int *lc = ws.lchain + rg.off, *rc = ws.rchain + rg.off;
        uint8_t *img = out + static_cast<size_t>(rg.page) * h * w * 3;
        for (int i0 = 0; i0 < rg.height; i0 += 32) {
            int2 sp = make_int2(INT_MAX, INT_MIN);
            if (i0 + lane < rg.height) sp = row_span(rg, e, lc, rc, i0 + lane);
            const int rows = min(32, rg.height - i0);
            for (int j = 0; j < rows; ++j) {
                const int lo = max(__shfl_sync(FULL, sp.x, j), 0), hi = min(__shfl_sync(FULL, sp.y, j), w - 1);
                uint8_t *r = img + static_cast<size_t>(rg.ymin + i0 + j) * w * 3;
                for (int x = lo + lane; x <= hi; x += 32) {
                    r[3 * x] = C0;
                    r[3 * x + 1] = C1;
                    r[3 * x + 2] = C2;
                }
            }
        }
    }
}

unsigned blocks(long long total) { return static_cast<unsigned>((total + LT - 1) / LT); }

}  // namespace

// zero when the sizes are out of range (pcb_text_region_hulls says why)
PCB_API size_t pcb_text_regions_workspace(int n, int h, int w) {
    if (n < 1 || n > 65535 || h < 1 || w < 1 || (static_cast<long long>(h) + 1) * (w + 1) > INT_MAX) return 0;
    return ws_bytes(n, h, w, nullptr, nullptr);
}

PCB_API int pcb_text_region_hulls(const uint8_t *text_mask, const float *page, int n, int h, int w, double area_threshold,
                                  void *workspace, uint8_t *out, pcb_stream_t stream) {
    const char *fn = "pcb_text_region_hulls";
    PCB_CHECK(text_mask && page && workspace && out, "%s: null pointer", fn);
    PCB_CHECK(n >= 1 && n <= 65535 && h >= 1 && w >= 1, "%s: page %dx3x%dx%d (1..65535 pages, no empty side)", fn, n, h, w);
    PCB_CHECK((static_cast<long long>(h) + 1) * (w + 1) <= INT_MAX, "%s: a %dx%d page is too large for int32 labels", fn, h, w);
    PCB_CHECK(static_cast<long long>(n) * h * w <= (1ll << 38), "%s: too many pixels", fn);
    PCB_CHECK((h + 8) / 8 <= 65535, "%s: page height %d too large", fn, h);
    PCB_CHECK(std::isfinite(area_threshold), "%s: non-finite area threshold", fn);
    PCB_CHECK(reinterpret_cast<uintptr_t>(workspace) % 256 == 0, "%s: workspace not aligned to 256 bytes", fn);
    Ws ws;
    ws_bytes(n, h, w, &ws, static_cast<char *>(workspace));
    const long long px = static_cast<long long>(n) * h * w;
    const unsigned rows = static_cast<unsigned>((static_cast<long long>(n) * h + RW - 1) / RW);
    const dim3 tile(32, 8);
    const dim3 wgrid((w + 1 + 31) / 32, (h + 1 + 7) / 8, n), pgrid((w + 31) / 32, (h + 7) / 8, n);
    const long long nreg = max_regions(n, h, w);
    const unsigned hull_blocks = static_cast<unsigned>(std::min<long long>(blocks(nreg), 8ll * pcb_num_sms()));
    const unsigned paint_blocks = static_cast<unsigned>(std::min<long long>((nreg + LT / 32 - 1) / (LT / 32), 16ll * pcb_num_sms()));
    runs_kernel<0><<<rows, LT, 0, ST>>>(text_mask, n, h, w, ws);
    PCB_LAUNCH_CHECK();
    merge_kernel<false><<<blocks(px), LT, 0, ST>>>(n, h, w, ws);
    PCB_LAUNCH_CHECK();
    compress_kernel<0><<<blocks(px), LT, 0, ST>>>(n, h, w, ws);
    PCB_LAUNCH_CHECK();
    runs_kernel<1><<<rows, LT, 0, ST>>>(text_mask, n, h, w, ws);
    PCB_LAUNCH_CHECK();
    merge_kernel<true><<<blocks(px), LT, 0, ST>>>(n, h, w, ws);
    PCB_LAUNCH_CHECK();
    compress_kernel<1><<<blocks(px), LT, 0, ST>>>(n, h, w, ws);
    PCB_LAUNCH_CHECK();
    stats_kernel<<<wgrid, tile, 0, ST>>>(h, w, ws);
    PCB_LAUNCH_CHECK();
    select_kernel<<<blocks(px), LT, 0, ST>>>(n, h, w, area_threshold, ws);
    PCB_LAUNCH_CHECK();
    extents_kernel<<<pgrid, tile, 0, ST>>>(page, h, w, ws, out);
    PCB_LAUNCH_CHECK();
    hull_kernel<<<hull_blocks, LT, 0, ST>>>(ws);
    PCB_LAUNCH_CHECK();
    paint_kernel<<<paint_blocks, LT, 0, ST>>>(h, w, ws, out);
    PCB_LAUNCH_CHECK();
    return 0;
}
