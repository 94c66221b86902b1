// Exact planar predicates and the Delaunay point-location step of the point-cloud warp (include/gspcd.h).
// Everything here is __host__ __device__: the CUDA library and the host test build compile the same code.
// It must be compiled without floating-point contraction (nvcc --fmad=false, g++ -ffp-contract=off): the
// error-free transformations below rely on every + and * rounding on its own.
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define PCD_HD __host__ __device__ __forceinline__
#else
#define PCD_HD inline
#endif

namespace pcd {

enum : int { ST_OK = 0, ST_EXACT_OVERFLOW = 1, ST_WALK_CAP = 2 };

// ---------------------------------------------------------------------------------------------------------------
// Expansion arithmetic (Shewchuk, "Adaptive precision floating-point arithmetic and fast robust geometric
// predicates", 1997): a value is an exact sum of non-overlapping doubles, smallest magnitude first.
PCD_HD void two_sum(double a, double b, double& x, double& y) {
    x = a + b; double bv = x - a; double av = x - bv; y = (a - av) + (b - bv);
}
PCD_HD void fast_two_sum(double a, double b, double& x, double& y) { x = a + b; y = b - (x - a); }
PCD_HD void two_diff(double a, double b, double& x, double& y) {
    x = a - b; double bv = a - x; double av = x + bv; y = (a - av) + (bv - b);
}
PCD_HD void two_prod(double a, double b, double& x, double& y) { x = a * b; y = fma(a, b, -x); }

// e (n terms) * b -> h, zero-eliminated; h holds up to 2n terms.
PCD_HD int scale_expansion(int n, const double* e, double b, double* h) {
    double Q, hh, p1, p0, sum; int k = 0;
    two_prod(e[0], b, Q, hh);
    if (hh != 0.0) h[k++] = hh;
    for (int i = 1; i < n; ++i) {
        two_prod(e[i], b, p1, p0);
        two_sum(Q, p0, sum, hh);
        if (hh != 0.0) h[k++] = hh;
        fast_two_sum(p1, sum, Q, hh);
        if (hh != 0.0) h[k++] = hh;
    }
    if (Q != 0.0 || k == 0) h[k++] = Q;
    return k;
}

// An exact accumulator of signed products of up to four doubles. CAP bounds the compressed expansion; an input
// whose exact value needs more terms (coordinates spanning hundreds of binary orders of magnitude) sets overflow.
struct ExactSum {
    static constexpr int CAP = 40;
    double v[CAP];
    int n = 0;
    bool overflow = false;

    PCD_HD void grow(double b) {                                  // Grow-Expansion with zero elimination, in place
        double Q = b, h; int k = 0;
        for (int i = 0; i < n; ++i) {
            two_sum(Q, v[i], Q, h);
            if (h != 0.0) v[k++] = h;
        }
        if (Q != 0.0 || k == 0) v[k++] = Q;
        n = k;
    }
    PCD_HD void compress() {
        if (n < 2) return;
        int bottom = n - 1; double Q = v[bottom], Qn, q;
        for (int i = n - 2; i >= 0; --i) {
            fast_two_sum(Q, v[i], Qn, q);
            if (q != 0.0) { v[bottom--] = Qn; Q = q; } else Q = Qn;
        }
        int top = 0;
        for (int i = bottom + 1; i < n; ++i) {
            fast_two_sum(v[i], Q, Qn, q);
            if (q != 0.0) v[top++] = q;
            Q = Qn;
        }
        v[top] = Q; n = top + 1;
    }
    // += sign * f[0] * ... * f[k-1]
    PCD_HD void add_product(const double* f, int k, double sign) {
        for (int i = 0; i < k; ++i) if (f[i] == 0.0) return;
        double a[8], b[8]; int na;
        two_prod(f[0], f[1], a[1], a[0]);
        na = a[0] != 0.0 ? 2 : (a[0] = a[1], 1);
        for (int i = 2; i < k; ++i) {
            int nb = scale_expansion(na, a, f[i], b);
            for (int j = 0; j < nb; ++j) a[j] = b[j];
            na = nb;
        }
        if (n + na > CAP) { compress(); if (n + na > CAP) { overflow = true; return; } }
        for (int j = 0; j < na; ++j) grow(sign * a[j]);
        if (n > CAP - 8) compress();
    }
    PCD_HD int sign() const { return n == 0 ? 0 : (v[n - 1] > 0.0) - (v[n - 1] < 0.0); }
};

struct Pt { double x, y; };

constexpr double EPS = 1.1102230246251565e-16;                    // 2^-53
constexpr double CCW_BOUND = (3.0 + 16.0 * EPS) * EPS;
constexpr double ICC_BOUND = (10.0 + 96.0 * EPS) * EPS;

// Sign of the orientation of (a, b, c): > 0 counter-clockwise (y up), exactly.
PCD_HD int orient(Pt a, Pt b, Pt c, int& status) {
    double l = (a.x - c.x) * (b.y - c.y), r = (a.y - c.y) * (b.x - c.x), det = l - r;
    double bound = CCW_BOUND * (fabs(l) + fabs(r));
    if (det > bound) return 1;
    if (-det > bound) return -1;
    double acx[2], acy[2], bcx[2], bcy[2];
    two_diff(a.x, c.x, acx[1], acx[0]); two_diff(a.y, c.y, acy[1], acy[0]);
    two_diff(b.x, c.x, bcx[1], bcx[0]); two_diff(b.y, c.y, bcy[1], bcy[0]);
    ExactSum s;
    for (int i = 0; i < 2; ++i)
        for (int j = 0; j < 2; ++j) {
            double f1[2] = {acx[i], bcy[j]}, f2[2] = {acy[i], bcx[j]};
            s.add_product(f1, 2, 1.0); s.add_product(f2, 2, -1.0);
        }
    if (s.overflow) status |= ST_EXACT_OVERFLOW;
    return s.sign();
}

// Sign of |p - a|^2 - |r - a|^2, exactly.
PCD_HD int cmp_dist(Pt a, Pt p, Pt r, int& status) {
    double pdx = p.x - a.x, pdy = p.y - a.y, rdx = r.x - a.x, rdy = r.y - a.y;
    double d1 = pdx * pdx + pdy * pdy, d2 = rdx * rdx + rdy * rdy, det = d1 - d2;
    double bound = 16.0 * EPS * (d1 + d2);
    if (det > bound) return 1;
    if (-det > bound) return -1;
    double d[4][2];
    two_diff(p.x, a.x, d[0][1], d[0][0]); two_diff(p.y, a.y, d[1][1], d[1][0]);
    two_diff(r.x, a.x, d[2][1], d[2][0]); two_diff(r.y, a.y, d[3][1], d[3][0]);
    ExactSum s;
    for (int c = 0; c < 4; ++c)
        for (int i = 0; i < 2; ++i)
            for (int j = 0; j < 2; ++j) {
                double f[2] = {d[c][i], d[c][j]};
                s.add_product(f, 2, c < 2 ? 1.0 : -1.0);
            }
    if (s.overflow) status |= ST_EXACT_OVERFLOW;
    return s.sign();
}

// In-circle determinant: > 0 when d lies inside the circle through a, b, c (counter-clockwise), exactly.
PCD_HD int incircle(Pt a, Pt b, Pt c, Pt d, int& status) {
    double adx = a.x - d.x, ady = a.y - d.y, bdx = b.x - d.x, bdy = b.y - d.y, cdx = c.x - d.x, cdy = c.y - d.y;
    double bdxcdy = bdx * cdy, cdxbdy = cdx * bdy, alift = adx * adx + ady * ady;
    double cdxady = cdx * ady, adxcdy = adx * cdy, blift = bdx * bdx + bdy * bdy;
    double adxbdy = adx * bdy, bdxady = bdx * ady, clift = cdx * cdx + cdy * cdy;
    double det = alift * (bdxcdy - cdxbdy) + blift * (cdxady - adxcdy) + clift * (adxbdy - bdxady);
    double perm = (fabs(bdxcdy) + fabs(cdxbdy)) * alift + (fabs(cdxady) + fabs(adxcdy)) * blift +
                  (fabs(adxbdy) + fabs(bdxady)) * clift;
    double bound = ICC_BOUND * perm;
    if (det > bound) return 1;
    if (-det > bound) return -1;
    double D[6][2];                                               // adx ady bdx bdy cdx cdy as two-term expansions
    two_diff(a.x, d.x, D[0][1], D[0][0]); two_diff(a.y, d.y, D[1][1], D[1][0]);
    two_diff(b.x, d.x, D[2][1], D[2][0]); two_diff(b.y, d.y, D[3][1], D[3][0]);
    two_diff(c.x, d.x, D[4][1], D[4][0]); two_diff(c.y, d.y, D[5][1], D[5][0]);
    // det = lift(u) * (x(v) y(w) - y(v) x(w)) summed over the cyclic triples (u, v, w) of (a, b, c)
    const int cyc[3][3] = {{0, 1, 2}, {1, 2, 0}, {2, 0, 1}};
    ExactSum s;
    for (int t = 0; t < 3; ++t) {
        const int u = cyc[t][0], v = cyc[t][1], w = cyc[t][2];
        for (int axis = 0; axis < 2; ++axis)
            for (int i = 0; i < 2; ++i)
                for (int j = 0; j < 2; ++j)
                    for (int k = 0; k < 2; ++k)
                        for (int l = 0; l < 2; ++l) {
                            double f1[4] = {D[2 * u + axis][i], D[2 * u + axis][j], D[2 * v][k], D[2 * w + 1][l]};
                            double f2[4] = {D[2 * u + axis][i], D[2 * u + axis][j], D[2 * v + 1][k], D[2 * w][l]};
                            s.add_product(f1, 4, 1.0); s.add_product(f2, 4, -1.0);
                        }
    }
    if (s.overflow) status |= ST_EXACT_OVERFLOW;
    return s.sign();
}

// In-circle with a fixed tie rule: each point's lift |p|^2 is lowered by an infinitesimal that is larger for a
// smaller index (simulation of simplicity). The result is never 0 for a non-degenerate triangle a, b, c; among
// cocircular points the lowest index wins, and of exactly duplicated points only the lowest index is a vertex.
PCD_HD int incircle_sos(Pt a, Pt b, Pt c, Pt d, int ia, int ib, int ic, int id, int& status) {
    int s = incircle(a, b, c, d, status);
    if (s != 0) return s;
    // d det / d lift: a -> +orient(b,c,d), b -> -orient(a,c,d), c -> +orient(a,b,d), d -> -orient(a,b,c)
    int idx[4] = {ia, ib, ic, id}, ord[4] = {0, 1, 2, 3};
    for (int i = 1; i < 4; ++i)
        for (int j = i; j > 0 && idx[ord[j]] < idx[ord[j - 1]]; --j) { int t = ord[j]; ord[j] = ord[j - 1]; ord[j - 1] = t; }
    for (int k = 0; k < 4; ++k) {
        int cof;
        switch (ord[k]) {
            case 0: cof = orient(b, c, d, status); break;
            case 1: cof = -orient(a, c, d, status); break;
            case 2: cof = orient(a, b, d, status); break;
            default: cof = -orient(a, b, c, status); break;
        }
        if (cof != 0) return -cof;                                  // lift lowered: det' = det - delta * cof
    }
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// Uniform cell grid over [0, W-1] x [0, H-1]. Points are stored cell by cell, ascending index within a cell.
struct Grid {
    int gw, gh;
    double s, inv_s;
    const int* cell_start;                                          // [gw*gh + 1]
    const double* x;                                                // [n] in cell order
    const double* y;
    const int* idx;                                                 // [n] point index (ascending = input order)
};

PCD_HD int cell_coord(double v, double inv_s, int g) {
    int c = (int)(v * inv_s);
    return c < 0 ? 0 : (c >= g ? g - 1 : c);
}

// Visits the cells in square rings of growing Chebyshev distance around the cell of (qx, qy). After ring k, every
// point not yet visited lies at least (k * s) away; visit(point) is called per point, and done(radius) after each
// ring. Returns true when done() stopped the search, false when the whole grid was visited.
template <typename Visit, typename Done>
PCD_HD bool ring_search(const Grid& g, double qx, double qy, Visit& visit, Done& done) {
    const int ci = cell_coord(qx, g.inv_s, g.gw), cj = cell_coord(qy, g.inv_s, g.gh);
    int kmax = ci;
    if (g.gw - 1 - ci > kmax) kmax = g.gw - 1 - ci;
    if (cj > kmax) kmax = cj;
    if (g.gh - 1 - cj > kmax) kmax = g.gh - 1 - cj;
    for (int k = 0; k <= kmax; ++k) {
        const int j0 = cj - k, j1 = cj + k;
        for (int j = (j0 < 0 ? 0 : j0); j <= (j1 >= g.gh ? g.gh - 1 : j1); ++j) {
            const bool edge_row = (j == j0 || j == j1);
            const int step = edge_row ? 1 : 2 * k;
            for (int i = ci - k; i <= ci + k; i += (step > 0 ? step : 1)) {
                if (i < 0 || i >= g.gw) continue;
                const int c = j * g.gw + i;
                for (int e = g.cell_start[c]; e < g.cell_start[c + 1]; ++e) visit(e);
            }
        }
        // slack for the rounding of the cell index of the query and of the points
        if (done((double)k * g.s * (1.0 - 1e-9) - 1e-9 * g.s)) return true;
    }
    return false;
}

struct NearestQuery {                                               // nearest point to q; ties by lowest index
    const Grid* g; Pt q; double best_d2; int best; int best_idx;
    PCD_HD void operator()(int e) {
        double dx = g->x[e] - q.x, dy = g->y[e] - q.y, d2 = dx * dx + dy * dy;
        if (best < 0 || d2 < best_d2 || (d2 == best_d2 && g->idx[e] < best_idx)) { best_d2 = d2; best = e; best_idx = g->idx[e]; }
    }
};
struct NearestDone {
    const NearestQuery* nq;
    PCD_HD bool operator()(double r) const {
        return nq->best >= 0 && sqrt(nq->best_d2) * (1.0 + 1e-9) < r;
    }
};

struct NeighbourQuery {                                             // exact nearest distinct point to a; ties by index
    const Grid* g; Pt a; int best; int best_idx; int* status;
    PCD_HD void operator()(int e) {
        Pt p = {g->x[e], g->y[e]};
        if (p.x == a.x && p.y == a.y) return;
        if (best < 0) { best = e; best_idx = g->idx[e]; return; }
        int c = cmp_dist(a, p, Pt{g->x[best], g->y[best]}, *status);
        if (c < 0 || (c == 0 && g->idx[e] < best_idx)) { best = e; best_idx = g->idx[e]; }
    }
};
struct NeighbourDone {
    const NeighbourQuery* nq;
    PCD_HD bool operator()(double r) const {
        if (nq->best < 0) return false;
        double dx = nq->g->x[nq->best] - nq->a.x, dy = nq->g->y[nq->best] - nq->a.y;
        return sqrt(dx * dx + dy * dy) * (1.0 + 1e-9) < r;
    }
};

// The third vertex of the Delaunay triangle left of the directed edge a -> b: the point strictly left of the edge
// whose circle through a and b holds no other such point (ties by incircle_sos).
struct ApexQuery {
    const Grid* g; Pt a, b; int ia, ib; int best; int* status;
    PCD_HD void operator()(int e) {
        Pt p = {g->x[e], g->y[e]};
        if (orient(a, b, p, *status) <= 0) return;
        if (best < 0) { best = e; return; }
        Pt c = {g->x[best], g->y[best]};
        if (incircle_sos(a, b, c, p, ia, ib, g->idx[best], g->idx[e], *status) > 0) best = e;
    }
};
struct ApexDone {
    const ApexQuery* aq; Pt m;
    PCD_HD bool operator()(double r) const {
        if (aq->best < 0) return false;
        const Pt a = aq->a, b = aq->b, c = {aq->g->x[aq->best], aq->g->y[aq->best]};
        // circumcentre relative to a
        double bx = b.x - a.x, by = b.y - a.y, cx = c.x - a.x, cy = c.y - a.y;
        double d = 2.0 * (bx * cy - by * cx);
        double b2 = bx * bx + by * by, c2 = cx * cx + cy * cy;
        double ox = (cy * b2 - by * c2) / d, oy = (bx * c2 - cx * b2) / d;
        double R = sqrt(ox * ox + oy * oy);
        double mx = ox + a.x - m.x, my = oy + a.y - m.y;
        double need = (sqrt(mx * mx + my * my) + R) * (1.0 + 1e-6) + 1e-9;
        return need < r;                                            // false for NaN / inf: keep searching
    }
};

PCD_HD int find_apex(const Grid& g, Pt a, Pt b, int ia, int ib, int& status) {
    ApexQuery aq{&g, a, b, ia, ib, -1, &status};
    ApexDone ad{&aq, Pt{0.5 * (a.x + b.x), 0.5 * (a.y + b.y)}};
    ring_search(g, ad.m.x, ad.m.y, aq, ad);
    return aq.best;
}

// ---------------------------------------------------------------------------------------------------------------
// Convex hull. Only points in cells near the extremes of their grid row or column can be hull vertices: a point
// with an occupied cell three or more rows above it in its own column is beaten, in every direction d with
// d.y >= |d.x|, by a point of that cell (it is higher by more than one cell and within one cell sideways); the same
// holds for the other three quadrants of directions. Three cells of margin cover the rounding of the cell index.
constexpr int HULL_BAND = 2;

PCD_HD bool in_hull_band(int i, int j, int top, int bot, int left, int right) {
    return j >= top - HULL_BAND || j <= bot + HULL_BAND || i <= left + HULL_BAND || i >= right - HULL_BAND;
}

PCD_HD bool xy_less(Pt a, int ia, Pt b, int ib) {
    return a.x < b.x || (a.x == b.x && (a.y < b.y || (a.y == b.y && ia < ib)));
}

// Andrew's monotone chain over m points given in ascending xy_less order (slots into x / y). Writes the hull
// counter-clockwise, without collinear or repeated vertices, into out (room for 2m + 1) and returns its vertex
// count; fewer than 3 means the points are collinear (or fewer than three distinct).
PCD_HD int monotone_chain(const double* x, const double* y, const int* order, int m, int* out, int& status) {
    if (m < 3) return 0;
    int k = 0;
    for (int t = 0; t < m; ++t) {
        const int e = order[t];
        while (k >= 2 && orient(Pt{x[out[k - 2]], y[out[k - 2]]}, Pt{x[out[k - 1]], y[out[k - 1]]}, Pt{x[e], y[e]},
                                status) <= 0) --k;
        out[k++] = e;
    }
    for (int t = m - 2, low = k + 1; t >= 0; --t) {
        const int e = order[t];
        while (k >= low && orient(Pt{x[out[k - 2]], y[out[k - 2]]}, Pt{x[out[k - 1]], y[out[k - 1]]}, Pt{x[e], y[e]},
                                  status) <= 0) --k;
        out[k++] = e;
    }
    return k - 1 >= 3 ? k - 1 : 0;                                   // the last vertex repeats the first
}

// q in the closed convex polygon (counter-clockwise, strictly convex, n >= 3), exactly: O(log n) orientations.
PCD_HD bool in_hull(const double* x, const double* y, const int* poly, int n, Pt q, int& status) {
    if (n < 3) return false;
    const Pt v0 = {x[poly[0]], y[poly[0]]};
    if (orient(v0, Pt{x[poly[1]], y[poly[1]]}, q, status) < 0) return false;
    if (orient(v0, Pt{x[poly[n - 1]], y[poly[n - 1]]}, q, status) > 0) return false;
    int lo = 1, hi = n - 2;                                         // largest k in [1, n-2] with orient(v0, vk, q) >= 0
    while (lo < hi) {
        const int mid = (lo + hi + 1) / 2;
        if (orient(v0, Pt{x[poly[mid]], y[poly[mid]]}, q, status) >= 0) lo = mid; else hi = mid - 1;
    }
    return orient(Pt{x[poly[lo]], y[poly[lo]]}, Pt{x[poly[lo + 1]], y[poly[lo + 1]]}, q, status) >= 0;
}

struct Located { int v[3]; };                                       // storage slots (cell order); v[0] < 0: outside

constexpr int WALK_CAP = 1 << 16;

// The triangle of the Delaunay triangulation of the grid's points (ties resolved as in incircle_sos) that contains
// q, closed. v[0] = -1 when q lies outside the convex hull, when there are fewer than three points, or when all
// points are collinear. A visibility walk from the nearest point over triangles built on demand.
PCD_HD Located locate(const Grid& g, int n, Pt q, int& status) {
    Located out{{-1, -1, -1}};
    if (n < 3) return out;
    NearestQuery nq{&g, q, 0.0, -1, 0};
    NearestDone nd{&nq};
    ring_search(g, q.x, q.y, nq, nd);
    int ea = nq.best;
    Pt a = {g.x[ea], g.y[ea]};
    NeighbourQuery bq{&g, a, -1, 0, &status};
    NeighbourDone bd{&bq};
    ring_search(g, a.x, a.y, bq, bd);
    if (bq.best < 0) return out;                                     // every point coincides
    int eb = bq.best;
    Pt b = {g.x[eb], g.y[eb]};
    int o = orient(a, b, q, status);
    if (o < 0) { int t = ea; ea = eb; eb = t; Pt tp = a; a = b; b = tp; }
    int ec = find_apex(g, a, b, g.idx[ea], g.idx[eb], status);
    if (ec < 0) {
        if (o != 0) return out;                                      // q strictly outside a hull edge
        int t = ea; ea = eb; eb = t; Pt tp = a; a = b; b = tp;       // q on the edge's line: try the other side
        ec = find_apex(g, a, b, g.idx[ea], g.idx[eb], status);
        if (ec < 0) return out;                                      // all points collinear
    }
    for (int step = 0; step < WALK_CAP; ++step) {
        Pt c = {g.x[ec], g.y[ec]};
        int o1 = orient(b, c, q, status), o2 = orient(c, a, q, status);
        if (o1 >= 0 && o2 >= 0) { out.v[0] = ea; out.v[1] = eb; out.v[2] = ec; return out; }
        // leave through an edge that has q strictly on its far side; the new edge keeps q on its left
        int na, nb;
        if (o1 < 0) { na = ec; nb = eb; } else { na = ea; nb = ec; }
        int nc = find_apex(g, Pt{g.x[na], g.y[na]}, Pt{g.x[nb], g.y[nb]}, g.idx[na], g.idx[nb], status);
        if (nc < 0) return out;                                      // crossed a hull edge: q is outside
        ea = na; eb = nb; ec = nc;
        a = Pt{g.x[ea], g.y[ea]}; b = Pt{g.x[eb], g.y[eb]};
    }
    status |= ST_WALK_CAP;
    return out;
}

}  // namespace pcd
