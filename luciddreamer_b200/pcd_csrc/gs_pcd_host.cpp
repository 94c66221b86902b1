// Host build of the exact predicates and the Delaunay locate step of gs_pcd_geom.cuh, for testing them against
// scipy.spatial.Delaunay without a GPU. Not used by the product path.
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "gs_pcd_geom.cuh"

extern "C" {

// tri[3*i .. 3*i+2]: the input indices of the triangle containing query i, or -1 when it lies outside the hull.
// Returns the OR of the status codes of all queries.
int gspcd_host_locate(const double* xy, int64_t n, const double* q, int64_t m, double cell, int32_t W, int32_t H,
                      int32_t* tri) {
    const double inv_s = 1.0 / cell;
    const int gw = (int)((double)(W - 1) * inv_s) + 1, gh = (int)((double)(H - 1) * inv_s) + 1;
    std::vector<int> start((size_t)gw * gh + 1, 0), idx(n), key(n);
    for (int64_t i = 0; i < n; ++i) {
        key[i] = pcd::cell_coord(xy[2 * i + 1], inv_s, gh) * gw + pcd::cell_coord(xy[2 * i], inv_s, gw);
        start[key[i] + 1]++;
    }
    for (size_t c = 0; c + 1 < start.size(); ++c) start[c + 1] += start[c];
    std::vector<int> cursor(start.begin(), start.end() - 1);
    for (int64_t i = 0; i < n; ++i) idx[cursor[key[i]]++] = (int)i;  // ascending index within a cell
    std::vector<double> x(n), y(n);
    for (int64_t e = 0; e < n; ++e) { x[e] = xy[2 * idx[e]]; y[e] = xy[2 * idx[e] + 1]; }
    pcd::Grid g{gw, gh, cell, inv_s, start.data(), x.data(), y.data(), idx.data()};
    int status = 0;
    // hull candidates: the points of the cells in the band near each grid row's and column's occupied extremes
    std::vector<int> top(gw, -1), bot(gw, gh), left(gh, gw), right(gh, -1), order, hull(2 * (size_t)n + 1);
    for (int c = 0; c < gw * gh; ++c)
        if (start[c + 1] > start[c]) {
            const int i = c % gw, j = c / gw;
            top[i] = std::max(top[i], j); bot[i] = std::min(bot[i], j);
            left[j] = std::min(left[j], i); right[j] = std::max(right[j], i);
        }
    for (int c = 0; c < gw * gh; ++c) {
        const int i = c % gw, j = c / gw;
        if (pcd::in_hull_band(i, j, top[i], bot[i], left[j], right[j]))
            for (int e = start[c]; e < start[c + 1]; ++e) order.push_back(e);
    }
    std::sort(order.begin(), order.end(), [&](int u, int v) {
        return pcd::xy_less(pcd::Pt{x[u], y[u]}, idx[u], pcd::Pt{x[v], y[v]}, idx[v]);
    });
    const int hn = pcd::monotone_chain(x.data(), y.data(), order.data(), (int)order.size(), hull.data(), status);
    for (int64_t i = 0; i < m; ++i) {
        const pcd::Pt qi{q[2 * i], q[2 * i + 1]};
        pcd::Located t{{-1, -1, -1}};
        if (pcd::in_hull(x.data(), y.data(), hull.data(), hn, qi, status)) t = pcd::locate(g, (int)n, qi, status);
        for (int k = 0; k < 3; ++k) tri[3 * i + k] = t.v[0] < 0 ? -1 : idx[t.v[k]];
    }
    return status;
}

int gspcd_host_orient(const double* a, const double* b, const double* c) {
    int st = 0;
    return pcd::orient(pcd::Pt{a[0], a[1]}, pcd::Pt{b[0], b[1]}, pcd::Pt{c[0], c[1]}, st);
}

int gspcd_host_incircle(const double* a, const double* b, const double* c, const double* d) {
    int st = 0;
    return pcd::incircle(pcd::Pt{a[0], a[1]}, pcd::Pt{b[0], b[1]}, pcd::Pt{c[0], c[1]}, pcd::Pt{d[0], d[1]}, st);
}

}  // extern "C"
