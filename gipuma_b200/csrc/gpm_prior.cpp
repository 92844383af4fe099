// gpm_prior.cpp — host side of the planar prior's construction (DESIGN.md §18): the Delaunay triangulation of the support
// points and the planes of its triangles.  oracle/pyprior.py restates both step for step.
#include <algorithm>
#include <array>
#include <cmath>
#include <stdexcept>
#include <vector>

namespace gpm {
namespace {

typedef long long i64;

struct Tri {
    int v[3];   // counter-clockwise: orient(v0, v1, v2) > 0
    int n[3];   // n[k]: the triangle across the edge opposite v[k], -1 on the hull
};

// Incremental Delaunay triangulation by edge flips (Lawson), exact in int64: at coordinates <= 4096 every difference
// is <= 2^12 and the in-circle determinant stays below 2^53.
struct Mesh {
    const int* xy;
    std::vector<Tri> t;
    int last = 0;

    i64 orient(int a, int b, int c) const
    {
        const i64 ax = xy[2 * a], ay = xy[2 * a + 1];
        return ((i64)xy[2 * b] - ax) * ((i64)xy[2 * c + 1] - ay) - ((i64)xy[2 * b + 1] - ay) * ((i64)xy[2 * c] - ax);
    }
    // d strictly inside the circle through the counter-clockwise a, b, c
    bool incircle(int a, int b, int c, int d) const
    {
        const i64 dx = xy[2 * d], dy = xy[2 * d + 1];
        const i64 adx = xy[2 * a] - dx, ady = xy[2 * a + 1] - dy;
        const i64 bdx = xy[2 * b] - dx, bdy = xy[2 * b + 1] - dy;
        const i64 cdx = xy[2 * c] - dx, cdy = xy[2 * c + 1] - dy;
        const i64 det = (adx * adx + ady * ady) * (bdx * cdy - cdx * bdy) + (bdx * bdx + bdy * bdy) * (cdx * ady - adx * cdy) +
                        (cdx * cdx + cdy * cdy) * (adx * bdy - bdx * ady);
        return det > 0;
    }
    int add(int a, int b, int c, int na, int nb, int nc)
    {
        t.push_back(Tri{{a, b, c}, {na, nb, nc}});
        return (int)t.size() - 1;
    }
    void relink(int x, int from, int to)
    {
        if (x < 0) return;
        for (int k = 0; k < 3; k++)
            if (t[x].n[k] == from) { t[x].n[k] = to;  return; }
    }
    // Flip the edge opposite p = t[i].v[0] while the vertex across it lies strictly inside the circle of t[i] (a
    // cocircular quadrilateral keeps its diagonal).  Depth first, in the order the triangles are given.
    void legalize(std::vector<int> stack)
    {
        std::reverse(stack.begin(), stack.end());
        while (!stack.empty()) {
            const int ti = stack.back();
            stack.pop_back();
            const int ui = t[ti].n[0];
            if (ui < 0) continue;
            const Tri T = t[ti], U = t[ui];
            int j = 0;
            while (U.n[j] != ti) j++;
            const int p = T.v[0], a = T.v[1], b = T.v[2], q = U.v[j];
            if (!incircle(p, a, b, q)) continue;
            const int nta = T.n[1], ntb = T.n[2], nua = U.n[(j + 2) % 3], nub = U.n[(j + 1) % 3];
            t[ti] = Tri{{p, a, q}, {nub, ui, ntb}};
            t[ui] = Tri{{p, q, b}, {nua, nta, ti}};
            relink(nta, ti, ui);
            relink(nub, ui, ti);
            stack.push_back(ui);
            stack.push_back(ti);
        }
    }
    // hull edge (t, k) = (v[k+1], v[k+2]); the hull edge after it (starting at its end) and before it (ending at its start)
    std::array<int, 2> next_hull(int ti, int k) const
    {
        const int b = t[ti].v[(k + 2) % 3];
        for (int cur = ti;;) {
            int m = 0;
            while (t[cur].v[m] != b) m++;
            const int e = (m + 2) % 3;
            if (t[cur].n[e] < 0) return {cur, e};
            cur = t[cur].n[e];
        }
    }
    std::array<int, 2> prev_hull(int ti, int k) const
    {
        const int a = t[ti].v[(k + 1) % 3];
        for (int cur = ti;;) {
            int m = 0;
            while (t[cur].v[m] != a) m++;
            const int e = (m + 1) % 3;
            if (t[cur].n[e] < 0) return {cur, e};
            cur = t[cur].n[e];
        }
    }
    bool sees(int ti, int k, int p) const { return orient(t[ti].v[(k + 1) % 3], t[ti].v[(k + 2) % 3], p) < 0; }

    void insert(int p)
    {
        // visibility walk from the triangle of the last insertion: leave through the first edge p lies strictly right of
        int cur = last, out = -1;
        for (size_t steps = 0;; steps++) {
            if (steps > 4 * t.size() + 16) throw std::runtime_error("Delaunay walk did not terminate");
            out = -1;
            for (int k = 0; k < 3 && out < 0; k++)
                if (orient(t[cur].v[(k + 1) % 3], t[cur].v[(k + 2) % 3], p) < 0) out = k;
            if (out < 0 || t[cur].n[out] < 0) break;
            cur = t[cur].n[out];
        }
        if (out >= 0) {                                          // outside the hull: a fan over every visible hull edge
            std::array<int, 2> first = {cur, out};
            for (;;) {
                const std::array<int, 2> pr = prev_hull(first[0], first[1]);
                if (pr == std::array<int, 2>{cur, out} || !sees(pr[0], pr[1], p)) break;
                first = pr;
            }
            std::vector<std::array<int, 2>> edges = {first};
            for (;;) {
                const std::array<int, 2> nx = next_hull(edges.back()[0], edges.back()[1]);
                if (nx == first || !sees(nx[0], nx[1], p)) break;
                edges.push_back(nx);
            }
            const int base = (int)t.size();
            std::vector<int> fresh;
            for (size_t e = 0; e < edges.size(); e++) {
                const int te = edges[e][0], ke = edges[e][1];
                const int a = t[te].v[(ke + 1) % 3], b = t[te].v[(ke + 2) % 3];
                const int prev = e > 0 ? base + (int)e - 1 : -1, next = e + 1 < edges.size() ? base + (int)e + 1 : -1;
                fresh.push_back(add(p, b, a, te, prev, next));
                t[te].n[ke] = fresh.back();
            }
            last = fresh[0];
            legalize(fresh);
            return;
        }
        const Tri T = t[cur];
        int zero = -1, nzero = 0;
        for (int k = 0; k < 3; k++)
            if (orient(T.v[(k + 1) % 3], T.v[(k + 2) % 3], p) == 0) { zero = k;  nzero++; }
        if (nzero > 1) throw std::runtime_error("Delaunay: duplicate point");
        last = cur;
        if (nzero == 0) {                                        // strictly inside: three triangles
            const int a = T.v[0], b = T.v[1], c = T.v[2];
            const int t1 = (int)t.size(), t2 = t1 + 1;
            t[cur] = Tri{{p, b, c}, {T.n[0], t1, t2}};
            add(p, c, a, T.n[1], t2, cur);
            add(p, a, b, T.n[2], cur, t1);
            relink(T.n[1], cur, t1);
            relink(T.n[2], cur, t2);
            legalize({cur, t1, t2});
            return;
        }
        // on the edge opposite T.v[zero]: two triangles on each side of it (one on the hull)
        const int i = zero, c = T.v[i], a = T.v[(i + 1) % 3], b = T.v[(i + 2) % 3];
        const int ui = T.n[i];
        const int t1 = (int)t.size(), u1 = ui >= 0 ? t1 + 1 : -1;
        t[cur] = Tri{{p, c, a}, {T.n[(i + 2) % 3], u1, t1}};
        add(p, b, c, T.n[(i + 1) % 3], cur, ui);
        relink(T.n[(i + 1) % 3], cur, t1);
        if (ui < 0) { legalize({cur, t1});  return; }
        const Tri U = t[ui];
        int j = 0;
        while (U.n[j] != cur) j++;
        const int d = U.v[j];
        t[ui] = Tri{{p, d, b}, {U.n[(j + 2) % 3], t1, u1}};
        add(p, a, d, U.n[(j + 1) % 3], ui, cur);
        relink(U.n[(j + 1) % 3], ui, u1);
        legalize({cur, t1, ui, u1});
    }
};

}  // namespace

// Delaunay triangulation of the n points xy (x0 y0 x1 y1 ..., distinct, 0 <= coordinate <= 4096), inserted in the given
// order.  Returns the triangles as counter-clockwise vertex-index triples, each rotated to start at its smallest index,
// sorted.  Until three points are not collinear nothing is triangulated; the first such point is joined to the collinear
// chain so far (a fan, which is Delaunay).
std::vector<std::array<int, 3>> delaunay(const std::vector<int>& xy)
{
    const int n = (int)xy.size() / 2;
    Mesh M;
    M.xy = xy.data();
    std::vector<int> chain;
    for (int p = 0; p < n; p++) {
        if (!M.t.empty()) { M.insert(p);  continue; }
        if (chain.size() < 2 || M.orient(chain[0], chain[1], p) == 0) { chain.push_back(p);  continue; }
        std::sort(chain.begin(), chain.end(), [&](int u, int v) {
            return xy[2 * u] != xy[2 * v] ? xy[2 * u] < xy[2 * v] : xy[2 * u + 1] < xy[2 * v + 1];
        });
        const bool left = M.orient(chain[0], chain[1], p) > 0;
        const int m = (int)chain.size() - 1;
        for (int k = 0; k < m; k++) {
            const int prev = k > 0 ? k - 1 : -1, next = k + 1 < m ? k + 1 : -1;
            if (left) M.add(p, chain[k], chain[k + 1], -1, next, prev);
            else M.add(p, chain[k + 1], chain[k], -1, prev, next);
        }
        M.last = 0;
    }
    std::vector<std::array<int, 3>> out;
    for (const Tri& T : M.t) {
        int r = 0;
        if (T.v[1] < T.v[r]) r = 1;
        if (T.v[2] < T.v[r]) r = 2;
        out.push_back({T.v[r], T.v[(r + 1) % 3], T.v[(r + 2) % 3]});
    }
    std::sort(out.begin(), out.end());
    return out;
}

// Plane (n.xyz, d) of the triangle through the points the support pixels (x, y) see on their own planes (float4: n.xyz, d):
// X_i = z_i K^-1 (x_i, y_i, 1) with z_i = -d_i / (n_i . K^-1 (x_i, y_i, 1)), in double; n = the unit cross product of
// X1 - X0 and X2 - X0, negated where it points along the sum of the three points (away from the camera, as the sweep
// orients its normals), d = -n . X0; rounded to float.  All-zero where the cross product is zero.
std::array<float, 4> triangle_plane(const float* Kinv, const int* x, const int* y, const float* const* plane)
{
    double X[3][3];
    for (int i = 0; i < 3; i++) {
        const double px = x[i], py = y[i];
        double r[3];
        for (int k = 0; k < 3; k++) r[k] = ((double)Kinv[3 * k] * px + (double)Kinv[3 * k + 1] * py) + (double)Kinv[3 * k + 2];
        const double nx = plane[i][0], ny = plane[i][1], nz = plane[i][2], d = plane[i][3];
        const double z = -d / ((nx * r[0] + ny * r[1]) + nz * r[2]);
        for (int k = 0; k < 3; k++) X[i][k] = z * r[k];
    }
    double e1[3], e2[3];
    for (int k = 0; k < 3; k++) { e1[k] = X[1][k] - X[0][k];  e2[k] = X[2][k] - X[0][k]; }
    double c[3] = {e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0]};
    const double len = std::sqrt((c[0] * c[0] + c[1] * c[1]) + c[2] * c[2]);
    if (len == 0.0) return {0.f, 0.f, 0.f, 0.f};
    for (int k = 0; k < 3; k++) c[k] = c[k] / len;
    double s[3];
    for (int k = 0; k < 3; k++) s[k] = (X[0][k] + X[1][k]) + X[2][k];
    if ((c[0] * s[0] + c[1] * s[1]) + c[2] * s[2] > 0.0)
        for (int k = 0; k < 3; k++) c[k] = -c[k];
    const double d = -((c[0] * X[0][0] + c[1] * X[0][1]) + c[2] * X[0][2]);
    return {(float)c[0], (float)c[1], (float)c[2], (float)d};
}

}  // namespace gpm
