// Internal: host-side decoder of one env's support graph (pct_get_support_graph, include/pct_b200.h) from a host copy of the env's
// records.  Plain C++ without device code: the C ABI runs it on the records it copied from the device, the host build of the
// stability routine (tests/host_emul/stab_host.cpp) on its own pools.  The records are data from elsewhere: every index is checked
// before it is followed, and a finding is reported as text instead of being walked into.
#pragma once
#include <cstdio>
#include <cstring>
#include "pct_kernels.h"

namespace pct {

struct GraphRecord {  // views into one env's records (host memory)
    int n_box, n_edge, n_poly;
    const uint16_t *e_off, *poly_off;
    const uint8_t *e_lower, *e_next, *first_in, *last_in;
    const Stack4 *e_st;
    const double *poly;       // [POLY_MAX][2]
    const Stack4 *box_st;     // the three arrays of EdgePoolA; nullptr outside the alias mode
    const uint8_t *e_upper;
    const uint32_t *e_alias;
};

#define PCT_GRAPH_FAIL(...) do { snprintf(err, cap, __VA_ARGS__); return false; } while (0)

inline bool decode_support_graph(const GraphRecord &r, pct_support_graph *g, char *err, size_t cap) {
    memset(g, 0, sizeof *g);
    const int nb = r.n_box, ne = r.n_edge;
    if (nb < 0 || nb > NB_MAX) PCT_GRAPH_FAIL("n_box = %d outside [0, %d]", nb, NB_MAX);
    if (ne < 0 || ne > EDGE_MAX) PCT_GRAPH_FAIL("n_edge = %d outside [0, %d]", ne, EDGE_MAX);
    if (r.n_poly < 0 || r.n_poly > POLY_MAX) PCT_GRAPH_FAIL("n_poly = %d outside [0, %d]", r.n_poly, POLY_MAX);
    g->n_box = nb; g->n_edge = ne; g->n_poly = r.n_poly; g->alias = r.box_st ? 1 : 0;
    // supports: CSR by upper box.  Edges at or behind e_off[n_box] belong to the box of a failed placement (index n_box)
    const int tail = (nb > 0 || ne > 0) ? (int)r.e_off[nb] : 0;
    if (tail > ne) PCT_GRAPH_FAIL("e_off[%d] = %d beyond n_edge = %d", nb, tail, ne);
    int upper_of[EDGE_MAX + 1];
    for (int u = 0; u < nb; u++) {
        const int a = r.e_off[u], b = r.e_off[u + 1];
        if (a > b || b > tail) PCT_GRAPH_FAIL("box %d: e_off %d .. %d not inside 0 .. %d", u, a, b, tail);
        if (u == 0 && a != 0) PCT_GRAPH_FAIL("box 0: e_off = %d, not 0", a);
        g->sup_off[u] = a;
        for (int q = a; q < b; q++) {
            if (r.e_lower[q] >= u) PCT_GRAPH_FAIL("box %d: support %d (edge %d) is not an earlier box", u, (int)r.e_lower[q], q);
            g->sup[q] = r.e_lower[q];
            upper_of[q] = u;
        }
    }
    g->sup_off[nb] = tail;
    for (int q = tail; q < ne; q++) {
        if (r.e_lower[q] >= nb) PCT_GRAPH_FAIL("box %d (failed placement): support %d (edge %d) is not a placed box", nb, (int)r.e_lower[q], q);
        upper_of[q] = nb;
    }
    // loads: the list of every placed box, in list order
    bool seen[EDGE_MAX + 1] = {};
    int n = 0;
    for (int t = 0; t < nb; t++) {
        g->load_off[t] = n;
        int q = r.first_in[t], prev = -1;
        while (q != EDGE_NIL) {
            if (q >= ne) PCT_GRAPH_FAIL("box %d: load list reaches edge %d beyond n_edge = %d (field e_next / first_in)", t, q, ne);
            if (seen[q]) PCT_GRAPH_FAIL("box %d: edge %d is filed twice (cycle or shared tail, field e_next)", t, q);
            if (q <= prev) PCT_GRAPH_FAIL("box %d: edge %d follows edge %d, list not in insertion order (field e_next)", t, q, prev);
            if (r.e_lower[q] != t) PCT_GRAPH_FAIL("box %d: edge %d in its load list rests on box %d (field e_next / e_lower)", t, q, (int)r.e_lower[q]);
            seen[q] = true;
            if (r.e_upper && r.e_upper[q] != upper_of[q])
                PCT_GRAPH_FAIL("box %d: edge %d comes from box %d by its position, e_upper says %d", t, q, upper_of[q], (int)r.e_upper[q]);
            g->load_upper[n] = upper_of[q];
            g->load_alias[n] = r.e_alias ? (int)((r.e_alias[q >> 5] >> (q & 31)) & 1u) : 0;
            const Stack4 &s = r.e_st[q];
            g->load[n][0] = s.cx; g->load[n][1] = s.cy; g->load[n][2] = s.cz; g->load[n][3] = s.m;
            n++;
            prev = q;
            q = r.e_next[q];
        }
        if (prev >= 0 && r.last_in[t] != prev) PCT_GRAPH_FAIL("box %d: load list ends at edge %d, last_in says %d", t, prev, (int)r.last_in[t]);
    }
    g->load_off[nb] = n;
    if (n != ne)
        for (int q = 0; q < ne; q++)
            if (!seen[q]) PCT_GRAPH_FAIL("edge %d (box %d on box %d) is in no load list (field e_next / first_in)", q, upper_of[q], (int)r.e_lower[q]);
    if (r.e_alias)
        for (int q = ne; q < EDGE_MAX + 1; q++) g->alias_stale += (int)((r.e_alias[q >> 5] >> (q & 31)) & 1u);
    // stored polygons: CSR by box; a box with two supports keeps its split direction behind the vertices
    const int ptail = nb > 0 ? (int)r.poly_off[nb] : 0;
    if (ptail > r.n_poly) PCT_GRAPH_FAIL("poly_off[%d] = %d beyond n_poly = %d", nb, ptail, r.n_poly);
    int m = 0;
    for (int u = 0; u < nb; u++) {
        const int a = r.poly_off[u], b = r.poly_off[u + 1], k = g->sup_off[u + 1] - g->sup_off[u];
        if (a > b || b > ptail) PCT_GRAPH_FAIL("box %d: poly_off %d .. %d not inside 0 .. %d", u, a, b, ptail);
        g->poly_off[u] = m; g->poly_pos[u] = a;
        if (b == a) continue;
        if (k < 2) PCT_GRAPH_FAIL("box %d: %d polygon entries stored for a box with %d support(s)", u, b - a, k);
        const int nv = b - a - (k == 2);
        if (nv < 3) PCT_GRAPH_FAIL("box %d: stored polygon has %d vertices", u, nv);
        for (int i = 0; i < nv; i++) { g->poly[m][0] = r.poly[2 * (a + i)]; g->poly[m][1] = r.poly[2 * (a + i) + 1]; m++; }
        if (k == 2) { g->has_split[u] = 1; g->split[u][0] = r.poly[2 * (b - 1)]; g->split[u][1] = r.poly[2 * (b - 1) + 1]; }
    }
    g->poly_off[nb] = m;
    if (r.box_st)
        for (int u = 0; u <= nb && u < NB_MAX + 1; u++) {
            const Stack4 &s = r.box_st[u];
            g->own_stack[u][0] = s.cx; g->own_stack[u][1] = s.cy; g->own_stack[u][2] = s.cz; g->own_stack[u][3] = s.m;
        }
    return true;
}
#undef PCT_GRAPH_FAIL

}  // namespace pct
