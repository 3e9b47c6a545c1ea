/* TEST INFRASTRUCTURE — CPU restatement ("oracle") of the reference's PCT environment hot path.
 * Not part of the product: only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load this.  See oracle/README.md for how it is pinned against the
 * unmodified Python reference (golden vectors under tests/golden/).
 *
 * Shared numeric helpers.  Every helper cites the reference lines it restates (paths relative to
 * /root/reference; D: = pct_envs/PctDiscrete0/, C: = pct_envs/PctContinuous0/).
 * Build with -ffp-contract=off: every * + - / below must be ONE IEEE-754 binary64 operation, as in
 * numpy's element-wise loops; the only fused operations are the explicit fma() calls that reproduce
 * OpenBLAS ddot on 2-vectors (SURVEY.md §8(a) "FP-parity facts").
 */
#ifndef PCT_ORACLE_COMMON_H
#define PCT_ORACLE_COMMON_H
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define PO_MAX_SUP 64   /* supports under one box (bottom_edges)            */
#define PO_MAX_UP 64    /* boxes resting directly on one box (up_edges)     */
#define PO_MAX_PTS (4 * PO_MAX_SUP)

/* np.dot(u, v) on 2-vectors = OpenBLAS ddot: fma(u1, v1, u0*v0)  (D:space.py:114-115,212-213) */
static inline double po_dot2(const double *u, const double *v) { return fma(u[1], v[1], u[0] * v[0]); }
/* np.linalg.norm(u) on a 2-vector = sqrt(dot(u,u))              (D:space.py:111,209) */
static inline double po_norm2(const double *u) { return sqrt(fma(u[1], u[1], u[0] * u[0])); }

/* ---- convex_hull.py:4-32  Line2D ------------------------------------------------------- */
static inline double po_slope(const double *p1, const double *p2) {
    if (p2[0] != p1[0]) return (p2[1] - p1[1]) / (p2[0] - p1[0]);
    return (p2[1] - p1[1]) * INFINITY; /* 0*inf = nan, as in the reference */
}
static inline int po_orientation(double slope1, double slope2) {
    if (fabs(slope1) == INFINITY && fabs(slope2) == INFINITY) return 0;
    double diff = slope2 - slope1;
    if (diff > 0) return -1;
    if (diff == 0) return 0;
    return 1; /* includes nan */
}

/* ---- convex_hull.py:39-95  ConvexHull --------------------------------------------------
 * in : n points (x,y);  out: hull polygon (lower chain minus its last + upper chain minus its last)
 * returns number of hull points.  The x-perturbation (x += y*1e-6, :43) stays in the output. */
static int po_convex_hull(const double (*pts_in)[2], int n, double (*out)[2]) {
    double pts[PO_MAX_PTS][2];
    int order[PO_MAX_PTS];
    for (int i = 0; i < n; i++) {
        double t = pts_in[i][1] * 1e-6;
        pts[i][0] = pts_in[i][0] + t;
        pts[i][1] = pts_in[i][1];
        order[i] = i;
    }
    /* sorted(key=x): stable insertion sort (:34-37) */
    for (int i = 1; i < n; i++) {
        int o = order[i];
        int j = i - 1;
        while (j >= 0 && pts[order[j]][0] > pts[o][0]) { order[j + 1] = order[j]; j--; }
        order[j + 1] = o;
    }
    double lower[PO_MAX_PTS + 1][2], upper[PO_MAX_PTS + 1][2];
    int nl = 0, nu = 0;
    for (int pass = 0; pass < 2; pass++) {
        double (*H)[2] = pass == 0 ? lower : upper;
        int nh = 0;
        double s1 = 0, s2 = 0; /* slopes of line1/line2; only read when nh>=2 (short-circuit at :56/:74) */
        for (int k = 0; k < n; k++) {
            const double *p = pts[order[pass == 0 ? k : n - 1 - k]];
            if (nh >= 2) {
                s1 = po_slope(H[nh - 2], H[nh - 1]);
                s2 = po_slope(H[nh - 1], p);
            }
            while (nh >= 2 && po_orientation(s1, s2) != -1) {
                nh--; /* pop */
                if (H[0][0] == H[nh - 1][0] && H[0][1] == H[nh - 1][1]) break; /* :58-59 list equality */
                s1 = po_slope(H[nh - 2], H[nh - 1]);
                s2 = po_slope(H[nh - 1], p);
            }
            H[nh][0] = p[0];
            H[nh][1] = p[1];
            nh++;
        }
        if (pass == 0) nl = nh; else nu = nh;
    }
    /* :89-92 drop the last of each chain, lower + upper */
    int m = 0;
    for (int i = 0; i < nl - 1; i++) { out[m][0] = lower[i][0]; out[m][1] = lower[i][1]; m++; }
    for (int i = 0; i < nu - 1; i++) { out[m][0] = upper[i][0]; out[m][1] = upper[i][1]; m++; }
    return m;
}

/* ---- D:space.py:341-345 / C:space.py:323-327  scale_down -------------------------------- */
static void po_scale_down(double (*poly)[2], int n) {
    double sx = 0, sy = 0;
    for (int i = 0; i < n; i++) { sx += poly[i][0]; sy += poly[i][1]; } /* np.mean axis 0: sequential */
    double cx = sx / (double)n, cy = sy / (double)n;
    for (int i = 0; i < n; i++) {
        double dx = poly[i][0] - cx, dy = poly[i][1] - cy;
        poly[i][0] = poly[i][0] - dx * 0.1;
        poly[i][1] = poly[i][1] - dy * 0.1;
    }
}

/* ---- convex_hull.py:97-112  point_in_polygen -------------------------------------------- */
static int po_point_in_polygon(double lat, double lon, const double (*c)[2], int n) {
    int j = n - 1, odd = 0;
    for (int i = 0; i < n; i++) {
        double a0 = c[i][0] - lat, a1 = c[i][1] - lon; /* coords[i] - point */
        double b0 = lat - c[j][0], b1 = lon - c[j][1]; /* point - coords[j] */
        double m1 = a0 * b1, m2 = a1 * b0;
        if (m1 - m2 == 0) return 0; /* np.cross == 0 -> False (:104-105) */
        if ((c[i][1] < lon && c[j][1] >= lon) || (c[j][1] < lon && c[i][1] >= lon)) {
            double t = (lon - c[i][1]) / (c[j][1] - c[i][1]);
            double u = t * (c[j][0] - c[i][0]);
            if (c[i][0] + u < lat) odd = !odd;
        }
        j = i;
    }
    return odd;
}

/* ---- np.linalg.lstsq(coefficient, value, rcond=None)[0]  (D:space.py:152,249) -------------
 * LAPACK dgelsd is an SVD-based minimum-norm solver and cannot be reproduced bit-for-bit.
 * Restatement: streaming Givens QR of the (k(k-1)/2+1) x k system (rows are generated one at a
 * time, only R (k x k) and the rotated right-hand side are kept), then a one-sided Jacobi SVD of R
 * and the same truncation rule (sigma <= eps*max(M,N)*sigma_max treated as zero).  The device code
 * in csrc/ performs the identical operation sequence so oracle and GPU agree bit-for-bit; agreement
 * with LAPACK is to rounding error (see tests/test_oracle_vs_reference.py for the measured rate).
 * Call protocol: po_ls_init, po_ls_add_row for every row (in order), po_ls_solve. */
typedef struct {
    int k;
    int rows;
    double R[PO_MAX_SUP][PO_MAX_SUP];
    double y[PO_MAX_SUP];
} po_ls;

static void po_ls_init(po_ls *s, int k) {
    s->k = k;
    s->rows = 0;
    for (int i = 0; i < k; i++) {
        s->y[i] = 0;
        for (int j = 0; j < k; j++) s->R[i][j] = 0;
    }
}
/* rotate (row, rhs) into R; row is destroyed */
static void po_ls_add_row(po_ls *s, double *row, double rhs) {
    int k = s->k;
    s->rows++;
    for (int i = 0; i < k; i++) {
        double b = row[i];
        if (b == 0) continue;
        double a = s->R[i][i];
        double r = sqrt(a * a + b * b);
        double c = a / r, sn = b / r;
        for (int j = i; j < k; j++) {
            double rij = s->R[i][j], vj = row[j];
            s->R[i][j] = c * rij + sn * vj;
            row[j] = c * vj - sn * rij;
        }
        double yi = s->y[i];
        s->y[i] = c * yi + sn * rhs;
        rhs = c * rhs - sn * yi;
    }
}
static void po_ls_solve(po_ls *s, double *x) {
    int k = s->k;
    double (*G)[PO_MAX_SUP] = s->R;
    {   /* full column rank and well conditioned (the usual case): least-squares solution of R x = y */
        double rmin = fabs(G[0][0]), rmax = rmin;
        for (int i = 1; i < k; i++) { double a = fabs(G[i][i]); rmin = fmin(rmin, a); rmax = fmax(rmax, a); }
        if (rmin * 1e4 > rmax) {
            for (int i = k - 1; i >= 0; i--) {
                double acc = s->y[i];
                for (int j = i + 1; j < k; j++) acc -= G[i][j] * x[j];
                x[i] = acc / G[i][i];
            }
            return;
        }
    }
    static __thread double V[PO_MAX_SUP][PO_MAX_SUP];
    for (int i = 0; i < k; i++)
        for (int j = 0; j < k; j++) V[i][j] = (i == j) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 60; sweep++) {
        int rotated = 0;
        for (int p = 0; p < k - 1; p++)
            for (int q = p + 1; q < k; q++) {
                double alpha = 0, beta = 0, gamma = 0;
                for (int i = 0; i < k; i++) {
                    alpha += G[i][p] * G[i][p];
                    beta += G[i][q] * G[i][q];
                    gamma += G[i][p] * G[i][q];
                }
                if (gamma == 0 || fabs(gamma) <= 1e-15 * sqrt(alpha * beta)) continue;
                rotated = 1;
                double zeta = (beta - alpha) / (2.0 * gamma);
                double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                double c = 1.0 / sqrt(1.0 + t * t), sn = c * t;
                for (int i = 0; i < k; i++) {
                    double gp = G[i][p], gq = G[i][q];
                    G[i][p] = c * gp - sn * gq;
                    G[i][q] = sn * gp + c * gq;
                    double vp = V[i][p], vq = V[i][q];
                    V[i][p] = c * vp - sn * vq;
                    V[i][q] = sn * vp + c * vq;
                }
            }
        if (!rotated) break;
    }
    double sig[PO_MAX_SUP], smax = 0;
    for (int j = 0; j < k; j++) {
        double a = 0;
        for (int i = 0; i < k; i++) a += G[i][j] * G[i][j];
        sig[j] = sqrt(a);
        if (sig[j] > smax) smax = sig[j];
    }
    int M = s->rows > k ? s->rows : k;
    double cutoff = 2.220446049250313e-16 * (double)M * smax;
    for (int i = 0; i < k; i++) x[i] = 0;
    for (int j = 0; j < k; j++) {
        if (!(sig[j] > cutoff)) continue;
        double uy = 0;
        for (int i = 0; i < k; i++) uy += G[i][j] * s->y[i];
        double coef = uy / (sig[j] * sig[j]); /* (u_j . y)/sigma_j with u_j = G_j/sigma_j */
        for (int i = 0; i < k; i++) x[i] += V[i][j] * coef;
    }
}

/* ---- CPython 3.12 set of 6-tuples: iteration-order emulation ------------------------------
 * Objects/tupleobject.c (xxHash-style tuplehash) + Objects/setobject.c (set_add_entry,
 * set_insert_clean, set_table_resize; LINEAR_PROBES 9, PERTURB_SHIFT 5).  Call sites:
 * D:space.py:535,565-569 and C:space.py:532,563-567.  Keys are compared as 6 x 64-bit words
 * (ints: the value; floats: the IEEE bit pattern — equal floats have equal bits here because no
 * -0.0/NaN coordinates occur). */
#define PO_XXP1 11400714785074694791ULL
#define PO_XXP2 14029467366897019727ULL
#define PO_XXP5 2870177450012600261ULL
static inline uint64_t po_tuple_hash6(const uint64_t lane[6]) {
    uint64_t acc = PO_XXP5;
    for (int i = 0; i < 6; i++) {
        acc += lane[i] * PO_XXP2;
        acc = (acc << 31) | (acc >> 33);
        acc *= PO_XXP1;
    }
    acc += 6ULL ^ (PO_XXP5 ^ 3527539ULL);
    if (acc == (uint64_t)-1) return 1546275796ULL;
    return acc;
}
/* tuplehash for an n-tuple of already hashed lanes (Objects/tupleobject.c) */
static inline uint64_t po_tuple_hash_n(const uint64_t *lane, int n) {
    uint64_t acc = PO_XXP5;
    for (int i = 0; i < n; i++) {
        acc += lane[i] * PO_XXP2;
        acc = (acc << 31) | (acc >> 33);
        acc *= PO_XXP1;
    }
    acc += (uint64_t)n ^ (PO_XXP5 ^ 3527539ULL);
    if (acc == (uint64_t)-1) return 1546275796ULL;
    return acc;
}
/* hash(int) for |v| < 2**61-1 */
static inline uint64_t po_hash_int(int64_t v) { return v == -1 ? (uint64_t)-2 : (uint64_t)v; }
/* _Py_HashDouble (Python/pyhash.c) for finite doubles */
static inline uint64_t po_hash_double(double v) {
    const uint64_t MOD = (1ULL << 61) - 1;
    int e, sign = 1;
    double m = frexp(v, &e);
    if (m < 0) { sign = -1; m = -m; }
    uint64_t x = 0;
    while (m) {
        x = ((x << 28) & MOD) | x >> (61 - 28);
        m *= 268435456.0; /* 2**28 */
        e -= 28;
        uint64_t y = (uint64_t)m;
        m -= (double)y;
        x += y;
        if (x >= MOD) x -= MOD;
    }
    e = e >= 0 ? e % 61 : 61 - 1 - ((-1 - e) % 61);
    x = ((x << e) & MOD) | x >> (61 - e);
    int64_t r = (int64_t)x * sign;
    if (r == -1) r = -2;
    return (uint64_t)r;
}

typedef struct {
    uint64_t (*keys)[6]; /* insertion-ordered unique keys   */
    uint64_t *hashes;
    int n, cap;
    int32_t *table; /* slot -> key index or -1         */
    uint64_t mask;
    int fill;
} po_pyset;

static void po_pyset_init(po_pyset *s) {
    s->cap = 64;
    s->keys = malloc(sizeof(uint64_t[6]) * s->cap);
    s->hashes = malloc(sizeof(uint64_t) * s->cap);
    s->n = 0;
    s->mask = 7;
    s->table = malloc(sizeof(int32_t) * 8);
    for (int i = 0; i < 8; i++) s->table[i] = -1;
    s->fill = 0;
}
static void po_pyset_free(po_pyset *s) { free(s->keys); free(s->hashes); free(s->table); }
/* set_insert_clean (setobject.c): same probe sequence, no key comparison */
static void po_pyset_insert_clean(int32_t *table, uint64_t mask, uint64_t hash, int idx) {
    uint64_t perturb = hash, i = hash & mask;
    for (;;) {
        int probes = (i + 9 <= mask) ? 9 : 0;
        for (int j = 0; j <= probes; j++)
            if (table[i + j] < 0) { table[i + j] = idx; return; }
        perturb >>= 5;
        i = (i * 5 + 1 + perturb) & mask;
    }
}
static void po_pyset_add(po_pyset *s, const uint64_t key[6]) {
    uint64_t hash = po_tuple_hash6(key);
    uint64_t perturb = hash, i = hash & s->mask;
    for (;;) {
        int probes = (i + 9 <= s->mask) ? 9 : 0;
        for (int j = 0; j <= probes; j++) {
            int32_t e = s->table[i + j];
            if (e < 0) {
                if (s->n == s->cap) {
                    s->cap *= 2;
                    s->keys = realloc(s->keys, sizeof(uint64_t[6]) * s->cap);
                    s->hashes = realloc(s->hashes, sizeof(uint64_t) * s->cap);
                }
                memcpy(s->keys[s->n], key, sizeof(uint64_t[6]));
                s->hashes[s->n] = hash;
                s->table[i + j] = s->n++;
                s->fill++;
                if ((uint64_t)s->fill * 5 < s->mask * 3) return;
                /* set_table_resize(so, used*4): smallest power of two > used*4 (used <= 50000) */
                uint64_t minused = (uint64_t)s->n * 4, newsize = 8;
                while (newsize <= minused) newsize <<= 1;
                int32_t *nt = malloc(sizeof(int32_t) * newsize);
                for (uint64_t t = 0; t < newsize; t++) nt[t] = -1;
                for (uint64_t t = 0; t <= s->mask; t++)
                    if (s->table[t] >= 0) po_pyset_insert_clean(nt, newsize - 1, s->hashes[s->table[t]], s->table[t]);
                free(s->table);
                s->table = nt;
                s->mask = newsize - 1;
                return;
            }
            if (s->hashes[e] == hash && memcmp(s->keys[e], key, sizeof(uint64_t[6])) == 0) return;
        }
        perturb >>= 5;
        i = (i * 5 + 1 + perturb) & s->mask;
    }
}
/* hash lanes and equality payload given separately (float tuples: lanes = float hashes, payload = value bits) */
static void po_pyset_add_kv(po_pyset *s, const uint64_t lanes[6], const uint64_t key[6]) {
    uint64_t hash = po_tuple_hash6(lanes);
    uint64_t perturb = hash, i = hash & s->mask;
    for (;;) {
        int probes = (i + 9 <= s->mask) ? 9 : 0;
        for (int j = 0; j <= probes; j++) {
            int32_t e = s->table[i + j];
            if (e < 0) {
                if (s->n == s->cap) {
                    s->cap *= 2;
                    s->keys = realloc(s->keys, sizeof(uint64_t[6]) * s->cap);
                    s->hashes = realloc(s->hashes, sizeof(uint64_t) * s->cap);
                }
                memcpy(s->keys[s->n], key, sizeof(uint64_t[6]));
                s->hashes[s->n] = hash;
                s->table[i + j] = s->n++;
                s->fill++;
                if ((uint64_t)s->fill * 5 < s->mask * 3) return;
                /* set_table_resize(so, used*4): smallest power of two > used*4 (used <= 50000) */
                uint64_t minused = (uint64_t)s->n * 4, newsize = 8;
                while (newsize <= minused) newsize <<= 1;
                int32_t *nt = malloc(sizeof(int32_t) * newsize);
                for (uint64_t t = 0; t < newsize; t++) nt[t] = -1;
                for (uint64_t t = 0; t <= s->mask; t++)
                    if (s->table[t] >= 0) po_pyset_insert_clean(nt, newsize - 1, s->hashes[s->table[t]], s->table[t]);
                free(s->table);
                s->table = nt;
                s->mask = newsize - 1;
                return;
            }
            if (s->hashes[e] == hash && memcmp(s->keys[e], key, sizeof(uint64_t[6])) == 0) return;
        }
        perturb >>= 5;
        i = (i * 5 + 1 + perturb) & s->mask;
    }
}
/* iterate in slot order: writes key indices, returns count */
static int po_pyset_order(const po_pyset *s, int *out) {
    int m = 0;
    for (uint64_t t = 0; t <= s->mask; t++)
        if (s->table[t] >= 0) out[m++] = s->table[t];
    return m;
}

/* ---- read-only export of the support graph an env keeps between steps (tests/harness.py "canonical support graph") ----------------
 * Both env types share the field names used here.  Per placed box u, in placement order:
 *   supports  be_box (bottom_edges order) with the contact centres c2d;   loads  up_edges in dict order: the upper box's placement index
 *   (n_boxes = the box whose real placement failed: its entries stay in the dicts and, found under no live box, keep their last value),
 *   the value calculate_new_com reads for the entry (the live stack of the upper box in alias mode, else the stored one), its alias bit;
 *   polygon  bottom_whole_contact_area;   own  thisStack.
 * hdr = {n_boxes, number of up_edges entries, the failed box has entries, its number of supports, its polygon length, alias_mode}.
 * Returns 0, or -1 when a caller array (cap_e edges, cap_p vertices) is too small / an entry's key belongs to no box. */
#define PO_DEFINE_GET_SUPPORT_GRAPH(fname, env_t, max_boxes)                                                                          \
    int fname(env_t *e, int *hdr, int *sup_off, int *sup, double *c2d, int *load_off, int *load_upper, int *load_alias, double *load4, \
              int *poly_off, double *poly2, double *own4, int cap_e, int cap_p) {                                                      \
        int ns = 0, nl = 0, np_ = 0, tail = 0;                                                                                         \
        const Box *fb = e->n_boxes < max_boxes ? &e->boxes[e->n_boxes] : NULL;                                                         \
        for (int u = 0; u < e->n_boxes; u++) {                                                                                         \
            const Box *b = &e->boxes[u];                                                                                               \
            sup_off[u] = ns; load_off[u] = nl; poly_off[u] = np_;                                                                      \
            if (ns + b->n_be > cap_e || nl + b->n_up > cap_e || np_ + b->n_poly > cap_p) return -1;                                    \
            for (int i = 0; i < b->n_be; i++, ns++) { sup[ns] = b->be_box[i]; c2d[2 * ns] = b->be_c2d[i][0]; c2d[2 * ns + 1] = b->be_c2d[i][1]; } \
            for (int i = 0; i < b->n_up; i++, nl++) {                                                                                  \
                const Box *ub = NULL;                                                                                                  \
                int idx = -1;                                                                                                          \
                for (int t = 0; t < e->n_boxes; t++)                                                                                   \
                    if (e->boxes[t].serial == b->up[i].key) { idx = t; ub = &e->boxes[t]; }                                            \
                if (idx < 0 && fb && fb->serial == b->up[i].key) { idx = e->n_boxes; tail = 1; }                                       \
                if (idx < 0) return -1;                                                                                                \
                const Stack *s = (e->alias_mode && b->up[i].alias && ub) ? &ub->thisStack : &b->up[i].s;                               \
                load_upper[nl] = idx; load_alias[nl] = b->up[i].alias;                                                                 \
                load4[4 * nl] = s->c[0]; load4[4 * nl + 1] = s->c[1]; load4[4 * nl + 2] = s->c[2]; load4[4 * nl + 3] = s->m;           \
            }                                                                                                                          \
            for (int i = 0; i < b->n_poly; i++, np_++) { poly2[2 * np_] = b->poly[i][0]; poly2[2 * np_ + 1] = b->poly[i][1]; }         \
            own4[4 * u] = b->thisStack.c[0]; own4[4 * u + 1] = b->thisStack.c[1]; own4[4 * u + 2] = b->thisStack.c[2]; own4[4 * u + 3] = b->thisStack.m; \
        }                                                                                                                              \
        sup_off[e->n_boxes] = ns; load_off[e->n_boxes] = nl; poly_off[e->n_boxes] = np_;                                               \
        hdr[0] = e->n_boxes; hdr[1] = nl; hdr[2] = tail; hdr[3] = tail ? fb->n_be : 0; hdr[4] = tail ? fb->n_poly : 0; hdr[5] = e->alias_mode; \
        return 0;                                                                                                                      \
    }

#endif
