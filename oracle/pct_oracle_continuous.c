/* TEST INFRASTRUCTURE — single-environment CPU restatement of the reference's CONTINUOUS PCT env.
 * Follows pct_envs/PctContinuous0/{bin3D.py,space.py,convex_hull.py} ("C:" below) of
 * alexfrom0815/Online-3D-BPP-PCT @ 5e088f2; same object structure as pct_oracle_discrete.c, float64 geometry with the
 * reference's 1e-6 tolerances and 6-decimal roundings.
 * Parity contract: actions are FLOAT64 leaf rows (rows of the float64 observation the reference env itself returns).
 * The float32 rows that VecPyTorch hands the reference (envs.py:168-180, train_tools.py:67) make the reference mix numpy
 * float32 / float64 scalars under NEP 50; that type-dependent arithmetic is NOT restated — float32 rows are widened to
 * float64 (DESIGN.md section 9).  sample_from_distribution draws come from the caller's stream (same values both sides).
 * Pinned by tests/golden/continuous_*.npz and, when /root/reference is mounted, live lock-step tests.
 */
#include "pct_oracle_common.h"
#include <stdio.h>

typedef struct { double c[3]; double m; } Stack;
typedef struct { int key; Stack s; int alias; } EdgeEnt; /* alias: the value IS the upper box's live Stack object */

typedef struct Box {
    int serial;
    double x, y, z, lx, ly, lz;
    double centre[3], mass; /* C:space.py:31,34 */
    int n_be;
    int be_box[PO_MAX_SUP];
    double be_area[PO_MAX_SUP][4];
    double be_c2d[PO_MAX_SUP][2];
    int n_poly;
    double poly[2 * PO_MAX_PTS][2];
    int n_up;
    EdgeEnt up[PO_MAX_UP];
    int n_vup;
    EdgeEnt vup[PO_MAX_UP];
    Stack thisStack, thisVStack;
    int involved;
} Box;

#define PC_MAX_BOXES 128
#define PC_MAX_EMS 1000 /* C:space.py:276 */
#define PC_MAX_CAND 8192

typedef struct pctc_env {
    int setting, nb_holder, nl_holder;
    double W, L, H, height;
    double low_bound;
    int n_boxes;
    Box *boxes;
    Box *vbox;
    Box *rbox;     /* the box a real drop_box is checking (not yet in boxes[0..n_boxes)) */
    int next_serial;
    double (*up_letter)[5]; /* C:space.py:273  [-lx,-ly,lx+x,ly+y,top] */
    int n_ems;
    double (*ems)[6];
    double *box_vec;
    const double *stream; int stream_len, stream_pos; int have_item;
    int alias_mode; /* 1: up_edges values that are the upper box's own Stack object are read live (pctc_set_alias_mode) */
    int traj_len; /* > 0: LoadBoxCreator.reset discipline, every reset jumps to the next trajectory boundary (C:binCreator.py:51-62) */
    int shuffle_on; uint64_t shuf_seed, shuf_gid; /* keyed candidate shuffle (pctc_set_shuffle), same definition as the discrete oracle */
    int use_rng; uint64_t rng_seed, rng_gid; double rng_lo, rng_hi; /* sample_from_distribution draws (C:bin3D.py:103-115), counter-based */
    double cur_item[4];
    double next_box[3];
    double next_den;
    int error, n_lstsq;
    int last_ncand;
    int last_ntmp; /* length of the last GENEMS intermediate list (survivors + children, before EliminateInscribedEMS) */
    double last_cand[PC_MAX_CAND][6];
    int last_feas[PC_MAX_CAND];
    int n_packed;
    double packed[PC_MAX_BOXES][7];
} pctc_env;

static double around6(double v) { return rint(v * 1e6) / 1e6; } /* np.around(v, 6) / round(np.float64, 6) */

static Box *box_by_serial(pctc_env *e, int serial) {
    if (e->vbox && e->vbox->serial == serial) return e->vbox;
    if (e->rbox && e->rbox->serial == serial) return e->rbox;
    for (int i = 0; i < e->n_boxes; i++)
        if (e->boxes[i].serial == serial) return &e->boxes[i];
    return NULL;
}
static int serial_involved(pctc_env *e, int serial) { Box *b = box_by_serial(e, serial); return b ? b->involved : 0; }

/* C:space.py:22-44 */
static void box_init(pctc_env *e, Box *b, double x, double y, double z, double lx, double ly, double lz, double density) {
    b->serial = e->next_serial++;
    b->x = x; b->y = y; b->z = z; b->lx = lx; b->ly = ly; b->lz = lz;
    b->centre[0] = lx + x / 2; b->centre[1] = ly + y / 2; b->centre[2] = lz + z / 2;
    b->mass = x * y * z * density;
    b->n_be = 0; b->n_poly = 0; b->n_up = 0; b->n_vup = 0;
    memcpy(b->thisStack.c, b->centre, sizeof b->centre); b->thisStack.m = b->mass;
    b->thisVStack = b->thisStack;
    b->involved = 0;
}

static void dict_set(EdgeEnt *d, int *n, int key, const Stack *s, int alias, int *err) {
    for (int i = 0; i < *n; i++)
        if (d[i].key == key) { d[i].s = *s; d[i].alias = alias; return; }
    if (*n >= PO_MAX_UP) { *err = 3; return; }
    d[*n].key = key; d[*n].s = *s; d[*n].alias = alias; (*n)++;
}
static void dict_pop(EdgeEnt *d, int *n, int key) {
    for (int i = 0; i < *n; i++)
        if (d[i].key == key) {
            memmove(&d[i], &d[i + 1], sizeof(EdgeEnt) * (*n - i - 1));
            (*n)--;
            return;
        }
}

/* C:space.py:47-67 calculate_new_com */
static void calculate_new_com(pctc_env *e, Box *b, int virt) {
    double c[3] = {b->centre[0] * b->mass, b->centre[1] * b->mass, b->centre[2] * b->mass};
    double m = b->mass;
    for (int i = 0; i < b->n_up; i++)
        if (!serial_involved(e, b->up[i].key)) {
            const Box *ub = (e->alias_mode && b->up[i].alias) ? box_by_serial(e, b->up[i].key) : NULL;
            const Stack *s = ub ? &ub->thisStack : &b->up[i].s; /* a box that was never added (its real check failed) keeps its last value */
            c[0] += s->c[0] * s->m; c[1] += s->c[1] * s->m; c[2] += s->c[2] * s->m;
            m += s->m;
        }
    for (int i = 0; i < b->n_vup; i++)
        if (serial_involved(e, b->vup[i].key)) {
            const Box *vb_ = (e->alias_mode && b->vup[i].alias) ? box_by_serial(e, b->vup[i].key) : NULL;
            const Stack *s = vb_ ? &vb_->thisVStack : &b->vup[i].s;
            c[0] += s->c[0] * s->m; c[1] += s->c[1] * s->m; c[2] += s->c[2] * s->m;
            m += s->m;
        }
    c[0] /= m; c[1] /= m; c[2] /= m;
    Stack *dst = virt ? &b->thisVStack : &b->thisStack;
    dst->c[0] = c[0]; dst->c[1] = c[1]; dst->c[2] = c[2]; dst->m = m;
}

/* C:space.py:69-160 (virt=0) and :162-263 (virt=1) */
static int calculated_impact(pctc_env *e, Box *b, int virt, int first) {
    if (virt) b->involved = 1;
    if (b->n_be == 0) { if (virt) b->involved = 0; return 1; }
    Stack *st = virt ? &b->thisVStack : &b->thisStack;
    if (!po_point_in_polygon(st->c[0], st->c[1], (const double (*)[2])b->poly, b->n_poly)) {
        if (virt) b->involved = 0;
        return 0;
    }
#define SUP(i) (&e->boxes[b->be_box[i]])
/* alias = 1: the reference stores the Stack OBJECT of the upper box (`up_edges[self] = self.thisStack`, space.py:82-83,98 / :179-180,195), whose
 * fields calculate_new_com later rewrites in place — a support that recomputes its centre of mass before that box's own calculated_impact
 * ran already sees the new load; alias = 0: a fresh Stack(...) object, i.e. a snapshot (:100,:121-122,:153 ...) */
#define SET_EDGE(i, stk, alias_) do { Box *s_ = SUP(i); if (virt) dict_set(s_->vup, &s_->n_vup, b->serial, (stk), (alias_), &e->error); \
                              else dict_set(s_->up, &s_->n_up, b->serial, (stk), (alias_), &e->error); \
                              calculate_new_com(e, s_, virt); } while (0)
    int k = b->n_be;
    if (k == 1) {
        SET_EDGE(0, st, 1);
        if (!calculated_impact(e, SUP(0), virt, 0)) { if (virt) b->involved = 0; return 0; }
    } else {
        int direct = -1;
        for (int i = 0; i < k; i++) {
            const double *a = b->be_area[i];
            if (st->c[0] - a[0] > 1e-6 && a[2] - st->c[0] > 1e-6 && st->c[1] - a[1] > 1e-6 && a[3] - st->c[1] > 1e-6) { direct = i; break; } /* C:space.py:85-86,182-183 */
        }
        if (direct >= 0) {
            for (int i = 0; i < k; i++) {
                if (i == direct) SET_EDGE(i, st, 1);
                else {
                    Stack z; /* real: Stack(thisStack.centre, 0) :100 ; virtual: Stack(self.centre, 0) :197 */
                    memcpy(z.c, virt ? b->centre : st->c, sizeof z.c);
                    z.m = 0;
                    SET_EDGE(i, &z, 0);
                }
            }
            for (int i = 0; i < k; i++)
                if (!calculated_impact(e, SUP(i), virt, 0)) { if (virt) b->involved = 0; return 0; }
        } else if (k == 2) {
            double line[2] = {b->be_c2d[0][0] - b->be_c2d[1][0], b->be_c2d[0][1] - b->be_c2d[1][1]};
            double len = po_norm2(line);
            double len2 = len * len; /* tri_base_len ** 2 */
            line[0] /= len2; line[1] /= len2;
            double d1[2] = {st->c[0] - b->be_c2d[1][0], st->c[1] - b->be_c2d[1][1]};
            double d0[2] = {st->c[0] - b->be_c2d[0][0], st->c[1] - b->be_c2d[0][1]};
            double ratio0 = fabs(po_dot2(d1, line));
            double ratio1 = fabs(po_dot2(d0, line));
            Stack s0 = {{b->be_c2d[0][0], b->be_c2d[0][1], st->c[2]}, st->m * ratio0};
            Stack s1 = {{b->be_c2d[1][0], b->be_c2d[1][1], st->c[2]}, st->m * ratio1};
            SET_EDGE(0, &s0, 0);
            SET_EDGE(1, &s1, 0);
            if (!calculated_impact(e, SUP(0), virt, 0)) { if (virt) b->involved = 0; return 0; }
            if (!calculated_impact(e, SUP(1), virt, 0)) { if (virt) b->involved = 0; return 0; }
        } else {
            e->n_lstsq++;
            po_ls ls;
            po_ls_init(&ls, k);
            double row[PO_MAX_SUP];
            for (int i = 0; i < k - 1; i++)
                for (int j = i + 1; j < k; j++) {
                    for (int t = 0; t < k; t++) row[t] = 0;
                    double line[2] = {b->be_c2d[i][0] - b->be_c2d[j][0], b->be_c2d[i][1] - b->be_c2d[j][1]};
                    double di[2] = {st->c[0] - b->be_c2d[i][0], st->c[1] - b->be_c2d[i][1]};
                    double molecular = po_dot2(di, line);
                    if (molecular != 0) {
                        double dj[2] = {st->c[0] - b->be_c2d[j][0], st->c[1] - b->be_c2d[j][1]};
                        double r = fabs(po_dot2(dj, line)) / molecular;
                        row[i] = 1;
                        row[j] = -r;
                    }
                    po_ls_add_row(&ls, row, 0.0);
                }
            for (int t = 0; t < k; t++) row[t] = 1;
            po_ls_add_row(&ls, row, 1.0);
            double ratio[PO_MAX_SUP];
            po_ls_solve(&ls, ratio);
            for (int i = 0; i < k; i++) {
                Stack s = {{b->be_c2d[i][0], b->be_c2d[i][1], st->c[2]}, st->m * ratio[i]};
                SET_EDGE(i, &s, 0);
            }
            for (int i = 0; i < k; i++)
                if (!calculated_impact(e, SUP(i), virt, 0)) { if (virt) b->involved = 0; return 0; }
        }
    }
    if (virt) {
        if (first)
            for (int i = 0; i < k; i++) { Box *s_ = SUP(i); dict_pop(s_->vup, &s_->n_vup, b->serial); }
        b->involved = 0;
    }
    return 1;
#undef SUP
#undef SET_EDGE
}


/* C:space.py:305-314 interSect2D: max top over the boxes whose (6-decimal rounded) footprint intersection is positive */
static double intersect2d(pctc_env *e, const double bi[5], int *idx, double (*area)[5], int *n_out) {
    int n = 0;
    double mh = 0;
    for (int i = 0; i < e->n_boxes; i++) {
        double it[5];
        for (int t = 0; t < 5; t++) it[t] = around6(fmin(bi[t], e->up_letter[i][t]));
        if ((it[0] + it[2] > 0) && (it[1] + it[3] > 0)) {
            if (n == 0 || e->up_letter[i][4] > mh) mh = e->up_letter[i][4];
            idx[n] = i; memcpy(area[n], it, sizeof it); n++;
        }
    }
    *n_out = n;
    return n ? mh : 0;
}

/* C:space.py:348-367 / 401-420 */
static void build_bottom(pctc_env *e, Box *b, double max_h, const int *idx, double (*area)[5], int n) {
    double pts[PO_MAX_PTS][2];
    int np_ = 0;
    for (int k = 0; k < n; k++) {
        Box *tmp = &e->boxes[idx[k]];
        if (!(fabs(tmp->lz + tmp->z - max_h) < 1e-6)) continue;
        if (b->n_be >= PO_MAX_SUP) { e->error = 3; return; }
        double x1 = -area[k][0], y1 = -area[k][1], x2 = area[k][2], y2 = area[k][3];
        int i = b->n_be++;
        b->be_box[i] = idx[k];
        b->be_area[i][0] = x1; b->be_area[i][1] = y1; b->be_area[i][2] = x2; b->be_area[i][3] = y2;
        b->be_c2d[i][0] = (x1 + x2) / 2; b->be_c2d[i][1] = (y1 + y2) / 2;
        pts[np_][0] = x1; pts[np_][1] = y1; np_++;
        pts[np_][0] = x1; pts[np_][1] = y2; np_++;
        pts[np_][0] = x2; pts[np_][1] = y1; np_++;
        pts[np_][0] = x2; pts[np_][1] = y2; np_++;
    }
    if (np_ > 0) {
        b->n_poly = po_convex_hull((const double (*)[2])pts, np_, b->poly);
        po_scale_down(b->poly, b->n_poly);
    }
}

/* C:space.py:428-439 */
static int check_box(pctc_env *e, double max_h, Box *b, int virt) {
    if (e->setting == 2) return 1;
    if (fabs(max_h) < 1e-6) return 1;
    return calculated_impact(e, b, virt, virt ? 1 : 0);
}

/* C:space.py:380-425 */
static int drop_box_virtual(pctc_env *e, double x, double y, double z, double lx, double ly, double density) {
    static __thread Box vb;
    static __thread int idx[PC_MAX_BOXES];
    static __thread double area[PC_MAX_BOXES][5];
    int check = 1, n;
    if (lx + x - 1e-6 > e->W || ly + y - 1e-6 > e->L) check = 0;
    if (lx + 1e-6 < 0 || ly + 1e-6 < 0) check = 0;
    double bi[5] = {-lx, -ly, lx + x, ly + y, 0};
    double max_h = intersect2d(e, bi, idx, area, &n);
    if (max_h + z - 1e-6 > e->height) check = 0;
    box_init(e, &vb, x, y, z, lx, ly, max_h, density);
    e->vbox = &vb;
    if (e->setting != 2 && check) build_bottom(e, &vb, max_h, idx, area, n);
    int ok = check && check_box(e, max_h, &vb, 1);
    e->vbox = NULL;
    for (int i = 0; i < vb.n_be; i++) { Box *s = &e->boxes[vb.be_box[i]]; dict_pop(s->vup, &s->n_vup, vb.serial); }
    return ok;
}

/* C:space.py:329-376 */
static int drop_box(pctc_env *e, double x, double y, double z, double lx, double ly, double density) {
    static __thread int idx[PC_MAX_BOXES];
    static __thread double area[PC_MAX_BOXES][5];
    int n;
    if (lx + x - 1e-6 > e->W || ly + y - 1e-6 > e->L) return 0;
    if (lx + 1e-6 < 0 || ly + 1e-6 < 0) return 0;
    double bi[5] = {-lx, -ly, lx + x, ly + y, 0};
    double max_h = intersect2d(e, bi, idx, area, &n);
    if (max_h + z - 1e-6 > e->height) return 0;
    bi[4] = max_h + z;
    if (e->n_boxes >= PC_MAX_BOXES - 1) { e->error = 1; return 0; }
    Box *b = &e->boxes[e->n_boxes];
    box_init(e, b, x, y, z, lx, ly, max_h, density);
    if (e->setting != 2) build_bottom(e, b, max_h, idx, area, n);
    e->rbox = b;
    const int stable = check_box(e, max_h, b, 0);
    e->rbox = NULL;
    if (!stable) return 0;
    if (e->n_boxes >= e->nb_holder) { e->error = 1; return 0; }
    memcpy(e->up_letter[e->n_boxes], bi, sizeof bi);
    double *r = &e->box_vec[e->n_boxes * 9];
    r[0] = lx; r[1] = ly; r[2] = max_h; r[3] = lx + x; r[4] = ly + y; r[5] = max_h + z; r[6] = 0; r[7] = 0; r[8] = 1; /* :372-373 */
    e->n_boxes++;
    return 1;
}

/* C:space.py:17-20 */
static int usable(double lb, double x1, double y1, double z1, double x2, double y2, double z2) {
    return (x2 - x1 + 1e-6 >= lb) && (y2 - y1 + 1e-6 >= lb) && (z2 - z1 + 1e-6 >= lb);
}
static void add_ems(pctc_env *e, double a, double b, double c, double x, double y, double z) {
    if (e->n_ems >= PC_MAX_EMS) { e->error = 3; return; }
    double *r = e->ems[e->n_ems++];
    r[0] = a; r[1] = b; r[2] = c; r[3] = x; r[4] = y; r[5] = z;
}

/* C:space.py:441-487 (+ Difference :490-502, EliminateInscribedEMS :508-528) */
static void genems(pctc_env *e, const double loc[6]) {
    int n0 = e->n_ems;
    char *del = calloc(n0 + 1, 1);
    int anydel = 0;
    double itn[6] = {-loc[0], -loc[1], -loc[2], loc[3], loc[4], loc[5]};
    for (int i = 0; i < n0; i++) {
        double *m = e->ems[i];
        double mn[6] = {-m[0], -m[1], -m[2], m[3], m[4], m[5]}, it[6];
        for (int t = 0; t < 6; t++) it[t] = around6(fmin(itn[t], mn[t]));
        if (!((it[0] + it[3] > 0) && (it[1] + it[4] > 0) && (it[2] + it[5] > 0))) continue;
        double x3 = -it[0], y3 = -it[1], x4 = it[3], y4 = it[4], z4 = it[5];
        (void)y3;
        double x1 = m[0], y1 = m[1], z1 = m[2], x2 = m[3], y2 = m[4], z2 = m[5], lb = e->low_bound;
        if (usable(lb, x1, y1, z1, x3, y2, z2)) add_ems(e, x1, y1, z1, x3, y2, z2);
        if (usable(lb, x4, y1, z1, x2, y2, z2)) add_ems(e, x4, y1, z1, x2, y2, z2);
        if (usable(lb, x1, y1, z1, x2, -it[1], z2)) add_ems(e, x1, y1, z1, x2, -it[1], z2);
        if (usable(lb, x1, y4, z1, x2, y2, z2)) add_ems(e, x1, y4, z1, x2, y2, z2);
        if (usable(lb, x1, y1, z4, x2, y2, z2)) add_ems(e, x1, y1, z4, x2, y2, z2);
        del[i] = 1; anydel = 1;
    }
    if (anydel) {
        int w = 0;
        for (int i = 0; i < e->n_ems; i++)
            if (i >= n0 || !del[i]) { if (w != i) memcpy(e->ems[w], e->ems[i], sizeof(double[6])); w++; }
        e->n_ems = w;
    }
    free(del);
    e->last_ntmp = e->n_ems;
    int n = e->n_ems;
    char *df = calloc(n + 1, 1);
    for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++) {
            if (i == j) continue;
            double *a = e->ems[i], *b = e->ems[j];
            if (a[0] >= b[0] && a[1] >= b[1] && a[2] >= b[2] && a[3] <= b[3] && a[4] <= b[4] && a[5] <= b[5]) { df[i] = 1; break; }
        }
    int w = 0;
    for (int i = 0; i < n; i++)
        if (!df[i]) { if (w != i) memcpy(e->ems[w], e->ems[i], sizeof(double[6])); w++; }
    e->n_ems = w;
    free(df);
}

/* C:space.py:531-568 — candidates in CPython-set order (set of float 6-tuples: hash = tuple hash of float hashes,
 * equality = float equality) */
static int ems_point(pctc_env *e, const double nb[3], double (*out)[6], int cap) {
    po_pyset set;
    po_pyset_init(&set);
    int vcap = 256, nv = 0;
    double (*vals)[6] = malloc(sizeof(double[6]) * vcap);
    int R = e->setting == 2 ? 6 : 2;
    for (int i = 0; i < e->n_ems; i++) {
        const double *m = e->ems[i];
        for (int rot = 0; rot < R; rot++) {
            double sx, sy, sz;
            switch (rot) {
            case 0: sx = nb[0]; sy = nb[1]; sz = nb[2]; break;
            case 1: sx = nb[1]; sy = nb[0]; sz = nb[2]; if (fabs(sx - sy) < 1e-6) continue; break;
            case 2: sx = nb[0]; sy = nb[2]; sz = nb[1]; if (fabs(sx - sy) < 1e-6 && fabs(sy - sz) < 1e-6) continue; break;
            case 3: sx = nb[1]; sy = nb[2]; sz = nb[0]; if (fabs(sx - sy) < 1e-6 && fabs(sy - sz) < 1e-6) continue; break;
            case 4: sx = nb[2]; sy = nb[0]; sz = nb[1]; if (fabs(sx - sy) < 1e-6) continue; break;
            default: sx = nb[2]; sy = nb[1]; sz = nb[0]; if (fabs(sx - sy) < 1e-6) continue; break;
            }
            if (m[3] - m[0] + 1e-6 >= sx && m[4] - m[1] + 1e-6 >= sy && m[5] - m[2] + 1e-6 >= sz) {
                double c[4][6] = {
                    {m[0], m[1], m[2], m[0] + sx, m[1] + sy, m[2] + sz},
                    {m[3] - sx, m[1], m[2], m[3], m[1] + sy, m[2] + sz},
                    {m[0], m[4] - sy, m[2], m[0] + sx, m[4], m[2] + sz},
                    {m[3] - sx, m[4] - sy, m[2], m[3], m[4], m[2] + sz}};
                for (int q = 0; q < 4; q++) {
                    uint64_t key[6];
                    for (int t = 0; t < 6; t++) {
                        double v = c[q][t] == 0 ? 0.0 : c[q][t]; /* -0.0 == 0.0 and hash(-0.0) == hash(0.0) */
                        memcpy(&key[t], &v, 8);                   /* equal floats <=> equal bits once zeros are canonical */
                    }
                    /* po_pyset hashes the lanes it is given: feed float hashes, compare by value bits */
                    uint64_t lanes[6];
                    for (int t = 0; t < 6; t++) lanes[t] = po_hash_double(c[q][t]);
                    int before = set.n;
                    po_pyset_add_kv(&set, lanes, key);
                    if (set.n != before) {
                        if (nv == vcap) { vcap *= 2; vals = realloc(vals, sizeof(double[6]) * vcap); }
                        memcpy(vals[nv++], c[q], sizeof(double[6]));
                    }
                }
            }
        }
    }
    int *order = malloc(sizeof(int) * (set.n + 1));
    int n = po_pyset_order(&set, order);
    if (n > cap) { e->error = 3; n = cap; }
    for (int i = 0; i < n; i++) memcpy(out[i], vals[order[i]], sizeof(double[6]));
    free(order); free(vals);
    po_pyset_free(&set);
    return n;
}

uint64_t pcto_rnd_u64(uint64_t seed, uint64_t a, uint64_t b);
static double rng_u01(const pctc_env *e, uint64_t salt, uint64_t d) { return (double)(pcto_rnd_u64(e->rng_seed ^ salt, e->rng_gid, d) >> 11) * (1.0 / 9007199254740992.0); }
static double round3(double v) { return rint(v * 1000.0) / 1000.0; }
static void creator_generate(pctc_env *e) {
    if (e->use_rng) { /* the same counter-based draws as the device generator (csrc/pct_continuous.cu draw_item_c) and make_continuous_stream */
        const uint64_t d = (uint64_t)e->stream_pos;
        const double lo = e->rng_lo, span = e->rng_hi - e->rng_lo;
        e->cur_item[0] = round3(lo + span * rng_u01(e, 0x11, d));
        e->cur_item[1] = round3(lo + span * rng_u01(e, 0x22, d));
        if (e->setting == 2) e->cur_item[2] = round3(lo + span * rng_u01(e, 0x33, d));
        else { static const double ch[5] = {0.1, 0.2, 0.3, 0.4, 0.5}; e->cur_item[2] = ch[pcto_rnd_u64(e->rng_seed ^ 0x44, e->rng_gid, d) % 5]; }
        uint64_t r = pcto_rnd_u64(e->rng_seed ^ 0xABCDEFULL, e->rng_gid, d) >> 11;
        if (r == 0) r = 1;
        e->cur_item[3] = (double)r * (1.0 / 9007199254740992.0);
        e->stream_pos++;
        e->have_item = 1;
        return;
    }
    const double *it = &e->stream[4 * (e->stream_pos % e->stream_len)];
    e->stream_pos++;
    memcpy(e->cur_item, it, sizeof e->cur_item);
    e->have_item = 1;
}

/* C:bin3D.py:78-100 + :118-148 */
static void cur_observation(pctc_env *e, double *obs) {
    if (!e->have_item) creator_generate(e);
    for (int i = 0; i < 3; i++) e->next_box[i] = e->cur_item[i];
    e->next_den = e->setting == 3 ? e->cur_item[3] : 1.0;
    int nbh = e->nb_holder, nlh = e->nl_holder;
    memcpy(obs, e->box_vec, sizeof(double) * 9 * nbh);
    double *leaf = obs + 9 * nbh;
    memset(leaf, 0, sizeof(double) * 9 * nlh);
    int nc = ems_point(e, e->next_box, e->last_cand, PC_MAX_CAND);
    if (e->shuffle_on && nc > 1) { /* C:bin3D.py:126-127; keyed permutation, see pct_oracle_discrete.c cur_observation */
        static __thread uint64_t keys[PC_MAX_CAND];
        static __thread int perm[PC_MAX_CAND];
        static __thread double tmpc[PC_MAX_CAND][6];
        for (int i = 0; i < nc; i++) { keys[i] = pcto_rnd_u64(e->shuf_seed ^ 0x5AFE5EEDULL, e->shuf_gid, ((uint64_t)e->stream_pos << 16) | (uint64_t)i); perm[i] = i; }
        for (int i = 1; i < nc; i++) {
            int v = perm[i], j = i - 1;
            while (j >= 0 && keys[perm[j]] > keys[v]) { perm[j + 1] = perm[j]; j--; }
            perm[j + 1] = v;
        }
        for (int i = 0; i < nc; i++) memcpy(tmpc[i], e->last_cand[perm[i]], sizeof(double[6]));
        memcpy(e->last_cand, tmpc, sizeof(double[6]) * nc);
    }
    e->last_ncand = nc;
    int nleaf = 0;
    for (int i = 0; i < nc; i++) e->last_feas[i] = -1;
    for (int i = 0; i < nc; i++) {
        double *p = e->last_cand[i];
        double x = p[3] - p[0], y = p[4] - p[1], z = p[5] - p[2];
        int ok = drop_box_virtual(e, x, y, z, p[0], p[1], e->next_den);
        e->last_feas[i] = ok;
        if (ok) {
            double *r = leaf + 9 * nleaf;
            r[0] = p[0]; r[1] = p[1]; r[2] = p[2]; r[3] = p[3]; r[4] = p[4]; r[5] = e->H; r[6] = 0; r[7] = 0; r[8] = 1;
            nleaf++;
        }
        if (nleaf >= nlh) break;
    }
    double *nx = leaf + 9 * nlh;
    double s[3] = {e->next_box[0], e->next_box[1], e->next_box[2]};
    for (int i = 0; i < 3; i++)
        for (int j = i + 1; j < 3; j++)
            if (s[j] < s[i]) { double t = s[i]; s[i] = s[j]; s[j] = t; }
    memset(nx, 0, sizeof(double) * 9);
    nx[0] = e->next_den; nx[3] = s[0]; nx[4] = s[1]; nx[5] = s[2]; nx[8] = 1;
}

pctc_env *pctc_create(int setting, double W, double L, double H, int nb_holder, int nl_holder, double low_bound) {
    pctc_env *e = calloc(1, sizeof(pctc_env));
    { const char *am = getenv("PCT_ORACLE_ALIAS"); e->alias_mode = am ? atoi(am) != 0 : 1; } /* default ON = the reference's object semantics (DESIGN.md section 3 (b)); PCT_ORACLE_ALIAS=0: snapshot semantics */
    e->setting = setting; e->W = W; e->L = L; e->H = H; e->height = H;
    e->nb_holder = nb_holder; e->nl_holder = nl_holder; e->low_bound = low_bound;
    e->boxes = calloc(PC_MAX_BOXES, sizeof(Box));
    e->up_letter = calloc(PC_MAX_BOXES, sizeof(double[5]));
    e->ems = calloc(PC_MAX_EMS, sizeof(double[6]));
    e->box_vec = calloc((size_t)nb_holder * 9, sizeof(double));
    return e;
}
void pctc_destroy(pctc_env *e) { free(e->boxes); free(e->up_letter); free(e->ems); free(e->box_vec); free(e); }
void pctc_set_stream(pctc_env *e, const double *items4, int n) { e->stream = items4; e->stream_len = n; e->stream_pos = 0; }
void pctc_set_random_sample(pctc_env *e, uint64_t seed, uint64_t gid, double lo, double hi) {
    e->use_rng = 1; e->rng_seed = seed; e->rng_gid = gid; e->rng_lo = lo; e->rng_hi = hi; e->stream_pos = 0;
}
int pctc_obs_len(pctc_env *e) { return (e->nb_holder + e->nl_holder + 1) * 9; }

/* C:bin3D.py:69-75 + C:space.py:281-303 */
void pctc_set_trajectory_length(pctc_env *e, int n) { e->traj_len = n; }
void pctc_set_alias_mode(pctc_env *e, int on) { e->alias_mode = on; }
void pctc_set_shuffle(pctc_env *e, int on, uint64_t seed, uint64_t gid) { e->shuffle_on = on; e->shuf_seed = seed; e->shuf_gid = gid; }
void pctc_reset(pctc_env *e, double *obs) {
    e->have_item = 0;
    if (e->traj_len > 0 && e->stream_pos % e->traj_len) e->stream_pos += e->traj_len - e->stream_pos % e->traj_len;
    e->n_packed = 0;
    memset(e->box_vec, 0, sizeof(double) * 9 * e->nb_holder);
    e->box_vec[8] = 1;
    e->n_ems = 1;
    e->ems[0][0] = e->ems[0][1] = e->ems[0][2] = 0; e->ems[0][3] = e->W; e->ems[0][4] = e->L; e->ems[0][5] = e->H;
    e->n_boxes = 0;
    e->error = 0;
    e->last_ntmp = 0;
    creator_generate(e);
    cur_observation(e, obs);
}
/* `env.next_box = item` and a fresh observation (heuristic.py assigns next_box and reads the env again): item4 becomes the current item on
 * the current state; no draw is consumed */
void pctc_set_next(pctc_env *e, const double *item4, double *obs) {
    memcpy(e->cur_item, item4, sizeof e->cur_item);
    e->have_item = 1;
    cur_observation(e, obs);
}

/* C:bin3D.py:151-207 */
int pctc_step(pctc_env *e, const double *action, int action_len, double *obs, double *reward, int *done, double *info) {
    double lx, ly, x, y, z;
    int rot = 0;
    const double *nb = e->next_box;
    if (action_len != 3) { /* LeafNode2Action :151-167 */
        double s = 0;
        for (int i = 0; i < 6; i++) s += action[i];
        if (s == 0) { lx = 0; ly = 0; x = nb[0]; y = nb[1]; z = nb[2]; }
        else {
            x = around6(action[3] - action[0]);
            y = around6(action[4] - action[1]);
            int rec[3] = {0, 1, 2}, n = 3;
            for (int i = 0; i < n; i++) if (fabs(x - nb[rec[i]]) < 1e-6) { memmove(&rec[i], &rec[i + 1], sizeof(int) * (n - i - 1)); n--; break; }
            for (int i = 0; i < n; i++) if (fabs(y - nb[rec[i]]) < 1e-6) { memmove(&rec[i], &rec[i + 1], sizeof(int) * (n - i - 1)); n--; break; }
            z = nb[rec[0]];
            lx = action[0]; ly = action[1];
        }
    } else {
        rot = (int)action[0]; lx = action[1]; ly = action[2];
        x = nb[0]; y = nb[1]; z = nb[2];
    }
    lx = around6(lx); ly = around6(ly); /* :173 */
    if (rot) { double t = x; x = y; y = t; }
    int ok = drop_box(e, x, y, z, lx, ly, e->next_den);
    double vol = 0; /* get_ratio :316-321 */
    for (int i = 0; i < e->n_boxes; i++) vol += e->boxes[i].x * e->boxes[i].y * e->boxes[i].z;
    double ratio = vol / (e->W * e->L * e->H);
    info[0] = e->n_boxes; info[1] = ratio; info[2] = ratio * 10;
    if (!ok) {
        *reward = 0.0; *done = 1;
        cur_observation(e, obs);
        return e->error;
    }
    Box *pb = &e->boxes[e->n_boxes - 1];
    double loc[6] = {pb->lx, pb->ly, pb->lz, around6(pb->lx + pb->x), around6(pb->ly + pb->y), around6(pb->lz + pb->z)};
    genems(e, loc);
    double *pk = e->packed[e->n_packed++];
    pk[0] = pb->x; pk[1] = pb->y; pk[2] = pb->z; pk[3] = pb->lx; pk[4] = pb->ly; pk[5] = pb->lz; pk[6] = 0;
    double box_ratio = (nb[0] * nb[1] * nb[2]) / (e->W * e->L * e->H);
    e->have_item = 0;
    creator_generate(e);
    *reward = box_ratio * 10;
    *done = 0;
    cur_observation(e, obs);
    return e->error;
}

int pctc_get_ems(pctc_env *e, double *out, int cap) { int n = e->n_ems < cap ? e->n_ems : cap; memcpy(out, e->ems, sizeof(double[6]) * n); return e->n_ems; }
int pctc_get_candidates(pctc_env *e, double *out6, int *feas, int cap) {
    int n = e->last_ncand < cap ? e->last_ncand : cap;
    memcpy(out6, e->last_cand, sizeof(double[6]) * n);
    memcpy(feas, e->last_feas, sizeof(int) * n);
    return e->last_ncand;
}
int pctc_get_packed(pctc_env *e, double *out7, int cap) { int n = e->n_packed < cap ? e->n_packed : cap; memcpy(out7, e->packed, sizeof(double[7]) * n); return e->n_packed; }
int pctc_n_lstsq(pctc_env *e) { return e->n_lstsq; }
int pctc_n_ems_intermediate(pctc_env *e) { return e->last_ntmp; }
PO_DEFINE_GET_SUPPORT_GRAPH(pctc_get_support_graph, pctc_env, PC_MAX_BOXES)

/* What heuristic.py reads from a PackingContinuous env (heuristic.py:163-166,190-193,387-416,541-567):
 * Space.drop_box_virtual(dims, (lx, ly), False, density, setting, returnH=True) (C:space.py:380-425; max_h is
 * interSect2D's, :391) and env.next_box / env.next_den. */
int pctc_drop_box_virtual(pctc_env *e, double x, double y, double z, double lx, double ly, double density, double *max_h) {
    static __thread int idx[PC_MAX_BOXES];
    static __thread double area[PC_MAX_BOXES][5];
    int n;
    double bi[5] = {-lx, -ly, lx + x, ly + y, 0};
    *max_h = intersect2d(e, bi, idx, area, &n);
    return drop_box_virtual(e, x, y, z, lx, ly, density);
}
void pctc_get_next(pctc_env *e, double *out4) { out4[0] = e->next_box[0]; out4[1] = e->next_box[1]; out4[2] = e->next_box[2]; out4[3] = e->next_den; }

/* debug / soak triage: the persisted stack (centre xyz, mass) of placed box i and its up_edges entries (serial, centre xyz, mass) */
int pctc_get_stack(pctc_env *e, int i, double *out4, double *up5, int cap) {
    if (i < 0 || i >= e->n_boxes) return -1;
    const Box *b = &e->boxes[i];
    out4[0] = b->thisStack.c[0]; out4[1] = b->thisStack.c[1]; out4[2] = b->thisStack.c[2]; out4[3] = b->thisStack.m;
    for (int k = 0; k < b->n_up && k < cap; k++) {
        up5[5 * k] = b->up[k].key; up5[5 * k + 1] = b->up[k].s.c[0]; up5[5 * k + 2] = b->up[k].s.c[1]; up5[5 * k + 3] = b->up[k].s.c[2]; up5[5 * k + 4] = b->up[k].s.m;
    }
    return b->n_up;
}
