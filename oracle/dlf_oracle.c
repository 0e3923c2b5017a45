/*
 * dlf_oracle.c — CPU restatement (plain scalar C) of the SVT-AV1 v0.8.6 deblocking loop filter: the 4/6/8/14-tap
 * edge filters (low and high bit depth), the per-edge parameter derivation and the frame loop.
 *
 * TEST INFRASTRUCTURE ONLY (see me_oracle.c).  Pinned bit-for-bit against svt_aom_[highbd_]lpf_* and
 * svt_av1_loop_filter_frame of the reference compiled into oracle/_ref — tests/test_oracle_dlf.py.
 * Reference paths are relative to /root/reference/Source/Lib.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/svt_av1_b200.h"
#include "oracle.h"

static inline int iabs(int v) { return v < 0 ? -v : v; }
static inline int sclamp(int v, int bd) { /* signed_char_clamp / signed_char_clamp_high */
    const int lo = -(128 << (bd - 8)), hi = (128 << (bd - 8)) - 1;
    return v < lo ? lo : (v > hi ? hi : v);
}

/* One sample position of an edge of nominal length `len` (4, 6, 8 or 14): px[] holds p6..p0 at [0..6] and q0..q6 at
 * [7..13] (only the taps the length needs are read/written).  Common/Codec/EbDeblockingCommon.c:148-924. */
static void lpf_sample(int *px, int len, int blimit, int limit, int thresh, int bd) {
    const int sh = bd - 8;
    int *p = px + 6, *q = px + 7; /* p[-i] = p_i, q[i] = q_i */
#define P(i) p[-(i)]
#define Q(i) q[(i)]
    const int lim = limit << sh, blim = blimit << sh, thr = thresh << sh, one = 1 << sh;
    int mask = iabs(P(1) - P(0)) <= lim && iabs(Q(1) - Q(0)) <= lim && iabs(P(0) - Q(0)) * 2 + iabs(P(1) - Q(1)) / 2 <= blim;
    if (len >= 6) mask = mask && iabs(P(2) - P(1)) <= lim && iabs(Q(2) - Q(1)) <= lim;
    if (len >= 8) mask = mask && iabs(P(3) - P(2)) <= lim && iabs(Q(3) - Q(2)) <= lim;
    int flat = 0, flat2 = 0;
    if (len >= 6) {
        flat = iabs(P(1) - P(0)) <= one && iabs(Q(1) - Q(0)) <= one && iabs(P(2) - P(0)) <= one && iabs(Q(2) - Q(0)) <= one;
        if (len >= 8) flat = flat && iabs(P(3) - P(0)) <= one && iabs(Q(3) - Q(0)) <= one;
    }
    if (len == 14)
        flat2 = iabs(P(4) - P(0)) <= one && iabs(Q(4) - Q(0)) <= one && iabs(P(5) - P(0)) <= one && iabs(Q(5) - Q(0)) <= one &&
            iabs(P(6) - P(0)) <= one && iabs(Q(6) - Q(0)) <= one;
    const int p0 = P(0), p1 = P(1), p2 = P(2), p3 = P(3), p4 = P(4), p5 = P(5), p6 = P(6);
    const int q0 = Q(0), q1 = Q(1), q2 = Q(2), q3 = Q(3), q4 = Q(4), q5 = Q(5), q6 = Q(6);
#define R(v, n) (((v) + (1 << ((n)-1))) >> (n))
    if (len == 14 && flat2 && flat && mask) { /* filter14 :810-842 */
        P(5) = R(p6 * 7 + p5 * 2 + p4 * 2 + p3 + p2 + p1 + p0 + q0, 4);
        P(4) = R(p6 * 5 + p5 * 2 + p4 * 2 + p3 * 2 + p2 + p1 + p0 + q0 + q1, 4);
        P(3) = R(p6 * 4 + p5 + p4 * 2 + p3 * 2 + p2 * 2 + p1 + p0 + q0 + q1 + q2, 4);
        P(2) = R(p6 * 3 + p5 + p4 + p3 * 2 + p2 * 2 + p1 * 2 + p0 + q0 + q1 + q2 + q3, 4);
        P(1) = R(p6 * 2 + p5 + p4 + p3 + p2 * 2 + p1 * 2 + p0 * 2 + q0 + q1 + q2 + q3 + q4, 4);
        P(0) = R(p6 + p5 + p4 + p3 + p2 + p1 * 2 + p0 * 2 + q0 * 2 + q1 + q2 + q3 + q4 + q5, 4);
        Q(0) = R(p5 + p4 + p3 + p2 + p1 + p0 * 2 + q0 * 2 + q1 * 2 + q2 + q3 + q4 + q5 + q6, 4);
        Q(1) = R(p4 + p3 + p2 + p1 + p0 + q0 * 2 + q1 * 2 + q2 * 2 + q3 + q4 + q5 + q6 * 2, 4);
        Q(2) = R(p3 + p2 + p1 + p0 + q0 + q1 * 2 + q2 * 2 + q3 * 2 + q4 + q5 + q6 * 3, 4);
        Q(3) = R(p2 + p1 + p0 + q0 + q1 + q2 * 2 + q3 * 2 + q4 * 2 + q5 + q6 * 4, 4);
        Q(4) = R(p1 + p0 + q0 + q1 + q2 + q3 * 2 + q4 * 2 + q5 * 2 + q6 * 5, 4);
        Q(5) = R(p0 + q0 + q1 + q2 + q3 + q4 * 2 + q5 * 2 + q6 * 7, 4);
        return;
    }
    if (len >= 8 && flat && mask) { /* filter8 :282-299 */
        P(2) = R(p3 + p3 + p3 + 2 * p2 + p1 + p0 + q0, 3);
        P(1) = R(p3 + p3 + p2 + 2 * p1 + p0 + q0 + q1, 3);
        P(0) = R(p3 + p2 + p1 + 2 * p0 + q0 + q1 + q2, 3);
        Q(0) = R(p2 + p1 + p0 + 2 * q0 + q1 + q2 + q3, 3);
        Q(1) = R(p1 + p0 + q0 + 2 * q1 + q2 + q3 + q3, 3);
        Q(2) = R(p0 + q0 + q1 + 2 * q2 + q3 + q3 + q3, 3);
        return;
    }
    if (len == 6 && flat && mask) { /* filter6 :266-280 */
        P(1) = R(p2 * 3 + p1 * 2 + p0 * 2 + q0, 3);
        P(0) = R(p2 + p1 * 2 + p0 * 2 + q0 * 2 + q1, 3);
        Q(0) = R(p1 + p0 * 2 + q0 * 2 + q1 * 2 + q2, 3);
        Q(1) = R(p0 + q0 * 2 + q1 * 2 + q2 * 3, 3);
        return;
    }
    { /* filter4 / highbd_filter4 :222-249, 449-481 */
        const int off = 0x80 << sh;
        const int ps1 = p1 - off, ps0 = p0 - off, qs0 = q0 - off, qs1 = q1 - off;
        const int hev = iabs(p1 - p0) > thr || iabs(q1 - q0) > thr;
        int f = hev ? sclamp(ps1 - qs1, bd) : 0;
        f = mask ? sclamp(f + 3 * (qs0 - ps0), bd) : 0;
        const int f1 = sclamp(f + 4, bd) >> 3, f2 = sclamp(f + 3, bd) >> 3;
        Q(0) = sclamp(qs0 - f1, bd) + off;
        P(0) = sclamp(ps0 + f2, bd) + off;
        const int f3 = hev ? 0 : ((f1 + 1) >> 1);
        Q(1) = sclamp(qs1 - f3, bd) + off;
        P(1) = sclamp(ps1 + f3, bd) + off;
    }
#undef P
#undef Q
#undef R
}

static int taps_of(int len) { return len == 4 ? 2 : len == 6 ? 3 : len == 8 ? 4 : 7; }

/* One 4-sample edge segment. `across`: element step across the edge, `along`: step along it. */
void orc_lpf_edge(void *s, int hbd, int across, int along, int len, int blimit, int limit, int thresh, int bd) {
    const int n = taps_of(len);
    for (int i = 0; i < 4; i++) {
        int px[14];
        memset(px, 0, sizeof(px));
        for (int t = 0; t < n; t++) {
            const ptrdiff_t op = (ptrdiff_t)i * along - (ptrdiff_t)(t + 1) * across, oq = (ptrdiff_t)i * along + (ptrdiff_t)t * across;
            px[6 - t] = hbd ? ((uint16_t *)s)[op] : ((uint8_t *)s)[op];
            px[7 + t] = hbd ? ((uint16_t *)s)[oq] : ((uint8_t *)s)[oq];
        }
        lpf_sample(px, len, blimit, limit, thresh, bd);
        for (int t = 0; t < n; t++) {
            const ptrdiff_t op = (ptrdiff_t)i * along - (ptrdiff_t)(t + 1) * across, oq = (ptrdiff_t)i * along + (ptrdiff_t)t * across;
            if (hbd) {
                ((uint16_t *)s)[op] = (uint16_t)px[6 - t];
                ((uint16_t *)s)[oq] = (uint16_t)px[7 + t];
            } else {
                ((uint8_t *)s)[op] = (uint8_t)px[6 - t];
                ((uint8_t *)s)[oq] = (uint8_t)px[7 + t];
            }
        }
    }
}

/* set_lpf_parameters (Encoder/Codec/EbDeblockingFilter.c:168-319) on the flattened mi summary.
 * Returns the filter length (0 = none) and the level of the edge at plane sample (x, y). */
static int edge_params(const SvtB200DlfParams *p, const SvtB200DlfMi *mi, int plane, int vert, int x, int y, int pw, int ph,
                       int *level) {
    if (x >= pw || y >= ph) return 0;
    const int ss = plane ? 1 : 0, c = plane ? 1 : 0;
    const int mi_row = ss | ((y << ss) >> 2), mi_col = ss | ((x << ss) >> 2);
    const SvtB200DlfMi *cur = mi + (size_t)mi_row * p->mi_stride + mi_col;
    const int ts = vert ? cur->tx_w[c] : cur->tx_h[c];
    const int coord = vert ? x : y;
    if (coord & (ts - 1)) return 0;
    if (!coord) return 0;
    const SvtB200DlfMi *prev = vert ? cur - (1 << ss) : cur - (size_t)(1 << ss) * p->mi_stride;
    const int pv_ts = vert ? prev->tx_w[c] : prev->tx_h[c];
    const int cl = plane == 0 ? cur->lvl_y[vert ? 0 : 1] : plane == 1 ? cur->lvl_u : cur->lvl_v;
    const int pl = plane == 0 ? prev->lvl_y[vert ? 0 : 1] : plane == 1 ? prev->lvl_u : prev->lvl_v;
    const int pu_edge = !(coord & ((vert ? cur->blk_w[c] : cur->blk_h[c]) - 1));
    if (!((cl || pl) && (!prev->skip_inter || !cur->skip_inter || pu_edge))) return 0;
    const int mn = ts < pv_ts ? ts : pv_ts;
    *level = cl ? cl : pl;
    if (mn <= 4) return 4;
    if (mn == 8) return plane ? 6 : 8;
    return plane ? 6 : 14;
}

static void thresholds(int level, int sharpness, int *blimit, int *limit, int *thresh) { /* update_sharpness :587, init :25-39 */
    int lim = level >> ((sharpness > 0) + (sharpness > 4));
    if (sharpness > 0 && lim > 9 - sharpness) lim = 9 - sharpness;
    if (lim < 1) lim = 1;
    *limit = lim;
    *blimit = 2 * (level + 2) + lim;
    *thresh = level >> 4;
}

/* svt_av1_loop_filter_frame (:711-753): the reference walks super-blocks filtering the vertical edges of SB n and
 * then the horizontal edges of SB n-1; no horizontal-edge filter touches a sample a later vertical-edge filter
 * reads and the edges of one direction are mutually independent, so "all vertical, then all horizontal" is the same
 * function (checked against the reference in the tests). */
void orc_dlf_frame(const SvtB200DlfParams *p, const SvtB200Frame *f, const SvtB200DlfMi *mi) {
    const int hbd = f->bit_depth > 8;
    for (int plane = p->plane_start; plane < p->plane_end; plane++) {
        if (plane == 0 && !p->filter_level[0] && !p->filter_level[1]) break;
        if (plane == 1 && !p->filter_level_u) continue;
        if (plane == 2 && !p->filter_level_v) continue;
        void *base = plane == 0 ? f->y : plane == 1 ? f->cb : f->cr;
        const int stride = plane ? f->stride_c : f->stride_y;
        const int pw = plane ? (p->mi_cols * 4) >> 1 : p->mi_cols * 4, ph = plane ? (p->mi_rows * 4) >> 1 : p->mi_rows * 4;
        for (int vert = 1; vert >= 0; vert--)
            for (int y = 0; y < ph; y += 4)
                for (int x = 0; x < pw; x += 4) {
                    int level = 0;
                    const int len = edge_params(p, mi, plane, vert, x, y, pw, ph, &level);
                    if (!len) continue;
                    int bl, l, t;
                    thresholds(level, p->sharpness, &bl, &l, &t);
                    void *s = hbd ? (void *)((uint16_t *)base + (size_t)y * stride + x) : (void *)((uint8_t *)base + (size_t)y * stride + x);
                    orc_lpf_edge(s, hbd, vert ? 1 : stride, vert ? stride : 1, len, bl, l, t, f->bit_depth);
                }
    }
}

void orc_frame_sse(const SvtB200Frame *a, const SvtB200Frame *b, uint64_t *sse) {
    for (int pl = 0; pl < 3; pl++) {
        const int w = pl ? (a->width + 1) >> 1 : a->width, h = pl ? (a->height + 1) >> 1 : a->height;
        const int sa = pl ? a->stride_c : a->stride_y, sb = pl ? b->stride_c : b->stride_y;
        const void *pa = pl == 0 ? a->y : pl == 1 ? a->cb : a->cr, *pb = pl == 0 ? b->y : pl == 1 ? b->cb : b->cr;
        uint64_t s = 0;
        for (int y = 0; y < h; y++)
            for (int x = 0; x < w; x++) {
                const int va = a->bit_depth > 8 ? ((const uint16_t *)pa)[(size_t)y * sa + x] : ((const uint8_t *)pa)[(size_t)y * sa + x];
                const int vb = b->bit_depth > 8 ? ((const uint16_t *)pb)[(size_t)y * sb + x] : ((const uint8_t *)pb)[(size_t)y * sb + x];
                s += (uint64_t)((va - vb) * (va - vb));
            }
        sse[pl] = s;
    }
}

/* ---- svt_av1_loop_filter_frame_init (Common/Codec/EbDeblockingCommon.c:78-145) as a table over the level class
 *      cls = segment_id * 16 + ref_frame[0] * 2 + mode_lf_lut[mode] -------------------------------------------- */
/* plane_start as frame_init's: a call that starts at a chroma plane fills that plane's table even when both luma levels
 * are 0 (the level search's chroma trials, svt_av1_loop_filter_frame(plane, plane + 1)). */
static void level_lut(const SvtB200LfFrameInit *init, const int32_t levels[4], int plane_start, uint8_t lut[3][2][128]) {
    static const int feature[3][2] = {{1, 2}, {3, 3}, {4, 4}}; /* seg_lvl_lf_lut */
    memset(lut, 0, 3 * 2 * 128);
    for (int plane = plane_start; plane < 3; plane++) {
        const int lv[2] = {plane == 0 ? levels[0] : levels[1 + plane], plane == 0 ? levels[1] : levels[1 + plane]};
        if (plane == 0 && !lv[0] && !lv[1]) break;
        if (plane && !lv[0]) continue;
        for (int cls = 0; cls < 128; cls++) {
            const int seg = cls >> 4, ref = (cls >> 1) & 7, mode = cls & 1;
            for (int dir = 0; dir < 2; dir++) {
                int l = lv[dir];
                if (init->segmentation_enabled && (init->seg_feature_mask[seg] >> feature[plane][dir] & 1)) {
                    l += init->seg_feature_data[seg][feature[plane][dir]];
                    l = l < 0 ? 0 : l > 63 ? 63 : l;
                }
                if (init->mode_ref_delta_enabled) {
                    const int scale = 1 << (l >> 5);
                    l += init->ref_deltas[ref] * scale + (ref ? init->mode_deltas[mode] * scale : 0);
                    l = l < 0 ? 0 : l > 63 ? 63 : l;
                }
                lut[plane][dir][cls] = (uint8_t)l;
            }
        }
    }
}
void orc_lf_level_lut(const SvtB200LfFrameInit *init, const int32_t levels[4], uint8_t lut[3][2][128]) {
    level_lut(init, levels, 0, lut);
}

/* ---- svt_av1_pick_filter_level (Encoder/Codec/EbDeblockingFilter.c:1193-1297) -------------------------------- */
typedef struct {
    const SvtB200LpfPickParams *p;
    const SvtB200Frame *recon, *source, *temp;
    const SvtB200DlfMi *mi;
    SvtB200DlfMi *mi_lv; /* copy of mi whose lvl_* fields carry the trial levels */
    int32_t hdr[4]; /* frm_hdr->loop_filter_params levels */
} PickState;

static void copy_plane(const SvtB200Frame *s, const SvtB200Frame *d, int plane) { /* svt_copy_buffer :756-823 */
    const int es = s->bit_depth > 8 ? 2 : 1, w = plane ? s->width >> 1 : s->width, h = plane ? s->height >> 1 : s->height;
    const uint8_t *sp = plane == 0 ? s->y : plane == 1 ? s->cb : s->cr;
    uint8_t *dp = plane == 0 ? d->y : plane == 1 ? d->cb : d->cr;
    const size_t ss = (size_t)(plane ? s->stride_c : s->stride_y) * es, ds = (size_t)(plane ? d->stride_c : d->stride_y) * es;
    for (int y = 0; y < h; y++) memcpy(dp + y * ds, sp + y * ss, (size_t)w * es);
}

static int64_t try_level(PickState *st, int level, int plane, int dir) { /* try_filter_frame :966-1026 */
    if (plane == 0) {
        if (dir == 0 || dir == 2) st->hdr[0] = level;
        if (dir == 1 || dir == 2) st->hdr[1] = level;
    } else {
        st->hdr[1 + plane] = level;
    }
    uint8_t lut[3][2][128];
    level_lut(&st->p->init, st->hdr, plane, lut);
    const SvtB200DlfParams *g = &st->p->dlf;
    for (int r = 0; r < g->mi_rows; r++)
        for (int c = 0; c < g->mi_cols; c++) {
            SvtB200DlfMi *m = &st->mi_lv[(size_t)r * g->mi_stride + c];
            const int cls = m->lvl_class & 127;
            m->lvl_y[0] = lut[0][0][cls], m->lvl_y[1] = lut[0][1][cls], m->lvl_u = lut[1][0][cls], m->lvl_v = lut[2][0][cls];
        }
    SvtB200DlfParams dp = *g;
    dp.sharpness = 0;
    dp.filter_level[0] = st->hdr[0], dp.filter_level[1] = st->hdr[1], dp.filter_level_u = st->hdr[2], dp.filter_level_v = st->hdr[3];
    dp.plane_start = plane, dp.plane_end = plane + 1;
    orc_dlf_frame(&dp, st->recon, st->mi_lv);
    uint64_t sse[3];
    orc_frame_sse(st->source, st->recon, sse); /* picture_sse_calculations :830-964 (one plane is used) */
    copy_plane(st->temp, st->recon, plane);
    return (int64_t)sse[plane];
}

static int search_level(PickState *st, int plane, int dir) { /* search_filter_level :1027-1191 */
    const int last = plane == 0 ? st->p->last_level[dir] : st->p->last_level[1 + plane];
    int mid = last < 0 ? 0 : last > 63 ? 63 : last, step = mid < 16 ? 4 : mid / 4, direction = 0;
    int64_t err[64];
    for (int i = 0; i < 64; i++) err[i] = -1;
    copy_plane(st->recon, st->temp, plane);
    int64_t best = err[mid] = try_level(st, mid, plane, dir);
    int pick = mid;
    const int once = st->p->loop_filter_mode <= 2;
    if (once) step = 2;
    while (step > 0) {
        const int hi = mid + step > 63 ? 63 : mid + step, lo = mid - step < 0 ? 0 : mid - step;
        int64_t bias = (best >> (15 - mid / 8)) * step;
        if (!st->p->tx_mode_only_4x4) bias >>= 1;
        if (direction <= 0 && lo != mid) {
            if (err[lo] < 0) err[lo] = try_level(st, lo, plane, dir);
            if (err[lo] < best + bias) {
                if (err[lo] < best) best = err[lo];
                pick = lo;
            }
        }
        if (direction >= 0 && hi != mid) {
            if (err[hi] < 0) err[hi] = try_level(st, hi, plane, dir);
            if (err[hi] < best - bias) {
                if (!once) best = err[hi];
                pick = hi;
            }
        }
        if (once) break;
        if (pick == mid) {
            step /= 2;
            direction = 0;
        } else {
            direction = pick < mid ? -1 : 1;
            mid = pick;
        }
    }
    return pick;
}

void orc_pick_filter_level(const SvtB200LpfPickParams *p, const SvtB200Frame *recon, const SvtB200Frame *source,
                           const SvtB200Frame *temp, const SvtB200DlfMi *mi, int32_t *levels_out) {
    if (p->method == 3) {
        levels_out[0] = levels_out[1] = 0;
        levels_out[2] = p->last_level[2], levels_out[3] = p->last_level[3];
        return;
    }
    if (p->method == 2) { /* LPF_PICK_FROM_Q :1209-1249 */
        const int bd = recon->bit_depth;
        const int64_t q = p->q_ac;
        int g;
        if (bd == 8) g = p->key_frame ? (int)((q * 17563 - 421574 + (1 << 17)) >> 18) : (int)((q * 6017 + 650707 + (1 << 17)) >> 18);
        else if (bd == 10) g = (int)((q * 20723 + 4060632 + (1 << 19)) >> 20);
        else g = (int)((q * 20723 + 16242526 + (1 << 21)) >> 22);
        if (bd != 8 && p->key_frame) g -= 4;
        g = g > 2 ? g - 2 : g > 1 ? g - 1 : g;
        const int gc = g > 1 ? g / 2 : g;
        levels_out[0] = levels_out[1] = g < 0 ? 0 : g > 63 ? 63 : g;
        levels_out[2] = levels_out[3] = gc < 0 ? 0 : gc > 63 ? 63 : gc;
        return;
    }
    PickState st = {p, recon, source, temp, mi, NULL, {p->last_level[0], p->last_level[1], p->last_level[2], p->last_level[3]}};
    const size_t n = (size_t)p->dlf.mi_rows * p->dlf.mi_stride;
    st.mi_lv = (SvtB200DlfMi *)malloc(n * sizeof(SvtB200DlfMi));
    memcpy(st.mi_lv, mi, n * sizeof(SvtB200DlfMi));
    st.hdr[0] = st.hdr[1] = search_level(&st, 0, 2);
    st.hdr[2] = search_level(&st, 1, 0);
    st.hdr[3] = search_level(&st, 2, 0);
    for (int i = 0; i < 4; i++) levels_out[i] = st.hdr[i];
    free(st.mi_lv);
}
