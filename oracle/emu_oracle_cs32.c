/*
 * TEST INFRASTRUCTURE ONLY -- the centre-surround model with a float32 photoreceptor state (cutoff_hz == 0), on top of
 * the scalar CPU oracle emu_oracle.c, which this file includes unchanged. Same rules: never linked, imported or executed
 * by the product package.
 *
 * At cutoff_hz == 0 low_pass_filter returns the float32 log frame unchanged (emulator_utils.py:75-77) and the surround
 * is its clone (emulator.py:1063), so every op of the reference's Euler step (emulator.py:1110-1120) and of
 * c_minus_s / diff (emulator.py:751-752) is float32; a Python-float alpha_p meets a float32 tensor, so it is rounded to
 * float32 first. max|change| is a float32 value compared with 1e-5 as a double.
 *
 * The library exports the entry points of emu_oracle.c under the same names and signatures. oracle_emu_first_frame and
 * oracle_emu_frame take the float32 branch below for a float32 centre-surround state (cfg->csdvs, !cfg->state_f64,
 * st->surround a float32 array) and call emu_oracle.c's own functions for everything else.
 *
 * Pinning: tests/test_oracle_csdvs_f32.py checks it against tests/golden/emu_cs32_*.npz, which
 * oracle/make_golden_cs32.py produced by running the unmodified reference (device="cpu").
 *
 * Build: gcc -O2 -ffp-contract=off -fPIC -shared (oracle/emu_oracle_cs32.py).
 */
#define oracle_emu_first_frame oracle_emu_first_frame_base
#define oracle_emu_frame oracle_emu_frame_base
#include "emu_oracle.c"
#undef oracle_emu_first_frame
#undef oracle_emu_frame

/* Deliberate error for the sensitivity tests, off by default: the float64 state's rule applied to a float32 state.
 * 1 computes p_term = alpha_p * (p - h) in float64 (and so the sum), 2 the sum change = p_term + h_term; the float64
 * change is then added to h in float64 and stored in the float32 state. */
static int g_f64_rule;
void oracle_set_cs_f64_rule(int f64_rule) { g_f64_rule = f64_rule; }

static int is_cs32(const OracleEmuCfg *cfg, const OracleEmuState *st) {
    return cfg->csdvs && !cfg->state_f64 && st->surround;
}

/* first frame: lp = base = log frame (emulator.py:684-691), surround = clone of lp, base = lp - surround (:714) */
int oracle_emu_first_frame(const OracleEmuCfg *cfg, OracleEmuState *st, const void *frame, double t_frame,
                           double t_previous) {
    int rc = oracle_emu_first_frame_base(cfg, st, frame, t_frame, t_previous);
    if (rc || !is_cs32(cfg, st)) return rc;
    long n = (long)cfg->width * cfg->height;
    float *lp = (float *)st->lp, *base = (float *)st->base, *h = (float *)st->surround;
    for (long i = 0; i < n; i++) {
        h[i] = lp[i];
        base[i] = lp[i] - h[i];
    }
    return 0;
}

/* Euler steps of h += float32(alpha_p)*(p - h) + float32(alpha_h)*lap(h) (emulator.py:1066-1124). Returns steps taken. */
static int csdvs_f32(const OracleEmuCfg *cfg, OracleEmuState *st, double delta_time) {
    long W = cfg->width, H = cfg->height, n = W * H;
    double tau_p = cfg->cs_tau_p_s, tau_h = cfg->cs_tau_h_s;
    double min_tau = tau_p < tau_h ? tau_p : tau_h;
    int num_steps = (int)ceil((delta_time / min_tau) * 5);
    double adt = delta_time / num_steps;
    double alpha_p = adt / tau_p, alpha_h = adt / tau_h;
    const float alpha_p_f = (float)alpha_p;
    float alpha_h_f = (float)alpha_h;
    for (int k = 0; k < g_perturb.alpha_h_ulps; k++) alpha_h_f = nextafterf(alpha_h_f, INFINITY);
    const float *p = (const float *)st->lp;
    float *h = (float *)st->surround;
    double *chg = (double *)malloc(sizeof(double) * n);
    double max_change = 2e-5;
    int steps = 0;
    while (steps < num_steps && max_change > 1e-5) {
        max_change = 0;
        for (long y = 0; y < H; y++) {
            for (long x = 0; x < W; x++) {
                long i = y * W + x;
                float h_term = alpha_h_f * lap_f32(h, H, W, y, x);
                float diff = p[i] - h[i];
                double c;
                if (g_f64_rule == 1) c = alpha_p * (double)diff + (double)h_term;
                else if (g_f64_rule == 2) c = (double)(alpha_p_f * diff) + (double)h_term;
                else c = (double)(alpha_p_f * diff + h_term);
                chg[i] = c;
                if (fabs(c) > max_change) max_change = fabs(c);
            }
        }
        for (long i = 0; i < n; i++) h[i] = g_f64_rule ? (float)((double)h[i] + chg[i]) : h[i] + (float)chg[i];
        steps++;
    }
    free(chg);
    return steps;
}

/* one frame after the first, float32 centre-surround state: emu_oracle.c's oracle_emu_frame with the float32 surround
 * (same outputs and contract; photoreceptor noise needs cutoff_hz > 0 and so never applies here) */
static long cs32_frame(const OracleEmuCfg *cfg, OracleEmuState *st, const void *frame, double t_frame,
                       double t_previous, const float *leak_randn, float *events, long cap, int32_t *iter_counts,
                       long iter_cap, int32_t *max_n_out, int32_t *final_pos_out, int32_t *final_neg_out,
                       int32_t *cs_steps_out) {
    long W = cfg->width, n = (long)cfg->width * cfg->height;
    double dt = t_frame - t_previous;
    float *lp = (float *)st->lp, *base = (float *)st->base, *h = (float *)st->surround;
    int32_t *pos_n = (int32_t *)malloc(sizeof(int32_t) * n);
    int32_t *neg_n = (int32_t *)malloc(sizeof(int32_t) * n);
    int32_t *fin_p = final_pos_out ? final_pos_out : (int32_t *)malloc(sizeof(int32_t) * n);
    int32_t *fin_n = final_neg_out ? final_neg_out : (int32_t *)malloc(sizeof(int32_t) * n);
    memset(fin_p, 0, sizeof(int32_t) * n);
    memset(fin_n, 0, sizeof(int32_t) * n);
    int32_t max_n = 0;
    /* low_pass_filter at cutoff 0: the log frame (emulator.py:686-691) */
    for (long i = 0; i < n; i++) lp[i] = log_new_f32(st, frame_value(frame, cfg->frame_dtype, i));
    *cs_steps_out = csdvs_f32(cfg, st, dt);
    /* SCIDVS, float32 (emulator.py:58-80, 719-725) */
    if (cfg->scidvs && st->hp) {
        float *hp = (float *)st->hp, *pv = (float *)st->prev_photo;
        for (long i = 0; i < n; i++) {
            float inv_tau = 1.0f / st->tau_arr[i];
            if (cfg->scidvs_first) { hp[i] = 0.0f; pv[i] = lp[i]; }
            float dvdt = inv_tau * sinhf(hp[i] / (float)(1 / 0.7));
            float d1 = lp[i] - pv[i], d2 = (float)dt * dvdt;
            hp[i] = hp[i] + (d1 - d2);
            pv[i] = lp[i];
        }
    }
    /* leak, c_minus_s, diff, event counts (emulator.py:734-775) */
    for (long i = 0; i < n; i++) {
        float thp = cfg->per_pixel_thres ? st->pos_thres[i] : (float)cfg->pos_thres_nominal;
        float thn = cfg->per_pixel_thres ? st->neg_thres[i] : (float)cfg->neg_thres_nominal;
        if (cfg->leak_rate_hz > 0) {
            float rate = ((float)cfg->leak_rate_hz * st->noise_rate[i]) *
                         (1.0f - (float)cfg->leak_jitter_fraction * leak_randn[i]);
            base[i] = base[i] - ((float)dt * rate) * thp;
        }
        float photo = (cfg->scidvs && st->hp) ? 2.0f * ((float *)st->hp)[i] : lp[i];
        photo = photo + 0.0f;                       /* + photoreceptor_noise_arr (zeros) */
        float c_minus_s = photo - h[i];
        float diff = c_minus_s - base[i];
        float pf = diff > 0 ? diff : 0.0f, nf = -diff > 0 ? -diff : 0.0f;
        pos_n[i] = (int32_t)div_floor_f32(pf, thp);
        neg_n[i] = (int32_t)div_floor_f32(nf, thn);
        if (pos_n[i] > max_n) max_n = pos_n[i];
        if (neg_n[i] > max_n) max_n = neg_n[i];
    }
    *max_n_out = max_n;
    /* iterations, refractory filter, emission (emulator.py:786-870), as in oracle_emu_frame */
    int64_t steps = max_n > 0 ? max_n : 1;
    double ts_step = dt / (double)steps;
    double start = t_previous + ts_step;
    int refr_on = cfg->refractory_period_s > ts_step;
    float refr_f = (float)cfg->refractory_period_s;
    long rows = 0;
    int fail = max_n > iter_cap;
    uint8_t *pc = (uint8_t *)malloc(n), *nc = (uint8_t *)malloc(n);
    for (int32_t it = 0; it < max_n && !fail; it++) {
        float ts = oracle_linspace_f32(start, t_frame, steps, it);
        for (long i = 0; i < n; i++) {
            int p = pos_n[i] >= it + 1, q = neg_n[i] >= it + 1;
            if (refr_on) {
                float tp = (p ? ts : 0.0f * ts) - st->tmem[i];
                float tn = (q ? ts : 0.0f * ts) - st->tmem[i];
                p = tp > refr_f;
                q = tn > refr_f;
                if (p) st->tmem[i] = ts;
                if (q) st->tmem[i] = ts;
            }
            pc[i] = (uint8_t)p;
            nc[i] = (uint8_t)q;
            fin_p[i] += p;
            fin_n[i] += q;
        }
        int32_t c_on = 0, c_off = 0;
        for (int pol = 0; pol < 2 && !fail; pol++) {
            const uint8_t *m = pol ? nc : pc;
            for (long i = 0; i < n; i++)
                if (m[i]) {
                    if (rows >= cap) { fail = 1; break; }
                    float *e = events + 4 * rows++;
                    e[0] = ts; e[1] = (float)(i % W); e[2] = (float)(i / W); e[3] = pol ? -1.0f : 1.0f;
                    if (pol) c_off++; else c_on++;
                }
        }
        iter_counts[2 * it] = c_on;
        iter_counts[2 * it + 1] = c_off;
    }
    /* base update: int32 * float32 products (emulator.py:936-937) */
    for (long i = 0; i < n; i++) {
        float thp = cfg->per_pixel_thres ? st->pos_thres[i] : (float)cfg->pos_thres_nominal;
        float thn = cfg->per_pixel_thres ? st->neg_thres[i] : (float)cfg->neg_thres_nominal;
        base[i] = base[i] + (float)fin_p[i] * thp;
        base[i] = base[i] - (float)fin_n[i] * thn;
    }
    free(pc);
    free(nc);
    free(pos_n);
    free(neg_n);
    if (!final_pos_out) free(fin_p);
    if (!final_neg_out) free(fin_n);
    return fail ? -1 : rows;
}

long oracle_emu_frame(const OracleEmuCfg *cfg, OracleEmuState *st, const void *frame, double t_frame,
                      double t_previous, const float *leak_randn, float *events, long cap, int32_t *iter_counts,
                      long iter_cap, int32_t *max_n_out, int32_t *final_pos_out, int32_t *final_neg_out,
                      int32_t *cs_steps_out) {
    if (!is_cs32(cfg, st))
        return oracle_emu_frame_base(cfg, st, frame, t_frame, t_previous, leak_randn, events, cap, iter_counts,
                                     iter_cap, max_n_out, final_pos_out, final_neg_out, cs_steps_out);
    return cs32_frame(cfg, st, frame, t_frame, t_previous, leak_randn, events, cap, iter_counts, iter_cap, max_n_out,
                      final_pos_out, final_neg_out, cs_steps_out);
}
