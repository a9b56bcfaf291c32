/*
 * TEST INFRASTRUCTURE ONLY -- scalar CPU restatement of the DVS pixel model.
 *
 * This file is the parity oracle for the CUDA emulator path. It must never be
 * linked, imported or executed by the product package (v2e_b200/); only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
 * may call it.
 *
 * What it restates (reference = SensorsINI/v2e, paths relative to /root/reference):
 *   lin_log                  v2ecore/emulator_utils.py:18-45
 *   rescale_intensity_frame  v2ecore/emulator_utils.py:48-54
 *   low_pass_filter          v2ecore/emulator_utils.py:57-109
 *   subtract_leak_current    v2ecore/emulator_utils.py:114-134
 *   compute_event_map        v2ecore/emulator_utils.py:137-173
 *   generate_shot_noise      v2ecore/emulator_utils.py:297-351
 *   generate_events body     v2ecore/emulator.py:619-1022 (steps 3-20 of SURVEY 3.3)
 *   _update_csdvs            v2ecore/emulator.py:1061-1124
 * plus the ATen semantics those Python lines rely on (third-party, torch 2.11):
 *   div(rounding_mode="floor") on floats  -> div_floor_floating()
 *   linspace(float32)                     -> linspace_f32()   (fused multiply-add
 *                                            form; verified against torch 2.11
 *                                            AVX512 CPU build, see DESIGN.md)
 *   Python-scalar x float32-tensor ops    -> scalar rounded to float32 first
 *
 * Pinning: tests/test_oracle_golden.py checks this file against
 * tests/golden/emu_*.npz, which oracle/make_golden.py produced by running the
 * unmodified reference (device="cpu") in the build container.
 *
 * Build: gcc -O2 -ffp-contract=off -fPIC -shared (see oracle/Makefile).
 * -ffp-contract=off matters: the reference evaluates every tensor op
 * separately, so no multiply-add may be fused except where stated.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct OracleEmuCfg {
    int32_t width, height;
    int32_t state_f64;          /* 1: lp/base are float64 (cutoff_hz>0 or hdr) */
    int32_t per_pixel_thres;    /* 1: pos/neg_thres arrays; 0: Python-float scalars */
    int32_t hdr;                /* log_input */
    int32_t frame_dtype;        /* 0 u8, 1 f32, 2 f64 */
    double pos_thres_nominal, neg_thres_nominal;
    double cutoff_hz;
    double leak_rate_hz, leak_jitter_fraction;
    double refractory_period_s;
    double shot_noise_rate_hz;
    double shot_inten_factor;   /* 0.25, emulator.py:213 */
    int32_t csdvs;              /* 1: centre-surround enabled (state->surround != NULL) */
    int32_t _pad;
    double cs_tau_p_s, cs_tau_h_s;  /* emulator.py:1069-1073 */
    int32_t scidvs;             /* emulator.py:308: nonlinear CR high-pass in front of the change amplifier */
    int32_t pr_noise;           /* emulator.py:192: Gaussian photoreceptor noise instead of injected shot events */
    int32_t scidvs_first;       /* this is the frame at which scidvs_highpass is created (emulator.py:720-722) */
    int32_t _pad2;
    double pr_vrms;             /* photoreceptor_noise_vrms of this frame (emulator.py:695-697), computed by the caller */
} OracleEmuCfg;

typedef struct OracleEmuState {
    void *lp;                   /* S[H*W] */
    void *base;                 /* S[H*W] */
    float *pos_thres, *neg_thres;   /* per-pixel or NULL */
    float *noise_rate;          /* or NULL when leak_rate_hz<=0 */
    float *tmem;                /* or NULL when refractory_period_s<=0 */
    double *surround;           /* CSDVS h, or NULL */
    const float *linlog_lut;    /* 256 entries built by the caller with the reference formula */
    void *hp;                   /* scidvs_highpass, S[H*W] (zeros_like(lp_log_frame)), or NULL */
    void *prev_photo;           /* scidvs_previous_photo, S[H*W] */
    const float *tau_arr;       /* scidvs_tau_arr float32 (emulator.py:480-483) */
    float *noise_arr;           /* photoreceptor_noise_arr float32 (zeros_like of the float32 log frame, :684) */
    const float *pr_randn;      /* this frame's torch.randn field (emulator.py:698) */
} OracleEmuState;

/* ---- ATen restatements ------------------------------------------------- */

/* aten/src/ATen/native/BinaryOps.h div_floor_floating (b>0 branch kept general) */
static double div_floor_f64(double a, double b) {
    if (b == 0) return a / b;
    double mod = fmod(a, b);
    double div = (a - mod) / b;
    if ((mod != 0) && ((b < 0) != (mod < 0))) div -= 1.0;
    double fl;
    if (div != 0) {
        fl = floor(div);
        if (div - fl > 0.5) fl += 1.0;
    } else {
        fl = copysign(0.0, a / b);
    }
    return fl;
}
static float div_floor_f32(float a, float b) {
    if (b == 0) return a / b;
    float mod = fmodf(a, b);
    float div = (a - mod) / b;
    if ((mod != 0) && ((b < 0) != (mod < 0))) div -= 1.0f;
    float fl;
    if (div != 0) {
        fl = floorf(div);
        if (div - fl > 0.5f) fl += 1.0f;
    } else {
        fl = copysignf(0.0f, a / b);
    }
    return fl;
}

/* torch.linspace(start, end, steps, dtype=float32) element i (emulator.py:793-796).
 * steps==1 -> fill(start). Otherwise ATen's CPU kernel evaluates
 *   i < steps/2 ? start + step*i : end - step*(steps-1-i)
 * and the AVX2/AVX512 builds contract both into a fused multiply-add. */
float oracle_linspace_f32(double start_d, double end_d, int64_t steps, int64_t i) {
    float start = (float)start_d, end = (float)end_d;
    if (steps == 1) return start;
    float step = (end - start) / (float)(steps - 1);
    if (i < steps / 2) return fmaf(step, (float)i, start);
    return fmaf(-step, (float)(steps - 1 - i), end);
}

/* lin_log for one value (emulator_utils.py:18-45), float64 in, float32 out */
static float lin_log_value(double x) {
    const double f = (1.0 / 20.0) * log(20.0);
    double y = (x <= 20.0) ? x * f : log(x);
    y = rint(y * 1e8) / 1e8;            /* torch.round = half-to-even */
    return (float)y;
}

static double frame_value(const void *frame, int dtype, long i) {
    if (dtype == 0) return (double)((const uint8_t *)frame)[i];
    if (dtype == 1) return (double)((const float *)frame)[i];
    return ((const double *)frame)[i];
}

static float log_new_f32(const OracleEmuState *st, double x) {
    if (x >= 0 && x <= 255 && x == floor(x)) return st->linlog_lut[(int)x];
    return lin_log_value(x);
}

/* ---- first frame: emulator.py:663-717 ---------------------------------- */
/* lp is seeded with log_new and still passes through the IIR once
 * (emulator.py:681-691); base = lp (minus surround for CSDVS). */
int oracle_emu_first_frame(const OracleEmuCfg *cfg, OracleEmuState *st,
                           const void *frame, double t_frame, double t_previous) {
    long n = (long)cfg->width * cfg->height;
    double dt = t_frame - t_previous;
    double tau = cfg->cutoff_hz > 0 ? 1.0 / (M_PI * 2 * cfg->cutoff_hz) : 0.0;
    for (long i = 0; i < n; i++) {
        double x = frame_value(frame, cfg->frame_dtype, i);
        if (cfg->state_f64) {
            double ln = cfg->hdr ? x : (double)log_new_f32(st, x);
            double lp = ln;
            if (cfg->cutoff_hz > 0) {
                double inten01 = (x + 20.0) / 275.0;
                double eps = inten01 * (dt / tau);
                if (eps > 1.0) eps = 1.0;
                lp = (1.0 - eps) * ln + eps * ln;
            }
            ((double *)st->lp)[i] = lp;
            if (st->surround) st->surround[i] = lp;   /* emulator.py:1062-1063 */
            ((double *)st->base)[i] = st->surround ? lp - st->surround[i] : lp;
        } else {
            float ln = log_new_f32(st, x);
            ((float *)st->lp)[i] = ln;
            ((float *)st->base)[i] = ln;
        }
    }
    return 0;
}

/* ---- float32 Laplacian: emulator.py:1115 -------------------------------- */
/* Deliberate errors for the sensitivity tests (tests/test_emulator_centre_surround.py), all off by default:
 * legacy_order restores the rule this file used to state (kernel order iff H*W >= 20000, no tail), alpha_h_ulps
 * moves the float32 alpha_h of the surround update up by that many ulps. */
static struct { int legacy_order, alpha_h_ulps; } g_perturb;
void oracle_set_cs_perturbation(int legacy_order, int alpha_h_ulps) {
    g_perturb.legacy_order = legacy_order;
    g_perturb.alpha_h_ulps = alpha_h_ulps;
}

/* torch.conv2d(ReplicationPad2d(1)(h), [[0,1,0],[1,-4,1],[0,1,0]]) on the CPU (torch 2.11, AVX-512 build) for a
 * [1,1,H,W] float32 field. Only the summation order of the five non-zero taps varies, by frame size and pixel:
 *  - padded input of more than 20480 elements, (H+2)*(W+2) > 20480: oneDNN (ATen's use_mkldnn size heuristic)
 *    accumulates in kernel order (((u+l)+c)+r)+d at every pixel;
 *  - otherwise ATen's native im2col + GEMM pairs the taps, (u+l)+(c+(r+d)), except in the last n mod 16 elements of
 *    the flattened output (the GEMM's 16-float vector remainder), which take kernel order again.
 * Measured by bisecting over frame sizes and pinned by tests/test_laplacian_order.py against
 * tests/golden/laplacian_conv2d.npz (oracle/make_golden_laplacian.py). i is the WHOLE frame's flattened index. */
int oracle_lap_kernel_order(long H, long W, long i) {
    if (g_perturb.legacy_order) return H * W >= 20000;
    if ((H + 2) * (W + 2) > 20480) return 1;
    return i >= (H * W) / 16 * 16;
}

static float lap_f32(const float *hf, long H, long W, long y, long x) {
    long ym = y > 0 ? y - 1 : 0, yp = y < H - 1 ? y + 1 : H - 1;
    long xm = x > 0 ? x - 1 : 0, xp = x < W - 1 ? x + 1 : W - 1;
    float uu = hf[ym * W + x], ll = hf[y * W + xm], cc = -4.0f * hf[y * W + x];
    float rr = hf[y * W + xp], dd = hf[yp * W + x];
    return oracle_lap_kernel_order(H, W, y * W + x) ? ((((uu + ll) + cc) + rr) + dd) : (uu + ll) + (cc + (rr + dd));
}

/* the whole Laplacian of an H x W float32 field, for the test against torch */
void oracle_laplacian_f32(const float *hf, long H, long W, float *out) {
    for (long y = 0; y < H; y++)
        for (long x = 0; x < W; x++) out[y * W + x] = lap_f32(hf, H, W, y, x);
}

/* ---- CSDVS surround: emulator.py:1061-1124 ----------------------------- */
/* Euler steps of h += alpha_p*(p-h) + alpha_h*lap(float32(h)), replicate pad,
 * until max|change| <= 1e-5 or num_steps. p,h float64; the 3x3 stencil is a
 * float32 conv2d (emulator.py:1115, lap_f32), products promoted back to float64.
 * Returns steps taken. */
int oracle_emu_csdvs(const OracleEmuCfg *cfg, OracleEmuState *st, double delta_time,
                     double tau_p, double tau_h) {
    long W = cfg->width, H = cfg->height, n = W * H;
    double min_tau = tau_p < tau_h ? tau_p : tau_h;
    int num_steps = (int)ceil((delta_time / min_tau) * 5);
    double adt = delta_time / num_steps;
    double alpha_p = adt / tau_p, alpha_h = adt / tau_h;
    const double *p = (const double *)st->lp;
    double *h = st->surround;
    float alpha_h_f = (float)alpha_h;
    for (int k = 0; k < g_perturb.alpha_h_ulps; k++) alpha_h_f = nextafterf(alpha_h_f, INFINITY);
    float *hf = (float *)malloc(sizeof(float) * n);
    double *chg = (double *)malloc(sizeof(double) * n);
    double max_change = 2e-5;
    int steps = 0;
    while (steps < num_steps && max_change > 1e-5) {
        for (long i = 0; i < n; i++) hf[i] = (float)h[i];
        max_change = 0;
        for (long y = 0; y < H; y++) {
            for (long x = 0; x < W; x++) {
                float acc = lap_f32(hf, H, W, y, x);
                /* alpha_h is a Python float meeting a float32 tensor: rounded to float32, float32 product */
                float h_term = alpha_h_f * acc;
                double c = alpha_p * (p[y * W + x] - h[y * W + x]) + (double)h_term;
                chg[y * W + x] = c;
                double a = fabs(c);
                if (a > max_change) max_change = a;
            }
        }
        for (long i = 0; i < n; i++) h[i] += chg[i];
        steps++;
    }
    free(hf);
    free(chg);
    return steps;
}

/* ---- one frame after the first ----------------------------------------- */
/*
 * Outputs, in the reference's pre-shuffle order (emulator.py:861-866, 1024-1059):
 *   for each iteration i: ON rows (row-major y,x) then OFF rows, all at ts[i];
 *   then shot-noise ON rows, shot-noise OFF rows at ts[-1] (emulator.py:906-919).
 * events: float32 [cap][4] rows [t, x, y, p]. iter_counts[2*i+{0,1}] = ON/OFF rows of
 * iteration i (caller needs them to replay torch.randperm, emulator.py:868).
 * Returns total rows, or -1 if cap / iter_cap is too small.
 * Phase split for RNG replay: the reference draws the shot-noise rand AFTER the
 * per-iteration randperm calls, whose sizes depend on this frame's events. So the
 * caller runs phase 1 (shot_rand==NULL, do_shot=0) to get iter_counts, replays
 * randperm, draws rand, then calls oracle_emu_shot().
 */
long oracle_emu_frame(const OracleEmuCfg *cfg, OracleEmuState *st, const void *frame,
                      double t_frame, double t_previous, const float *leak_randn,
                      float *events, long cap, int32_t *iter_counts, long iter_cap,
                      int32_t *max_n_out, int32_t *final_pos_out, int32_t *final_neg_out,
                      int32_t *cs_steps_out) {
    long W = cfg->width, n = (long)cfg->width * cfg->height;
    double dt = t_frame - t_previous;
    double tau = cfg->cutoff_hz > 0 ? 1.0 / (M_PI * 2 * cfg->cutoff_hz) : 0.0;
    int32_t *pos_n = (int32_t *)malloc(sizeof(int32_t) * n);
    int32_t *neg_n = (int32_t *)malloc(sizeof(int32_t) * n);
    int32_t *fin_p = final_pos_out ? final_pos_out : (int32_t *)calloc(n, sizeof(int32_t));
    int32_t *fin_n = final_neg_out ? final_neg_out : (int32_t *)calloc(n, sizeof(int32_t));
    memset(fin_p, 0, sizeof(int32_t) * n);
    memset(fin_n, 0, sizeof(int32_t) * n);
    int32_t max_n = 0;

    /* pass A: photoreceptor low-pass (emulator.py:686-691) */
    for (long i = 0; i < n; i++) {
        double x = frame_value(frame, cfg->frame_dtype, i);
        if (cfg->state_f64) {
            double *lp = (double *)st->lp;
            double ln = cfg->hdr ? x : (double)log_new_f32(st, x);
            if (cfg->cutoff_hz > 0) {
                double inten01 = (x + 20.0) / 275.0;
                double eps = inten01 * (dt / tau);
                if (eps > 1.0) eps = 1.0;
                lp[i] = (1.0 - eps) * lp[i] + eps * ln;
            } else {
                lp[i] = ln;
            }
        } else {
            ((float *)st->lp)[i] = log_new_f32(st, x);
        }
    }
    /* photoreceptor noise (emulator.py:694-703): noise = vrms * randn (Python float x float32 tensor ->
     * float32 product), then low_pass_filter(noise, arr, None, dt, cutoff): eps = dt/tau is a Python float,
     * so (1-eps) and eps meet a float32 tensor and are rounded to float32; no clamp (emulator_utils.py:96-99) */
    if (cfg->pr_noise && st->noise_arr) {
        float vr = (float)cfg->pr_vrms;
        for (long i = 0; i < n; i++) {
            float noise = vr * st->pr_randn[i];
            if (cfg->cutoff_hz > 0) {
                double eps = dt / tau;
                float ome = (float)(1.0 - eps), ef = (float)eps;
                float a = ome * st->noise_arr[i], b = ef * noise;
                st->noise_arr[i] = a + b;
            } else {
                st->noise_arr[i] = noise;
            }
        }
    }
    /* surround diffusion needs the whole lp field (emulator.py:707-708) */
    if (cfg->csdvs && st->surround)
        *cs_steps_out = oracle_emu_csdvs(cfg, st, dt, cfg->cs_tau_p_s, cfg->cs_tau_h_s);
    /* SCIDVS (emulator.py:58-80, 719-725): hp += (lp - lp_prev) - dt * (1/tau_px) * sinh(hp / efold);
     * 1/tau_px is a float32 tensor, hp/efold and sinh are evaluated in hp's dtype */
    if (cfg->scidvs && st->hp) {
        const double efold = 1 / 0.7;
        for (long i = 0; i < n; i++) {
            float inv_tau = 1.0f / st->tau_arr[i];
            if (cfg->state_f64) {
                double *hp = (double *)st->hp, *pv = (double *)st->prev_photo, lp = ((double *)st->lp)[i];
                if (cfg->scidvs_first) { hp[i] = 0.0; pv[i] = lp; }
                double dvdt = (double)inv_tau * sinh(hp[i] / efold);
                double d1 = lp - pv[i], d2 = dt * dvdt;
                hp[i] = hp[i] + (d1 - d2);
                pv[i] = lp;
            } else {
                float *hp = (float *)st->hp, *pv = (float *)st->prev_photo, lp = ((float *)st->lp)[i];
                if (cfg->scidvs_first) { hp[i] = 0.0f; pv[i] = lp; }
                float dvdt = inv_tau * sinhf(hp[i] / (float)efold);
                float d1 = lp - pv[i], d2 = (float)dt * dvdt;
                hp[i] = hp[i] + (d1 - d2);
                pv[i] = lp;
            }
        }
    }
    /* pass B: leak, difference, event counts (emulator.py:734-775) */
    for (long i = 0; i < n; i++) {
        float thp_f = cfg->per_pixel_thres ? st->pos_thres[i] : (float)cfg->pos_thres_nominal;
        float thn_f = cfg->per_pixel_thres ? st->neg_thres[i] : (float)cfg->neg_thres_nominal;
        /* leak delta: all float32 products, emulator_utils.py:126-129 */
        float delta_leak = 0.0f;
        if (cfg->leak_rate_hz > 0) {
            float rate = ((float)cfg->leak_rate_hz * st->noise_rate[i]) *
                         (1.0f - (float)cfg->leak_jitter_fraction * leak_randn[i]);
            delta_leak = ((float)dt * rate) * thp_f;
        }
        if (cfg->state_f64) {
            double *lp = (double *)st->lp, *base = (double *)st->base;
            if (cfg->leak_rate_hz > 0) base[i] = base[i] - (double)delta_leak;
            /* photoreceptor + photoreceptor_noise_arr (a float32 tensor, zeros when the option is off) */
            double photo = (cfg->scidvs && st->hp) ? 2.0 * ((double *)st->hp)[i] : lp[i];
            photo = photo + (double)((cfg->pr_noise && st->noise_arr) ? st->noise_arr[i] : 0.0f);
            double diff = (cfg->csdvs && st->surround) ? (photo - st->surround[i]) - base[i]
                                                       : photo - base[i];
            /* a Python-float threshold stays float64 against a float64 tensor */
            double thp = cfg->per_pixel_thres ? (double)thp_f : cfg->pos_thres_nominal;
            double thn = cfg->per_pixel_thres ? (double)thn_f : cfg->neg_thres_nominal;
            double pf = diff > 0 ? diff : 0.0, nf = -diff > 0 ? -diff : 0.0;
            pos_n[i] = (int32_t)div_floor_f64(pf, thp);
            neg_n[i] = (int32_t)div_floor_f64(nf, thn);
        } else {
            float *lp = (float *)st->lp, *base = (float *)st->base;
            if (cfg->leak_rate_hz > 0) base[i] = base[i] - delta_leak;
            float photo = (cfg->scidvs && st->hp) ? 2.0f * ((float *)st->hp)[i] : lp[i];
            photo = photo + 0.0f;
            float diff = photo - base[i];
            float pf = diff > 0 ? diff : 0.0f, nf = -diff > 0 ? -diff : 0.0f;
            pos_n[i] = (int32_t)div_floor_f32(pf, thp_f);
            neg_n[i] = (int32_t)div_floor_f32(nf, thn_f);
        }
        if (pos_n[i] > max_n) max_n = pos_n[i];
        if (neg_n[i] > max_n) max_n = neg_n[i];
    }
    *max_n_out = max_n;

    int64_t steps = max_n > 0 ? max_n : 1;
    double ts_step = dt / (double)steps;
    double start = t_previous + ts_step;
    int refr_on = cfg->refractory_period_s > ts_step;
    float refr_f = (float)cfg->refractory_period_s;
    long rows = 0;
    int fail = 0;
    if (max_n > iter_cap) fail = 1;
    for (int32_t it = 0; it < max_n && !fail; it++) {
        float ts = oracle_linspace_f32(start, t_frame, steps, it);
        uint8_t *pc = (uint8_t *)malloc(n), *nc = (uint8_t *)malloc(n);
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
        for (long i = 0; i < n && !fail; i++)
            if (pc[i]) {
                if (rows >= cap) { fail = 1; break; }
                float *e = events + 4 * rows++;
                e[0] = ts; e[1] = (float)(i % W); e[2] = (float)(i / W); e[3] = 1.0f;
                c_on++;
            }
        for (long i = 0; i < n && !fail; i++)
            if (nc[i]) {
                if (rows >= cap) { fail = 1; break; }
                float *e = events + 4 * rows++;
                e[0] = ts; e[1] = (float)(i % W); e[2] = (float)(i / W); e[3] = -1.0f;
                c_off++;
            }
        iter_counts[2 * it] = c_on;
        iter_counts[2 * it + 1] = c_off;
        free(pc);
        free(nc);
    }

    /* base update: int32*float32 product is float32, emulator.py:936-937 */
    for (long i = 0; i < n; i++) {
        float thp_f = cfg->per_pixel_thres ? st->pos_thres[i] : (float)cfg->pos_thres_nominal;
        float thn_f = cfg->per_pixel_thres ? st->neg_thres[i] : (float)cfg->neg_thres_nominal;
        float up = (float)fin_p[i] * thp_f, dn = (float)fin_n[i] * thn_f;
        if (cfg->state_f64) {
            double *base = (double *)st->base;
            base[i] = base[i] + (double)up;
            base[i] = base[i] - (double)dn;
        } else {
            float *base = (float *)st->base;
            base[i] = base[i] + up;
            base[i] = base[i] - dn;
        }
    }
    free(pos_n);
    free(neg_n);
    if (!final_pos_out) free(fin_p);
    if (!final_neg_out) free(fin_n);
    return fail ? -1 : rows;
}

/* shot noise of the same frame (emulator.py:893-923, 940-942; emulator_utils.py:297-351).
 * Must run after oracle_emu_frame() of that frame. max_n is that frame's value.
 * Appends ON rows then OFF rows at ts[-1]; resets base to lp on those pixels.
 * counts[0]=ON rows, counts[1]=OFF rows. */
long oracle_emu_shot(const OracleEmuCfg *cfg, OracleEmuState *st, const void *frame,
                     double t_frame, double t_previous, int32_t max_n, const float *rand01,
                     float *events, long cap, int32_t *counts) {
    long W = cfg->width, n = (long)cfg->width * cfg->height;
    double dt = t_frame - t_previous;
    int64_t steps = max_n > 0 ? max_n : 1;
    double start = t_previous + dt / (double)steps;
    float ts_last = oracle_linspace_f32(start, t_frame, steps, steps - 1);
    double c = (cfg->shot_noise_rate_hz / 2) * dt;
    uint8_t *on = (uint8_t *)malloc(n), *off = (uint8_t *)malloc(n);
    for (long i = 0; i < n; i++) {
        double x = frame_value(frame, cfg->frame_dtype, i);
        double inten01 = (x + 20.0) / 275.0;
        double factor = c * ((cfg->shot_inten_factor - 1) * inten01 + 1);
        double pre_on, pre_off;
        if (cfg->per_pixel_thres) {
            pre_on = (double)((float)cfg->pos_thres_nominal / st->pos_thres[i]);
            pre_off = (double)((float)cfg->neg_thres_nominal / st->neg_thres[i]);
        } else {
            pre_on = (double)(float)(cfg->pos_thres_nominal / cfg->pos_thres_nominal);
            pre_off = (double)(float)(cfg->neg_thres_nominal / cfg->neg_thres_nominal);
        }
        double r = (double)rand01[i];
        on[i] = r > 1 - factor * pre_on;
        off[i] = r < factor * pre_off;
    }
    long rows = 0;
    int fail = 0;
    counts[0] = counts[1] = 0;
    for (long i = 0; i < n && !fail; i++)
        if (on[i]) {
            if (rows >= cap) { fail = 1; break; }
            float *e = events + 4 * rows++;
            e[0] = ts_last; e[1] = (float)(i % W); e[2] = (float)(i / W); e[3] = 1.0f;
            counts[0]++;
        }
    for (long i = 0; i < n && !fail; i++)
        if (off[i]) {
            if (rows >= cap) { fail = 1; break; }
            float *e = events + 4 * rows++;
            e[0] = ts_last; e[1] = (float)(i % W); e[2] = (float)(i / W); e[3] = -1.0f;
            counts[1]++;
        }
    for (long i = 0; i < n; i++)
        if (on[i] || off[i]) {
            if (cfg->state_f64) ((double *)st->base)[i] = ((double *)st->lp)[i];
            else ((float *)st->base)[i] = ((float *)st->lp)[i];
        }
    free(on);
    free(off);
    return fail ? -1 : rows;
}
