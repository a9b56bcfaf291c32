/*
 * v2e_b200 -- C ABI of the H100-native (sm_90a) hot paths of SensorsINI/v2e.
 *
 * The reference is pure Python and has no FFI; its boundary for these paths is two
 * Python classes (SURVEY.md 8b). This header is the boundary a maintainer binds
 * (ctypes / cffi, see INTEGRATION.md) to put the sm_90a kernels behind
 *   v2ecore/emulator.py:35   class EventEmulator  (generate_events, :619)
 *   v2ecore/slomo.py:37      class SuperSloMo     (interpolate, :231)
 *
 * Conventions: every function returns 0 (V2E_OK) or a negative V2eStatus; no C++
 * exception crosses the ABI; v2e_last_error() gives a message for the calling
 * thread. Pointers named *_dev are CUDA device pointers, *_host are host pointers.
 * All work is enqueued on the cudaStream_t passed as `stream` (a void* here so
 * that the header needs no CUDA include); functions never synchronise unless their
 * comment says so. A handle is not thread-safe (like the reference's objects).
 */
#ifndef V2E_B200_H
#define V2E_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum V2eStatus {
    V2E_OK = 0,
    V2E_E_INVALID = -1,      /* bad argument */
    V2E_E_CUDA = -2,         /* CUDA runtime error, see v2e_last_error() */
    V2E_E_CAPACITY = -3,     /* event buffer too small; state is resumable, see v2e_emu_step */
    V2E_E_ITER_CAP = -4,     /* a pixel produced more events in one frame than iter_cap */
    V2E_E_STATE = -5,        /* call order violated (e.g. step before first frame) */
    V2E_E_UNSUPPORTED = -6,
    V2E_E_FALLBACK = -7      /* v2e_emu_collect after v2e_emu_fused_*: the chunk must be replayed frame by frame */
} V2eStatus;

typedef enum V2eFrameDtype { V2E_U8 = 0, V2E_F32 = 1, V2E_F64 = 2 } V2eFrameDtype;

const char *v2e_last_error(void);
int v2e_version(void);
/* ABI guard for bindings that mirror the structs (ctypes): version and the sizes of V2eEmuCfg / V2eFrameInfo /
 * V2eUNetWeights as this library was compiled. A binding whose own sizes differ must refuse to load. */
int v2e_abi_info(int *version, int *emu_cfg_size, int *frame_info_size, int *unet_weights_size);

/* ------------------------------------------------------------------------- */
/* DVS pixel model: replaces EventEmulator.generate_events (emulator.py:619-1022)
 * and the tensor helpers it calls (emulator_utils.py:18-173, 297-351).           */
/* ------------------------------------------------------------------------- */

typedef struct V2eEmuCfg {
    int32_t width, height;          /* emulator.py: output_width / output_height */
    int32_t per_pixel_thres;        /* 1 when sigma_thres > 0 (emulator.py:459-472); else the
                                       nominal thresholds act as Python floats */
    int32_t hdr;                    /* emulator.py:110 hdr / log_input */
    double pos_thres_nominal;       /* emulator.py:88 */
    double neg_thres_nominal;       /* emulator.py:89 */
    double cutoff_hz;               /* emulator.py:91 ; >0 (or hdr) makes lp/base (and surround) float64 */
    double leak_rate_hz;            /* emulator.py:92 */
    double leak_jitter_fraction;    /* emulator.py:96 */
    double refractory_period_s;     /* emulator.py:93 */
    double shot_noise_rate_hz;      /* emulator.py:94 */
    double shot_inten_factor;       /* emulator.py:213 SHOT_NOISE_INTEN_FACTOR = 0.25 */
    int32_t rng_mode;               /* 0 = replay: caller uploads the per-frame random fields the
                                           reference would draw (bit-exact with torch's CPU generator);
                                       1 = device: counter-based Philox4x32-7 inside the kernels */
    int32_t iter_cap;               /* max events per pixel per frame that can be emitted (>=1) */
    uint64_t seed;                  /* rng_mode 1 only */
    int32_t csdvs;                  /* 1: centre-surround model enabled (emulator.py:245-265) */
    int32_t max_frames_per_step;    /* upper bound of T in v2e_emu_step (control-block slots) */
    double cs_tau_p_s, cs_tau_h_s;  /* emulator.py:1069-1073 (already floored at 1e-9) */
    int32_t scidvs;                 /* emulator.py:114, 719-725: nonlinear CR high-pass before the change amplifier */
    int32_t photoreceptor_noise;    /* emulator.py:95, 694-703: Gaussian photoreceptor noise instead of injected
                                       shot events (needs shot_noise_rate_hz > 0 and cutoff_hz > 0, :196-204) */
    uint32_t rng_pixel_offset;      /* index, in the WHOLE frame, of this handle's pixel 0. 0 unless the handle owns a
                                       row band of a pixel-sharded clip (y0 * width): the Philox counters (rng_mode 1)
                                       and the centre-surround Laplacian's summation order use whole-frame pixel
                                       indices, so the bands compute what one GPU would compute */
    uint32_t full_frame_px;         /* pixels of the WHOLE frame when the handle owns a row band (0: width * height;
                                       a band has the frame's width): the reference's float32 conv2d sums in an order
                                       that depends on the frame's size and the pixel's index (centre-surround) */
    int32_t own_row0, own_rows;     /* rows [own_row0, own_row0 + own_rows) of the handle emit events; the rest are halo
                                       rows of a pixel-sharded centre-surround handle (own_rows = 0: all rows) */
    int32_t cs_halo_rows;           /* K > 0: pixel-sharded centre-surround model -- K halo rows either side of the own
                                       rows (absent at the image border), Euler steps in chunks of K between halo
                                       exchanges (v2e_emu_cs_*); 0: single-GPU surround */
    int32_t reserved1;
} V2eEmuCfg;

typedef struct V2eEmu V2eEmu;

/* per-frame record the host reads back after a step (host copy of the device control block) */
typedef struct V2eFrameInfo {
    int32_t max_n;                  /* max_num_events_any_pixel, emulator.py:773-775 */
    int32_t filter_active;          /* refractory_period_s > ts_step, emulator.py:830 */
    uint32_t n_on, n_off;           /* rows emitted for this frame incl. shot noise */
    uint32_t n_shot_on, n_shot_off;
    uint32_t n_events;              /* n_on + n_off */
    int32_t cs_steps;               /* Euler steps taken by the surround, emulator.py:1123 */
    uint64_t ev_base;               /* row offset of this frame's first event in events_out */
} V2eFrameInfo;

int v2e_emu_create(const V2eEmuCfg *cfg, V2eEmu **out);
int v2e_emu_destroy(V2eEmu *h);

/* Uploads the 256-entry lin_log table for integer-valued input (emulator_utils.py:18-45
 * evaluated by the caller with the reference expression, so it is exact by construction). */
int v2e_emu_set_linlog_lut(V2eEmu *h, const float *lut256_host, void *stream);

/* Per-pixel fields drawn at the first frame (emulator.py:439-511). Any pointer may be NULL
 * when the feature is off. Host pointers, [H*W] float32. Synchronous copy. */
int v2e_emu_set_fields(V2eEmu *h, const float *pos_thres_host, const float *neg_thres_host,
                       const float *noise_rate_host);

/* SCIDVS per-pixel time constants (emulator.py:480-483), host pointer, [H*W] float32. Synchronous copy. */
int v2e_emu_set_scidvs_tau(V2eEmu *h, const float *tau_host);
/* Photoreceptor noise inputs of the NEXT v2e_emu_step (T frames) or v2e_emu_phase_count (T = 1):
 * vrms_host[T] = photoreceptor_noise_vrms per frame (emulator.py:695-697, a host-side calibration the caller
 * runs); pr_randn_dev [T][H*W] float32 = the values torch.randn would return (emulator.py:698), required in
 * rng_mode 0, ignored (may be NULL) in rng_mode 1. */
int v2e_emu_set_pr_noise(V2eEmu *h, const float *pr_randn_dev, const double *vrms_host, int T);

/* First frame (emulator.py:663-717): seeds lp / base / surround / timestamp_mem. Emits nothing.
 * t_previous stays unchanged, as in the reference (it returns before emulator.py:1011). */
int v2e_emu_first_frame(V2eEmu *h, const void *frame_dev, int frame_dtype, double t_frame,
                        double t_previous, void *stream);

/* T frames after the first. frames_dev: [T][H][W] of frame_dtype. t_frames_host[T]: absolute
 * times; t_previous: time of the frame before frames[0].
 * leak_randn_dev / shot_rand_dev: [T][H*W] float32, used in rng_mode 0 when the respective
 * noise is on (the values torch.randn / torch.rand would return, emulator_utils.py:122-124,
 * 340-343); NULL otherwise. NOTE: in the reference the shot draw of a frame happens after that
 * frame's randperm calls; a caller that needs seed parity with noise on therefore steps one
 * frame at a time with the phase functions below.
 * events_out_dev: [capacity][4] float32 rows [t, x, y, p] (emulator.py:1020); rows of frame f
 * start at info[f].ev_base; ev_base_start is the row at which this step starts writing.
 * Groups are iteration-major, ON before OFF, shot noise (ON, then OFF) last. The order of the rows inside a group
 * is set by option 2 of v2e_emu_set_option:
 *   0 (default): as emitted -- it can differ from run to run;
 *   1 canonical: by pixel index y * width + x ascending, the reference's order before its randperm
 *     (emulator.py:861-870, 1024-1059);
 *   2 shuffled: the ON and OFF rows of one (frame, iteration) are mixed, in ascending order of a 64-bit key that is
 *     uniform and a pure function of (seed, Philox frame index, iteration, pixel, polarity) -- what the reference's
 *     randperm does (emulator.py:866-870), though not its permutation; shot-noise rows stay canonical and last.
 * With 1 or 2 the rows are identical from run to run and whatever kernels, chunk sizes, replays or capacity resumes
 * produced them; v2e_emu_collect enqueues the ordering on `stream` once every frame of the step is emitted.
 * Enqueues everything on `stream`, no host synchronisation.
 * If the buffer is too small at frame f, that frame's emission and everything after it is
 * skipped on the device (sticky abort), state is left as "frame f counted, not emitted";
 * v2e_emu_collect() then reports V2E_E_CAPACITY with frames_done = f, and the caller resumes
 * with v2e_emu_step(..., first = f, resume_emit = 1) into a larger buffer. */
int v2e_emu_step(V2eEmu *h, const void *frames_dev, int frame_dtype, int T,
                 const double *t_frames_host, double t_previous,
                 const float *leak_randn_dev, const float *shot_rand_dev,
                 float *events_out_dev, uint64_t capacity, uint64_t ev_base_start,
                 int first, int resume_emit, void *stream);

/* Multi-frame fast path. v2e_emu_step takes it by itself when it can (T >= 2, uint8 frames, plain pixel model --
 * no hdr / csdvs / scidvs / photoreceptor noise --, rng_mode 1 or no per-frame noise): per-pixel state stays in
 * registers across the T frames, per-frame work is one byte read per pixel plus a 16-bit record per active pixel;
 * rows, counters and state are identical to the frame-by-frame kernels'. It relies on the refractory filter not
 * running (refractory_period_s <= dt / max_n in every frame, emulator.py:830) and on max_n <= 31; a chunk that
 * breaks this is rejected on the device (nothing emitted, state untouched) and v2e_emu_collect replays it frame by
 * frame before it returns. option 0 of v2e_emu_set_option: 0 = never take the fast path (A/B tests), 1 = default.
 * option 1: 1 = the photoreceptor-noise Philox counters (rng_mode 1) use rng_pixel_offset + pixel like the leak and
 * shot counters, so that a row band of a pixel-sharded clip draws what one GPU draws; 0 = the handle's own pixel index
 * (default).
 * option 2: row order inside a group, see v2e_emu_step: 0 = as emitted (default; nothing is launched or allocated for
 * ordering), 1 = canonical, 2 = shuffled (rng_mode 1 only). The shuffled key of a row is the first two words, high
 * word first, of Philox4x32-7 with the seed as key and the counter (2 * pixel + (p < 0), Philox frame index, iteration,
 * 0x726f7264 "rord"), pixel = rng_pixel_offset + y * width + x; equal keys are ordered by 2 * pixel + (p < 0). A row
 * band of a pixel-sharded clip therefore sorts by the whole frame's keys: its rows are a subsequence of the one-GPU
 * order. The canonical key is (p < 0) << 32 | pixel. */
int v2e_emu_set_option(V2eEmu *h, int option, int value);
/* Row order 1 or 2: keys_dev (nullable; uint64, one entry per row of events_out_dev, indexed like it) receives the key
 * of every row v2e_emu_collect orders from now on. */
int v2e_emu_set_key_buffer(V2eEmu *h, uint64_t *keys_dev);
/* Device memory held for ordering (0 until a step has been ordered) and rows ordered so far. */
int v2e_emu_order_stats(V2eEmu *h, uint64_t *scratch_bytes, long long *rows_ordered);
/* The fast path in two halves for a pixel-sharded clip (SURVEY.md 8e): v2e_emu_fused_count enqueues the register-
 * resident update of the T frames and the per-frame counts; the caller all-reduces (MAX) the T int32 at
 * v2e_emu_max_vec_dev() over the ranks on the same stream; v2e_emu_fused_emit plans with the reduced maxima, emits and
 * commits the state. v2e_emu_collect then returns V2E_E_FALLBACK if the chunk was rejected (identically on every
 * rank: the decision uses only the reduced maxima and the frame times) and the caller replays it frame by frame
 * (v2e_emu_phase_*). V2E_E_UNSUPPORTED when the configuration does not qualify. */
int v2e_emu_fused_count(V2eEmu *h, const void *frames_dev, int frame_dtype, int T, const double *t_frames_host,
                        double t_previous, void *stream);
int32_t *v2e_emu_max_vec_dev(V2eEmu *h);
int v2e_emu_fused_emit(V2eEmu *h, float *events_out_dev, uint64_t capacity, uint64_t ev_base_start, void *stream);
/* counters: chunks that went through the fast path / chunks it rejected */
int v2e_emu_fused_stats(V2eEmu *h, long long *chunks, long long *rejected);
/* frames of the steps that took the fast path: how many went through multi-frame segments and how many (those
 * breaking the assumption, and lone frames between them) through the frame-by-frame kernels */
int v2e_emu_fused_frames(V2eEmu *h, long long *frames_multi, long long *frames_single);
/* diagnostics: the frame (index in its chunk) at which the last rejected chunk broke the assumption, and that frame's
 * max_num_events_any_pixel */
int v2e_emu_fused_last_reject(V2eEmu *h, int *frame, int *max_n);
/* Measurement: K repetitions of the fast path of one chunk (update, count, plan, emit; no commit, so the state is
 * left untouched and every repetition does the same work) between one CUDA-event pair, and K repetitions of the
 * update kernel alone between another. Returns microseconds per chunk. Synchronises. */
int v2e_emu_time_fused(V2eEmu *h, const void *frames_dev, int frame_dtype, int T, const double *t_frames_host,
                       double t_previous, float *events_out_dev, uint64_t capacity, int K, float *us_chunk,
                       float *us_update, void *stream);

/* Copies the per-frame control blocks of the last step to the host. Synchronises `stream`.
 * info_host[T]. *frames_done = number of frames fully emitted. Returns V2E_OK,
 * V2E_E_CAPACITY or V2E_E_ITER_CAP. With a row order set (option 2) and V2E_OK, the kernels that order the step's rows
 * in place are enqueued on `stream` after the synchronisation: work enqueued later on that stream sees ordered rows. */
int v2e_emu_collect(V2eEmu *h, V2eFrameInfo *info_host, int T, int *frames_done,
                    uint64_t *rows_total, void *stream);

/* ---- single-frame phases (what v2e_emu_step enqueues per frame), exposed so that a host
 * that must replay torch's CPU generator can interleave its draws (SURVEY.md 7, RNG parity) */
/* phase 1: low-pass, leak, event counts, global max (emulator.py:663-775) and, when the
 * refractory filter applies, the filtered per-iteration counts. Ends with the emission plan
 * unless shot_pending. */
int v2e_emu_phase_count(V2eEmu *h, const void *frame_dev, int frame_dtype, double t_frame,
                        double t_previous, const float *leak_randn_dev,
                        const float *shot_rand_dev, int shot_pending, uint64_t capacity,
                        uint64_t ev_base_start, void *stream);
/* Pixel-sharded operation (one clip's rows split over GPUs, SURVEY.md 8e): max_num_events_any_pixel is
 * frame-global (emulator.py:773-775), so a rank runs phase_update on its band, all-reduces (MAX) the
 * int32 at v2e_emu_max_n_dev() over the ranks on the same stream, then phase_filter (refractory filter
 * with the global maximum, and the emission plan when do_plan != 0), then phase_shot / phase_emit. */
int v2e_emu_phase_update(V2eEmu *h, const void *frame_dev, int frame_dtype, double t_frame,
                         double t_previous, const float *leak_randn_dev, const float *shot_rand_dev,
                         uint64_t capacity, uint64_t ev_base_start, void *stream);
int32_t *v2e_emu_max_n_dev(V2eEmu *h);
/* Pixel-sharded centre-surround model (emulator.py:1061-1124 over row bands; BASELINE config 5). The handle holds
 * the rank's own rows plus cs_halo_rows = K rows of each neighbour; lp is computed on all of them (it is a per-pixel
 * function of the frames), the surround on the halo rows comes from the neighbours. Per frame:
 *   v2e_emu_cs_begin      low-pass of the band, Euler-step plan (*num_steps, emulator.py:1076-1078)
 *   for chunks [s0, s1) of at most K steps:
 *       v2e_emu_cs_pack        own edge rows of the current surround -> v2e_emu_cs_send_dev()  [2][K][W] of the
 *                              state dtype (float64 when v2e_emu_state_is_f64, else float32)
 *                              ([0] = the top K own rows, [1] = the bottom K)
 *       (caller: exchange with the neighbours, e.g. one all-gather of every rank's send buffer)
 *       v2e_emu_cs_unpack_from the neighbours' rows -> halo rows, read where the exchange left them:
 *                              rows_above_dev = the upper neighbour's bottom K rows [K][W], rows_below_dev = the lower
 *                              neighbour's top K rows (state dtype); NULL at the image border
 *       v2e_emu_cs_chunk      steps s0 .. s1-1 (each into its own ring buffer; maxima over the own rows)
 *       (caller: all-reduce MAX of the uint64 at v2e_emu_cs_max_dev()[s0 .. s1) -- non-negative doubles order
 *        like their bit patterns; a float32 state's maxima are float32 magnitudes widened to double, exactly)
 *       v2e_emu_cs_advance     first step with max|change| <= 1e-5 ends the iteration (device side, no host sync)
 *   v2e_emu_cs_update     the update kernel on the converged surround (then v2e_emu_max_n_dev ... as above)
 * Everything is enqueued on `stream`; nothing synchronises. */
int v2e_emu_cs_begin(V2eEmu *h, const void *frame_dev, int frame_dtype, double t_frame, double t_previous,
                     uint64_t capacity, uint64_t ev_base_start, int *num_steps, void *stream);
int v2e_emu_cs_pack(V2eEmu *h, void *stream);
int v2e_emu_cs_unpack_from(V2eEmu *h, const void *rows_above_dev, const void *rows_below_dev, void *stream);
void *v2e_emu_cs_send_dev(V2eEmu *h);
int v2e_emu_cs_chunk(V2eEmu *h, int s0, int s1, void *stream);
uint64_t *v2e_emu_cs_max_dev(V2eEmu *h);
int v2e_emu_cs_advance(V2eEmu *h, int s0, int s1, void *stream);
int v2e_emu_cs_update(V2eEmu *h, const void *frame_dev, int frame_dtype, const float *leak_randn_dev,
                      const float *shot_rand_dev, void *stream);
/* counters: surround Euler iterations (one per frame; one per chunk when pixel-sharded) that ran as one cooperative
 * launch / as one kernel per step (the cooperative launch was refused, or V2E_CS_COOP=0 at the first use) */
int v2e_emu_cs_paths(V2eEmu *h, long long *coop, long long *per_step);
int v2e_emu_phase_filter(V2eEmu *h, double t_frame, double t_previous, uint64_t capacity, int do_plan,
                         void *stream);
/* per-(iteration,polarity) row counts of the frame just counted: counts_host[2*max_n]
 * (ON, OFF interleaved). Synchronises. Returns max_n in *max_n. */
int v2e_emu_read_counts(V2eEmu *h, int32_t *max_n, uint32_t *counts_host, int counts_cap,
                        void *stream);
/* phase 2 (rng_mode 0, shot noise on): flags from the uploaded uniform field
 * (emulator_utils.py:326-349), then the emission plan. */
int v2e_emu_phase_shot(V2eEmu *h, const void *frame_dev, int frame_dtype, double t_frame,
                       double t_previous, const float *shot_rand_dev, uint64_t capacity,
                       void *stream);
/* phase 3: emission + state update (emulator.py:810-870, 906-942). */
int v2e_emu_phase_emit(V2eEmu *h, double t_frame, double t_previous, float *events_out_dev,
                       uint64_t capacity, void *stream);

/* Measurement hooks: when enabled, v2e_emu_step brackets each of its kernels with CUDA events on
 * `stream`. v2e_emu_profile_read4 synchronises and returns, for the last step, the summed device
 * time (ms) and launch count of the {update, filter, emit} kernels, and a fourth entry: the event
 * bracket around an empty kernel launched once per frame while profiling -- the floor of this
 * measurement method (launch + event processing), so that a reader can tell a kernel's duration
 * from the cost of observing it. */
int v2e_emu_profile(V2eEmu *h, int enable);
int v2e_emu_profile_read4(V2eEmu *h, float *ms_sum4, int *launches4, void *stream);

/* State access for parity probes (emulator.py:756-764 reads them by name): the device pointer of a state
 * array, for zero-copy views, or NULL when this configuration has none. which:
 * 0 lp_log_frame, 1 base_log_frame, 2 pos_thres, 3 neg_thres, 4 noise_rate_array,
 * 5 timestamp_mem, 6 cs_surround_frame (state dtype), 7 scidvs_highpass (state dtype), 8 photoreceptor_noise_arr
 * (float32), 9 scidvs_tau_arr (float32). lp, base, the surround and the high-pass have the state dtype: float64 when
 * v2e_emu_state_is_f64, else float32 (cutoff_hz == 0 without hdr, as in the reference); the others are float32. */
int v2e_emu_state_is_f64(V2eEmu *h);
void *v2e_emu_state_ptr(V2eEmu *h, int which);

/* Test hook, rng_mode 1 (not used by the stepping functions): the Philox draws of Philox frame index `frame_index`
 * for every pixel of the handle, from the same device functions the kernels use. Each non-null output is a device
 * array of H*W float32 indexed by the handle's pixel index: leak_randn the leak-jitter normal, shot_u01 the full
 * shot-noise uniform (the kernels only complete it for prefix candidates), pr_randn the photoreceptor-noise normal.
 * Leak and shot counters use rng_pixel_offset + pixel, like the kernels; the photoreceptor counters too after
 * v2e_emu_set_option(h, 1, 1), else the handle's pixel. Frame k >= 1 of a clip (frame 0 only
 * initialises) is drawn with frame_index k - 1. Asynchronous on `stream`. */
int v2e_emu_draw_noise(V2eEmu *h, uint32_t frame_index, float *leak_randn, float *shot_u01, float *pr_randn,
                       void *stream);

/* ------------------------------------------------------------------------- */
/* SuperSloMo network pieces: replace v2ecore/model.py (UNet :158-226, backWarp :229-300)
 * and the per-frame tensor code of v2ecore/slomo.py:330-444.                      */
/* ------------------------------------------------------------------------- */

/* conv2d(stride 1, "same" zero padding) + bias + LeakyReLU(slope) as a wgmma implicit GEMM
 * (model.py:72-76, 145-154, 213-225: every conv of the UNet is followed by leaky_relu(0.1)).
 * Activations: NHWC fp16, channel counts padded to a multiple of 16 (padding channels zero).
 *   x1_dev [N,H,W,C1], optional x2_dev [N,H,W,C2] (C2 = 0: none) -- the logical input is
 *   cat(x1, x2) along channels (model.py:150-153) without materialising it.
 * wgt_dev: fp16 [Cout_pad][KH*KW*(C1+C2)], K index = (r*KW+s)*(C1+C2) + c. bias_dev: fp32 [Cout_pad].
 * Cout_pad in {16,32,64} or a multiple of 128.
 * out_mode 0: out_dev fp16 NHWC with channel stride out_cstride (>= Cout_pad);
 * out_mode 1: out_dev fp32 [N,H,W,8], the first 8 output channels (network heads). */
int v2e_conv2d_lrelu_sm100(const void *x1_dev, int C1, const void *x2_dev, int C2,
                           const void *wgt_dev, const float *bias_dev, int Cout_pad, int KH, int KW,
                           int N, int H, int W, void *out_dev, int out_cstride, int out_mode,
                           int co_real, float slope, void *stream);

/* Per-tap tiles of v2e_conv2d_lrelu_sm100 (output pixels x output channels per CTA). AUTO: the tile
 * v2e_conv_pick_tile chooses for the layer on the current device, what v2e_conv2d_lrelu_sm100 and the SloMo
 * networks run (the multicast argument is then ignored). LEGACY: 128 x min(Cout_pad, 128). The wide tiles need
 * 64-channel slabs (C1, C2 multiples of 64), fp16 output (out_mode 0) and Cout_pad a multiple of their width; with
 * multicast != 0 their CTAs run in pairs (clusters of 2) that share one weight slab per stage. Every tile gives the
 * same output bit for bit. */
enum {
    V2E_CONV_TILE_AUTO = -1,
    V2E_CONV_TILE_LEGACY = 0,
    V2E_CONV_TILE_256x128 = 1,        /* 16x16 pixels x 128 channels */
    V2E_CONV_TILE_128x256 = 2         /* 8x16 pixels x 256 channels */
};
int v2e_conv2d_lrelu_sm100_tile(const void *x1_dev, int C1, const void *x2_dev, int C2,
                                const void *wgt_dev, const float *bias_dev, int Cout_pad, int KH, int KW,
                                int N, int H, int W, void *out_dev, int out_cstride, int out_mode,
                                int co_real, float slope, int tile, int multicast, void *stream);
/* The tile AUTO picks for a layer on a device with n_sms SMs (wave-aware cost; no GPU needed). */
int v2e_conv_pick_tile(int C1, int C2, int Cout_pad, int KH, int KW, int N, int H, int W, int n_sms);

/* Same operation through the strip kernel (full-resolution layers: W >= 128, Cout_pad <= 128, the
 * whole weight tensor resident in shared memory): a CTA walks down a 128-pixel-wide column strip with a
 * ring of input rows in shared memory; one new input row per output row, filter taps are descriptor
 * offsets. wgt_row_dev: fp16 [slabs][KH*KW][Cout_pad][KC], slabs = (C1+C2)/KC, KC from
 * v2e_conv_strip_pick_kc (0 = the layer does not qualify). */
int v2e_conv2d_lrelu_sm100_strip(const void *x1_dev, int C1, const void *x2_dev, int C2,
                                 const void *wgt_row_dev, const float *bias_dev, int Cout_pad, int KH,
                                 int KW, int N, int H, int W, void *out_dev, int out_cstride,
                                 int out_mode, int co_real, float slope, void *stream);
int v2e_conv_strip_pick_kc(int C1, int C2, int Cout_pad, int KH, int KW, int W);

/* conv2d 3x3 (+bias +LeakyReLU) over the x2 bilinear up-sampling (align_corners=False) of x_low, i.e. the first
 * convolution of an up block (model.py:140-147: interpolate -> conv1 -> leaky_relu) WITHOUT materialising the
 * up-sampled tensor: the up-sampling is folded into four phase-specific 3x3 filters over the low-resolution
 * tensor (v2e_conv_up2_fold_weights), a 2-pixel frame is rewritten by a direct kernel.
 *   x_low_dev [N, H_out/2, W_out/2, C] fp16 NHWC, C a multiple of 64; out_dev [N, H_out, W_out, out_cstride] fp16.
 *   wgt_fold_dev: output of v2e_conv_up2_fold_weights copied to the device; wgt_plain_dev: the layout of
 *   v2e_conv2d_lrelu_sm100 ([Cout_pad][9*C]), used for the frame. Cout_pad must be 32, 0 <= slope <= 1.
 * v2e_conv_up2_supported_c returns 1 when a layer qualifies (weights resident in shared memory). */
int v2e_conv2d_up2_lrelu_sm100(const void *x_low_dev, int C, const void *wgt_fold_dev, const void *wgt_plain_dev,
                               const float *bias_dev, int Cout_pad, int N, int H_out, int W_out, void *out_dev,
                               int out_cstride, float slope, void *stream);
/* w_host: float32 [cout][cin][3][3]; out_host: fp16 [C_pad/64][2][3][6][Cout_pad][64] (host buffers). */
int v2e_conv_up2_fold_weights(const float *w_host, int cout, int cin, int Cout_pad, int C_pad, void *out_host);
int v2e_conv_up2_supported_c(int C, int Cout_pad, int W_out);

/* The 23 convolutions of one UNet (model.py:184-196) in forward order: conv1, conv2,
 * down1..down5 {conv1, conv2}, up1..up5 {conv1, conv2}, conv3. Host pointers to the float32
 * tensors of the reference's state_dict ([Cout][Cin][KH][KW] weights, [Cout] biases), i.e. what
 * torch.load(ckpt)['state_dictFC' / 'state_dictAT'] holds (slomo.py:225-227). */
typedef struct V2eUNetWeights {
    const float *w[23];
    const float *b[23];
} V2eUNetWeights;

typedef struct V2eSlomo V2eSlomo;

/* H, W: network resolution (multiples of 32, dataloader.py:122-123). Packs the weights to fp16
 * on the device and allocates activations for max_batch frame pairs. Synchronous. */
int v2e_slomo_create(int H, int W, int max_batch, const V2eUNetWeights *flow,
                     const V2eUNetWeights *interp, V2eSlomo **out);
int v2e_slomo_destroy(V2eSlomo *h);
/* frames_u8_dev: [B+1][H][W] consecutive source frames at network resolution. Normalises them
 * (slomo.py:148-162, CUDA branch: x/255 - 0.428) and runs the flow UNet for the B pairs
 * (slomo.py:338-345). Enqueue only. */
int v2e_slomo_set_pairs(V2eSlomo *h, const uint8_t *frames_u8_dev, int B, void *stream);
/* max over the batch of the flow magnitudes (slomo.py:358-366). Synchronises. */
int v2e_slomo_max_flow(V2eSlomo *h, float *max_speed_host, void *stream);
/* One intermediate frame per pair at fraction t in (0,1) (slomo.py:404-437).
 * out_u8_dev: [B][H][W] = uint8((Ft_p + 0.428) * 255) as torchvision's ToPILImage computes it;
 * out_f32_dev: optional [B][H][W] float32 Ft_p before quantisation (parity probe), may be NULL. */
int v2e_slomo_interp(V2eSlomo *h, double t, uint8_t *out_u8_dev, float *out_f32_dev, void *stream);
/* fp16 range guard: *nonfinite_host = 1 if, since the last call, any fp32 network head (flows, residual flows,
 * visibility) or blended pixel was inf / nan -- what fp16 activations beyond 65504 turn into. Resets the flag.
 * Synchronises. The Python class raises FloatingPointError on it (no silent garbage frames). */
int v2e_slomo_check_finite(V2eSlomo *h, int *nonfinite_host, void *stream);
/* option 0: force the per-tap convolution kernel for every layer; option 1: do not fold the up-sampling into
 * up5.conv1; option 2: do not fuse the average pools into the epilogues of conv2 / down1.conv2 (A/B measurements
 * and bit-identity tests: the fused pool must equal the separate kernel exactly), value 0/1;
 * option 3: plan every later launch (per-tap tile pick, strip and up-sampling grids and their segmentation) as if
 * the device had `value` SMs, 1 <= value <= the device's count; 0 restores the device's count (the default). A test
 * hook: the outputs must not depend on it. Other values: V2E_E_INVALID. */
int v2e_slomo_set_option(V2eSlomo *h, int option, int value);
/* Measurement hooks: bracket every convolution launch with CUDA events; profile_read synchronises
 * and returns the summed device time, the number of launches and their algorithmic FLOPs
 * (2 x MACs over the unpadded channel counts) since the last read. */
int v2e_slomo_profile(V2eSlomo *h, int enable);
int v2e_slomo_profile_read(V2eSlomo *h, float *conv_ms, int *conv_launches, double *conv_flops, void *stream);
/* Same, split by UNet layer (forward order of V2eUNetWeights; flow and interpolation networks summed): device
 * time, launches and algorithmic FLOPs of each of the 23 layers since the last read; the totals are optional. */
int v2e_slomo_profile_read_layers(V2eSlomo *h, float *ms23, int *launches23, double *flops23, float *conv_ms,
                                  int *conv_launches, double *conv_flops, void *stream);
/* device pointers of the last flow / interpolation network outputs, fp32 [B][H][W][8] */
const float *v2e_slomo_flow_ptr(V2eSlomo *h);
const float *v2e_slomo_intrp_ptr(V2eSlomo *h);
/* Test hooks: read-only views of the engine's internals, for checking every layer in its production
 * configuration. Neither adds a launch or a synchronisation to set_pairs / interp.
 * v2e_slomo_buffer_ptr: device pointer of an activation buffer (NHWC fp16, sized for max_batch; img: fp32
 * [B+1][H][W]). index selects the level l (0..4, 1/2^(l+1) resolution) of pool / da / s and the up block k
 * (0..4, 1/2^(4-k) resolution) of up / ua / ub; it is ignored otherwise. The flow and interpolation networks share
 * the buffers, and up[k] is left stale when up block k ran the fused up-sampling convolution. NULL: unknown name. */
typedef enum V2eSlomoBuffer {
    V2E_SLOMO_BUF_IN16 = 0, V2E_SLOMO_BUF_X0 = 1, V2E_SLOMO_BUF_S1 = 2, V2E_SLOMO_BUF_POOL = 3, V2E_SLOMO_BUF_DA = 4,
    V2E_SLOMO_BUF_S = 5, V2E_SLOMO_BUF_UP = 6, V2E_SLOMO_BUF_UA = 7, V2E_SLOMO_BUF_UB = 8, V2E_SLOMO_BUF_IMG = 9
} V2eSlomoBuffer;
void *v2e_slomo_buffer_ptr(V2eSlomo *h, int which, int index);
/* Which kernel computed layer 0..22 (forward order of V2eUNetWeights) of net 0 (flow) / 1 (interpolation) in its
 * last forward pass, as launched (options and V2E_NO_FUSED_* overrides applied). < 0: bad argument. */
typedef enum V2eSlomoKernel {
    V2E_SLOMO_KERNEL_NONE = 0,        /* not run yet */
    V2E_SLOMO_KERNEL_TAP = 1,         /* per-tap implicit GEMM (v2e_conv2d_lrelu_sm100) */
    V2E_SLOMO_KERNEL_STRIP = 2,       /* strip kernel (v2e_conv2d_lrelu_sm100_strip) */
    V2E_SLOMO_KERNEL_STRIP_POOL = 3,  /* strip kernel writing the following 2x2 average pool from its epilogue */
    V2E_SLOMO_KERNEL_UP2 = 4          /* fused x2 bilinear up-sampling convolution (v2e_conv2d_up2_lrelu_sm100) */
} V2eSlomoKernel;
int v2e_slomo_layer_kernel(V2eSlomo *h, int net, int layer);

/* Pillow-exact 8-bit resampling of 'L' images (Pillow Resample.c; dataloader.py:142 uses LANCZOS,
 * slomo.py:438 BILINEAR). filter: 0 = BILINEAR, 1 = LANCZOS. Images are [n][h][w] uint8. */
typedef struct V2eResizer V2eResizer;
int v2e_resize_create(int src_w, int src_h, int dst_w, int dst_h, int filter, int max_images,
                      V2eResizer **out);
int v2e_resize_destroy(V2eResizer *r);
int v2e_resize_run(V2eResizer *r, const uint8_t *src_dev, uint8_t *dst_dev, int n_images, void *stream);
/* Same, destination image i at dst_dev + i * dst_image_stride bytes (>= dst_w * dst_h): the interpolated frame of
 * pair b at time step k goes straight to its place U*b + k of the output clip (slomo.py:440), no gather copy. */
int v2e_resize_run_strided(V2eResizer *r, const uint8_t *src_dev, uint8_t *dst_dev, int n_images,
                           long dst_image_stride, void *stream);

/* ------------------------------------------------------------------------- */
/* Stage-1 input preparation (SURVEY.md 8f rank 2; v2e.py:687-737): crop, cv2.resize(INTER_AREA), BGR -> luma for
 * 8-bit frames, bit-exact with OpenCV 4.x. src_dev: [n][src_h][src_w][channels] uint8 (channels 1 = grey, 3 = BGR as
 * cv2 delivers); crop_* as v2e's --crop (pixels removed at the left / right / top / bottom, <= 0: none);
 * dst_dev: [n][dst_h][dst_w] uint8 luma -- what v2e.py:733-737 saves as source frames. Shrinking (or equal size)
 * only: OpenCV treats an INTER_AREA enlargement as bilinear, which is not built (V2E_E_UNSUPPORTED). */
/* ------------------------------------------------------------------------- */
typedef struct V2ePrep V2ePrep;
int v2e_prep_create(int src_w, int src_h, int channels, int crop_left, int crop_right, int crop_top, int crop_bottom,
                    int dst_w, int dst_h, V2ePrep **out);
int v2e_prep_destroy(V2ePrep *h);
int v2e_prep_run(V2ePrep *h, const uint8_t *src_dev, int n_images, uint8_t *dst_dev, void *stream);

/* ------------------------------------------------------------------------- */
/* Event-sink row conversions (SURVEY.md 8f): packed rows [t, x, y, p] float32 -> what the reference's writers
 * store. events_dev: [n][4] float32, 16-byte aligned. Enqueue only.                                             */
/* ------------------------------------------------------------------------- */
/* HDF5 "events" dataset rows (emulator.py:953-959): rows_dev [n][4] uint32 = [t * 1e6 (float32 product,
 * truncated), x, y, p with -1 -> 0]. */
int v2e_events_to_h5_rows(const float *events_dev, uint64_t n, uint32_t *rows_dev, void *stream);
/* AEDAT-2.0 body (v2ecore/output/aedat2_output.py:133-168): words_dev [2n] uint32 = per event the address
 * x << x_shift | y << y_shift | p01 << pol_shift (x, y flipped about size-1 when asked) and the int32 microsecond
 * timestamp, both big endian, ready for file.write(). The shifts / flips of the three supported cameras are in
 * aedat2_output.py:38-60. labels_dev (nullable): [n] uint8, 0 = shot noise; a noise row's address ORs in the
 * special-event bit 1 << 10 (label_signal_noise, :154-158), even where that bit overlaps x (640x480).
 * n_on_dev (nullable): += number of ON events (numOnEvents, :176). */
int v2e_events_to_aedat2(const float *events_dev, uint64_t n, int size_x, int size_y, int x_shift, int y_shift,
                         int pol_shift, int flip_x, int flip_y, const uint8_t *labels_dev, uint32_t *words_dev,
                         uint64_t *n_on_dev, void *stream);
/* DVS text body (RPG events.txt, v2ecore/output/ae_text_output.py:89-101), one line per row:
 *   '{} {} {} {}\n'.format(float(t), int(x), int(y), int((p + 1) / 2))
 * where float(t) is Python's repr() of the float32 timestamp widened to double (shortest round trip: "0.1000000015"
 * style 17 digits, "4.8999998398358e-05" below 1e-4, "1e+16" from 1e16 up, "0.0", "inf", "nan"), x, y and p are cast
 * to int32 by truncation and (p + 1) / 2 is evaluated in float32. labels_dev (nullable): [n] uint8; when given, each
 * line ends ' {label}' before the newline (label_signal_noise: 1 = signal, 0 = shot noise). Lines are at most 64 bytes.
 * Two calls:
 *   v2e_events_to_text_layout: block_offsets_dev [v2e_events_to_text_scratch(n)] uint64 receives the byte offset of
 *     every 256-row block and, in its last entry, the total length of the body. Read that entry (the only
 *     synchronisation) to size text_dev.
 *   v2e_events_to_text: writes the body, total bytes, to text_dev (no alignment needed).  */
uint64_t v2e_events_to_text_scratch(uint64_t n);
int v2e_events_to_text_layout(const float *events_dev, uint64_t n, const uint8_t *labels_dev,
                              uint64_t *block_offsets_dev, void *stream);
int v2e_events_to_text(const float *events_dev, uint64_t n, const uint8_t *labels_dev,
                       const uint64_t *block_offsets_dev, uint8_t *text_dev, void *stream);
/* Signal / shot-noise labels of a chunk of frames (emulator.py:889-923): frame f holds rows
 * [offsets_dev[f], offsets_dev[f + 1]) and its last n_noise_dev[f] rows are shot noise (V2eFrameInfo n_shot_on +
 * n_shot_off: every path emits them after the frame's signal rows). labels_dev [n_rows] uint8 = 1 for signal, 0 for
 * noise; n_rows = offsets_dev[n_frames]. */
int v2e_signnoise_labels(const int64_t *offsets_dev, const uint32_t *n_noise_dev, int n_frames, uint64_t n_rows,
                         uint8_t *labels_dev, void *stream);

/* ------------------------------------------------------------------------- */
/* DVS frame rendering (SURVEY.md 8f rank 4): the histogram of EventRenderer.render_events_to_frames
 * (v2ecore/renderer.py:392-430, v2ecore/v2e_utils.py:474-486). Frame f takes the event rows
 * [starts_dev[f], ends_dev[f]) of events_dev ([n][4] float32 [t, x, y, p]; slices may overlap, as the reference's do):
 * ON minus OFF per pixel, clipped to +-full_scale_count. acc_dev: [n_frames][H][W] int32 scratch;
 * frames_f64_dev (nullable): (frame + fs) / (2 fs) float64, what the reference returns; frames_u8_dev (nullable):
 * uint8(img * 255), what it writes to the AVI (renderer.py:345-347). max_events_per_frame sizes the grid. */
/* ------------------------------------------------------------------------- */
/* ExposureMode.AREA_COUNT (renderer.py:246-261): frame slices of one packet -- a frame ends when a cell of
 * area_dimension x area_dimension pixels has collected area_count events. counts_dev: [cells_w][cells_h] int32,
 * persistent between packets (zero it once). Sequential by definition: one thread walks the packet.
 * *n_frames_dev = finished frames (their slices in starts_dev / ends_dev), or -1 if more than max_frames. */
int v2e_render_area_scan(const float *events_dev, int64_t n, int area_dimension, int area_count, int cells_w, int cells_h,
                         int32_t *counts_dev, int64_t *starts_dev, int64_t *ends_dev, int max_frames,
                         int32_t *n_frames_dev, void *stream);
int v2e_render_frames(const float *events_dev, const int64_t *starts_dev, const int64_t *ends_dev, int n_frames,
                      int64_t max_events_per_frame, int height, int width, int full_scale_count, int32_t *acc_dev,
                      double *frames_f64_dev, uint8_t *frames_u8_dev, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* V2E_B200_H */
