/*
 * dspi_b200.h — C ABI of the CUDA-native (H100, sm_90a) DSPi signal-chain engine.
 *
 * Drop-in boundary for the per-sample DSP hot path of WeebLabs/DSPi
 * (SURVEY.md §8b).  The reference has no FFI layer: the path is reached through
 * plain C functions over global arrays.  Every entry point below names the
 * reference function (file:line under /root/reference/firmware/DSPi) whose role
 * it takes for MANY independent channels / device instances at once.
 *
 * Conventions
 *   - plain pointers and sizes only; records are byte-for-byte the reference's
 *     (sizes asserted below; checked against the compiled reference in tests);
 *   - every function returns 0 on success or a negative DSPI_E* code, never
 *     aborts; dspi_last_error() gives a per-thread message;
 *   - an engine belongs to one CUDA device and one stream; calls on one engine
 *     must be serialised by the caller (the firmware's single processing
 *     thread, main.c:743), different engines are independent;
 *   - there is NO CPU fallback: if no sm_90 device is present, create fails
 *     with DSPI_ENODEV.
 */
#ifndef DSPI_B200_H
#define DSPI_B200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DSPI_MAX_BANDS        12   /* config.h:329 MAX_BANDS — row stride of filters[][]          */
#define DSPI_NUM_BANDS        10   /* dsp_pipeline.c:36-44 channel_band_counts                     */
#define DSPI_LA_SAMPLES      480   /* leveller.h:36                                                */
#define DSPI_PACKET_MAX      192   /* usb_audio.c:273,588                                          */

enum {
    DSPI_OK       = 0,
    DSPI_EINVAL   = -22,   /* bad argument                                   */
    DSPI_ENOMEM   = -12,   /* host or device allocation failed               */
    DSPI_ENODEV   = -19,   /* no sm_90 CUDA device / CUDA runtime unusable   */
    DSPI_ECUDA    = -5,    /* a CUDA call failed (message in dspi_last_error) */
    DSPI_ERANGE   = -34    /* index / size outside the engine's shape        */
};

/* arithmetic of an engine (SURVEY.md §8c "Build flags for the oracle") */
enum {
    DSPI_ARITH_F32_FUSED  = 0,  /* RP2350 float path as arm-none-eabi-gcc contracts it (VFMA) */
    DSPI_ARITH_F32_STRICT = 1,  /* RP2350 float path, every operation rounded separately       */
    DSPI_ARITH_Q28        = 2   /* RP2040 Q28 fixed point (dsp_process_rp2040.S), bit-exact    */
};

/* filter types, config.h:440-443 */
enum { DSPI_FILTER_FLAT = 0, DSPI_FILTER_PEAKING = 1, DSPI_FILTER_LOWSHELF = 2,
       DSPI_FILTER_HIGHSHELF = 3, DSPI_FILTER_LOWPASS = 4, DSPI_FILTER_HIGHPASS = 5 };

/* ---- records shared with the reference (same bytes) ----------------------- */

/* Biquad, RP2350 build — config.h:418-431 (68 bytes) */
typedef struct {
    float b0, b1, b2, a1, a2;
    float s1, s2;
    float sva1, sva2, sva3;
    float svm0, svm1, svm2;
    float svic1eq, svic2eq;
    uint32_t svf_type;
    uint8_t use_svf;
    uint8_t bypass;
} dspi_biquad_f32;

/* Biquad, RP2040 build — config.h:433-437, dsp_process_rp2040.S:6-14 (32 bytes) */
typedef struct {
    int32_t b0, b1, b2, a1, a2;
    int32_t s1, s2;
    uint8_t bypass;
} dspi_biquad_q28;

/* EqParamPacket — config.h:445-453 (packed, 16 bytes) */
typedef struct __attribute__((packed)) {
    uint8_t channel, band, type, reserved;
    float freq, Q, gain_db;
} dspi_eq_param;

#ifdef __cplusplus
static_assert(sizeof(dspi_biquad_f32) == 68 && sizeof(dspi_biquad_q28) == 32 && sizeof(dspi_eq_param) == 16, "reference layouts");
#else
_Static_assert(sizeof(dspi_biquad_f32) == 68 && sizeof(dspi_biquad_q28) == 32 && sizeof(dspi_eq_param) == 16, "reference layouts");
#endif

/* ---- library ---------------------------------------------------------------- */
const char *dspi_last_error(void);
/* number of visible CUDA devices that can run the engine (compute capability 10.x) */
int dspi_device_count(void);

/* ---- host-side parameter API (no GPU needed) -------------------------------- */
/* dsp_compute_coefficients(), dsp_pipeline.c:61-175.  `p` is clamped in place
 * exactly like the reference does (:78-81).  The float store keeps SVF/biquad
 * path selection and the state reset on a path flip (:87-92). */
void dspi_compute_coefficients_f32(dspi_eq_param *p, dspi_biquad_f32 *bq, float sample_rate);
void dspi_compute_coefficients_q28(dspi_eq_param *p, dspi_biquad_q28 *bq, float sample_rate);

/* ---- EQ engine: many independent cascades ---------------------------------- */
/* One row of filters[][] per channel: dsp_process_channel_block()
 * (float dsp_pipeline.c:281-365, Q28 dsp_process_rp2040.S:225-394) applied to
 * n_channels channels in one launch. */
typedef struct dspi_eq dspi_eq;

typedef struct {
    uint32_t arith;          /* DSPI_ARITH_*                                          */
    uint32_t n_channels;     /* independent EQ channels (rows of filters[][])         */
    uint32_t n_bands;        /* bands processed per channel, 1..DSPI_MAX_BANDS (10)   */
    int32_t  device;         /* CUDA device ordinal                                   */
    uint32_t flags;          /* 0                                                     */
} dspi_eq_desc;

/* A new engine holds, in every band of every channel, the record dsp_compute_coefficients() makes of a flat recipe
 * (dsp_init_default_filters(), dsp_pipeline.c:177-199): bypass set, b0 = 1, all other coefficients and the state zero.
 * It passes audio through until coefficients are uploaded, and dspi_eq_set_param on it gives a one-band EQ.  Chain
 * engines start the same way: instances whose biquads were never uploaded run with every filter row bypassed. */
int dspi_eq_create(dspi_eq **out, const dspi_eq_desc *desc);
int dspi_eq_destroy(dspi_eq *e);

/* Coefficients + state in the reference's own layout:
 * biquads[n][DSPI_MAX_BANDS] of dspi_biquad_f32 (float engines) or
 * dspi_biquad_q28 (Q28 engines) — i.e. n rows of the firmware's filters[][].
 * upload == writing filters[][] between packets (main.c:843-856 semantics:
 * takes effect for the next process call); download returns coefficients and
 * the CURRENT filter state, so a run can be checkpointed bit-exactly. */
int dspi_eq_upload_biquads(dspi_eq *e, uint32_t ch0, uint32_t n, const void *biquads);
int dspi_eq_download_biquads(dspi_eq *e, uint32_t ch0, uint32_t n, void *biquads);
/* REQ_SET_EQ_PARAM path (usb_audio.c:1641-1649 + main.c:826-857): recompute one
 * band of one channel from its recipe and upload it.  p->channel is ignored
 * (8 bits on the wire); `channel` selects the row, p->band the band. */
int dspi_eq_set_param(dspi_eq *e, uint32_t channel, dspi_eq_param *p, float sample_rate);
/* Mass reconfiguration (SURVEY 8 f-1, device part): dsp_compute_coefficients() for all 12 bands of channels
 * [ch0, ch0 + n) ON THE GPU, straight into the engine's stores - recipes[n][DSPI_MAX_BANDS] (host memory) are
 * clamped in place like the reference does (dsp_pipeline.c:78-81); filter state is kept unless a band's
 * topology flips (:87-92).  Arithmetic is the reference's float arithmetic operation by operation; its libm
 * calls (powf, tanf, sinf, cosf) are evaluated in double and rounded once ("libm policy", DESIGN.md 6), which
 * can differ from a host libm's float functions in a last bit - use dspi_compute_coefficients_* +
 * dspi_eq_upload_biquads when coefficients must be those of a particular host libm. */
int dspi_eq_set_params_device(dspi_eq *e, uint32_t ch0, uint32_t n, dspi_eq_param *recipes, float sample_rate);

/* Process T samples of every channel, in place.
 *   *_device: samples is a DEVICE pointer, channel-major [n_channels][ld]
 *             (row stride `ld` elements, float32 or int32); asynchronous on the
 *             engine's stream.
 *   *_host:   samples is a HOST pointer [n_channels][T]; copies in, processes,
 *             copies out (chunked, overlapped) and returns when the data is back.
 *             Pinned memory (dspi_host_alloc) gives full PCIe bandwidth.
 * Equivalent reference loop: for each channel, dsp_process_channel_block(
 * filters[ch], samples[ch], T, ch) — packet size does not change the values. */
int dspi_eq_process_device(dspi_eq *e, void *d_samples, uint32_t T, uint32_t ld);
/* The same for channels [ch0, ch0 + n) only: d_rows points at the row of channel ch0 ([n][ld], device memory); ch0 must be a
 * multiple of 64, n may be any count.  Channels outside [ch0, ch0 + n) are left untouched: their samples and their filter
 * state.  For callers that stream a large block through in pieces (dspi_b200/sharding.py pipelines NCCL transfers
 * against it).  Asynchronous on the engine's stream. */
int dspi_eq_process_device_range(dspi_eq *e, void *d_rows, uint32_t T, uint32_t ld, uint32_t ch0, uint32_t n);
/* Host block: staged through the device in 48 MiB channel chunks (DSPI_HOST_CHUNK_MB in the environment overrides). */
int dspi_eq_process_host(dspi_eq *e, void *h_samples, uint32_t T);
int dspi_eq_sync(dspi_eq *e);
/* cudaStream_t of the engine (so callers can order their own work / events) */
void *dspi_eq_stream(dspi_eq *e);
/* number of kernel launches issued by this engine so far */
uint64_t dspi_eq_launch_count(dspi_eq *e);
/* Which K1/K2 kernel the next dspi_eq_process_* call will run, as text ("jit sig=0x...", "aot
 * straight-line biquad", "aot generic ...").  Float engines whose channels share one band-topology
 * vector get a kernel compiled for that vector at run time (NVRTC); this call triggers that
 * compilation if it is pending.  Results never depend on the choice.  No reference counterpart. */
int dspi_eq_kernel_info(dspi_eq *e, char *buf, size_t cap);

/* ---- EQ engine over several GPUs of one box, one process (SURVEY 8b `devices[], n_devices`, 8e) ------ */
/* Channels shard into contiguous ranges, one per listed device (dspi_eqx_shard_range: 64-channel boundaries); all
 * coefficients and filter state of a range stay on its owner and no data is exchanged between devices - the firmware's
 * own two-core split is the same idea (disjoint output ranges, config.h:350-357).  Results are bit-identical to a
 * single engine over all channels.  upload / download address channels of the whole group. */
#define DSPI_MAX_DEVICES 8
typedef struct dspi_eqx dspi_eqx;
typedef struct {
    uint32_t arith;                     /* DSPI_ARITH_*                                     */
    uint32_t n_channels;                /* over the whole group                             */
    uint32_t n_bands;
    uint32_t n_devices;                 /* 1..DSPI_MAX_DEVICES                              */
    int32_t  devices[DSPI_MAX_DEVICES]; /* CUDA ordinals; devices[0] is the root            */
    uint32_t flags;                     /* 0                                                */
} dspi_eqx_desc;
int dspi_eqx_create(dspi_eqx **out, const dspi_eqx_desc *desc);
int dspi_eqx_destroy(dspi_eqx *x);
int dspi_eqx_shard_range(uint32_t n_channels, uint32_t n_devices, uint32_t k, uint32_t *lo, uint32_t *hi);
int dspi_eqx_upload_biquads(dspi_eqx *x, uint32_t ch0, uint32_t n, const void *biquads);
int dspi_eqx_download_biquads(dspi_eqx *x, uint32_t ch0, uint32_t n, void *biquads);
/* samples [n_channels][T] in HOST memory (pinned: dspi_host_alloc): every device runs its staged PCIe pipeline on its
 * rows concurrently; returns when all rows are back. */
int dspi_eqx_process_host(dspi_eqx *x, void *h_samples, uint32_t T);
/* samples [n_channels][T] resident on devices[0]: the root processes its rows in place, the other devices pull theirs
 * over NVLink (peer access), process and push them back, chunked so that transfers in both directions overlap the
 * kernels.  Returns when the block on the root is complete. */
int dspi_eqx_process_root(dspi_eqx *x, void *d_samples_on_root, uint32_t T, uint32_t ld);
uint64_t dspi_eqx_launch_count(dspi_eqx *x);

/* ---- one rank per GPU: frames that originate on one rank, over NCCL (SURVEY 8e) ------------------------- */
/* Multi-PROCESS form of dspi_eqx_process_root: every rank owns an EQ engine over its shard
 * [lo_r, hi_r) = dspi_eqx_shard_range(total, world, r); the block [total][T] lives on the root rank.  dspi_sg_process
 * scatters it in row chunks with grouped ncclSend / ncclRecv: step j carries chunk j out and chunk j-L back in the same
 * NCCL group (both NVLink directions busy) while the engines work on the chunks in between, each chunk's kernel on a
 * stream of its own (a cascade kernel takes as long as its rows are long however few rows it gets, but a chunk fills only
 * a few SMs); the results end up in the root's block.  n_chunks = 0 lets the library choose chunk count and lag from the
 * transfer / kernel time ratio.  libnccl.so.2 is dlopen'ed at first use.  The 128-byte unique id comes from
 * dspi_nccl_unique_id() on one rank and is
 * handed to the others by the caller (dspi_b200/sharding.py broadcasts it with torch.distributed). */
typedef struct dspi_sg dspi_sg;
int dspi_nccl_unique_id(void *id128);
int dspi_sg_create(dspi_sg **out, dspi_eq *engine, int device, const void *id128, int rank, int world, int root);
int dspi_sg_destroy(dspi_sg *g);
int dspi_sg_process(dspi_sg *g, void *d_full_on_root, uint32_t total_channels, uint32_t T, uint32_t n_chunks);

/* ---- full signal chain: many independent DSPi device instances ------------------------------ */
/* One instance = process_audio_packet() of one RP2350-shape device (usb_audio.c:500-1317, float
 * pipeline :560-967, single-core branch :874-960): 2 inputs -> preamp -> loudness -> master EQ ->
 * leveller -> crossfeed -> 2x9 matrix -> per-output EQ, gain, delay -> 4 S/PDIF stereo pairs
 * (24-bit words) + the PDM sub through the 2nd-order delta-sigma modulator (pdm_generator.c:351-397). */
#define DSPI_CHAIN_OUTPUTS      9    /* config.h:321 NUM_OUTPUT_CHANNELS                            */
#define DSPI_CHAIN_EQ_CHANNELS 11    /* config.h:322 NUM_CHANNELS: master L, R, Out1..9             */
#define DSPI_CHAIN_MAX_DELAY 4096    /* config.h:84  MAX_DELAY_SAMPLES                              */

/* LoudnessCoeffs (RP2350), loudness.h:11-17 (28 bytes) */
typedef struct { float sva1, sva2, sva3, svm0, svm1, svm2; uint8_t bypass; } dspi_loudness_coeffs_f32;
/* CrossfeedState (RP2350), crossfeed.h:46-51 (28 bytes) */
typedef struct { float lp_a0, lp_b1, lp_state_L, lp_state_R, ap_a, ap_state_L, ap_state_R; } dspi_crossfeed_state_f32;
/* LevellerCoeffs, leveller.h:81-99 (36 bytes) */
typedef struct {
    float alpha_rms, alpha_attack, alpha_release;
    float threshold_db, ratio, knee_width_db, makeup_db, gate_threshold_db, max_gain_db;
} dspi_leveller_coeffs;
/* MatrixCrosspoint / OutputChannel / MatrixMixer, config.h:383-406 (12 / 20 / 396 bytes) */
typedef struct __attribute__((packed)) { uint8_t enabled, phase_invert, reserved[2]; float gain_db, gain_linear; } dspi_matrix_crosspoint;
typedef struct __attribute__((packed)) { uint8_t enabled, mute, reserved[2]; float gain_db, gain_linear, delay_ms; int32_t delay_samples; } dspi_output_channel;
typedef struct {
    dspi_matrix_crosspoint crosspoints[2][DSPI_CHAIN_OUTPUTS];
    dspi_output_channel outputs[DSPI_CHAIN_OUTPUTS];
} dspi_matrix_mixer_f32;
/* SystemStatusPacket, config.h:455-460 (26 bytes): peaks are Q15, clip_flags sticky */
typedef struct { uint16_t peaks[DSPI_CHAIN_EQ_CHANNELS]; uint8_t cpu0_load, cpu1_load; uint16_t clip_flags; } dspi_status;

/* Everything process_audio_packet() reads besides filters[][]: the globals of usb_audio.c:148-211
 * for one instance, with the coefficient records in the reference's own layouts. */
typedef struct {
    uint8_t bypass_master_eq;        /* usb_audio.c:48                                             */
    uint8_t loudness_enabled;        /* loud_on && current_loudness_coeffs != NULL, :579-580        */
    uint8_t crossfeed_enabled;       /* !crossfeed_bypassed                                         */
    uint8_t leveller_enabled;        /* !leveller_bypassed                                          */
    uint8_t host_mute;               /* audio_state.mute                                            */
    uint8_t leveller_lookahead;      /* leveller_config.lookahead                                   */
    uint8_t reserved0[2];
    int16_t host_vol_mul;            /* audio_state.vol_mul - an int16: 0 dB gives -32768 (quirk)   */
    int16_t reserved1;
    float preset_mute_gain;          /* update_preset_mute_envelope(), 1.0 when no preset loads     */
    float master_volume_linear;      /* usb_audio.c:161                                             */
    float preamp_linear[2];          /* global_preamp_linear[]                                      */
    dspi_loudness_coeffs_f32 loudness[2];   /* the selected row of loudness_active_table            */
    dspi_crossfeed_state_f32 crossfeed;     /* coefficients AND state (crossfeed_compute_coefficients clears state) */
    dspi_leveller_coeffs leveller;
    dspi_matrix_mixer_f32 matrix;    /* outputs[o].delay_samples is channel_delay_samples[o]        */
} dspi_chain_params_f32;

#ifdef __cplusplus
static_assert(sizeof(dspi_loudness_coeffs_f32) == 28 && sizeof(dspi_crossfeed_state_f32) == 28 && sizeof(dspi_leveller_coeffs) == 36 &&
              sizeof(dspi_matrix_mixer_f32) == 396 && sizeof(dspi_status) == 26, "reference layouts");
#else
_Static_assert(sizeof(dspi_loudness_coeffs_f32) == 28 && sizeof(dspi_crossfeed_state_f32) == 28 && sizeof(dspi_leveller_coeffs) == 36 &&
               sizeof(dspi_matrix_mixer_f32) == 396 && sizeof(dspi_status) == 26, "reference layouts");
#endif

/* CrossfeedConfig, crossfeed.h:26-32 (12 bytes) and LevellerConfig, leveller.h:59-66 (24 bytes) */
typedef struct { uint8_t enabled, itd_enabled, preset; float custom_fc, custom_feed_db; } dspi_crossfeed_config;
typedef struct { uint8_t enabled; float amount; uint8_t speed; float max_gain_db; uint8_t lookahead; float gate_threshold_db; } dspi_leveller_config;
/* host-side parameter functions of the chain (no GPU needed; host libm, like the firmware's main loop):
 * crossfeed_compute_coefficients() crossfeed.c:35-127 (clears the filter state),
 * leveller_compute_coefficients() leveller.c:42-89, loudness_recompute_table() loudness.c:169-217
 * (table[volume step 0..60][low shelf, high shelf]) and audio_set_volume() usb_audio.c:428-440
 * (returns audio_state.vol_mul and the loudness table row). */
void dspi_crossfeed_compute_coefficients_f32(dspi_crossfeed_state_f32 *st, const dspi_crossfeed_config *cfg, float sample_rate);
void dspi_leveller_compute_coefficients(dspi_leveller_coeffs *out, const dspi_leveller_config *cfg, float sample_rate);
void dspi_loudness_compute_table_f32(dspi_loudness_coeffs_f32 table[61][2], float ref_spl, float intensity_pct, float sample_rate);
int16_t dspi_host_volume(int16_t volume_8_8, uint8_t *table_index);
/* update_preamp() usb_audio.c:244-250 and update_master_volume() :255-269: dB -> the gains the packet loop reads
 * (float for the RP2350 shape, Q28 / Q15 for the RP2040 shape).  Return -1 for NaN / Inf like the firmware's guard. */
int dspi_preamp(float db, float *linear_out, int32_t *q28_out);
int dspi_master_volume(float db, float *linear_out, int32_t *q15_out);
/* The preset-mute envelope, update_preset_mute_envelope() usb_audio.c:456-498: state of one instance and its
 * per-packet step (host side; dspi_chain(q)_set_preset_mute runs the same recurrence on the device). */
typedef struct {
    uint8_t  loading;                /* preset_loading, flash_storage.c:255                          */
    uint8_t  reserved[3];
    uint32_t counter;                /* preset_mute_counter, flash_storage.c:256                     */
    float    smooth_gain;            /* preset_mute_smooth_gain, usb_audio.c:457 (1.0 = full level)  */
} dspi_preset_mute;
void  dspi_preset_mute_arm(dspi_preset_mute *m, uint32_t sample_rate_hz);    /* flash_storage.c:272-276, 347-348 */
float dspi_preset_mute_step(dspi_preset_mute *m, uint32_t sample_count, uint32_t sample_rate_hz);

typedef struct dspi_chain dspi_chain;
typedef struct {
    uint32_t arith;          /* DSPI_ARITH_F32_FUSED or DSPI_ARITH_F32_STRICT                       */
    uint32_t n_instances;
    uint32_t n_bands;        /* channel_band_counts[] value (10)                                    */
    int32_t  device;
    uint32_t max_frames;     /* most frames of one process call (sum of its packet lengths)         */
} dspi_chain_desc;

int dspi_chain_create(dspi_chain **out, const dspi_chain_desc *desc);
int dspi_chain_destroy(dspi_chain *c);
/* bulk_params_apply()-style update between packets (bulk_params.c:178-377 + main.c:1126-1162):
 * params[n] for instances [inst0, inst0+n).  Filter, delay-line, leveller and PDM state are kept; so is the crossfeed
 * filter state unless the record's crossfeed COEFFICIENTS differ from the ones in force - then the record's state rows
 * are taken, i.e. the zeros crossfeed_compute_coefficients() leaves (crossfeed.c:35-127 is the only place the firmware
 * resets that state; audio_set_volume and the mute / matrix handlers never do). */
int dspi_chain_set_params(dspi_chain *c, uint32_t inst0, uint32_t n, const dspi_chain_params_f32 *params);
/* filters[NUM_CHANNELS][MAX_BANDS] of n instances: biquads[n][11][12] (master L, R, Out1..9) */
int dspi_chain_upload_biquads(dspi_chain *c, uint32_t inst0, uint32_t n, const dspi_biquad_f32 *biquads);
int dspi_chain_download_biquads(dspi_chain *c, uint32_t inst0, uint32_t n, dspi_biquad_f32 *biquads);
/* dsp_recalculate_all_filters() for n instances on the GPU: recipes[n][11][DSPI_MAX_BANDS] = filter_recipes[][] of each
 * instance (host memory, clamped in place); see dspi_eq_set_params_device for the arithmetic and the libm policy */
int dspi_chain_set_eq_params_device(dspi_chain *c, uint32_t inst0, uint32_t n, dspi_eq_param *recipes, float sample_rate);
/* Pipeline reset of every instance: leveller state (leveller_reset_state(): envelopes and smoothed gain cleared, gains 1,
 * look-ahead buffer and index cleared), the modulator's state (pdm_processing_loop() restart path: integrators and error
 * cleared, dither seed 123456789), loudness shelf state, delay lines and their write index, and the meters (peaks and
 * sticky clip flags).  Kept: the EQ filter state (part of the biquads), the crossfeed state, the preset-mute envelope and
 * the S/PDIF transmitter state (block position and channel status, dspi_chain_set_spdif_tx).
 * Ordered after earlier asynchronous process calls on the engine stream. */
int dspi_chain_reset_state(dspi_chain *c);
/* The preset-mute envelope inside the engine (update_preset_mute_envelope(), usb_audio.c:466-498, called once per packet
 * at :532): states[n] puts instances [inst0, inst0+n) into envelope mode - from then on every packet of every process
 * call advances the instance's envelope and uses its gain where process_audio_packet() uses preset_mute_gain (:570), so a
 * fade runs across the packets of one call and across calls.  Arm a mute with dspi_preset_mute_arm() as the firmware's
 * flash operations do.  states == NULL leaves envelope mode: the constant preset_mute_gain of dspi_chain_set_params
 * applies again.  _get_ returns the current state (it is part of the state blob too). */
/* Mass reconfiguration of the dynamics stages ON THE GPU (SURVEY 8 f-1): per instance what the firmware's main loop does
 * when crossfeed_update_pending / leveller_update_pending / loudness_recompute_pending are set (main.c:868-895) -
 * crossfeed_compute_coefficients() (crossfeed.c:35-127: new coefficients, filter state cleared), leveller_compute_coefficients()
 * (leveller.c:42-89), loudness_recompute_table() (loudness.c:169-217) for the row audio_set_volume() selects - followed by
 * audio_set_volume() (usb_audio.c:428-440): the host volume becomes vol_mul (the int16 quirk included) and the output gains
 * follow.  cfgs[n] is host memory.  Arithmetic and libm policy as dspi_eq_set_params_device.  The bypass flags, preamp,
 * master volume, matrix and delays stay as dspi_chain_set_params left them. */
typedef struct {
    dspi_crossfeed_config crossfeed;     /* crossfeed_config, usb_audio.c:187-193                       */
    dspi_leveller_config  leveller;      /* leveller_config, usb_audio.c:199-206                        */
    float   loudness_ref_spl;            /* loudness_ref_spl, usb_audio.c:175                           */
    float   loudness_intensity_pct;      /* loudness_intensity_pct, usb_audio.c:176                     */
    uint8_t loudness_enabled;            /* loudness_enabled, usb_audio.c:174                           */
    uint8_t host_mute;                   /* audio_state.mute                                            */
    int16_t volume_8_8;                  /* audio_state.volume: UAC1 volume in 1/256 dB, 0 = full scale */
} dspi_dynamics_config;
int dspi_chain_set_dynamics_device(dspi_chain *c, uint32_t inst0, uint32_t n, const dspi_dynamics_config *cfgs, float sample_rate);
int dspi_chain_set_preset_mute(dspi_chain *c, uint32_t inst0, uint32_t n, const dspi_preset_mute *states, uint32_t sample_rate_hz);
int dspi_chain_get_preset_mute(dspi_chain *c, uint32_t inst0, uint32_t n, dspi_preset_mute *states);
/* Checkpoint / resume (the dspi_state_export/import of SURVEY 8 b): everything a later process call depends on besides
 * dspi_chain_set_params' records - filter coefficients and state, loudness / crossfeed / leveller state, look-ahead and
 * delay rings, write index, modulator state, meters.  The blob is private to this library (header + raw arrays) and only
 * loads into an engine of the same shape.  It records the K1 stage geometry (DSPI_F32_CPL) it was written under and
 * loads into an engine created under either one.  The S/PDIF transmitter state is not in the blob (its format is
 * unchanged): a resume that continues the S/PDIF stream needs dspi_chain_state_import followed by
 * dspi_chain_set_spdif_tx with what dspi_chain_get_spdif_tx returned at the checkpoint. */
size_t dspi_chain_state_size(dspi_chain *c);
int dspi_chain_state_export(dspi_chain *c, void *blob, size_t cap);
int dspi_chain_state_import(dspi_chain *c, const void *blob, size_t len);
/* Per-instance lifecycle: restart, checkpoint or move one device without touching the others.  An instance image holds
 * everything of ONE instance that a later call depends on: its parameter rows (those _set_params, _set_dynamics_device
 * and _apply_bulk_device write), its 11 (Q28: 7) x 12 biquads with their current state (reference layout), loudness /
 * crossfeed / leveller state, look-ahead and delay rings with the write index, modulator state, meters, preset-mute
 * envelope and mode, S/PDIF transmitter (block position, channel status), and the wire configuration record (packet body,
 * host record, DSPI_BULK_* mark).  Private, versioned format (header: magic, version, arith, n_bands, size; no CRC).  It
 * loads into any engine of the same arith and n_bands on any device, at any instance index: it does not depend on
 * n_instances, max_frames, the K1 geometry (DSPI_F32_CPL) or the SM partition.  _instance_image_size gives its size
 * (0 for a NULL engine): about 164 KB for the float engine, 51 KB for Q28, most of it the delay rings.
 * images is host memory; image i is at images + i * image_stride, image_stride >= the image size (as preset images).
 * The calls stage through a bounded device buffer in instance chunks (32 MiB, DSPI_HOST_CHUNK_MB in the environment
 * overrides; shared with the _response_host staging), one copy kernel and one copy each way per chunk.
 *   _export_instances: images of instances [inst0, inst0+n).  Read-only; ordered behind everything issued earlier on the
 *     engine stream, asynchronous process calls included; returns when the images are in the caller's memory.
 *   _import_instances: instances [inst0, inst0+n) become the instances the images were exported from, from the next
 *     process call on (a continuation gives the bytes the source engine would have given).  All or nothing: every
 *     header is checked first - magic, version, arith, n_bands, size - and any mismatch gives DSPI_EINVAL with nothing
 *     written.  Ordered behind earlier work; every instance outside the range is left untouched, its EQ coefficients and
 *     state in 32- and 64-channel groups shared with the range included.  The configuration record and its mark come
 *     from the image (a stale or unset instance stays so).  Returns when the engine is updated.
 *   _reset_instances: _reset_state for instances [inst0, inst0+n) only - the same fields cleared, the same kept (EQ
 *     state, crossfeed state, preset-mute envelope, S/PDIF transmitter), and the parameters and configuration record
 *     kept too.  Ordered behind earlier work; returns when done.
 * A freed slot returns to power-on state by importing an image exported from a freshly created engine of the same arith
 * and n_bands: parameters, state and transmitter of a new engine's instance, mark DSPI_BULK_UNSET.
 * Errors: DSPI_EINVAL for a NULL pointer or an image_stride below the image size; DSPI_ERANGE for a range past the end of
 * the engine (also one whose end wraps in 32 bits); nothing is written then.  n == 0 does nothing. */
size_t dspi_chain_instance_image_size(dspi_chain *c);
int dspi_chain_export_instances(dspi_chain *c, uint32_t inst0, uint32_t n, void *images, size_t image_stride);
int dspi_chain_import_instances(dspi_chain *c, uint32_t inst0, uint32_t n, const void *images, size_t image_stride);
int dspi_chain_reset_instances(dspi_chain *c, uint32_t inst0, uint32_t n);
/* Copy instances within one engine on the GPU, so a host can repack its clock groups into contiguous ranges (or clone
 * one configured device into many slots) without sending images over the bus.
 *   src[n] and dst[n] are host memory, read during the call.  After it, instance dst[k] is, byte for byte, what
 *   _export_instances(src[k], 1) followed by _import_instances(dst[k], 1) would have made of it: everything an instance
 *   image holds (parameter rows, the 11 (Q28: 7) x 12 biquads with their current state, loudness / crossfeed / leveller
 *   state, look-ahead and delay rings with the write index, modulator state, meters, preset-mute envelope and mode,
 *   S/PDIF transmitter, configuration record, host record and DSPI_BULK_* mark).  A later process call on dst[k] gives
 *   the bytes the source would have given.  The data moves device to device; no image is formed.
 *   Sources are left exactly as they were, and so is every instance not in dst, its EQ coefficients and state in 32- and
 *   64-channel groups shared with a destination included.
 *   src may repeat (one instance cloned into many slots).  dst entries must be distinct and no index may be in both
 *   lists, so every copy reads a source no copy of the call writes.  To shift a group onto slots that overlap its own,
 *   call in steps whose sources and destinations do not overlap (e.g. through free slots, or one block at a time).
 *   Ordered behind everything issued earlier on the engine stream, asynchronous process calls included; returns when
 *   the engine is updated.  The engine's count of envelope-mode instances follows the copied modes.
 * Errors: DSPI_EINVAL for a NULL engine, src or dst, a destination named twice, or an index in both lists; DSPI_ERANGE
 * for an index at or above n_instances.  Every check runs before anything is written, and nothing is written on an
 * error.  n == 0 does nothing. */
int dspi_chain_copy_instances(dspi_chain *c, uint32_t n, const uint32_t *src, const uint32_t *dst);
/* n_packets USB packets of frames_per_packet (<= 192) frames for every instance.
 *   pcm:       [n_instances][n_packets * frames_per_packet] interleaved L,R little-endian frames,
 *              bit_depth 16 (4 bytes / frame) or 24 (packed, 6 bytes / frame)      (HOST memory)
 *   spdif_out: [n_instances][4][n_frames][2] int32 - the four pico_audio producer buffers
 *   pdm_out:   [n_instances][n_frames][8] uint32 - 256 PDM bits per frame, MSB first; the rows of
 *              instances whose sub output is disabled are zero.  The _device forms write the rows of
 *              instances with the sub enabled only and leave the others as the caller left them.
 *   status:    [n_instances], peaks of the LAST packet, clip flags OR-ed in (sticky)
 * Any of the three outputs may be NULL. */
int dspi_chain_process_host(dspi_chain *c, const void *pcm, uint32_t bit_depth, uint32_t n_packets, uint32_t frames_per_packet,
                            int32_t *spdif_out, uint32_t *pdm_out, dspi_status *status);
/* same with DEVICE pointers; asynchronous on the engine stream */
int dspi_chain_process_device(dspi_chain *c, const void *d_pcm, uint32_t bit_depth, uint32_t n_packets, uint32_t frames_per_packet,
                              int32_t *d_spdif_out, uint32_t *d_pdm_out, dspi_status *d_status);
/* n_packets USB packets whose lengths are packet_frames[0 .. n_packets) (each 1..DSPI_PACKET_MAX; HOST memory, read
 * during the call, reusable by the caller as soon as the call returns).  The schedule is shared by every instance of the
 * call.  F = sum of packet_frames <= max_frames; pcm, spdif_out, pdm_out and status are laid out as for
 * dspi_chain_process_host with n_frames = F.  usb_audio.c:500 with data_len = packet_frames[p] * bytes per frame: the
 * leveller's block gain, the preset-mute envelope step and the last-packet peaks follow each packet's own length, so a
 * 44.1 kHz stream (nine 44-frame packets, then one of 45) or a feedback-paced one (n-1, n or n+1 frames) runs bit-exact
 * in one call.  dspi_chain_process_* with frames_per_packet is this call with n_packets equal lengths.
 * Per-instance schedules (different lengths for different instances of one call) are not supported: every row of the
 * call's EQ stages would need its own length.
 * Errors: DSPI_EINVAL for a NULL table, n_packets == 0, a length of 0 or above DSPI_PACKET_MAX, or a bit depth other than
 * 16 or 24; DSPI_ERANGE when the lengths add up to more than max_frames.  The _device form stays asynchronous on the
 * engine stream and never waits for the device (the packet offsets travel as kernel parameters). */
int dspi_chain_process_packets_host  (dspi_chain *c, const void *pcm, uint32_t bit_depth, uint32_t n_packets, const uint16_t *packet_frames,
                                      int32_t *spdif_out, uint32_t *pdm_out, dspi_status *status);
int dspi_chain_process_packets_device(dspi_chain *c, const void *d_pcm, uint32_t bit_depth, uint32_t n_packets, const uint16_t *packet_frames,
                                      int32_t *d_spdif_out, uint32_t *d_pdm_out, dspi_status *d_status);
/* dspi_chain_process_packets_* over the instances [inst0, inst0 + n) only, with this call's own packet_frames: a host packs
 * its connected devices (or each group of devices on one clock) into contiguous ranges with the instance image calls and
 * serves each range as its packets arrive, so idle slots cost nothing and a 44.1 kHz group, a 48 kHz group and a
 * feedback-paced group share one engine.  The schedule stays one per call (see above).
 *   Layout: every buffer is laid out for n instances - pcm [n][F * bytes per frame], spdif_out [n][4][F][2], pdm_out
 *   [n][F][8], status [n] - and row i belongs to instance inst0 + i.  F = sum of packet_frames <= max_frames.  PDM rows as
 *   for the whole engine: _host zeroes the rows of instances whose sub is off, _device leaves them as they were.
 *   Inside the range everything happens as in a whole-engine call: filter, loudness, crossfeed and leveller state, the
 *   look-ahead and delay rings and their write index, modulator state, meters, the preset-mute envelope step per packet,
 *   the S/PDIF block position advancing by F.
 *   Outside the range nothing changes: state, envelope, transmitter, meters, and the EQ coefficients and state of
 *   instances that share a K1 / K2 channel group with the range.  A later call on them gives the bytes it would have given
 *   without this call.
 *   Rules: inst0 is a multiple of 64 (DSPI_EINVAL otherwise); n is any count and n == 0 does nothing; a range past the end
 *   of the engine (also one whose end wraps in 32 bits) is DSPI_ERANGE; the table, bit depth and NULL checks are those of
 *   dspi_chain_process_packets_*.  Nothing is written on any error.
 *   The _device form is asynchronous on the engine stream and never waits for the device; consecutive calls on one engine
 *   run in issue order.  The whole-engine calls are this call with inst0 = 0, n = n_instances. */
int dspi_chain_process_packets_range_host  (dspi_chain *c, uint32_t inst0, uint32_t n, const void *pcm, uint32_t bit_depth, uint32_t n_packets,
                                            const uint16_t *packet_frames, int32_t *spdif_out, uint32_t *pdm_out, dspi_status *status);
int dspi_chain_process_packets_range_device(dspi_chain *c, uint32_t inst0, uint32_t n, const void *d_pcm, uint32_t bit_depth, uint32_t n_packets,
                                            const uint16_t *packet_frames, int32_t *d_spdif_out, uint32_t *d_pdm_out, dspi_status *d_status);
int dspi_chain_sync(dspi_chain *c);
void *dspi_chain_stream(dspi_chain *c);
uint64_t dspi_chain_launch_count(dspi_chain *c);
/* How the engine split the GPU for this chain: the delta-sigma modulator (one serial chain per instance, latency-bound)
 * runs alone on pdm_sms SMs, every other stage on rest_sms (CUDA green contexts; 0 / 0 when the driver offers none or
 * DSPI_PDM_SMS=0 is set - results never depend on it).  No reference counterpart: the firmware gives the modulator
 * core 1 (pdm_generator.c:691-721). */
int dspi_chain_sm_partition(dspi_chain *c, uint32_t *pdm_sms, uint32_t *rest_sms);
/* dsp_update_delay_samples() for one output, dsp_pipeline.c:216-239 (is_last adds SUB_ALIGN_SAMPLES) */
int32_t dspi_delay_samples(float delay_ms, float sample_rate, int is_last);

/* ---- full signal chain, RP2040 arithmetic (Q28 fixed point, 2 in -> 5 out) ---------------------- */
/* process_audio_packet(), usb_audio.c:968-1283 (single-core branch :1191-1276): every stage in
 * 32-bit wrapping Q28/Q15 arithmetic (fast_mul_q28 dsp_pipeline.c:47-58, fast_mul_q15
 * config.h:556-567), crossfeed.c:161-180, leveller.c:275-389; bit-exact. */
#define DSPI_CHAINQ_OUTPUTS      5    /* config.h:326                                               */
#define DSPI_CHAINQ_EQ_CHANNELS  7    /* config.h:327                                               */
#define DSPI_CHAINQ_MAX_DELAY 2048    /* config.h:86                                                */

/* LoudnessCoeffs (RP2040), loudness.h:21 (24 bytes); CrossfeedState (RP2040), crossfeed.h:53-58 */
typedef struct { int32_t b0, b1, b2, a1, a2; uint8_t bypass; } dspi_loudness_coeffs_q28;
typedef struct { int32_t lp_a0, lp_b1, lp_state_L, lp_state_R, ap_a, ap_state_L, ap_state_R; } dspi_crossfeed_state_q28;
/* MatrixMixer (RP2040), config.h:403-406 (220 bytes); SystemStatusPacket (RP2040, 18 bytes) */
typedef struct {
    dspi_matrix_crosspoint crosspoints[2][DSPI_CHAINQ_OUTPUTS];
    dspi_output_channel outputs[DSPI_CHAINQ_OUTPUTS];
} dspi_matrix_mixer_q28;
typedef struct { uint16_t peaks[DSPI_CHAINQ_EQ_CHANNELS]; uint8_t cpu0_load, cpu1_load; uint16_t clip_flags; } dspi_status_q28;

typedef struct {
    uint8_t bypass_master_eq, loudness_enabled, crossfeed_enabled, leveller_enabled;
    uint8_t host_mute, leveller_lookahead, reserved0[2];
    int16_t host_vol_mul;            /* audio_state.vol_mul (int16: 0 dB gives -32768)              */
    int16_t reserved1;
    float preset_mute_gain;          /* quantised to Q15 per packet, usb_audio.c:976-978            */
    int32_t master_volume_q15;       /* usb_audio.c:162                                             */
    int32_t preamp_q28[2];           /* global_preamp_mul[]                                         */
    dspi_loudness_coeffs_q28 loudness[2];
    dspi_crossfeed_state_q28 crossfeed;
    dspi_leveller_coeffs leveller;
    dspi_matrix_mixer_q28 matrix;
} dspi_chain_params_q28;

#ifdef __cplusplus
static_assert(sizeof(dspi_loudness_coeffs_q28) == 24 && sizeof(dspi_crossfeed_state_q28) == 28 && sizeof(dspi_matrix_mixer_q28) == 220 &&
              sizeof(dspi_status_q28) == 18, "reference layouts");
#else
_Static_assert(sizeof(dspi_loudness_coeffs_q28) == 24 && sizeof(dspi_crossfeed_state_q28) == 28 && sizeof(dspi_matrix_mixer_q28) == 220 &&
               sizeof(dspi_status_q28) == 18, "reference layouts");
#endif

typedef struct dspi_chainq dspi_chainq;
int dspi_chainq_create(dspi_chainq **out, const dspi_chain_desc *desc);      /* desc->arith must be DSPI_ARITH_Q28 */
int dspi_chainq_destroy(dspi_chainq *c);
int dspi_chainq_set_params(dspi_chainq *c, uint32_t inst0, uint32_t n, const dspi_chain_params_q28 *params);
/* filters[7][12] per instance: biquads[n][7][12] (master L, R, Out1..4, sub) */
int dspi_chainq_upload_biquads(dspi_chainq *c, uint32_t inst0, uint32_t n, const dspi_biquad_q28 *biquads);
int dspi_chainq_download_biquads(dspi_chainq *c, uint32_t inst0, uint32_t n, dspi_biquad_q28 *biquads);
int dspi_chainq_set_eq_params_device(dspi_chainq *c, uint32_t inst0, uint32_t n, dspi_eq_param *recipes, float sample_rate);   /* recipes[n][7][12] */
int dspi_chainq_reset_state(dspi_chainq *c);                                  /* as dspi_chain_reset_state */
int dspi_chainq_set_dynamics_device(dspi_chainq *c, uint32_t inst0, uint32_t n, const dspi_dynamics_config *cfgs, float sample_rate);
int dspi_chainq_set_preset_mute(dspi_chainq *c, uint32_t inst0, uint32_t n, const dspi_preset_mute *states, uint32_t sample_rate_hz);   /* Q15 use of the gain: usb_audio.c:976-980 */
int dspi_chainq_get_preset_mute(dspi_chainq *c, uint32_t inst0, uint32_t n, dspi_preset_mute *states);
size_t dspi_chainq_state_size(dspi_chainq *c);
int dspi_chainq_state_export(dspi_chainq *c, void *blob, size_t cap);
int dspi_chainq_state_import(dspi_chainq *c, const void *blob, size_t len);   /* + dspi_chainq_set_spdif_tx, as dspi_chain_* */
/* per-instance images and reset, as dspi_chain_* */
size_t dspi_chainq_instance_image_size(dspi_chainq *c);
int dspi_chainq_export_instances(dspi_chainq *c, uint32_t inst0, uint32_t n, void *images, size_t image_stride);
int dspi_chainq_import_instances(dspi_chainq *c, uint32_t inst0, uint32_t n, const void *images, size_t image_stride);
int dspi_chainq_reset_instances(dspi_chainq *c, uint32_t inst0, uint32_t n);
int dspi_chainq_copy_instances(dspi_chainq *c, uint32_t n, const uint32_t *src, const uint32_t *dst);
/* pcm as for dspi_chain_process_host; spdif_out [n_instances][2][n_frames][2]; pdm_out [n_instances][n_frames][8] */
int dspi_chainq_process_host(dspi_chainq *c, const void *pcm, uint32_t bit_depth, uint32_t n_packets, uint32_t frames_per_packet,
                             int32_t *spdif_out, uint32_t *pdm_out, dspi_status_q28 *status);
int dspi_chainq_process_device(dspi_chainq *c, const void *d_pcm, uint32_t bit_depth, uint32_t n_packets, uint32_t frames_per_packet,
                               int32_t *d_spdif_out, uint32_t *d_pdm_out, dspi_status_q28 *d_status);
/* a packet_frames[n_packets] schedule, as dspi_chain_process_packets_* (usb_audio.c:968 with data_len per packet) */
int dspi_chainq_process_packets_host  (dspi_chainq *c, const void *pcm, uint32_t bit_depth, uint32_t n_packets, const uint16_t *packet_frames,
                                       int32_t *spdif_out, uint32_t *pdm_out, dspi_status_q28 *status);
int dspi_chainq_process_packets_device(dspi_chainq *c, const void *d_pcm, uint32_t bit_depth, uint32_t n_packets, const uint16_t *packet_frames,
                                       int32_t *d_spdif_out, uint32_t *d_pdm_out, dspi_status_q28 *d_status);
/* instances [inst0, inst0 + n) only, as dspi_chain_process_packets_range_*; spdif_out [n][2][F][2] */
int dspi_chainq_process_packets_range_host  (dspi_chainq *c, uint32_t inst0, uint32_t n, const void *pcm, uint32_t bit_depth, uint32_t n_packets,
                                             const uint16_t *packet_frames, int32_t *spdif_out, uint32_t *pdm_out, dspi_status_q28 *status);
int dspi_chainq_process_packets_range_device(dspi_chainq *c, uint32_t inst0, uint32_t n, const void *d_pcm, uint32_t bit_depth, uint32_t n_packets,
                                             const uint16_t *packet_frames, int32_t *d_spdif_out, uint32_t *d_pdm_out, dspi_status_q28 *d_status);
int dspi_chainq_sync(dspi_chainq *c);
void *dspi_chainq_stream(dspi_chainq *c);
uint64_t dspi_chainq_launch_count(dspi_chainq *c);
int dspi_chainq_sm_partition(dspi_chainq *c, uint32_t *pdm_sms, uint32_t *rest_sms);
/* Q28 stores of the crossfeed and loudness parameter functions (crossfeed.c:116-119, loudness.c:131-162) */
void dspi_crossfeed_compute_coefficients_q28(dspi_crossfeed_state_q28 *st, const dspi_crossfeed_config *cfg, float sample_rate);
void dspi_loudness_compute_table_q28(dspi_loudness_coeffs_q28 table[61][2], float ref_spl, float intensity_pct, float sample_rate);

/* ---- bulk parameter ingest (host side; SURVEY.md 8 f-1 / the dspi_set_bulk_params of 8 b) ------- */
/* WireBulkParams, bulk_params.h:40-205: the 2896-byte little-endian packet the DSPi Console sends with
 * REQ_SET_ALL_PARAMS and reads with REQ_GET_ALL_PARAMS.  Byte-identical layout. */
#define DSPI_WIRE_MAX_CHANNELS 11
#define DSPI_WIRE_MAX_OUTPUTS  9
#define DSPI_WIRE_FORMAT_VERSION 6
#define DSPI_PLATFORM_RP2040 0
#define DSPI_PLATFORM_RP2350 1
typedef struct __attribute__((packed)) {
    struct __attribute__((packed)) { uint8_t format_version, platform_id, num_channels, num_output_channels, num_input_channels, max_bands;
                                     uint16_t payload_length, fw_version_major, fw_version_minor; uint32_t reserved; } header;          /*  16 */
    struct __attribute__((packed)) { float preamp_gain_db; uint8_t bypass, loudness_enabled, reserved[2];
                                     float loudness_ref_spl, loudness_intensity_pct; } global;                                        /*  16 */
    struct __attribute__((packed)) { uint8_t enabled, preset, itd_enabled, reserved; float custom_fc, custom_feed_db; uint32_t reserved2; } crossfeed;   /* 16 */
    struct __attribute__((packed)) { float gain_db[3]; uint8_t mute[3], reserved; } legacy;                                           /*  16 */
    struct __attribute__((packed)) { float delay_ms[DSPI_WIRE_MAX_CHANNELS]; } delays;                                                /*  44 */
    struct __attribute__((packed)) { uint8_t enabled, phase_invert, reserved[2]; float gain_db; } crosspoints[2][DSPI_WIRE_MAX_OUTPUTS];   /* 144 */
    struct __attribute__((packed)) { uint8_t enabled, mute, reserved[2]; float gain_db, delay_ms; } outputs[DSPI_WIRE_MAX_OUTPUTS];   /* 108 */
    struct __attribute__((packed)) { uint8_t num_pin_outputs, pins[5], reserved[2]; } pins;                                           /*   8 */
    struct __attribute__((packed)) { uint8_t type, reserved[3]; float freq, q, gain_db; } eq[DSPI_WIRE_MAX_CHANNELS][DSPI_MAX_BANDS]; /* 2112 */
    char channel_names[DSPI_WIRE_MAX_CHANNELS][32];                                                                                    /* 352 */
    struct __attribute__((packed)) { uint8_t output_types[4], bck_pin, mck_pin, mck_enabled, mck_multiplier, reserved[8]; } i2s_config;    /* 16 */
    struct __attribute__((packed)) { uint8_t enabled, speed, lookahead, reserved; float amount, max_gain_db, gate_threshold_db; } leveller; /* 16 */
    struct __attribute__((packed)) { float preamp_db[2]; uint8_t reserved[8]; } preamp;                                               /*  16 */
    struct __attribute__((packed)) { float master_volume_db; uint8_t reserved[12]; } master_volume;                                   /*  16 */
} dspi_wire_bulk_params;
#ifdef __cplusplus
static_assert(sizeof(dspi_wire_bulk_params) == 2896, "WireBulkParams");
#else
_Static_assert(sizeof(dspi_wire_bulk_params) == 2896, "WireBulkParams");
#endif

/* The globals bulk_params_apply() writes that feed the DSP path (bulk_params.c:22-43), for one device. */
typedef struct {
    int32_t platform;                        /* DSPI_PLATFORM_*: 11 channels / 9 outputs or 7 / 5                  */
    float preamp_db[2], preamp_linear[2]; int32_t preamp_q28[2];          /* global_preamp_db / _linear / _mul     */
    float master_volume_db, master_volume_linear; int32_t master_volume_q15;
    uint8_t bypass_master_eq, loudness_enabled, reserved0[2];
    float loudness_ref_spl, loudness_intensity_pct;
    dspi_crossfeed_config crossfeed;
    dspi_leveller_config leveller;
    float legacy_gain_db[3], legacy_gain_linear[3]; int32_t legacy_gain_mul[3]; uint8_t legacy_mute[3], reserved1;
    float channel_delays_ms[DSPI_WIRE_MAX_CHANNELS];
    dspi_matrix_crosspoint crosspoints[2][DSPI_WIRE_MAX_OUTPUTS];        /* gain_linear by the firmware's db_to_linear */
    dspi_output_channel outputs[DSPI_WIRE_MAX_OUTPUTS];                  /* delay_samples is filled by dspi_bulk_state_to_chain_* */
    dspi_eq_param recipes[DSPI_WIRE_MAX_CHANNELS][DSPI_MAX_BANDS];       /* filter_recipes[][]                      */
} dspi_bulk_state;

/* power-on values of those globals (usb_audio.c:148-211, leveller.h:69-74, matrix defaults config.h) */
void dspi_bulk_state_defaults(dspi_bulk_state *st, int platform);
/* bulk_params_apply(), bulk_params.c:178-377, on `st` instead of the firmware's globals.  Same return codes:
 * 0 ok, -1 format version, -2 platform, -3 channel counts, -4 payload length.  Gains go through the
 * firmware's own db_to_linear (a 4-term Taylor series clamped to [-60, +20] dB, bulk_params.c:49-56;
 * SURVEY quirk 2) unless exact_db != 0 (then 10^(dB/20)); master volume always uses powf (:361-374). */
int dspi_bulk_params_apply(const dspi_wire_bulk_params *in, dspi_bulk_state *st, int exact_db);
/* bulk_params_collect(), bulk_params.c:62-172 (pins, names and I2S sections are control plane: zero) */
void dspi_bulk_params_collect(const dspi_bulk_state *st, dspi_wire_bulk_params *out);
/* What the main loop derives after a successful apply (main.c:1137-1139 and the pending-flag handlers):
 * dsp_recalculate_all_filters, dsp_update_delay_samples, loudness table + row for the host volume,
 * crossfeed and leveller coefficients.  `previous` (may be NULL) supplies the filters whose state must
 * survive (dsp_compute_coefficients only clears state on a topology flip). */
int dspi_bulk_state_to_chain_f32(const dspi_bulk_state *st, float sample_rate, int16_t host_volume_8_8, int host_mute,
                                 dspi_chain_params_f32 *params, dspi_biquad_f32 biquads[11][DSPI_MAX_BANDS]);
int dspi_bulk_state_to_chain_q28(const dspi_bulk_state *st, float sample_rate, int16_t host_volume_8_8, int host_mute,
                                 dspi_chain_params_q28 *params, dspi_biquad_q28 biquads[7][DSPI_MAX_BANDS]);

/* ---- bulk parameter ingest on the device (SURVEY.md 8 f-1) ------------------------------------- */
/* audio_state of one device: the host volume and mute are USB audio-class controls, not part of the wire packet */
typedef struct { int16_t volume_8_8; uint8_t host_mute; uint8_t reserved; } dspi_bulk_host;
#ifdef __cplusplus
static_assert(sizeof(dspi_bulk_host) == 4, "dspi_bulk_host");
#else
_Static_assert(sizeof(dspi_bulk_host) == 4, "dspi_bulk_host");
#endif
/* REQ_SET_ALL_PARAMS for instances [inst0, inst0+n) of a chain engine, from wire bytes to engine records ON THE GPU:
 * packets[n], host[n] and results[n] are host memory.  Per instance this is bulk_params_apply() (bulk_params.c:178-377)
 * followed by what the main loop derives from it (dsp_recalculate_all_filters, dsp_update_delay_samples, the crossfeed /
 * leveller / loudness handlers, audio_set_volume), i.e. dspi_bulk_params_apply + dspi_bulk_state_to_chain_* +
 * dspi_chain(q)_set_params + _upload_biquads, except that
 *   - results[i] is the firmware's code (0, -1 .. -4; the platform and the channel counts are the engine's shape) and a
 *     rejected packet changes nothing of its instance - the firmware returns before its first write.  The call still
 *     returns DSPI_OK;
 *   - below format version 6 the master volume in force stays (the packet has none); the preamp comes from the legacy field;
 *   - EQ filter state is kept unless a band's topology flips, as dsp_compute_coefficients does; the crossfeed filter state
 *     is ALWAYS cleared, as crossfeed_compute_coefficients() does after a bulk apply (the rule of _set_dynamics_device).
 *     The host route through _set_params differs in this one point: it keeps that state when the coefficients did not change;
 *   - leveller, loudness-shelf, delay-line and modulator state, the meters, the preset-mute gain and envelope mode and the
 *     S/PDIF transmitter state are left alone.
 * Gains go through the firmware's Taylor db_to_linear (exact 0 dB -> 1.0, clamped to [-60, +20] dB) unless exact_db != 0
 * (then 10^(dB/20)); the master volume always uses the exact conversion.  Arithmetic and libm policy as
 * dspi_eq_set_params_device: coefficients are the oracle's policy coefficients bit for bit and within the documented libm
 * distance of the host route's.  Ordered behind process calls issued earlier on the engine stream; returns when the engine
 * is reconfigured.  DSPI_EINVAL for a NULL pointer or a sample_rate that is not positive and finite, DSPI_ERANGE for a
 * range past the end of the engine; nothing is written then.  Preset slot images load with _apply_preset_device below.
 * The older route dspi_preset_slot_apply -> dspi_bulk_params_collect -> this call with exact_db = 1 differs from it for
 * gains <= -120 dB (flash gives 0, exact gives 10^(dB/20)) and >= 80 dB (flash clamps to 80 dB). */
int dspi_chain_apply_bulk_device (dspi_chain *c,  uint32_t inst0, uint32_t n, const dspi_wire_bulk_params *packets, const dspi_bulk_host *host,
                                  int exact_db, float sample_rate, int32_t *results);
int dspi_chainq_apply_bulk_device(dspi_chainq *c, uint32_t inst0, uint32_t n, const dspi_wire_bulk_params *packets, const dspi_bulk_host *host,
                                  int exact_db, float sample_rate, int32_t *results);

/* REQ_GET_ALL_PARAMS for instances [inst0, inst0+n) of a chain engine: what bulk_params_collect() (bulk_params.c:62-172)
 * would read from the firmware's globals, from a configuration record the engine keeps per instance in device memory.
 * packets[n], host[n] and results[n] are host memory; host and results may be NULL.  results[i] is one of */
#define DSPI_BULK_CURRENT 0   /* the packet describes what the instance runs                       */
#define DSPI_BULK_STALE   1   /* records were replaced by set_params / upload_biquads since         */
#define DSPI_BULK_UNSET   2   /* never configured through a wire packet: packet bytes are all zero  */
/* For a current or stale instance packets[i] is byte for byte what dspi_bulk_params_collect returns for the dspi_bulk_state
 * the same sequence of calls would have left on the host: format version 6, the engine's platform id and channel counts,
 * the full payload length, firmware version 1.1, pins.num_pin_outputs 5 or 3, everything else of the pins / names / I2S
 * sections and all reserved bytes zero, rows past the shape's channel and output counts zero.  host[i] is the
 * dspi_bulk_host the instance was last given.  Who writes the record:
 *   - _apply_bulk_device: for an accepted packet exactly what bulk_params_apply() writes, under its version gates (legacy
 *     preamp field first, leveller fields from version 4 and the fixed defaults below, per-side preamp and master volume
 *     from version 6 - below 6 the master volume in force stays -, the master volume made finite and clamped to
 *     [-128, 0] dB, channel_delays_ms overwritten by the output delays), then the recipes with the clamps
 *     dsp_compute_coefficients() writes back (dsp_pipeline.c:78-81), as a GET_ALL_PARAMS after a SET_ALL_PARAMS shows
 *     them.  The instance becomes DSPI_BULK_CURRENT.  A rejected packet leaves record and mark alone;
 *   - _set_eq_params_device: the clamped recipes; _set_dynamics_device: the crossfeed, leveller and loudness fields and
 *     the host volume / mute.  Both keep the mark the instance has;
 *   - _set_params and _upload_biquads take derived records (linear gains, coefficients) that dB values and recipes cannot
 *     be recovered from: they leave the record alone and turn a current instance DSPI_BULK_STALE.  An instance that never
 *     had an accepted packet stays DSPI_BULK_UNSET whatever else it was given, and collects zero bytes and a zero host
 *     record.
 * The record is not part of the state blob, and _reset_state leaves it alone.  The call is ordered behind everything issued
 * earlier on the engine stream, asynchronous process calls included, returns when the packets are in the caller's memory,
 * and changes nothing a process call reads.  DSPI_EINVAL for a NULL engine or packets, DSPI_ERANGE for a range past the
 * end of the engine (also one whose end wraps in 32 bits); nothing is written then.  n == 0 does nothing.
 * Preset slot images come from _collect_preset_device below, which gives the bytes of the route this call ->
 * dspi_bulk_params_apply(packet, st, exact_db = 1) -> dspi_preset_slot_collect without a host loop. */
int dspi_chain_collect_bulk_device (dspi_chain *c,  uint32_t inst0, uint32_t n, dspi_wire_bulk_params *packets, dspi_bulk_host *host,
                                    int32_t *results);
int dspi_chainq_collect_bulk_device(dspi_chainq *c, uint32_t inst0, uint32_t n, dspi_wire_bulk_params *packets, dspi_bulk_host *host,
                                    int32_t *results);

/* perform_rate_change() (main.c:132-171) for instances [inst0, inst0+n) ON THE GPU, from each instance's configuration
 * record: the USB host switched those devices to new sample rates.  sample_rates[n] (host memory) gives each instance its
 * own rate fs_i; results[n] (host memory, may be NULL) gets each instance's DSPI_BULK_* mark.
 *   - Only DSPI_BULK_CURRENT instances switch.  A DSPI_BULK_STALE or DSPI_BULK_UNSET instance is left exactly as it was:
 *     its derived records came from _set_params / _upload_biquads, which the record cannot reproduce.  The call still
 *     returns DSPI_OK.
 *   - A switched instance gets, at fs_i: dsp_recalculate_all_filters(fs_i) over all 11 (Q28: 7) x 12 bands from the
 *     record's recipes, the clamps written back into the record (dsp_pipeline.c:78-81: a band a 44.1 kHz switch clamped to
 *     19845 Hz stays there after a switch back to 96 kHz), filter state kept unless a band's topology flips (SVF below
 *     fs / 7.5, TDF2 above); dsp_update_delay_samples(fs_i) from the record's output delays in ms (the sub's
 *     SUB_ALIGN_SAMPLES term, the clamp to [0, MAX], dly == MAX still aliasing to no delay) and the any_delay bit of its
 *     flag word recomputed, delay-line contents and write index kept; crossfeed_compute_coefficients(cfg, fs_i) with the
 *     crossfeed filter state cleared; leveller_compute_coefficients(cfg, fs_i) with leveller state kept; the loudness row
 *     loudness_recompute_table(ref_spl, intensity, fs_i) selects for the record's host volume, shelf state kept.
 *   - Left alone: every gain (preamp, matrix crosspoints, output gains, master volume, vol_mul), the flags and skip rows
 *     that do not depend on the rate, modulator state, meters, the preset-mute envelope, the S/PDIF transmitter (block
 *     position and channel status), the mark and the host record.  Of the record only the eq section changes: the
 *     recipes, clamped at fs_i.
 *   - The rest of a rate change is the caller's, through the calls that do it: channel-status byte 3 (the rate code) with
 *     _set_spdif_tx, a fade with _set_preset_mute, a pipeline reset with _reset_instances.  Whether perform_rate_change()
 *     does any of these was not checked against main.c; this call does none of them.
 * Arithmetic and libm policy as dspi_eq_set_params_device / _set_dynamics_device: coefficients are the oracle's policy
 * coefficients bit for bit.  Ordered behind everything issued earlier on the engine stream, asynchronous process calls
 * included; returns when the engine is reconfigured.  DSPI_EINVAL for a NULL engine or sample_rates, or any rate that is
 * not positive and finite (every rate is checked before the first write); DSPI_ERANGE for a range past the end of the
 * engine (also one whose end wraps in 32 bits); nothing is written then.  n == 0 does nothing. */
int dspi_chain_set_rate_device (dspi_chain *c,  uint32_t inst0, uint32_t n, const float *sample_rates, int32_t *results);
int dspi_chainq_set_rate_device(dspi_chainq *c, uint32_t inst0, uint32_t n, const float *sample_rates, int32_t *results);

/* One edit: `length` bytes at `offset` of an instance's configuration, in the address space
 *   [0, 2896)      dspi_wire_bulk_params (the packet _collect_bulk_device returns)
 *   [2896, 2900)   dspi_bulk_host        (host volume_8_8, host_mute) */
typedef struct { uint32_t instance; uint16_t offset; uint8_t length; uint8_t reserved; uint8_t bytes[24]; } dspi_bulk_edit;  /* 32 B */
#ifdef __cplusplus
static_assert(sizeof(dspi_bulk_edit) == 32, "dspi_bulk_edit");
#else
_Static_assert(sizeof(dspi_bulk_edit) == 32, "dspi_bulk_edit");
#endif
/* Single fields of many instances' configuration, edited ON THE GPU: what a DSPi Console sends while a user drags an EQ
 * band, a fader, an output gain, a mute or a crosspoint.  edits[n_edits] and results[n_edits] are host memory; results
 * may be NULL.
 *   - Reference semantics.  Take a DSPI_BULK_CURRENT instance, P the packet _collect_bulk_device returns for it and H its
 *     host record.  Write the call's edits for that instance over (P, H) in list order (the last write to a byte wins).
 *     The instance's configuration record, host record and mark then become exactly what _apply_bulk_device(P', H',
 *     exact_db, sample_rate) would leave, and so do its derived rows for every field an edit touched.
 *   - A field is touched when any edit writes any byte of it, whatever the value.  The record is normalised as
 *     _apply_bulk_device leaves it: flags 0 / 1, reserved bytes zero, global.preamp_gain_db mirroring preamp_db[0],
 *     channel_delays_ms following the output delays, the master volume finite and clamped to [-128, 0] dB, rows past the
 *     shape's channel and output counts zero.
 *   - What a touched field re-derives (the rows bulk_params_apply() and the main loop's handlers write from it):
 *       crosspoint                          its gain row
 *       output enabled / mute               every output's flags (the partner's pair-off bit), the sub-on flag bit, skip rows
 *       output gain_db                      its linear gain
 *       output delay_ms                     its delay in samples at sample_rate, the any_delay flag bit
 *       preamp_db[side]                     that preamp row
 *       master_volume_db                    the master gain, always with the exact conversion
 *       output enable / mute / gain, master volume, host volume or mute:   the output gain rows (audio_set_volume())
 *       host volume_8_8                     also the loudness row it selects
 *       global.bypass                       its flag bit, the master skip rows and the output skip rows
 *       loudness enabled / ref / intensity  its flag bit and the loudness row
 *       any crossfeed byte                  coefficients at sample_rate with the filter state cleared, its flag bit
 *       any leveller byte                   coefficients at sample_rate, its flag bits
 *       eq[ch][b]                           that band's coefficients at sample_rate, its clamped recipe written back
 *     Legacy fields and the master channels' delays.delay_ms[0..1] change the record only, as an apply does with them.
 *   - A field no edit touched is not re-derived: gains keep the values they have, whichever conversion made them (Taylor,
 *     exact or preset flash), and untouched bands keep coefficients and state byte for byte, even when sample_rate differs
 *     from the rate they were computed at.
 *   - Running state: EQ state is kept unless a touched band flips between SVF and TDF2; the crossfeed filter state is
 *     cleared only when a crossfeed byte is touched, so unlike _apply_bulk_device and _set_dynamics_device a host-volume or
 *     gain edit keeps it; leveller, loudness-shelf, delay-line and modulator state, the meters, the preset-mute gain,
 *     envelope and mode and the S/PDIF transmitter are left alone.
 *   - Edits for a DSPI_BULK_STALE or DSPI_BULK_UNSET instance change nothing of it; results[k] is the mark of edit k's
 *     instance at the call's point in the stream.  The call still returns DSPI_OK.
 *   - Errors, all checked before anything is written: DSPI_EINVAL for a NULL engine or edits, a sample_rate that is not
 *     positive and finite, a length of 0 or above 24, a non-zero reserved byte, a span past 2900 bytes, or a span that
 *     touches the header, pins, channel_names or i2s_config (control plane: the record keeps them zero and collect stamps
 *     them); DSPI_ERANGE for an instance at or above n_instances.  n_edits == 0 does nothing.
 * Arithmetic and libm policy as _apply_bulk_device.  One sample_rate per call: a farm issues one call per clock group.
 * Ordered behind everything issued earlier on the engine stream, asynchronous process calls included; returns when the
 * engine is updated, and edits can be reused then. */
int dspi_chain_edit_bulk_device (dspi_chain *c,  uint32_t n_edits, const dspi_bulk_edit *edits, int exact_db, float sample_rate, int32_t *results);
int dspi_chainq_edit_bulk_device(dspi_chainq *c, uint32_t n_edits, const dspi_bulk_edit *edits, int exact_db, float sample_rate, int32_t *results);

/* ---- preset slot images (SURVEY.md 8 f-4): PresetSlot v12, flash_storage.c:139-189 ------------ */
/* One flash sector per slot: 12-byte header (magic "DSP3", data version, slot index, CRC-32 of everything
 * after the header) + the packed DSP state.  Device preset dumps load directly into a dspi_bulk_state and
 * from there (dspi_bulk_state_to_chain_*) into a chain engine. */
#define DSPI_PRESET_SLOT_MAGIC   0x44535033u     /* flash_storage.c:67 */
#define DSPI_PRESET_SLOT_VERSION 12              /* :71 */
#define DSPI_PRESET_OK       0                   /* config.h:262-266 */
#define DSPI_PRESET_ERR_CRC  3
size_t dspi_preset_slot_size(int platform);                       /* sizeof(PresetSlot) on that platform */
uint32_t dspi_crc32(const void *data, size_t len);               /* flash_storage.c:282-291 (reflected 0xEDB88320) */
/* validate_slot() (:750-760) + apply_slot_to_live() (:597-744) + apply_master_volume_from_mode() (:580-590),
 * i.e. the state part of preset_load(): DSPI_PRESET_OK, or DSPI_PRESET_ERR_CRC when magic, slot index or CRC
 * do not match (state untouched).  Gains use flash_storage.c's db_to_linear (powf, :302-306), not the Taylor
 * series of the bulk path.  master_volume_mode / dir_master_volume_db are the directory's settings
 * (MASTER_VOLUME_MODE_INDEPENDENT = 0: use dir_master_volume_db; 1: the slot's own value when version >= 12). */
int dspi_preset_slot_apply(const void *slot, size_t len, uint8_t slot_index, uint8_t master_volume_mode, float dir_master_volume_db,
                           dspi_bulk_state *st);
/* collect_live_state() (:464-556): writes dspi_preset_slot_size(st->platform) bytes with a valid header and CRC.
 * dspi_bulk_state carries the DSP state only: output pins, channel names, output types and the I2S fields are written as
 * ZERO, so the image is for exchanging DSP state between hosts of this library (apply ignores those fields) - do NOT
 * flash it onto a device, which would load the zeros over its pin / name / I2S configuration. */
int dspi_preset_slot_collect(const dspi_bulk_state *st, uint8_t slot_index, void *out, size_t cap);

/* ---- preset slot images on the device: preset_load() / preset_save() for many chain instances ----- */
/* Per instance, what preset_load() gets from its caller and the preset directory. */
typedef struct { uint8_t slot_index, master_volume_mode, reserved[2]; float dir_master_volume_db; } dspi_preset_load;
#ifdef __cplusplus
static_assert(sizeof(dspi_preset_load) == 8, "dspi_preset_load");
#else
_Static_assert(sizeof(dspi_preset_load) == 8, "dspi_preset_load");
#endif
/* preset_load() for instances [inst0, inst0+n) of a chain engine, from slot images to engine records ON THE GPU.  Image i
 * starts at images + i * image_stride (image_stride >= dspi_preset_slot_size(platform): 2864 B RP2350, 1840 B RP2040, so
 * 4 KiB flash sectors can be passed as dumped); images, load[n], host[n] and results[n] are host memory.  Per instance this
 * is dspi_preset_slot_apply(image, slot size, load.slot_index, load.master_volume_mode, load.dir_master_volume_db, st)
 * followed by what the main loop derives from it, with the contract of _apply_bulk_device:
 *   - results[i] is DSPI_PRESET_OK, or DSPI_PRESET_ERR_CRC for a wrong magic, slot index or CRC-32 (checked on the
 *     device); a rejected image changes nothing of its instance, and the call still returns DSPI_OK;
 *   - version gates as the host: leveller fields from version 10 (fixed defaults below), per-side preamp and the slot's
 *     master volume from version 12; master_volume_mode 1 takes the slot's master volume from version 12, otherwise
 *     dir_master_volume_db is used;
 *   - every gain uses flash_storage.c's db_to_linear (powf; <= -120 dB gives 0, >= 80 dB is clamped to 80 dB); the
 *     master volume is made finite and clamped to [-128, 0] dB;
 *   - coefficients, arithmetic and libm policy as dspi_eq_set_params_device; running state as _apply_bulk_device (EQ
 *     state kept unless a band's topology flips, crossfeed state cleared, everything else left alone - arming the
 *     preset-mute fade is dspi_chain(q)_set_preset_mute's job);
 *   - the instance becomes DSPI_BULK_CURRENT: _collect_bulk_device then returns what dspi_bulk_params_collect returns for
 *     the state dspi_preset_slot_apply left, and host[i] is its host record.
 * Ordered behind earlier work on the engine stream; returns when the engine is reconfigured.  DSPI_EINVAL for a NULL
 * pointer, an image_stride below the slot size or a sample_rate that is not positive and finite, DSPI_ERANGE for a range
 * past the end of the engine (also one whose end wraps in 32 bits); nothing is written then.  n == 0 does nothing. */
int dspi_chain_apply_preset_device (dspi_chain *c,  uint32_t inst0, uint32_t n, const void *images, size_t image_stride,
                                    const dspi_preset_load *load, const dspi_bulk_host *host, float sample_rate, int32_t *results);
int dspi_chainq_apply_preset_device(dspi_chainq *c, uint32_t inst0, uint32_t n, const void *images, size_t image_stride,
                                    const dspi_preset_load *load, const dspi_bulk_host *host, float sample_rate, int32_t *results);
/* The state part of preset_save() for instances [inst0, inst0+n): writes dspi_preset_slot_size(platform) bytes at
 * images + i * image_stride - magic, version 12, slot_indices[i], CRC-32 - and leaves the rest of each stride as it was.
 * For a current or stale instance the bytes are those of _collect_bulk_device -> dspi_bulk_params_apply(packet, st,
 * exact_db = 1) on dspi_bulk_state_defaults -> dspi_preset_slot_collect(st, slot_indices[i]): pins, names, I2S fields and
 * padding zero, recipes carrying (channel, band) = (ch, b).  An unset instance gives an all-zero image, which an apply
 * rejects.  results[i] (results may be NULL) is the instance's DSPI_BULK_* mark.  Read-only; ordered behind everything
 * issued earlier on the engine stream, asynchronous process calls included; returns when the images are in the caller's
 * memory.  Argument errors as the apply call (there is no sample rate). */
int dspi_chain_collect_preset_device (dspi_chain *c,  uint32_t inst0, uint32_t n, const uint8_t *slot_indices, void *images, size_t image_stride,
                                      int32_t *results);
int dspi_chainq_collect_preset_device(dspi_chainq *c, uint32_t inst0, uint32_t n, const uint8_t *slot_indices, void *images, size_t image_stride,
                                      int32_t *results);

/* ---- S/PDIF (IEC 60958) subframe encoder: the step after the chain -------------------------- */
/* What stereo_to_spdif_producer_give_s32() does with every S/PDIF producer buffer
 * (pico_audio_spdif_multi/sample_encoding.cpp:42-50 -> spdif_update_subframe,
 * include/pico/audio_spdif/sample_encoding.h:27-50), together with the preamble / channel-status /
 * validity-user-status-parity stamping of init_spdif_buffer (audio_spdif.c:99-114) and the
 * block-position fix-up at DMA start (:372-388): 24-bit words in, 64-bit biphase-mark subframes out,
 * ready for the 2-bits-per-cell PIO serialiser. */
typedef struct { uint32_t l, h; } dspi_spdif_subframe;           /* spdif_subframe_t, sample_encoding.h:20-23 */
/* the reference's 256-entry table (audio_spdif.c:141-153), for hosts that keep its table-driven encoder */
void dspi_spdif_lookup_table(uint32_t table[256]);
/* words: [n_streams][frames][2] int32 (bits 23:0 used) - the layout dspi_chain_process_* writes with
 * n_streams = 4 * n_instances; subframes: [n_streams][frames][2] {l, h}.  Frame n of every stream sits at
 * block position (block_pos0 + n) % 192; channel_status = the 5 consumer status bytes (audio_spdif.c:82-88).
 * _device is asynchronous on `cuda_stream` (a cudaStream_t, may be NULL); _host copies in and out. */
int dspi_spdif_encode_device(int device, const int32_t *d_words, uint64_t n_streams, uint32_t frames, uint32_t block_pos0,
                             const uint8_t channel_status[5], dspi_spdif_subframe *d_subframes, void *cuda_stream);
int dspi_spdif_encode_host(int device, const int32_t *words, uint64_t n_streams, uint32_t frames, uint32_t block_pos0,
                           const uint8_t channel_status[5], dspi_spdif_subframe *subframes);

/* ---- S/PDIF subframes straight from the chain engines ------------------------------------------ */
/* Every chain instance has one S/PDIF transmitter (audio_spdif.c:82-88, :372-388), shared by all its pairs - four on the
 * RP2350 shape, two on the RP2040 shape (the firmware starts them together and feeds them the same frames): a block
 * position block_pos (0..191) and the 5 consumer channel-status bytes.  Frame T of a call (0-based over the call's F
 * frames) sits at block position (block_pos + T) % 192 on every pair of the instance.  EVERY process call - words form,
 * subframe form, outputs NULL or not - advances block_pos to (block_pos + F) % 192: the transmitter sends every frame the
 * chain produces.  A new engine starts each instance at block_pos 0 with the bytes init_spdif_buffer() stamps
 * { 0x04, 0x00, 0x00, 0x00, 0x0B } (byte 3 is the sample-rate code: set it for the instance's rate).  The engine keeps it
 * across calls; dspi_chain(q)_reset_state leaves it alone; it is not part of the state blob. */
typedef struct { uint8_t channel_status[5]; uint8_t block_pos; uint8_t reserved[2]; } dspi_spdif_tx;   /* 8 bytes */
#ifdef __cplusplus
static_assert(sizeof(dspi_spdif_tx) == 8, "dspi_spdif_tx");
#else
_Static_assert(sizeof(dspi_spdif_tx) == 8, "dspi_spdif_tx");
#endif
/* tx[n] for instances [inst0, inst0+n).  _set_ runs on the engine stream behind earlier asynchronous process calls (it
 * applies from the next call on) and has finished when it returns; _get_ waits for the engine stream, so it returns the
 * state after the last call issued.  Errors: DSPI_ERANGE for a range past the end (also one whose end wraps in 32 bits),
 * DSPI_EINVAL for NULL records or a block_pos >= 192 (nothing is written then); n = 0 does nothing. */
int dspi_chain_set_spdif_tx (dspi_chain *c,  uint32_t inst0, uint32_t n, const dspi_spdif_tx *tx);
int dspi_chain_get_spdif_tx (dspi_chain *c,  uint32_t inst0, uint32_t n, dspi_spdif_tx *tx);
int dspi_chainq_set_spdif_tx(dspi_chainq *c, uint32_t inst0, uint32_t n, const dspi_spdif_tx *tx);
int dspi_chainq_get_spdif_tx(dspi_chainq *c, uint32_t inst0, uint32_t n, dspi_spdif_tx *tx);
/* As dspi_chain(q)_process_packets_*, with the S/PDIF output as subframes written by the output stage itself:
 * subframes [n_instances][4 (Q28: 2)][F][2] dspi_spdif_subframe, i.e. exactly what dspi_spdif_encode_* makes of the
 * [n_instances * pairs][F][2] words the words form writes, at each instance's own block position and channel status.
 * Pairs whose two outputs are both disabled carry encoded zero words, as in the two-pass path.  No words buffer and no
 * second pass.  Arguments are checked as for the _packets_ forms; d_subframes must be 16-byte aligned.  Any output may be
 * NULL (the block position still advances). */
int dspi_chain_process_subframes_host   (dspi_chain *c,  const void *pcm,   uint32_t bit_depth, uint32_t n_packets, const uint16_t *packet_frames,
                                         dspi_spdif_subframe *subframes,   uint32_t *pdm_out,   dspi_status *status);
int dspi_chain_process_subframes_device (dspi_chain *c,  const void *d_pcm, uint32_t bit_depth, uint32_t n_packets, const uint16_t *packet_frames,
                                         dspi_spdif_subframe *d_subframes, uint32_t *d_pdm_out, dspi_status *d_status);
int dspi_chainq_process_subframes_host  (dspi_chainq *c, const void *pcm,   uint32_t bit_depth, uint32_t n_packets, const uint16_t *packet_frames,
                                         dspi_spdif_subframe *subframes,   uint32_t *pdm_out,   dspi_status_q28 *status);
int dspi_chainq_process_subframes_device(dspi_chainq *c, const void *d_pcm, uint32_t bit_depth, uint32_t n_packets, const uint16_t *packet_frames,
                                         dspi_spdif_subframe *d_subframes, uint32_t *d_pdm_out, dspi_status_q28 *d_status);
/* instances [inst0, inst0 + n) only, as dspi_chain(q)_process_packets_range_*: subframes [n][4 (Q28: 2)][F][2], row i for
 * instance inst0 + i; each instance encoded at its own block position and channel status; d_subframes 16-byte aligned */
int dspi_chain_process_subframes_range_host   (dspi_chain *c,  uint32_t inst0, uint32_t n, const void *pcm,   uint32_t bit_depth, uint32_t n_packets,
                                               const uint16_t *packet_frames, dspi_spdif_subframe *subframes,   uint32_t *pdm_out,   dspi_status *status);
int dspi_chain_process_subframes_range_device (dspi_chain *c,  uint32_t inst0, uint32_t n, const void *d_pcm, uint32_t bit_depth, uint32_t n_packets,
                                               const uint16_t *packet_frames, dspi_spdif_subframe *d_subframes, uint32_t *d_pdm_out, dspi_status *d_status);
int dspi_chainq_process_subframes_range_host  (dspi_chainq *c, uint32_t inst0, uint32_t n, const void *pcm,   uint32_t bit_depth, uint32_t n_packets,
                                               const uint16_t *packet_frames, dspi_spdif_subframe *subframes,   uint32_t *pdm_out,   dspi_status_q28 *status);
int dspi_chainq_process_subframes_range_device(dspi_chainq *c, uint32_t inst0, uint32_t n, const void *d_pcm, uint32_t bit_depth, uint32_t n_packets,
                                               const uint16_t *packet_frames, dspi_spdif_subframe *d_subframes, uint32_t *d_pdm_out, dspi_status_q28 *d_status);

/* ---- lanes: range calls of several clock groups running side by side ------------------------------ */
/* A lane is an issue queue of one engine, bound to a window of instances, with stage streams and a packet schedule of its
 * own.  Calls on different lanes run concurrently on the GPU: a farm opens one lane per clock group and serves each group's
 * packets on its lane, so that the small calls of several groups share the GPU instead of adding their times.  The lanes'
 * stage streams run in the engine's own SM partition (dspi_chain_sm_partition).
 *   Window.  _lane_open reserves instances [inst0, inst0 + n) and returns the lane's id in *lane.  inst0 is a multiple of 64,
 *   n > 0, and the window overlaps no open lane's window.  At most DSPI_CHAIN_MAX_LANES lanes are open at once; a closed
 *   lane's id may be handed out again.
 *   Calls.  _lane_process_packets_device / _lane_process_subframes_device run over any [inst0, inst0 + n) inside the lane's
 *   window (inst0 a multiple of 64, n == 0 does nothing).  Arguments, buffer layout and results are exactly those of
 *   dspi_chain(q)_process_packets_range_device / _process_subframes_range_device over that range.  Their host-memory forms
 *   are the lane host calls below.
 *   Ordering.  Calls on one lane run in issue order.  A lane call runs after every engine-level call issued before it, and
 *   every engine-level call runs after every lane call issued before it.  An engine-level call is any call taking the
 *   engine that is not a lane call: process, range process, set / edit / apply / collect, copy / export / import / reset,
 *   response, state, the S/PDIF and preset-mute getters and setters, dspi_chain_sync and destroy.  So engine-level calls
 *   are barriers across lanes, and lane calls are ordered only against them, never against other lanes.
 *   _lane_stream is where a lane's outputs (S/PDIF, PDM, status) become visible; dspi_chain_stream does not carry lane
 *   work.  _lane_sync waits for the lane's calls.
 *   Result.  Outputs, state, meters, envelope, S/PDIF transmitter and configuration record are byte for byte those of the
 *   same calls issued in the same order as range calls on the engine stream.
 *   No lane open.  Every other call issues exactly the work it issues without lanes (dspi_chain_launch_count included).
 *   Close.  _lane_close waits for the lane's calls and frees its streams; destroying the engine closes its lanes.
 *   Threads.  One host thread issues the calls of an engine and its lanes.  Lane calls do not wait for the device, with one
 *   exception: a call with more packets than any envelope-mode call before it grows the envelope table, and first waits
 *   for every lane and the engine stream.
 *   Errors (nothing is written on any error): DSPI_EINVAL for a NULL engine or lane pointer, a misaligned inst0, n == 0 or an
 *   overlapping window at _lane_open, an unknown or closed lane id, and every check of the range calls; DSPI_ERANGE for a
 *   window past the end of the engine (also one whose end wraps in 32 bits), a call range outside its lane's window, or a
 *   lane beyond DSPI_CHAIN_MAX_LANES.  _lane_stream returns NULL for an unknown or closed lane. */
#define DSPI_CHAIN_MAX_LANES 16
int   dspi_chain_lane_open (dspi_chain *c, uint32_t inst0, uint32_t n, uint32_t *lane);
int   dspi_chain_lane_close(dspi_chain *c, uint32_t lane);
int   dspi_chain_lane_process_packets_device  (dspi_chain *c, uint32_t lane, uint32_t inst0, uint32_t n, const void *d_pcm,
                                               uint32_t bit_depth, uint32_t n_packets, const uint16_t *packet_frames,
                                               int32_t *d_spdif_out, uint32_t *d_pdm_out, dspi_status *d_status);
int   dspi_chain_lane_process_subframes_device(dspi_chain *c, uint32_t lane, uint32_t inst0, uint32_t n, const void *d_pcm,
                                               uint32_t bit_depth, uint32_t n_packets, const uint16_t *packet_frames,
                                               dspi_spdif_subframe *d_subframes, uint32_t *d_pdm_out, dspi_status *d_status);
void *dspi_chain_lane_stream(dspi_chain *c, uint32_t lane);
int   dspi_chain_lane_sync  (dspi_chain *c, uint32_t lane);
int   dspi_chainq_lane_open (dspi_chainq *c, uint32_t inst0, uint32_t n, uint32_t *lane);
int   dspi_chainq_lane_close(dspi_chainq *c, uint32_t lane);
int   dspi_chainq_lane_process_packets_device  (dspi_chainq *c, uint32_t lane, uint32_t inst0, uint32_t n, const void *d_pcm,
                                                uint32_t bit_depth, uint32_t n_packets, const uint16_t *packet_frames,
                                                int32_t *d_spdif_out, uint32_t *d_pdm_out, dspi_status_q28 *d_status);
int   dspi_chainq_lane_process_subframes_device(dspi_chainq *c, uint32_t lane, uint32_t inst0, uint32_t n, const void *d_pcm,
                                                uint32_t bit_depth, uint32_t n_packets, const uint16_t *packet_frames,
                                                dspi_spdif_subframe *d_subframes, uint32_t *d_pdm_out, dspi_status_q28 *d_status);
void *dspi_chainq_lane_stream(dspi_chainq *c, uint32_t lane);
int   dspi_chainq_lane_sync  (dspi_chainq *c, uint32_t lane);

/* Lane host calls: a clock group's packets served from host memory on its lane (PCM from USB or the network, S/PDIF and PDM
 * back to the transmitters), so that a host-resident farm neither waits for nor holds up the other groups, and the copies
 * run while the stages do.
 *   Semantics.  _lane_process_packets_host / _lane_process_subframes_host have exactly the layouts, argument checks and
 *   results of dspi_chain(q)_process_packets_range_host / _process_subframes_range_host over [inst0, inst0 + n): the range
 *   lies inside the lane's window and inst0 is a multiple of 64; PDM rows of instances whose sub is off come back as zeros
 *   on every call.  Outputs, state, meters, envelope, transmitter and configuration record are byte for byte those of the
 *   same sequence with these calls issued as the engine-level range host calls.
 *   Memory.  pcm, spdif_out / subframes, pdm_out and status are page-locked host memory (dspi_host_alloc, cudaHostAlloc,
 *   cudaHostRegister, a pinned torch tensor); every output may be NULL.  Each non-NULL buffer is checked at its first byte
 *   and a pageable one is refused with DSPI_EINVAL before anything is issued: a lane call never waits, and a copy from
 *   pageable memory would.  The caller keeps the whole extent of every buffer page-locked until the call has completed.
 *   Ordering and lifetime.  Ordered as the lane process calls are: behind its lane's calls in issue order and against
 *   engine-level calls, never against another lane.  The call returns without waiting for the device.  packet_frames is
 *   read during the call.  pcm is read, and the outputs written, on the lane's timeline: pcm may be rewritten, and the
 *   outputs read, only once the lane has reached the end of the call, which an event recorded on _lane_stream after the
 *   call (or _lane_sync) shows.  This differs from the lane control calls, which read their inputs during the call.
 *   Pipelining.  The call runs over the packet slices of the stage pipeline.  Each slice's PCM frames are copied in on a
 *   copy stream of the lane just before its front stage, its S/PDIF frames leave after its output stage and its PDM frames
 *   after its modulator, on a second copy stream; the status leaves after the call.  So the copies overlap the stages
 *   and one another, and the device time hides under the link time.  Consecutive calls of one lane do not overlap.
 *   Staging.  Each lane has its own device staging, sized for its whole window at max_frames so that no later call grows
 *   it, and two copy streams.  The lane's first host call allocates the PCM (6 bytes per instance-frame) and status
 *   staging and the streams, its first call with PDM out the PDM staging (32 bytes per instance-frame), its first call with
 *   words the S/PDIF staging at 8 bytes per pair frame (32 per float, 16 per Q28 instance-frame) and its first call with
 *   subframes at 16 (64 / 32), replacing a words staging; each of these first waits for every lane and the engine stream.
 *   _lane_close frees them.  A 1024-instance float window at 6144 frames takes about 0.44 GB for words + PDM, 0.64 GB for
 *   subframes + PDM.
 *   Errors (nothing is issued on any error): every refusal of the range host calls, a pageable buffer and an unknown or
 *   closed lane with DSPI_EINVAL; a range outside the lane's window with DSPI_ERANGE.
 *   No lane host call made.  Every other call issues exactly the work it issues without them; the engine-level host calls
 *   stay barriers that return when their outputs are in host memory. */
int dspi_chain_lane_process_packets_host    (dspi_chain *c, uint32_t lane, uint32_t inst0, uint32_t n, const void *pcm, uint32_t bit_depth,
                                             uint32_t n_packets, const uint16_t *packet_frames, int32_t *spdif_out, uint32_t *pdm_out,
                                             dspi_status *status);
int dspi_chain_lane_process_subframes_host  (dspi_chain *c, uint32_t lane, uint32_t inst0, uint32_t n, const void *pcm, uint32_t bit_depth,
                                             uint32_t n_packets, const uint16_t *packet_frames, dspi_spdif_subframe *subframes,
                                             uint32_t *pdm_out, dspi_status *status);
int dspi_chainq_lane_process_packets_host   (dspi_chainq *c, uint32_t lane, uint32_t inst0, uint32_t n, const void *pcm, uint32_t bit_depth,
                                             uint32_t n_packets, const uint16_t *packet_frames, int32_t *spdif_out, uint32_t *pdm_out,
                                             dspi_status_q28 *status);
int dspi_chainq_lane_process_subframes_host (dspi_chainq *c, uint32_t lane, uint32_t inst0, uint32_t n, const void *pcm, uint32_t bit_depth,
                                             uint32_t n_packets, const uint16_t *packet_frames, dspi_spdif_subframe *subframes,
                                             uint32_t *pdm_out, dspi_status_q28 *status);

/* Lane control calls: the control calls a running clock group needs (a Console edit, a preset-change fade, a transmitter
 * restamp, a device restart, a device connecting, a preset recall, a session rate change), issued on the group's lane so
 * that they neither wait for nor hold up the other groups.
 *   Semantics.  Each call means exactly what its engine-level counterpart means over the same instances:
 *   _lane_edit_bulk_device is _edit_bulk_device, _lane_set_preset_mute is _set_preset_mute, _lane_set_spdif_tx is
 *   _set_spdif_tx, _lane_reset_instances is _reset_instances, _lane_apply_bulk_device is _apply_bulk_device,
 *   _lane_apply_preset_device is _apply_preset_device and _lane_set_rate_device is _set_rate_device, with the same argument
 *   checks, result codes, state rules, gain modes and libm policy; a rejected packet or image changes nothing.  Outputs,
 *   biquads, state, meters, envelope, transmitter, configuration record, host record and marks are byte for byte what the
 *   same sequence gives on the engine stream: every lane's calls in issue order, with the control calls issued as
 *   engine-level calls.
 *   Window.  Every instance a call names lies inside the lane's window: each edits[k].instance, or [inst0, inst0 + n) for
 *   the others (inst0 has no alignment rule beyond that).  Otherwise the call fails with DSPI_ERANGE.
 *   Ordering.  A lane control call is ordered against its lane's calls in issue order, and against engine-level calls as
 *   lane process calls are; never against another lane.
 *   No host wait.  The call returns without waiting for the device.  edits, states, tx, packets, host, images (at any
 *   stride >= the slot size), load and sample_rates are read during the call and may be reused as soon as it returns.
 *   Exceptions, each a growth of a buffer: a lane's first edit, first apply or rate switch, and first preset apply
 *   allocate its staging, and an engine whose skip rows were never set (no set_params, apply, import, copy or edit yet)
 *   remasks every row once; these first wait for every lane and the engine stream.  Uploads go through a ring of 8 pinned
 *   host buffers per lane: a call waits when the buffer it takes is still read by a copy 8 uploads back (an apply or
 *   preset apply takes one per 1024 instances), and a buffer that has to grow for a larger upload than it carried before
 *   is a pinned allocation, which may wait for the device.  A fade arm can make the lane's next process call grow the
 *   envelope table (see Threads above).
 *   Results.  d_results is device memory, written on the lane stream at the call's point and visible on _lane_stream:
 *   [n_edits] marks of each edit's instance (may be NULL); [n] firmware codes of a bulk apply and DSPI_PRESET_* codes of a
 *   preset apply (required, as results is for the engine-level calls); [n] DSPI_BULK_* marks of a rate switch (may be
 *   NULL).
 *   K1 kernel choice.  Lane edits, applies, preset applies and rate switches re-pack EQ rows but leave the K1 kernel that
 *   float engines selected for the topology of their rows, since other lanes may be running it; the next engine-level
 *   call waits for the lanes and selects it again.  Only speed depends on the choice.
 *   Errors (nothing is written on any error): every refusal of the engine-level call, and an unknown or closed lane, with
 *   DSPI_EINVAL; a window violation with DSPI_ERANGE.
 *   No lane control call made.  Every other call issues exactly the work it issues without them.
 * Left as barriers: _download_biquads (an instance image carries the biquads with their state), the state blob
 * (_state_export / _state_import), and the writes _set_params, _upload_biquads, _set_eq_params_device and
 * _set_dynamics_device, since the wire-packet routes above cover what a Console or a preset sends.  The reads a running
 * group needs have lane forms (the lane read calls below), and so do the moves of a device into a group's window (the
 * lane move calls below). */
int dspi_chain_lane_edit_bulk_device  (dspi_chain *c, uint32_t lane, uint32_t n_edits, const dspi_bulk_edit *edits, int exact_db,
                                       float sample_rate, int32_t *d_results);
int dspi_chain_lane_set_preset_mute   (dspi_chain *c, uint32_t lane, uint32_t inst0, uint32_t n, const dspi_preset_mute *states,
                                       uint32_t sample_rate_hz);
int dspi_chain_lane_set_spdif_tx      (dspi_chain *c, uint32_t lane, uint32_t inst0, uint32_t n, const dspi_spdif_tx *tx);
int dspi_chain_lane_reset_instances   (dspi_chain *c, uint32_t lane, uint32_t inst0, uint32_t n);
int dspi_chainq_lane_edit_bulk_device (dspi_chainq *c, uint32_t lane, uint32_t n_edits, const dspi_bulk_edit *edits, int exact_db,
                                       float sample_rate, int32_t *d_results);
int dspi_chainq_lane_set_preset_mute  (dspi_chainq *c, uint32_t lane, uint32_t inst0, uint32_t n, const dspi_preset_mute *states,
                                       uint32_t sample_rate_hz);
int dspi_chainq_lane_set_spdif_tx     (dspi_chainq *c, uint32_t lane, uint32_t inst0, uint32_t n, const dspi_spdif_tx *tx);
int dspi_chainq_lane_reset_instances  (dspi_chainq *c, uint32_t lane, uint32_t inst0, uint32_t n);
int dspi_chain_lane_apply_bulk_device   (dspi_chain *c, uint32_t lane, uint32_t inst0, uint32_t n, const dspi_wire_bulk_params *packets,
                                        const dspi_bulk_host *host, int exact_db, float sample_rate, int32_t *d_results);
int dspi_chain_lane_apply_preset_device (dspi_chain *c, uint32_t lane, uint32_t inst0, uint32_t n, const void *images, size_t image_stride,
                                        const dspi_preset_load *load, const dspi_bulk_host *host, float sample_rate, int32_t *d_results);
int dspi_chain_lane_set_rate_device     (dspi_chain *c, uint32_t lane, uint32_t inst0, uint32_t n, const float *sample_rates,
                                        int32_t *d_results);
int dspi_chainq_lane_apply_bulk_device  (dspi_chainq *c, uint32_t lane, uint32_t inst0, uint32_t n, const dspi_wire_bulk_params *packets,
                                        const dspi_bulk_host *host, int exact_db, float sample_rate, int32_t *d_results);
int dspi_chainq_lane_apply_preset_device(dspi_chainq *c, uint32_t lane, uint32_t inst0, uint32_t n, const void *images, size_t image_stride,
                                        const dspi_preset_load *load, const dspi_bulk_host *host, float sample_rate, int32_t *d_results);
int dspi_chainq_lane_set_rate_device    (dspi_chainq *c, uint32_t lane, uint32_t inst0, uint32_t n, const float *sample_rates,
                                        int32_t *d_results);

/* Lane read calls: the reads a running clock group needs (a Console connecting reads REQ_GET_ALL_PARAMS, a preset save, a
 * Console's EQ curve, a checkpoint or a move of a device to another engine, a poll of a fade or a transmitter), issued on
 * the group's lane so that they neither wait for nor hold up the other groups.
 *   Semantics.  Each call returns byte for byte what its engine-level counterpart returns over the same instances at the
 *   same point of the call sequence, after every call issued earlier on the lane and every engine-level call issued before
 *   it: _lane_collect_bulk_device is _collect_bulk_device (packets, host records, DSPI_BULK_* marks),
 *   _lane_collect_preset_device is _collect_preset_device (slot images; the stride tail is left as it was),
 *   _lane_export_instances is _export_instances (instance images with their header; the stride tail is left as it was),
 *   _lane_response_device is _response_device ({re, im} arrays), _lane_get_preset_mute is _get_preset_mute and
 *   _lane_get_spdif_tx is _get_spdif_tx (records with their reserved bytes zero).
 *   Read-only.  A later call on any lane or on the engine gives the bytes it would have given without the read.
 *   Window.  [inst0, inst0 + n) lies inside the lane's window (inst0 has no alignment rule beyond that); otherwise the call
 *   fails with DSPI_ERANGE.  n == 0 does nothing.
 *   Ordering and no host wait.  Ordered as the lane control calls are: behind its lane's calls and the engine-level calls
 *   issued before it, never against another lane.  The call returns without waiting for the device.
 *   Outputs.  d_packets, d_host, d_results, d_images, d_out, d_states and d_tx are device memory, written on the lane
 *   stream and visible on _lane_stream.  d_host and d_results may be NULL, as on the engine-level calls; every other
 *   output is required.  d_packets may hold any address: packets at a 16-byte aligned address are written in place,
 *   others go through the lane's staging and a device-to-device copy.  d_out must be 8-byte aligned ({re, im} float
 *   pairs are stored as such).  slot_indices and freqs_hz are host memory, read during the call: they may be reused as
 *   soon as it returns.
 *   Exceptions, each a growth of a buffer: a lane's first preset collect, first export, first response and first collect
 *   into packets that are not 16-byte aligned allocate its preset staging, image staging, frequency table (256 KiB) and
 *   bulk staging (unless an apply, rate switch or edit did); these first wait for every lane and the engine stream.  The
 *   image staging holds chunks of the whole window, so that no later export grows it: one instance image per instance of
 *   the window, at most 32 MiB (DSPI_HOST_CHUNK_MB), kept until the lane closes even if the lane only ever exports one
 *   instance.  Slot indices go through the lane's ring of pinned host buffers (see the lane control calls).
 *   Errors (nothing is written on any error): every refusal of the engine-level call, a NULL required output, a d_out
 *   that is not 8-byte aligned, and an unknown or closed lane, with DSPI_EINVAL; a window violation with DSPI_ERANGE.
 *   No lane read call made.  Every other call issues exactly the work it issues without them; the engine-level getters
 *   stay barriers. */
int dspi_chain_lane_collect_bulk_device   (dspi_chain *c, uint32_t lane, uint32_t inst0, uint32_t n, dspi_wire_bulk_params *d_packets,
                                          dspi_bulk_host *d_host, int32_t *d_results);
int dspi_chain_lane_collect_preset_device (dspi_chain *c, uint32_t lane, uint32_t inst0, uint32_t n, const uint8_t *slot_indices,
                                          void *d_images, size_t image_stride, int32_t *d_results);
int dspi_chain_lane_export_instances      (dspi_chain *c, uint32_t lane, uint32_t inst0, uint32_t n, void *d_images, size_t image_stride);
int dspi_chain_lane_response_device       (dspi_chain *c, uint32_t lane, uint32_t inst0, uint32_t n, const float *freqs_hz,
                                          uint32_t n_freqs, float sample_rate, float *d_out);
int dspi_chain_lane_get_preset_mute       (dspi_chain *c, uint32_t lane, uint32_t inst0, uint32_t n, dspi_preset_mute *d_states);
int dspi_chain_lane_get_spdif_tx          (dspi_chain *c, uint32_t lane, uint32_t inst0, uint32_t n, dspi_spdif_tx *d_tx);
int dspi_chainq_lane_collect_bulk_device  (dspi_chainq *c, uint32_t lane, uint32_t inst0, uint32_t n, dspi_wire_bulk_params *d_packets,
                                          dspi_bulk_host *d_host, int32_t *d_results);
int dspi_chainq_lane_collect_preset_device(dspi_chainq *c, uint32_t lane, uint32_t inst0, uint32_t n, const uint8_t *slot_indices,
                                          void *d_images, size_t image_stride, int32_t *d_results);
int dspi_chainq_lane_export_instances     (dspi_chainq *c, uint32_t lane, uint32_t inst0, uint32_t n, void *d_images, size_t image_stride);
int dspi_chainq_lane_response_device      (dspi_chainq *c, uint32_t lane, uint32_t inst0, uint32_t n, const float *freqs_hz,
                                          uint32_t n_freqs, float sample_rate, float *d_out);
int dspi_chainq_lane_get_preset_mute      (dspi_chainq *c, uint32_t lane, uint32_t inst0, uint32_t n, dspi_preset_mute *d_states);
int dspi_chainq_lane_get_spdif_tx         (dspi_chainq *c, uint32_t lane, uint32_t inst0, uint32_t n, dspi_spdif_tx *d_tx);

/* Lane move calls: the writes a device needs when it moves (a rate change moves it into another clock group's window, a
 * move to another engine or GPU imports its image there, a checkpoint is restored into a running group), issued on the
 * groups' lanes so that they neither wait for nor hold up the other groups.
 *   Semantics.  _lane_import_instances is _import_instances over [inst0, inst0 + n); _lane_copy_instances is
 *   _copy_instances(n, src, dst), with the same argument checks and the same all-or-nothing header check: src may repeat,
 *   dst is distinct and shares no index with src.  Outputs, biquads, running state, meters, envelope, transmitter,
 *   configuration record and marks are byte for byte what the same sequence gives with these calls issued as engine-level
 *   calls.
 *   Window.  Import: [inst0, inst0 + n) lies inside the lane's window.  Copy: every src[k] lies inside src_lane's window and
 *   every dst[k] inside dst_lane's; src_lane == dst_lane repacks within one group.  Otherwise the call fails with
 *   DSPI_ERANGE.  n == 0 does nothing.
 *   Ordering.  An import is ordered as the lane control calls are.  A copy is ordered against both of its lanes: it runs
 *   after every call issued earlier on either lane and after the engine-level calls issued before it, and every later call
 *   on either lane runs after it; it is never ordered against a third lane.  So the source lane may free the old slot right
 *   after the copy (with _lane_reset_instances, say) and the destination still gets the bytes from before the reset.
 *   Images.  images is host memory (an image from _export_instances, or from _lane_export_instances copied to the host),
 *   read during the call: it may be reused as soon as the call returns.  Any image_stride >= dspi_chain_instance_image_size
 *   is accepted.  Host memory lets the call check every header before anything is written, and keep its count of
 *   envelope-mode instances from the images without reading the device.
 *   No host wait.  Both calls return without waiting for the device.  src and dst are read during the call.  Exceptions,
 *   each a growth of a buffer that first waits for every lane and the engine stream: a lane's first import allocates its
 *   image staging (the one its exports use, sized for its whole window, at most 32 MiB, DSPI_HOST_CHUNK_MB), unless an
 *   export did; a lane's first copy as destination allocates its instance lists, sized for its window so that no later
 *   copy grows them; and an engine whose skip rows were never set remasks every row once.  Images and lists go through the
 *   lane's ring of 8 pinned host buffers (see the lane control calls; a copy's lists through the destination's): one
 *   buffer carries one staging chunk of images, at most 32 MiB (DSPI_HOST_CHUNK_MB) or one image if that is larger, or
 *   the 8 n bytes of a copy's lists.
 *   K1 kernel choice.  As for the lane control calls: both re-pack EQ rows and leave the choice to the next engine-level
 *   call.
 *   Errors (nothing is written on any error): every refusal of the engine-level call (NULL images or lists, a stride below
 *   the image size, a bad magic or version, an image of another arith, band count or size, a duplicate dst, an index
 *   both a source and a destination), and an unknown or closed lane, with DSPI_EINVAL; a window violation with
 *   DSPI_ERANGE.
 *   No lane move made.  Every other call issues exactly the work it issues without them; _import_instances and
 *   _copy_instances keep their copies, synchronisations and launches. */
int dspi_chain_lane_import_instances (dspi_chain  *c, uint32_t lane, uint32_t inst0, uint32_t n, const void *images, size_t image_stride);
int dspi_chain_lane_copy_instances   (dspi_chain  *c, uint32_t src_lane, uint32_t dst_lane, uint32_t n, const uint32_t *src, const uint32_t *dst);
int dspi_chainq_lane_import_instances(dspi_chainq *c, uint32_t lane, uint32_t inst0, uint32_t n, const void *images, size_t image_stride);
int dspi_chainq_lane_copy_instances  (dspi_chainq *c, uint32_t src_lane, uint32_t dst_lane, uint32_t n, const uint32_t *src, const uint32_t *dst);

/* ---- frequency response of EQ channels and chain instances ------------------------------------ */
/* The complex transfer function H(e^{j omega}) of the linear, time-invariant part of the path the NEXT process call applies,
 * read from the engine's device-resident coefficients and parameters at the point of the engine stream where the call is
 * issued (so after every upload, set_params, device-side generation and process call issued before it) and evaluated at
 * the caller's frequencies.  Read-only: it changes no coefficient, state, meter, envelope or S/PDIF transmitter field and
 * never touches the packed K1 / K2 stores; a process call after it gives the same bytes as one without it.
 * Every stage is taken from its recurrence as the processing runs it, as a 2-state model (DESIGN.md 4), formed and evaluated
 * in double; each output value is rounded once to float.
 *   EQ row: product over bands b < n_bands that are not bypassed - TDF2 (b0 + b1 z^-1 + b2 z^-2) / (1 + a1 z^-1 + a2 z^-2)
 *     with the firmware's signs (s1 = b1 x - a1 y + s2), or the SVF of dsp_pipeline.c:290-345 with its svf_type's output mix;
 *     Q28 coefficients enter as value / 2^28.  Bands >= n_bands are not processed and not included.
 *   Float chain, input side s (unpacked sample, full scale 1.0) -> output o (float value before the 24-bit / Q28 conversion):
 *     preamp; the loudness shelves if loudness is on (each shelf's bypass honoured); master EQ unless bypass_master_eq; the
 *     leveller, when enabled with look-ahead, as its 480-sample delay at 0 dB gain - exact for signals under its gate once
 *     the gain has settled, its level-dependent gain is not modelled; crossfeed if on, L' = (1 - LP) L + AP LP R with
 *     LP = a0 / (1 - b1 z^-1), AP = (a + z^-1) / (1 + a z^-1); the matrix crosspoints (enabled, phase invert); the output EQ
 *     (skipped for a muted or disabled output); the output gain gain_linear * vol_mul_master - host mute, the int16 volume
 *     quirk (0 dB gives -1), master volume and the preset-mute gain: the constant preset_mute_gain outside envelope mode, the
 *     envelope's current smooth gain inside it (during a fade: the gain reached so far, not the next packet's step); the
 *     delay z^-(dly mod MAX) for dly > 0, so dly == MAX is no delay, as the ring does.  Disabled outputs are exactly 0; the
 *     sub (output 9) is the value fed to the modulator.
 *   Q28 chain: the same in the RP2040's quantities (ratios of Q28 values): preamp_q28, Q28 TDF2 loudness shelves, Q28
 *     crossfeed, matrix gains as the Q15 integers the packet loop forms ((int32)(g * 32768)), the output gain as the Q15
 *     integer of usb_audio.c:1204-1205, MAX = 2048, and output EQs skipped while the master EQ is bypassed (quirk 3).
 *   Not modelled: float rounding, Q28 truncation, the leveller's level-dependent gain, the modulator's noise shaping.
 * freqs_hz[n_freqs] (host memory, read during the call and reusable as soon as it returns; 0 <= f <= sample_rate / 2,
 * finite), sample_rate > 0.  Output: interleaved float {re, im} pairs.
 *   *_device: d_out is device memory; asynchronous on the engine stream.
 *   *_host:   returns when the data is back; staged through a bounded device buffer in channel / instance chunks (32 MiB,
 *             DSPI_HOST_CHUNK_MB in the environment overrides), never n x n_freqs at once.
 * Errors: DSPI_EINVAL for NULL pointers, n_freqs == 0 or above 65536, a frequency that is NaN, negative or above Nyquist, a
 * sample_rate that is not positive and finite; DSPI_ERANGE for a range past the end (also one whose end wraps in 32 bits);
 * nothing is written then.  n == 0 does nothing.  All three EQ arithmetics are supported. */
int dspi_eq_response_host       (dspi_eq *e,     uint32_t ch0,   uint32_t n, const float *freqs_hz, uint32_t n_freqs, float sample_rate, float *out);    /* [n][n_freqs][2] */
int dspi_eq_response_device     (dspi_eq *e,     uint32_t ch0,   uint32_t n, const float *freqs_hz, uint32_t n_freqs, float sample_rate, float *d_out);
int dspi_chain_response_host    (dspi_chain *c,  uint32_t inst0, uint32_t n, const float *freqs_hz, uint32_t n_freqs, float sample_rate, float *out);    /* [n][9][2 inputs][n_freqs][2] */
int dspi_chain_response_device  (dspi_chain *c,  uint32_t inst0, uint32_t n, const float *freqs_hz, uint32_t n_freqs, float sample_rate, float *d_out);
int dspi_chainq_response_host   (dspi_chainq *c, uint32_t inst0, uint32_t n, const float *freqs_hz, uint32_t n_freqs, float sample_rate, float *out);    /* [n][5][2][n_freqs][2] */
int dspi_chainq_response_device (dspi_chainq *c, uint32_t inst0, uint32_t n, const float *freqs_hz, uint32_t n_freqs, float sample_rate, float *d_out);

/* pinned host memory helpers */
void *dspi_host_alloc(size_t bytes);
void dspi_host_free(void *p);
/* Bind the calling thread - and the memory it allocates from now on - to the NUMA node of the device's PCIe link
 * (sysfs numa_node + sched_setaffinity + set_mempolicy), so that staging memory allocated afterwards is local to the
 * link.  Returns the node, or -1 when the topology is not exposed (nothing changed).  Call before dspi_host_alloc. */
int dspi_bind_host_to_device(int device);

#ifdef __cplusplus
}
#endif
#endif /* DSPI_B200_H */
