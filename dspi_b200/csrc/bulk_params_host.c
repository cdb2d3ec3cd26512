/* bulk_params_host.c — host-side ingest of the firmware's bulk parameter packet (no GPU needed).
 *
 * Reference: bulk_params.c (apply :178-377, collect :62-172, db_to_linear :49-56), the main-loop
 * work that follows a successful apply (main.c:1126-1162: dsp_recalculate_all_filters,
 * dsp_update_delay_samples) and the pending-flag handlers (loudness table, crossfeed and leveller
 * coefficients, main.c:876-900).  State that the firmware keeps in globals lives in dspi_bulk_state;
 * everything derived from it is produced with the library's own host parameter functions
 * (host_params.c), so a wire packet becomes exactly the records dspi_chain_set_params /
 * dspi_chain_upload_biquads take.  Built with gcc -ffp-contract=off like host_params.c. */
#include <math.h>
#include <string.h>

#include "dspi_b200.h"
#include "preset_slot.h"

enum { CH_OUT_1 = 2 };                                   /* config.h:310 */

static int n_channels(int platform) { return platform == DSPI_PLATFORM_RP2350 ? 11 : 7; }      /* config.h:322 / :327 */
static int n_outputs(int platform) { return platform == DSPI_PLATFORM_RP2350 ? 9 : 5; }        /* :321 / :326 */

/* bulk_params.c:49-56 — the firmware's own conversion: 4-term Taylor series of exp(), clamped */
static float db_to_linear_fw(float db)
{
    if (db == 0.0f) return 1.0f;
    if (db < -60.0f) db = -60.0f;
    if (db > 20.0f) db = 20.0f;
    float x = db * 0.1151292546f;
    float linear = 1.0f + x + x * x * 0.5f + x * x * x * 0.1666667f + x * x * x * x * 0.0416667f;
    return (linear < 0.0f) ? 0.0f : linear;
}

static float db_to_linear(float db, int exact)
{
    return exact ? powf(10.0f, db / 20.0f) : db_to_linear_fw(db);
}

/* C float -> int32 conversions in the firmware run on ARM (saturating); keep the same definition here */
static int32_t f2i_sat(float x)
{
    if (x != x) return 0;
    if (x >= 2147483648.0f) return INT32_MAX;
    if (x <= -2147483648.0f) return INT32_MIN;
    return (int32_t)x;
}

void dspi_bulk_state_defaults(dspi_bulk_state *st, int platform)
{
    memset(st, 0, sizeof(*st));
    st->platform = platform;
    for (int i = 0; i < 2; i++) { st->preamp_linear[i] = 1.0f; st->preamp_q28[i] = 1 << 28; }       /* usb_audio.c:150-152 */
    st->master_volume_linear = 1.0f;                                                               /* :160-162 */
    st->master_volume_q15 = 32768;
    st->loudness_ref_spl = 83.0f;                                                                  /* loudness.h defaults, usb_audio.c:175-176 */
    st->loudness_intensity_pct = 100.0f;
    st->crossfeed.custom_fc = 700.0f;                                                              /* crossfeed.h defaults */
    st->crossfeed.custom_feed_db = 4.5f;
    st->crossfeed.itd_enabled = 1;
    st->leveller.amount = 50.0f;                                                                   /* leveller.h:69-74 */
    st->leveller.max_gain_db = 15.0f;
    st->leveller.lookahead = 1;
    st->leveller.gate_threshold_db = -96.0f;
    for (int i = 0; i < 3; i++) { st->legacy_gain_linear[i] = 1.0f; st->legacy_gain_mul[i] = 32768; }
    for (int in = 0; in < 2; in++)
        for (int o = 0; o < DSPI_WIRE_MAX_OUTPUTS; o++) st->crosspoints[in][o].gain_linear = 1.0f;
    for (int o = 0; o < DSPI_WIRE_MAX_OUTPUTS; o++) st->outputs[o].gain_linear = 1.0f;
    for (int ch = 0; ch < DSPI_WIRE_MAX_CHANNELS; ch++)
        for (int b = 0; b < DSPI_MAX_BANDS; b++) {                                                 /* dsp_pipeline.c:177-199: flat */
            dspi_eq_param *r = &st->recipes[ch][b];
            r->channel = (uint8_t)ch; r->band = (uint8_t)b; r->type = 0; r->freq = 1000.0f; r->Q = 0.707f; r->gain_db = 0.0f;
        }
}

int dspi_bulk_params_apply(const dspi_wire_bulk_params *in, dspi_bulk_state *st, int exact_db)
{
    if (!in || !st) return DSPI_EINVAL;
    const int NC = n_channels(st->platform), NO = n_outputs(st->platform);
    /* :179-203 */
    if (in->header.format_version < 2 || in->header.format_version > DSPI_WIRE_FORMAT_VERSION) return -1;
    if (in->header.platform_id != (st->platform == DSPI_PLATFORM_RP2350 ? 1 : 0)) return -2;
    if (in->header.num_channels != NC) return -3;
    if (in->header.num_output_channels != NO) return -3;
    const uint16_t v5_size = (uint16_t)(sizeof(dspi_wire_bulk_params) - 16 - 16);
    const uint16_t v2_size = (uint16_t)(v5_size - 16 - 16);
    if (in->header.payload_length < v2_size || in->header.payload_length > sizeof(dspi_wire_bulk_params)) return -4;

    {   /* :206-215: legacy preamp field first */
        const float db = in->global.preamp_gain_db, lin = db_to_linear(db, exact_db);
        for (int i = 0; i < 2; i++) { st->preamp_db[i] = db; st->preamp_q28[i] = f2i_sat(lin * (float)(1 << 28)); st->preamp_linear[i] = lin; }
    }
    st->bypass_master_eq = in->global.bypass != 0;                                                 /* :217 */
    st->loudness_enabled = in->global.loudness_enabled != 0;                                       /* :219-222 */
    st->loudness_ref_spl = in->global.loudness_ref_spl;
    st->loudness_intensity_pct = in->global.loudness_intensity_pct;
    st->crossfeed.enabled = in->crossfeed.enabled != 0;                                            /* :225-230 */
    st->crossfeed.preset = in->crossfeed.preset;
    st->crossfeed.itd_enabled = in->crossfeed.itd_enabled != 0;
    st->crossfeed.custom_fc = in->crossfeed.custom_fc;
    st->crossfeed.custom_feed_db = in->crossfeed.custom_feed_db;
    for (int i = 0; i < 3; i++) {                                                                  /* :233-239 */
        st->legacy_gain_db[i] = in->legacy.gain_db[i];
        const float g = db_to_linear(in->legacy.gain_db[i], exact_db);
        st->legacy_gain_mul[i] = f2i_sat(g * 32768.0f);
        st->legacy_gain_linear[i] = g;
        st->legacy_mute[i] = in->legacy.mute[i] != 0;
    }
    for (int i = 0; i < NC; i++) st->channel_delays_ms[i] = in->delays.delay_ms[i];                /* :242-244 */
    for (int inp = 0; inp < 2; inp++)                                                              /* :247-254 */
        for (int o = 0; o < NO; o++) {
            dspi_matrix_crosspoint *x = &st->crosspoints[inp][o];
            x->enabled = in->crosspoints[inp][o].enabled;
            x->phase_invert = in->crosspoints[inp][o].phase_invert;
            x->gain_db = in->crosspoints[inp][o].gain_db;
            x->gain_linear = db_to_linear(in->crosspoints[inp][o].gain_db, exact_db);
        }
    for (int o = 0; o < NO; o++) {                                                                 /* :257-264 */
        dspi_output_channel *oc = &st->outputs[o];
        oc->enabled = in->outputs[o].enabled;
        oc->mute = in->outputs[o].mute;
        oc->gain_db = in->outputs[o].gain_db;
        oc->gain_linear = db_to_linear(in->outputs[o].gain_db, exact_db);
        oc->delay_ms = in->outputs[o].delay_ms;
        st->channel_delays_ms[CH_OUT_1 + o] = in->outputs[o].delay_ms;
    }
    for (int ch = 0; ch < NC; ch++)                                                                /* :291-300 */
        for (int b = 0; b < DSPI_MAX_BANDS; b++) {
            dspi_eq_param *r = &st->recipes[ch][b];
            r->channel = (uint8_t)ch;
            r->band = (uint8_t)b;
            r->type = in->eq[ch][b].type;
            r->freq = in->eq[ch][b].freq;
            r->Q = in->eq[ch][b].q;
            r->gain_db = in->eq[ch][b].gain_db;
        }
    if (in->header.format_version >= 4) {                                                          /* :330-346 */
        st->leveller.enabled = in->leveller.enabled != 0;
        st->leveller.speed = in->leveller.speed;
        st->leveller.lookahead = in->leveller.lookahead != 0;
        st->leveller.amount = in->leveller.amount;
        st->leveller.max_gain_db = in->leveller.max_gain_db;
        st->leveller.gate_threshold_db = in->leveller.gate_threshold_db;
    } else {
        st->leveller.enabled = 0;
        st->leveller.amount = 50.0f;
        st->leveller.speed = 0;
        st->leveller.max_gain_db = 15.0f;
        st->leveller.lookahead = 1;
        st->leveller.gate_threshold_db = -96.0f;
    }
    if (in->header.format_version >= 6) {                                                          /* :351-375 */
        for (int i = 0; i < 2; i++) {
            const float db = in->preamp.preamp_db[i], lin = db_to_linear(db, exact_db);
            st->preamp_db[i] = db;
            st->preamp_q28[i] = f2i_sat(lin * (float)(1 << 28));
            st->preamp_linear[i] = lin;
        }
        float db = in->master_volume.master_volume_db;
        if (!isfinite(db)) db = 0.0f;
        if (db < -128.0f) db = -128.0f;
        if (db > 0.0f) db = 0.0f;
        st->master_volume_db = db;
        if (db <= -128.0f) { st->master_volume_linear = 0.0f; st->master_volume_q15 = 0; }
        else {
            const float lin = powf(10.0f, db / 20.0f);
            st->master_volume_linear = lin;
            st->master_volume_q15 = f2i_sat(lin * 32768.0f);
        }
    }
    return 0;
}

void dspi_bulk_params_collect(const dspi_bulk_state *st, dspi_wire_bulk_params *out)
{
    const int NC = n_channels(st->platform), NO = n_outputs(st->platform);
    memset(out, 0, sizeof(*out));
    out->header.format_version = DSPI_WIRE_FORMAT_VERSION;                                         /* :66-78 */
    out->header.platform_id = st->platform == DSPI_PLATFORM_RP2350 ? 1 : 0;
    out->header.num_channels = (uint8_t)NC;
    out->header.num_output_channels = (uint8_t)NO;
    out->header.num_input_channels = 2;
    out->header.max_bands = DSPI_MAX_BANDS;
    out->header.payload_length = (uint16_t)sizeof(*out);
    out->header.fw_version_major = 1;                                                              /* config.h:273-274 */
    out->header.fw_version_minor = 1;
    out->global.preamp_gain_db = st->preamp_db[0];                                                 /* :81-85 */
    out->global.bypass = st->bypass_master_eq ? 1 : 0;
    out->global.loudness_enabled = st->loudness_enabled ? 1 : 0;
    out->global.loudness_ref_spl = st->loudness_ref_spl;
    out->global.loudness_intensity_pct = st->loudness_intensity_pct;
    out->crossfeed.enabled = st->crossfeed.enabled ? 1 : 0;                                        /* :88-92 */
    out->crossfeed.preset = st->crossfeed.preset;
    out->crossfeed.itd_enabled = st->crossfeed.itd_enabled ? 1 : 0;
    out->crossfeed.custom_fc = st->crossfeed.custom_fc;
    out->crossfeed.custom_feed_db = st->crossfeed.custom_feed_db;
    for (int i = 0; i < 3; i++) { out->legacy.gain_db[i] = st->legacy_gain_db[i]; out->legacy.mute[i] = st->legacy_mute[i] ? 1 : 0; }
    for (int i = 0; i < NC; i++) out->delays.delay_ms[i] = st->channel_delays_ms[i];
    for (int inp = 0; inp < 2; inp++)
        for (int o = 0; o < NO; o++) {
            out->crosspoints[inp][o].enabled = st->crosspoints[inp][o].enabled;
            out->crosspoints[inp][o].phase_invert = st->crosspoints[inp][o].phase_invert;
            out->crosspoints[inp][o].gain_db = st->crosspoints[inp][o].gain_db;
        }
    for (int o = 0; o < NO; o++) {
        out->outputs[o].enabled = st->outputs[o].enabled;
        out->outputs[o].mute = st->outputs[o].mute;
        out->outputs[o].gain_db = st->outputs[o].gain_db;
        out->outputs[o].delay_ms = st->outputs[o].delay_ms;
    }
    out->pins.num_pin_outputs = st->platform == DSPI_PLATFORM_RP2350 ? 5 : 3;                       /* :123 (pin numbers: control plane) */
    for (int ch = 0; ch < NC; ch++)
        for (int b = 0; b < DSPI_MAX_BANDS; b++) {
            out->eq[ch][b].type = st->recipes[ch][b].type;
            out->eq[ch][b].freq = st->recipes[ch][b].freq;
            out->eq[ch][b].q = st->recipes[ch][b].Q;
            out->eq[ch][b].gain_db = st->recipes[ch][b].gain_db;
        }
    out->leveller.enabled = st->leveller.enabled ? 1 : 0;                                          /* :158-163 */
    out->leveller.speed = st->leveller.speed;
    out->leveller.lookahead = st->leveller.lookahead ? 1 : 0;
    out->leveller.amount = st->leveller.amount;
    out->leveller.max_gain_db = st->leveller.max_gain_db;
    out->leveller.gate_threshold_db = st->leveller.gate_threshold_db;
    for (int i = 0; i < 2; i++) out->preamp.preamp_db[i] = st->preamp_db[i];
    out->master_volume.master_volume_db = st->master_volume_db;
}

/* dsp_update_delay_samples(), dsp_pipeline.c:216-239, for one output */
static int32_t delay_samples(const dspi_bulk_state *st, int o, int n_out, float fs, int32_t max_delay)
{
    float delay_ms = st->channel_delays_ms[CH_OUT_1 + o];
    if (o == n_out - 1) delay_ms += (float)128 / fs * 1000.0f;                                     /* SUB_ALIGN_SAMPLES, config.h:93-95 */
    int32_t s = f2i_sat(delay_ms * fs / 1000.0f);
    if (s > max_delay) s = max_delay;
    if (s < 0) s = 0;
    return s;
}

int dspi_bulk_state_to_chain_f32(const dspi_bulk_state *st, float fs, int16_t host_volume_8_8, int host_mute,
                                 dspi_chain_params_f32 *p, dspi_biquad_f32 biquads[11][DSPI_MAX_BANDS])
{
    if (!st || !p || !biquads) return DSPI_EINVAL;
    if (st->platform != DSPI_PLATFORM_RP2350) return DSPI_EINVAL;
    memset(p, 0, sizeof(*p));
    uint8_t row = 0;
    p->host_vol_mul = dspi_host_volume(host_volume_8_8, &row);                                     /* audio_set_volume(), usb_audio.c:428-440 */
    p->host_mute = host_mute != 0;
    p->bypass_master_eq = st->bypass_master_eq;
    p->loudness_enabled = st->loudness_enabled;
    p->crossfeed_enabled = st->crossfeed.enabled;                                                  /* crossfeed_bypassed = !enabled, main.c:882 */
    p->leveller_enabled = st->leveller.enabled;                                                    /* main.c:893 */
    p->leveller_lookahead = st->leveller.lookahead;
    p->preset_mute_gain = 1.0f;
    p->master_volume_linear = st->master_volume_linear;
    p->preamp_linear[0] = st->preamp_linear[0];
    p->preamp_linear[1] = st->preamp_linear[1];
    {
        static _Thread_local dspi_loudness_coeffs_f32 table[61][2];
        dspi_loudness_compute_table_f32(table, st->loudness_ref_spl, st->loudness_intensity_pct, fs);   /* loudness_recompute_pending */
        p->loudness[0] = table[row][0];
        p->loudness[1] = table[row][1];
    }
    dspi_crossfeed_compute_coefficients_f32(&p->crossfeed, &st->crossfeed, fs);                    /* crossfeed_update_pending */
    dspi_leveller_compute_coefficients(&p->leveller, &st->leveller, fs);                           /* leveller_update_pending */
    for (int inp = 0; inp < 2; inp++)
        for (int o = 0; o < 9; o++) p->matrix.crosspoints[inp][o] = st->crosspoints[inp][o];
    for (int o = 0; o < 9; o++) {
        p->matrix.outputs[o] = st->outputs[o];
        p->matrix.outputs[o].delay_samples = delay_samples(st, o, 9, fs, DSPI_CHAIN_MAX_DELAY);
    }
    for (int ch = 0; ch < 11; ch++)                                                                /* dsp_recalculate_all_filters */
        for (int b = 0; b < DSPI_MAX_BANDS; b++) {
            dspi_eq_param r = st->recipes[ch][b];
            dspi_compute_coefficients_f32(&r, &biquads[ch][b], fs);
        }
    return DSPI_OK;
}

int dspi_bulk_state_to_chain_q28(const dspi_bulk_state *st, float fs, int16_t host_volume_8_8, int host_mute,
                                 dspi_chain_params_q28 *p, dspi_biquad_q28 biquads[7][DSPI_MAX_BANDS])
{
    if (!st || !p || !biquads) return DSPI_EINVAL;
    if (st->platform != DSPI_PLATFORM_RP2040) return DSPI_EINVAL;
    memset(p, 0, sizeof(*p));
    uint8_t row = 0;
    p->host_vol_mul = dspi_host_volume(host_volume_8_8, &row);
    p->host_mute = host_mute != 0;
    p->bypass_master_eq = st->bypass_master_eq;
    p->loudness_enabled = st->loudness_enabled;
    p->crossfeed_enabled = st->crossfeed.enabled;
    p->leveller_enabled = st->leveller.enabled;
    p->leveller_lookahead = st->leveller.lookahead;
    p->preset_mute_gain = 1.0f;
    p->master_volume_q15 = st->master_volume_q15;
    p->preamp_q28[0] = st->preamp_q28[0];
    p->preamp_q28[1] = st->preamp_q28[1];
    {
        static _Thread_local dspi_loudness_coeffs_q28 table[61][2];
        dspi_loudness_compute_table_q28(table, st->loudness_ref_spl, st->loudness_intensity_pct, fs);
        p->loudness[0] = table[row][0];
        p->loudness[1] = table[row][1];
    }
    dspi_crossfeed_compute_coefficients_q28(&p->crossfeed, &st->crossfeed, fs);
    dspi_leveller_compute_coefficients(&p->leveller, &st->leveller, fs);
    for (int inp = 0; inp < 2; inp++)
        for (int o = 0; o < 5; o++) p->matrix.crosspoints[inp][o] = st->crosspoints[inp][o];
    for (int o = 0; o < 5; o++) {
        p->matrix.outputs[o] = st->outputs[o];
        p->matrix.outputs[o].delay_samples = delay_samples(st, o, 5, fs, DSPI_CHAINQ_MAX_DELAY);
    }
    for (int ch = 0; ch < 7; ch++)
        for (int b = 0; b < DSPI_MAX_BANDS; b++) {
            dspi_eq_param r = st->recipes[ch][b];
            dspi_compute_coefficients_q28(&r, &biquads[ch][b], fs);
        }
    return DSPI_OK;
}

/* ================================================================================================
 * Preset slot images — flash_storage.c (PresetSlot v12 :139-189, crc32 :282-291, db_to_linear :302-306,
 * collect_live_state :464-556, apply_master_volume_db :558-571, apply_master_volume_from_mode :580-590,
 * apply_slot_to_live :597-744, validate_slot :750-760)
 * ================================================================================================ */
uint32_t dspi_crc32(const void *data, size_t len)
{
    const uint8_t *p = (const uint8_t *)data;
    uint32_t crc = 0xFFFFFFFFu;
    for (size_t i = 0; i < len; i++) {
        crc ^= p[i];
        for (int j = 0; j < 8; j++) crc = (crc >> 1) ^ (0xEDB88320u & (0u - (crc & 1u)));
    }
    return ~crc;
}

/* flash_storage.c:302-306 */
static float db_to_linear_flash(float db)
{
    if (db <= -120.0f) return 0.0f;
    if (db >= 80.0f) db = 80.0f;
    return powf(10.0f, db / 20.0f);
}

size_t dspi_preset_slot_size(int platform) { return platform == DSPI_PLATFORM_RP2350 ? sizeof(slot_rp2350) : sizeof(slot_rp2040); }

/* flash_storage.c:558-571 */
static void apply_master_volume_db(dspi_bulk_state *st, float db)
{
    if (!isfinite(db)) db = 0.0f;
    if (db < -128.0f) db = -128.0f;
    if (db > 0.0f) db = 0.0f;
    st->master_volume_db = db;
    if (db <= -128.0f) { st->master_volume_linear = 0.0f; st->master_volume_q15 = 0; }
    else {
        const float lin = powf(10.0f, db / 20.0f);
        st->master_volume_linear = lin;
        st->master_volume_q15 = f2i_sat(lin * 32768.0f);
    }
}

#define SLOT_IMPL(SUF, TYPE, NC, NO)                                                                                 \
    static int apply_##SUF(const TYPE *s, uint8_t slot_index, uint8_t mv_mode, float dir_mv_db, dspi_bulk_state *st) \
    {                                                                                                                \
        if (s->magic != DSPI_PRESET_SLOT_MAGIC) return DSPI_PRESET_ERR_CRC;                         /* :752 */        \
        if (s->slot_index != slot_index) return DSPI_PRESET_ERR_CRC;                                /* :753 */        \
        if (dspi_crc32(&s->filter_recipes, sizeof(TYPE) - offsetof(TYPE, filter_recipes)) != s->crc32) return DSPI_PRESET_ERR_CRC;   /* :755-757 */ \
        memcpy(st->recipes, s->filter_recipes, sizeof(s->filter_recipes));                          /* :599 */        \
        for (int i = 0; i < 2; i++) {                                                               /* :602-617 */    \
            const float db = s->version >= 12 ? s->preamp_db_per_ch[i] : s->preamp_db, lin = db_to_linear_flash(db);  \
            st->preamp_db[i] = db; st->preamp_q28[i] = f2i_sat(lin * (float)(1 << 28)); st->preamp_linear[i] = lin;   \
        }                                                                                                            \
        st->bypass_master_eq = s->bypass != 0;                                                      /* :620 */        \
        memcpy(st->channel_delays_ms, s->delays_ms, sizeof(s->delays_ms));                          /* :623 */        \
        for (int i = 0; i < 3; i++) {                                                               /* :626-631 */    \
            st->legacy_gain_db[i] = s->channel_gain_db[i];                                                           \
            st->legacy_gain_mul[i] = f2i_sat(db_to_linear_flash(s->channel_gain_db[i]) * 32768.0f);                  \
            st->legacy_mute[i] = s->channel_mute[i] != 0;                                                            \
        }                                                                                                            \
        st->loudness_enabled = s->loudness_enabled != 0;                                            /* :634-637 */    \
        st->loudness_ref_spl = s->loudness_ref_spl;                                                                  \
        st->loudness_intensity_pct = s->loudness_intensity_pct;                                                      \
        st->crossfeed.enabled = s->crossfeed_enabled != 0;                                          /* :640-645 */    \
        st->crossfeed.preset = s->crossfeed_preset;                                                                  \
        st->crossfeed.itd_enabled = s->crossfeed_itd_enabled != 0;                                                   \
        st->crossfeed.custom_fc = s->crossfeed_custom_fc;                                                            \
        st->crossfeed.custom_feed_db = s->crossfeed_custom_feed_db;                                                  \
        for (int in = 0; in < 2; in++)                                                              /* :648-655 */    \
            for (int o = 0; o < NO; o++) {                                                                           \
                dspi_matrix_crosspoint *x = &st->crosspoints[in][o];                                                 \
                x->enabled = s->matrix_crosspoints[in][o].enabled;                                                   \
                x->phase_invert = s->matrix_crosspoints[in][o].phase_invert;                                         \
                x->gain_db = s->matrix_crosspoints[in][o].gain_db;                                                   \
                x->gain_linear = db_to_linear_flash(s->matrix_crosspoints[in][o].gain_db);                           \
            }                                                                                                        \
        for (int o = 0; o < NO; o++) {                                                              /* :656-663 */    \
            dspi_output_channel *oc = &st->outputs[o];                                                               \
            oc->enabled = s->matrix_outputs[o].enabled;                                                              \
            oc->mute = s->matrix_outputs[o].mute;                                                                    \
            oc->gain_db = s->matrix_outputs[o].gain_db;                                                              \
            oc->gain_linear = db_to_linear_flash(s->matrix_outputs[o].gain_db);                                      \
            oc->delay_ms = s->matrix_outputs[o].delay_ms;                                                            \
            st->channel_delays_ms[CH_OUT_1 + o] = s->matrix_outputs[o].delay_ms;                                     \
        }                                                                                                            \
        if (s->version >= 10) {                                                                     /* :724-741 */    \
            st->leveller.enabled = s->leveller_enabled != 0;                                                         \
            st->leveller.speed = s->leveller_speed;                                                                  \
            st->leveller.lookahead = s->leveller_lookahead != 0;                                                     \
            st->leveller.amount = s->leveller_amount;                                                                \
            st->leveller.max_gain_db = s->leveller_max_gain_db;                                                      \
            st->leveller.gate_threshold_db = s->leveller_gate_threshold_db;                                          \
        } else {                                                                                                     \
            st->leveller.enabled = 0; st->leveller.amount = 50.0f; st->leveller.speed = 0;                           \
            st->leveller.max_gain_db = 15.0f; st->leveller.lookahead = 1; st->leveller.gate_threshold_db = -96.0f;   \
        }                                                                                                            \
        apply_master_volume_db(st, (mv_mode == 1 && s->version >= 12) ? s->master_volume_db : dir_mv_db);   /* :580-590 */ \
        return DSPI_PRESET_OK;                                                                                       \
    }                                                                                                                \
    static void collect_##SUF(const dspi_bulk_state *st, uint8_t slot_index, TYPE *s)                                \
    {                                                                                                                \
        memset(s, 0, sizeof(*s));                                                                                    \
        s->magic = DSPI_PRESET_SLOT_MAGIC; s->version = DSPI_PRESET_SLOT_VERSION; s->slot_index = slot_index;        \
        memcpy(s->filter_recipes, st->recipes, sizeof(s->filter_recipes));                                           \
        s->preamp_db = st->preamp_db[0];                                                                             \
        s->bypass = st->bypass_master_eq ? 1 : 0;                                                                    \
        memcpy(s->delays_ms, st->channel_delays_ms, sizeof(s->delays_ms));                                           \
        for (int i = 0; i < 3; i++) { s->channel_gain_db[i] = st->legacy_gain_db[i]; s->channel_mute[i] = st->legacy_mute[i] ? 1 : 0; } \
        s->loudness_enabled = st->loudness_enabled ? 1 : 0;                                                          \
        s->loudness_ref_spl = st->loudness_ref_spl; s->loudness_intensity_pct = st->loudness_intensity_pct;          \
        s->crossfeed_enabled = st->crossfeed.enabled ? 1 : 0; s->crossfeed_preset = st->crossfeed.preset;            \
        s->crossfeed_itd_enabled = st->crossfeed.itd_enabled ? 1 : 0;                                                \
        s->crossfeed_custom_fc = st->crossfeed.custom_fc; s->crossfeed_custom_feed_db = st->crossfeed.custom_feed_db; \
        for (int in = 0; in < 2; in++)                                                                               \
            for (int o = 0; o < NO; o++) {                                                                           \
                s->matrix_crosspoints[in][o].enabled = st->crosspoints[in][o].enabled;                               \
                s->matrix_crosspoints[in][o].phase_invert = st->crosspoints[in][o].phase_invert;                     \
                s->matrix_crosspoints[in][o].gain_db = st->crosspoints[in][o].gain_db;                               \
            }                                                                                                        \
        for (int o = 0; o < NO; o++) {                                                                               \
            s->matrix_outputs[o].enabled = st->outputs[o].enabled; s->matrix_outputs[o].mute = st->outputs[o].mute;  \
            s->matrix_outputs[o].gain_db = st->outputs[o].gain_db; s->matrix_outputs[o].delay_ms = st->outputs[o].delay_ms; \
        }                                                                                                            \
        s->leveller_enabled = st->leveller.enabled ? 1 : 0; s->leveller_speed = st->leveller.speed;                  \
        s->leveller_lookahead = st->leveller.lookahead ? 1 : 0; s->leveller_amount = st->leveller.amount;            \
        s->leveller_max_gain_db = st->leveller.max_gain_db; s->leveller_gate_threshold_db = st->leveller.gate_threshold_db; \
        for (int i = 0; i < 2; i++) s->preamp_db_per_ch[i] = st->preamp_db[i];                                       \
        s->master_volume_db = st->master_volume_db;                                                                  \
        s->crc32 = dspi_crc32(&s->filter_recipes, sizeof(TYPE) - offsetof(TYPE, filter_recipes));                    \
    }

SLOT_IMPL(rp2350, slot_rp2350, 11, 9)
SLOT_IMPL(rp2040, slot_rp2040, 7, 5)

int dspi_preset_slot_apply(const void *slot, size_t len, uint8_t slot_index, uint8_t master_volume_mode, float dir_master_volume_db,
                           dspi_bulk_state *st)
{
    if (!slot || !st) return DSPI_EINVAL;
    if (len < dspi_preset_slot_size(st->platform)) return DSPI_PRESET_ERR_CRC;
    if (st->platform == DSPI_PLATFORM_RP2350) return apply_rp2350((const slot_rp2350 *)slot, slot_index, master_volume_mode, dir_master_volume_db, st);
    return apply_rp2040((const slot_rp2040 *)slot, slot_index, master_volume_mode, dir_master_volume_db, st);
}

int dspi_preset_slot_collect(const dspi_bulk_state *st, uint8_t slot_index, void *out, size_t cap)
{
    if (!st || !out) return DSPI_EINVAL;
    if (cap < dspi_preset_slot_size(st->platform)) return DSPI_ERANGE;
    if (st->platform == DSPI_PLATFORM_RP2350) collect_rp2350(st, slot_index, (slot_rp2350 *)out);
    else collect_rp2040(st, slot_index, (slot_rp2040 *)out);
    return DSPI_OK;
}
