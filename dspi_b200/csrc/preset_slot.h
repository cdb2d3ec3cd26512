/* preset_slot.h — PresetSlot v12 of flash_storage.c (:139-189), one packed layout per platform, shared by the host
 * preset functions (bulk_params_host.c) and the device preset kernels (bulk_ingest.cuh). */
#pragma once
#include <stdint.h>

#include "dspi_b200.h"

#define DSPI_SLOT_STRUCT(NAME, NC, NO, NPIN)                                                                         \
    typedef struct __attribute__((packed)) {                                                                         \
        uint32_t magic; uint16_t version, slot_index; uint32_t crc32;                                                \
        dspi_eq_param filter_recipes[NC][DSPI_MAX_BANDS];                                                            \
        float preamp_db; uint8_t bypass, padding[3];                                                                 \
        float delays_ms[NC];                                                                                         \
        float channel_gain_db[3]; uint8_t channel_mute[3], padding2;                                                 \
        uint8_t loudness_enabled, padding3[3]; float loudness_ref_spl, loudness_intensity_pct;                       \
        uint8_t crossfeed_enabled, crossfeed_preset, crossfeed_itd_enabled, padding4; float crossfeed_custom_fc, crossfeed_custom_feed_db; \
        struct __attribute__((packed)) { uint8_t enabled, phase_invert, reserved[2]; float gain_db; } matrix_crosspoints[2][NO]; \
        struct __attribute__((packed)) { uint8_t enabled, mute, reserved[2]; float gain_db, delay_ms; } matrix_outputs[NO]; \
        uint8_t output_pins[NPIN], pin_padding[8 - NPIN];                                                            \
        char channel_names[NC][32];                                                                                  \
        uint8_t output_types[4], i2s_bck_pin, i2s_mck_pin, i2s_mck_enabled, i2s_mck_multiplier;                      \
        uint8_t leveller_enabled, leveller_speed, leveller_lookahead, leveller_padding;                              \
        float leveller_amount, leveller_max_gain_db, leveller_gate_threshold_db;                                     \
        float preamp_db_per_ch[2]; float master_volume_db;                                                           \
    } NAME

DSPI_SLOT_STRUCT(slot_rp2350, 11, 9, 5);
DSPI_SLOT_STRUCT(slot_rp2040, 7, 5, 3);
