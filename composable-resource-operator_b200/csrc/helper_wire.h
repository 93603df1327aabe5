/*
 * helper_wire.h — the argv and stdout of croprobe-cli's -raw commands, stated once for both sides: the library, which
 * writes the argv and reads the frames, and croprobe-cli, which reads the argv and writes the frames.  Plain C, so that
 * croprobe_cli.c and the C++ units both include it; internal, so nothing here is exported or part of croprobe.h.
 *
 * argv: croprobe-cli <cmd> <uuid> [<seed_base>] <field 0> ... <field n-1> <cap>, each field a decimal of the option
 * it names.  The options not on argv are the reserved ones and deadline_ms (the library keeps the deadline).
 *
 * stdout: one frame per result, see cro_wire_frame.
 */
#ifndef CRO_HELPER_WIRE_H
#define CRO_HELPER_WIRE_H

#include <inttypes.h>
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/croprobe.h"

/* One option on argv: its offset and size in its cro_*_opts struct, and whether its type is signed. */
typedef struct cro_wire_field {
    uint16_t at;
    uint8_t size;
    uint8_t is_signed;
} cro_wire_field;

/* The field f of T, its size and signedness taken from its type (compared with 1, not 0: no type-limits warning). */
#define CRO_WIRE_TYPE(T, f) __typeof__(((T *)0)->f)
#define CRO_WIRE_FIELD(T, f) {offsetof(T, f), sizeof(((T *)0)->f), (CRO_WIRE_TYPE(T, f))-1 < (CRO_WIRE_TYPE(T, f))1}
/* Where the count field f of T is in a frame's head: its offset and width. */
#define CRO_WIRE_AT(T, f) offsetof(T, f), sizeof(((T *)0)->f)

/* One check's frame: the result; `counts` uint64_t counts of the helper's own; the per-SM block of max_sms entries of
 * sm bytes (none when max_sms is 0), n_sms of them filled; then n records of rec bytes.  n_sms and n are the
 * little-endian integers of n_sms_width and n_width bytes at n_sms_at and n_at in the head, in the result or in the
 * counts (n_sms_width 0: no per-SM list). */
typedef struct cro_wire_frame {
    uint32_t result, counts, sm, max_sms, rec;
    uint32_t n_sms_at, n_sms_width, n_at, n_width;
} cro_wire_frame;

/* The compute, precision, sparse, warp-MMA and L2 frames: the counts n_sms and n follow the result. */
#define CRO_WIRE_SM_FRAME(R, S, F, MAX) {sizeof(R), 2, sizeof(S), MAX, sizeof(F), sizeof(R), 8, sizeof(R) + 8, 8}

/* One -raw command: its name, whether argv[3] is cro_opts.seed_base (the device seed is seed_base | minor, as in
 * process), its option fields in argv order, and its frame. */
typedef struct cro_wire {
    const char *cmd;
    int seeded;
    uint32_t n_fields;
    const cro_wire_field *fields;
    cro_wire_frame frame;
} cro_wire;

#define CRO_WIRE_FIELDS(a) (uint32_t)(sizeof(a) / sizeof *(a)), a

static const cro_wire_field cro_wire_scan_fields[] = {
    CRO_WIRE_FIELD(cro_scan_opts, max_bytes),        CRO_WIRE_FIELD(cro_scan_opts, reserve_bytes),
    CRO_WIRE_FIELD(cro_scan_opts, seed),             CRO_WIRE_FIELD(cro_scan_opts, test_chunk_bytes),
    CRO_WIRE_FIELD(cro_scan_opts, test_force_first), CRO_WIRE_FIELD(cro_scan_opts, test_force_count),
    CRO_WIRE_FIELD(cro_scan_opts, test_force_and),   CRO_WIRE_FIELD(cro_scan_opts, test_force_or),
};
static const cro_wire cro_wire_scan = {"scan-raw", 0, CRO_WIRE_FIELDS(cro_wire_scan_fields),
                                       {sizeof(cro_scan_report), 0, 0, 0, sizeof(cro_fault_word), 0, 0,
                                        CRO_WIRE_AT(cro_scan_report, recorded)}};

static const cro_wire_field cro_wire_sram_fields[] = {
    CRO_WIRE_FIELD(cro_sram_opts, legs),
    CRO_WIRE_FIELD(cro_sram_opts, iterations),
    CRO_WIRE_FIELD(cro_sram_opts, cluster),
    CRO_WIRE_FIELD(cro_sram_opts, max_rounds),
    CRO_WIRE_FIELD(cro_sram_opts, test_inject_leg),
    CRO_WIRE_FIELD(cro_sram_opts, test_inject_sm),
    CRO_WIRE_FIELD(cro_sram_opts, test_inject_element),
    CRO_WIRE_FIELD(cro_sram_opts, test_inject_iteration),
    CRO_WIRE_FIELD(cro_sram_opts, test_inject_word),
    CRO_WIRE_FIELD(cro_sram_opts, test_inject_mask),
};
static const cro_wire cro_wire_sram = {"sram-raw", 0, CRO_WIRE_FIELDS(cro_wire_sram_fields),
                                       {sizeof(cro_sram_result), 0, sizeof(cro_sram_sm), CRO_SRAM_MAX_SMS,
                                        sizeof(cro_sram_fault), CRO_WIRE_AT(cro_sram_result, sms_listed),
                                        CRO_WIRE_AT(cro_sram_result, recorded)}};

static const cro_wire_field cro_wire_link_fields[] = {
    CRO_WIRE_FIELD(cro_link_opts, bytes),
    CRO_WIRE_FIELD(cro_link_opts, hops),
    CRO_WIRE_FIELD(cro_link_opts, ctas),
    CRO_WIRE_FIELD(cro_link_opts, test_inject_check),
    CRO_WIRE_FIELD(cro_link_opts, test_inject_word),
    CRO_WIRE_FIELD(cro_link_opts, test_inject_mask),
};
static const cro_wire cro_wire_link = {"link-raw", 1, CRO_WIRE_FIELDS(cro_wire_link_fields),
                                       {sizeof(cro_link_result), 1, 0, 0, sizeof(cro_link_fault), 0, 0,
                                        sizeof(cro_link_result), 8}};

static const cro_wire_field cro_wire_compute_fields[] = {
    CRO_WIRE_FIELD(cro_compute_opts, iterations),
    CRO_WIRE_FIELD(cro_compute_opts, alu_iterations),
    CRO_WIRE_FIELD(cro_compute_opts, legs),
    CRO_WIRE_FIELD(cro_compute_opts, max_rounds),
    CRO_WIRE_FIELD(cro_compute_opts, test_inject_leg),
    CRO_WIRE_FIELD(cro_compute_opts, test_inject_sm),
    CRO_WIRE_FIELD(cro_compute_opts, test_inject_iteration),
    CRO_WIRE_FIELD(cro_compute_opts, test_inject_row),
    CRO_WIRE_FIELD(cro_compute_opts, test_inject_col),
    CRO_WIRE_FIELD(cro_compute_opts, test_inject_mask),
};
static const cro_wire cro_wire_compute = {
    "compute-raw", 1, CRO_WIRE_FIELDS(cro_wire_compute_fields),
    CRO_WIRE_SM_FRAME(cro_compute_result, cro_compute_sm, cro_compute_fault, CRO_COMPUTE_MAX_SMS)};

static const cro_wire_field cro_wire_precision_fields[] = {
    CRO_WIRE_FIELD(cro_precision_opts, iterations),
    CRO_WIRE_FIELD(cro_precision_opts, alu_iterations),
    CRO_WIRE_FIELD(cro_precision_opts, legs),
    CRO_WIRE_FIELD(cro_precision_opts, max_rounds),
    CRO_WIRE_FIELD(cro_precision_opts, test_inject_leg),
    CRO_WIRE_FIELD(cro_precision_opts, test_inject_sm),
    CRO_WIRE_FIELD(cro_precision_opts, test_inject_iteration),
    CRO_WIRE_FIELD(cro_precision_opts, test_inject_row),
    CRO_WIRE_FIELD(cro_precision_opts, test_inject_col),
    CRO_WIRE_FIELD(cro_precision_opts, test_inject_mask),
};
static const cro_wire cro_wire_precision = {
    "precision-raw", 1, CRO_WIRE_FIELDS(cro_wire_precision_fields),
    CRO_WIRE_SM_FRAME(cro_precision_result, cro_precision_sm, cro_precision_fault, CRO_PRECISION_MAX_SMS)};

static const cro_wire_field cro_wire_sparse_fields[] = {
    CRO_WIRE_FIELD(cro_sparse_opts, iterations),
    CRO_WIRE_FIELD(cro_sparse_opts, legs),
    CRO_WIRE_FIELD(cro_sparse_opts, max_rounds),
    CRO_WIRE_FIELD(cro_sparse_opts, test_inject_leg),
    CRO_WIRE_FIELD(cro_sparse_opts, test_inject_sm),
    CRO_WIRE_FIELD(cro_sparse_opts, test_inject_iteration),
    CRO_WIRE_FIELD(cro_sparse_opts, test_inject_row),
    CRO_WIRE_FIELD(cro_sparse_opts, test_inject_col),
    CRO_WIRE_FIELD(cro_sparse_opts, test_inject_mask),
    CRO_WIRE_FIELD(cro_sparse_opts, test_meta),
    CRO_WIRE_FIELD(cro_sparse_opts, test_meta_leg),
    CRO_WIRE_FIELD(cro_sparse_opts, test_meta_sm),
    CRO_WIRE_FIELD(cro_sparse_opts, test_meta_iteration),
    CRO_WIRE_FIELD(cro_sparse_opts, test_meta_row),
    CRO_WIRE_FIELD(cro_sparse_opts, test_meta_group),
};
static const cro_wire cro_wire_sparse = {
    "sparse-raw", 1, CRO_WIRE_FIELDS(cro_wire_sparse_fields),
    CRO_WIRE_SM_FRAME(cro_sparse_result, cro_sparse_sm, cro_sparse_fault, CRO_SPARSE_MAX_SMS)};

static const cro_wire_field cro_wire_warpmma_fields[] = {
    CRO_WIRE_FIELD(cro_warpmma_opts, iterations),
    CRO_WIRE_FIELD(cro_warpmma_opts, legs),
    CRO_WIRE_FIELD(cro_warpmma_opts, max_rounds),
    CRO_WIRE_FIELD(cro_warpmma_opts, test_inject_leg),
    CRO_WIRE_FIELD(cro_warpmma_opts, test_inject_sm),
    CRO_WIRE_FIELD(cro_warpmma_opts, test_inject_iteration),
    CRO_WIRE_FIELD(cro_warpmma_opts, test_inject_row),
    CRO_WIRE_FIELD(cro_warpmma_opts, test_inject_col),
    CRO_WIRE_FIELD(cro_warpmma_opts, test_inject_mask),
    CRO_WIRE_FIELD(cro_warpmma_opts, test_addr),
    CRO_WIRE_FIELD(cro_warpmma_opts, test_addr_leg),
    CRO_WIRE_FIELD(cro_warpmma_opts, test_addr_sm),
    CRO_WIRE_FIELD(cro_warpmma_opts, test_addr_iteration),
    CRO_WIRE_FIELD(cro_warpmma_opts, test_addr_row),
    CRO_WIRE_FIELD(cro_warpmma_opts, test_addr_kstep),
};
static const cro_wire cro_wire_warpmma = {
    "warpmma-raw", 1, CRO_WIRE_FIELDS(cro_wire_warpmma_fields),
    CRO_WIRE_SM_FRAME(cro_warpmma_result, cro_warpmma_sm, cro_warpmma_fault, CRO_WARPMMA_MAX_SMS)};

static const cro_wire_field cro_wire_l2_fields[] = {
    CRO_WIRE_FIELD(cro_l2_opts, bytes),
    CRO_WIRE_FIELD(cro_l2_opts, iterations),
    CRO_WIRE_FIELD(cro_l2_opts, a1_counters),
    CRO_WIRE_FIELD(cro_l2_opts, a2_counters),
    CRO_WIRE_FIELD(cro_l2_opts, test_inject_leg),
    CRO_WIRE_FIELD(cro_l2_opts, test_inject_sm),
    CRO_WIRE_FIELD(cro_l2_opts, test_inject_element),
    CRO_WIRE_FIELD(cro_l2_opts, test_inject_iteration),
    CRO_WIRE_FIELD(cro_l2_opts, test_inject_word),
    CRO_WIRE_FIELD(cro_l2_opts, test_inject_mask),
};
static const cro_wire cro_wire_l2 = {"l2-raw", 1, CRO_WIRE_FIELDS(cro_wire_l2_fields),
                                     CRO_WIRE_SM_FRAME(cro_l2_result, cro_l2_sm, cro_l2_fault, CRO_L2_MAX_SMS)};

static const cro_wire_field cro_wire_regfile_fields[] = {
    CRO_WIRE_FIELD(cro_regfile_opts, iterations),
    CRO_WIRE_FIELD(cro_regfile_opts, max_rounds),
    CRO_WIRE_FIELD(cro_regfile_opts, test_inject_sm),
    CRO_WIRE_FIELD(cro_regfile_opts, test_inject_warp),
    CRO_WIRE_FIELD(cro_regfile_opts, test_inject_lane),
    CRO_WIRE_FIELD(cro_regfile_opts, test_inject_slot),
    CRO_WIRE_FIELD(cro_regfile_opts, test_inject_element),
    CRO_WIRE_FIELD(cro_regfile_opts, test_inject_iteration),
    CRO_WIRE_FIELD(cro_regfile_opts, test_inject_mask),
};
/* The register-file frame: the result, then CRO_REGFILE_MAX_SMS cro_regfile_sm entries (sms_listed of them filled) and
 * `recorded` cro_regfile_fault records. */
static const cro_wire cro_wire_regfile = {"regfile-raw", 1, CRO_WIRE_FIELDS(cro_wire_regfile_fields),
                                          {sizeof(cro_regfile_result), 0, sizeof(cro_regfile_sm), CRO_REGFILE_MAX_SMS,
                                           sizeof(cro_regfile_fault), CRO_WIRE_AT(cro_regfile_result, sms_listed),
                                           CRO_WIRE_AT(cro_regfile_result, recorded)}};

static const cro_wire_field cro_wire_xlane_fields[] = {
    CRO_WIRE_FIELD(cro_xlane_opts, iterations),
    CRO_WIRE_FIELD(cro_xlane_opts, legs),
    CRO_WIRE_FIELD(cro_xlane_opts, max_rounds),
    CRO_WIRE_FIELD(cro_xlane_opts, test_inject_leg),
    CRO_WIRE_FIELD(cro_xlane_opts, test_inject_sm),
    CRO_WIRE_FIELD(cro_xlane_opts, test_inject_warp),
    CRO_WIRE_FIELD(cro_xlane_opts, test_inject_lane),
    CRO_WIRE_FIELD(cro_xlane_opts, test_inject_op),
    CRO_WIRE_FIELD(cro_xlane_opts, test_inject_iteration),
    CRO_WIRE_FIELD(cro_xlane_opts, test_inject_mask),
};
/* The cross-lane frame: the result, then CRO_XLANE_MAX_SMS cro_xlane_sm entries (sms_listed of them filled) and
 * `recorded` cro_xlane_fault records. */
static const cro_wire cro_wire_xlane = {"xlane-raw", 1, CRO_WIRE_FIELDS(cro_wire_xlane_fields),
                                        {sizeof(cro_xlane_result), 0, sizeof(cro_xlane_sm), CRO_XLANE_MAX_SMS,
                                         sizeof(cro_xlane_fault), CRO_WIRE_AT(cro_xlane_result, sms_listed),
                                         CRO_WIRE_AT(cro_xlane_result, recorded)}};

static const cro_wire_field cro_wire_alu_fields[] = {
    CRO_WIRE_FIELD(cro_alu_opts, iterations),
    CRO_WIRE_FIELD(cro_alu_opts, legs),
    CRO_WIRE_FIELD(cro_alu_opts, max_rounds),
    CRO_WIRE_FIELD(cro_alu_opts, test_inject_leg),
    CRO_WIRE_FIELD(cro_alu_opts, test_inject_sm),
    CRO_WIRE_FIELD(cro_alu_opts, test_inject_warp),
    CRO_WIRE_FIELD(cro_alu_opts, test_inject_lane),
    CRO_WIRE_FIELD(cro_alu_opts, test_inject_op),
    CRO_WIRE_FIELD(cro_alu_opts, test_inject_iteration),
    CRO_WIRE_FIELD(cro_alu_opts, test_inject_operand),
    CRO_WIRE_FIELD(cro_alu_opts, test_inject_mask),
};
/* The ALU frame: the result, then CRO_ALU_MAX_SMS cro_alu_sm entries (sms_listed of them filled) and `recorded`
 * cro_alu_fault records. */
static const cro_wire cro_wire_alu = {"alu-raw", 1, CRO_WIRE_FIELDS(cro_wire_alu_fields),
                                      {sizeof(cro_alu_result), 0, sizeof(cro_alu_sm), CRO_ALU_MAX_SMS, sizeof(cro_alu_fault),
                                       CRO_WIRE_AT(cro_alu_result, sms_listed), CRO_WIRE_AT(cro_alu_result, recorded)}};

static const cro_wire_field cro_wire_barrier_fields[] = {
    CRO_WIRE_FIELD(cro_barrier_opts, iterations),
    CRO_WIRE_FIELD(cro_barrier_opts, legs),
    CRO_WIRE_FIELD(cro_barrier_opts, max_rounds),
    CRO_WIRE_FIELD(cro_barrier_opts, cluster),
    CRO_WIRE_FIELD(cro_barrier_opts, test_inject_leg),
    CRO_WIRE_FIELD(cro_barrier_opts, test_inject_sm),
    CRO_WIRE_FIELD(cro_barrier_opts, test_inject_warp),
    CRO_WIRE_FIELD(cro_barrier_opts, test_inject_lane),
    CRO_WIRE_FIELD(cro_barrier_opts, test_inject_op),
    CRO_WIRE_FIELD(cro_barrier_opts, test_inject_iteration),
    CRO_WIRE_FIELD(cro_barrier_opts, test_inject_mask),
};
/* The barrier frame: the result, then CRO_BARRIER_MAX_SMS cro_barrier_sm entries (sms_listed of them filled) and
 * `recorded` cro_barrier_fault records. */
static const cro_wire cro_wire_barrier = {"barrier-raw", 1, CRO_WIRE_FIELDS(cro_wire_barrier_fields),
                                          {sizeof(cro_barrier_result), 0, sizeof(cro_barrier_sm), CRO_BARRIER_MAX_SMS,
                                           sizeof(cro_barrier_fault), CRO_WIRE_AT(cro_barrier_result, sms_listed),
                                           CRO_WIRE_AT(cro_barrier_result, recorded)}};

/* health-raw: <uuid> <seed_base> <checks>, then each check's fields and cap in run order (the CRO_HEALTH_* bit order).
 * Its stdout: the cro_health_result, then the frame of each check that ran, in run order.  opts_at and result_at:
 * where the check's options and result are in cro_health_opts and cro_health_result. */
typedef struct cro_wire_part {
    const cro_wire *wire;
    uint32_t opts_at, result_at;
} cro_wire_part;

static const cro_wire_part cro_wire_health[CRO_HEALTH_CHECKS] = {
    {&cro_wire_compute, offsetof(cro_health_opts, compute), offsetof(cro_health_result, compute)},
    {&cro_wire_precision, offsetof(cro_health_opts, precision), offsetof(cro_health_result, precision)},
    {&cro_wire_sram, offsetof(cro_health_opts, sram), offsetof(cro_health_result, sram)},
    {&cro_wire_l2, offsetof(cro_health_opts, l2), offsetof(cro_health_result, l2)},
    {&cro_wire_link, offsetof(cro_health_opts, link), offsetof(cro_health_result, link)},
    {&cro_wire_scan, offsetof(cro_health_opts, scan), offsetof(cro_health_result, scan)},
};

/* The argc croprobe-cli takes for w: croprobe-cli <cmd> <uuid> [<seed_base>] <fields> <cap>. */
static inline int cro_wire_argc(const cro_wire *w) { return 4 + w->seeded + (int)w->n_fields; }

/* health-raw's argv index of check k's first field: after <uuid> <seed_base> <checks>, each earlier check's fields and
 * cap.  cro_wire_health_at(CRO_HEALTH_CHECKS) is its argc. */
static inline int cro_wire_health_at(int k) {
    int at = 5;
    for (int j = 0; j < k; ++j) at += (int)cro_wire_health[j].wire->n_fields + 1;
    return at;
}

/* A frame's bytes before its records. */
static inline size_t cro_wire_head(const cro_wire_frame *f) {
    return (size_t)f->result + f->counts * sizeof(uint64_t) + (size_t)f->max_sms * f->sm;
}

/* Field i of w's options at opts as a decimal, into s (24 bytes hold any).  Both sides are little-endian, as the
 * frames' counts assume. */
static inline void cro_wire_format(const cro_wire *w, uint32_t i, const void *opts, char *s, size_t cap) {
    const cro_wire_field *f = &w->fields[i];
    uint64_t u = 0;
    memcpy(&u, (const unsigned char *)opts + f->at, f->size);
    if (f->is_signed && f->size < 8 && (u >> (8 * f->size - 1) & 1)) u |= ~0ull << (8 * f->size);
    if (f->is_signed) snprintf(s, cap, "%" PRId64, (int64_t)u);
    else snprintf(s, cap, "%" PRIu64, u);
}

/* Field i of w's options at opts from the decimal s (as strtoll or strtoull reads it, cut to the field's size). */
static inline void cro_wire_parse(const cro_wire *w, uint32_t i, const char *s, void *opts) {
    const cro_wire_field *f = &w->fields[i];
    const uint64_t u = f->is_signed ? (uint64_t)strtoll(s, NULL, 10) : (uint64_t)strtoull(s, NULL, 10);
    memcpy((unsigned char *)opts + f->at, &u, f->size);
}

#endif
