/*
 * croprobe-cli — libcroprobe as a one-shot helper process.
 *
 * Why a helper: CUDA fixes its device list at cuInit, so a long-lived operator process cannot see a GPU that is
 * hot-plugged later (SURVEY.md §7 "freshly hot-plugged GPU"); the reference gets around the same problem by
 * exec'ing nvidia-smi in a pod on every reconcile (internal/utils/gpus.go:886).  libcroprobe keeps the node's
 * inventory fresh by re-reading the driver's registry, and when a device shows up that its CUDA contexts do not
 * cover, cro_probe_uuid runs THIS program for it (`probe-raw`, CUDA_VISIBLE_DEVICES=<uuid>): a fresh cuInit that
 * sees exactly that GPU.  The cold start it pays (cuInit + one primary context + cudaMalloc) is what `cold` prints.
 *
 *   croprobe-cli csv <query>            what `nvidia-smi --query-gpu=<query> --format=csv,noheader,nounits` prints
 *   croprobe-cli enumerate              JSON array of the devices (minor, uuid, bus id, name)
 *   croprobe-cli probe <uuid|index> [sweep_MiB]      one full probe; JSON annotations on stdout, exit 0 iff status ok
 *   croprobe-cli probe-raw <uuid> [sweep_MiB]        the same, the 512-byte cro_probe_result on stdout (for the library)
 *   croprobe-cli cold <uuid|index> [sweep_MiB] [nvml] timings: init, first (cold) probe, second (warm) probe
 *   croprobe-cli scan <uuid|index> [max_MiB]         whole-HBM scan of the free memory (all of it but 1 GiB unless
 *                                                    max_MiB bounds it); JSON annotations, exit 0 iff status ok
 *   croprobe-cli scan-raw <uuid> <max_bytes> <reserve_bytes> <seed> <chunk_bytes> <force_first> <force_count>
 *                         <force_and> <force_or> <cap>
 *                                                    the same with every cro_scan_opts field; cro_scan_report and
 *                                                    its `recorded` cro_fault_word records (at most cap) on stdout
 *   croprobe-cli sram-raw <uuid> <legs> <iterations> <cluster> <max_rounds> <inject_leg> <inject_sm> <inject_element>
 *                         <inject_iteration> <inject_word> <inject_mask> <cap>
 *                                                    the SRAM probe with every cro_sram_opts field; cro_sram_result,
 *                                                    CRO_SRAM_MAX_SMS cro_sram_sm entries (sms_listed of them filled)
 *                                                    and its `recorded` cro_sram_fault records (at most cap) on stdout
 *   croprobe-cli link-raw <uuid> <seed_base> <bytes> <hops> <ctas> <inject_check> <inject_word> <inject_mask> <cap>
 *                                                    the host link probe with every cro_link_opts field, its sweep
 *                                                    region L (256 MiB when bytes is 0) and NVML on for the replay
 *                                                    counters; cro_link_result, a uint64_t n, then n cro_link_fault
 *                                                    records (at most cap) on stdout
 *   croprobe-cli compute-raw <uuid> <seed_base> <iterations> <alu_iterations> <legs> <max_rounds> <inject_leg>
 *                            <inject_sm> <inject_iteration> <inject_row> <inject_col> <inject_mask> <cap>
 *                                                    the compute probe with every cro_compute_opts field, no sweep
 *                                                    region and no NVML; cro_compute_result, uint64_t n_sms and n,
 *                                                    CRO_COMPUTE_MAX_SMS cro_compute_sm entries (n_sms of them filled),
 *                                                    then n cro_compute_fault records (at most cap) on stdout
 *   croprobe-cli precision-raw <uuid> <seed_base> <iterations> <alu_iterations> <legs> <max_rounds> <inject_leg>
 *                              <inject_sm> <inject_iteration> <inject_row> <inject_col> <inject_mask> <cap>
 *                                                    the precision probe with every cro_precision_opts field, as
 *                                                    compute-raw: cro_precision_result, uint64_t n_sms and n,
 *                                                    CRO_PRECISION_MAX_SMS cro_precision_sm entries, then n
 *                                                    cro_precision_fault records (at most cap) on stdout
 *   croprobe-cli sparse-raw <uuid> <seed_base> <iterations> <legs> <max_rounds> <inject_leg> <inject_sm>
 *                           <inject_iteration> <inject_row> <inject_col> <inject_mask> <meta> <meta_leg> <meta_sm>
 *                           <meta_iteration> <meta_row> <meta_group> <cap>
 *                                                    the sparse probe with every cro_sparse_opts field, as compute-raw:
 *                                                    cro_sparse_result, uint64_t n_sms and n, CRO_SPARSE_MAX_SMS
 *                                                    cro_sparse_sm entries, then n cro_sparse_fault records (at most
 *                                                    cap) on stdout
 *   croprobe-cli warpmma-raw <uuid> <seed_base> <iterations> <legs> <max_rounds> <inject_leg> <inject_sm>
 *                            <inject_iteration> <inject_row> <inject_col> <inject_mask> <addr> <addr_leg> <addr_sm>
 *                            <addr_iteration> <addr_row> <addr_kstep> <cap>
 *                                                    the warp-MMA probe with every cro_warpmma_opts field, as
 *                                                    compute-raw: cro_warpmma_result, uint64_t n_sms and n,
 *                                                    CRO_WARPMMA_MAX_SMS cro_warpmma_sm entries, then n
 *                                                    cro_warpmma_fault records (at most cap) on stdout
 *   croprobe-cli l2-raw <uuid> <seed_base> <bytes> <iterations> <a1_counters> <a2_counters> <inject_leg> <inject_sm>
 *                       <inject_element> <inject_iteration> <inject_word> <inject_mask> <cap>
 *                                                    the L2 probe with every cro_l2_opts field but the deadline, NVML on
 *                                                    for its health record; cro_l2_result, uint64_t n_sms and n,
 *                                                    CRO_L2_MAX_SMS cro_l2_sm entries (n_sms of them filled), then n
 *                                                    cro_l2_fault records (at most cap) on stdout
 *   croprobe-cli regfile-raw <uuid> <seed_base> <iterations> <max_rounds> <inject_sm> <inject_warp> <inject_lane>
 *                            <inject_slot> <inject_element> <inject_iteration> <inject_mask> <cap>
 *                                                    the register-file probe with every cro_regfile_opts field but the
 *                                                    deadline, NVML on for its health record; cro_regfile_result,
 *                                                    CRO_REGFILE_MAX_SMS cro_regfile_sm entries (sms_listed of them
 *                                                    filled) and its `recorded` cro_regfile_fault records (at most cap)
 *                                                    on stdout
 *   croprobe-cli xlane-raw <uuid> <seed_base> <iterations> <legs> <max_rounds> <inject_leg> <inject_sm> <inject_warp>
 *                          <inject_lane> <inject_op> <inject_iteration> <inject_mask> <cap>
 *                                                    the cross-lane probe with every cro_xlane_opts field but the
 *                                                    deadline; cro_xlane_result, CRO_XLANE_MAX_SMS cro_xlane_sm entries
 *                                                    (sms_listed of them filled) and its `recorded` cro_xlane_fault
 *                                                    records (at most cap) on stdout
 *   croprobe-cli alu-raw <uuid> <seed_base> <iterations> <legs> <max_rounds> <inject_leg> <inject_sm> <inject_warp>
 *                        <inject_lane> <inject_op> <inject_iteration> <inject_operand> <inject_mask> <cap>
 *                                                    the ALU probe with every cro_alu_opts field but the deadline;
 *                                                    cro_alu_result, CRO_ALU_MAX_SMS cro_alu_sm entries (sms_listed of
 *                                                    them filled) and its `recorded` cro_alu_fault records (at most
 *                                                    cap) on stdout
 *   croprobe-cli barrier-raw <uuid> <seed_base> <iterations> <legs> <max_rounds> <cluster> <inject_leg> <inject_sm>
 *                            <inject_warp> <inject_lane> <inject_op> <inject_iteration> <inject_mask> <cap>
 *                                                    the barrier probe with every cro_barrier_opts field but the
 *                                                    deadline; cro_barrier_result, CRO_BARRIER_MAX_SMS cro_barrier_sm
 *                                                    entries (sms_listed of them filled) and its `recorded`
 *                                                    cro_barrier_fault records (at most cap) on stdout
 *   croprobe-cli health-raw <uuid> <seed_base> <checks> <compute-raw's options and cap> <precision-raw's> <sram-raw's>
 *                           <l2-raw's> <link-raw's> <scan-raw's>
 *                                                    the health check (cro_check_health) with every option of every
 *                                                    check, each as its own -raw command takes them after the uuid (and
 *                                                    the seed base), its sweep region L, NVML on; the cro_health_result,
 *                                                    then each check that ran, in run order, as its own -raw writes it
 *   croprobe-cli health <uuid|index>                 the health check with defaults; JSON annotations, exit 0 iff ok
 *   link-raw, compute-raw, precision-raw, sparse-raw, warpmma-raw, l2-raw, regfile-raw, xlane-raw, alu-raw, barrier-raw and health-raw take
 *   cro_opts.seed_base from argv (the device seed is seed_base | minor, as in process), so that the library can give
 *   every helper call fresh patterns and operands; their counts are the helper's own, because neither result says how many records follow.
 * Exit 3: the device is not visible to this (fresh) process — the reference's found=false.  The raw commands exit 0
 * iff the probe's status is CRO_OK, 1 for any other status (the result on stdout says which), 64 for a wrong argument
 * count.
 *
 * Plain C against include/croprobe.h — the same surface the cgo shim binds.
 */
#define _POSIX_C_SOURCE 200809L
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <unistd.h>

#include "croprobe.h"
#include "helper_wire.h"

static double now_s(void) {
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

static int fail(cro_ctx *ctx, const char *what, int rc) {
    char msg[1024] = {0};
    cro_last_error(ctx, msg, sizeof msg);
    fprintf(stderr, "croprobe-cli: %s: %s%s%s\n", what, cro_strerror(rc), msg[0] ? ": " : "", msg);
    return 2;
}

static char buf[1 << 16];

/* A raw command's stdout, the result whatever its status (the library reads why from it): one frame per result, laid
 * out as its cro_wire_frame says, the counts the result does not hold written after it (put_frame: 0, or 2 when stdout
 * takes less).  Then end_frames exits 0 iff the status is CRO_OK and 1 for any other, skipping the teardown (it costs as
 * much as a probe): the process's buffers and allocations go with it. */
static int put_frame(const cro_wire_frame *w, const void *result, const void *sms, uint64_t n_sms, const void *records, uint64_t n) {
    unsigned char counts[2 * sizeof(uint64_t)] = {0};
    if (w->n_sms_width && w->n_sms_at >= w->result) memcpy(counts + (w->n_sms_at - w->result), &n_sms, w->n_sms_width);
    if (w->n_width && w->n_at >= w->result) memcpy(counts + (w->n_at - w->result), &n, w->n_width);
    const size_t sms_bytes = (size_t)w->max_sms * w->sm;
    if (fwrite(result, w->result, 1, stdout) != 1 || (w->counts && fwrite(counts, sizeof(uint64_t), w->counts, stdout) != w->counts) ||
        (sms_bytes && fwrite(sms, sms_bytes, 1, stdout) != 1) || (n && fwrite(records, w->rec, (size_t)n, stdout) != (size_t)n))
        return 2;
    return 0;
}
static int end_frames(int status) {
    fflush(stdout);
    _exit(status == CRO_OK ? 0 : 1);
}

/* w's options from argv, a[0] its first, into opts; the cap that follows them. */
static int opts_at(const cro_wire *w, char **a, void *opts) {
    for (uint32_t i = 0; i < w->n_fields; ++i) cro_wire_parse(w, i, a[i], opts);
    return atoi(a[w->n_fields]);
}
/* A raw command's options, after its uuid and seed base. */
static int raw_opts(const cro_wire *w, char **argv, void *opts) { return opts_at(w, argv + 3 + w->seeded, opts); }

/* The raw commands: each fills its probe's options from argv, runs the probe on device idx and writes its frame. */
static int scan_raw(cro_ctx *ctx, int idx, char **argv) {
    static cro_scan_opts so;
    const int cap = raw_opts(&cro_wire_scan, argv, &so);
    static cro_scan_report sr;
    cro_fault_word *words = (cro_fault_word *)calloc(cap > 0 ? (size_t)cap : 1, sizeof *words);
    int got = 0;
    if (!words) return 2;
    cro_scan_hbm(ctx, idx, &so, &sr, words, cap, &got);
    return put_frame(&cro_wire_scan.frame, &sr, NULL, 0, words, (uint64_t)got) ? 2 : end_frames(sr.status);
}

static int sram_raw(cro_ctx *ctx, int idx, char **argv) {
    static cro_sram_opts so;
    const int cap = raw_opts(&cro_wire_sram, argv, &so);
    static cro_sram_result sr;
    static cro_sram_sm sms[CRO_SRAM_MAX_SMS];
    cro_sram_fault *faults = (cro_sram_fault *)calloc(cap > 0 ? (size_t)cap : 1, sizeof *faults);
    int n_sms = 0, got = 0;
    if (!faults) return 2;
    cro_probe_sram(ctx, idx, &so, &sr, sms, CRO_SRAM_MAX_SMS, &n_sms, faults, cap > 0 ? cap : 0, &got);
    return put_frame(&cro_wire_sram.frame, &sr, sms, (uint64_t)n_sms, faults, (uint64_t)got) ? 2 : end_frames(sr.status);
}

static int link_raw(cro_ctx *ctx, int idx, char **argv) {
    static cro_link_opts lo;
    const int cap = raw_opts(&cro_wire_link, argv, &lo);
    static cro_link_result lr;
    cro_link_fault *faults = (cro_link_fault *)calloc(cap > 0 ? (size_t)cap : 1, sizeof *faults);
    int got = 0;
    if (!faults) return 2;
    cro_probe_host_link(ctx, idx, &lo, &lr, faults, cap > 0 ? cap : 0, &got);
    return put_frame(&cro_wire_link.frame, &lr, NULL, 0, faults, (uint64_t)got) ? 2 : end_frames(lr.status);
}

static int compute_raw(cro_ctx *ctx, int idx, char **argv) {
    static cro_compute_opts co;
    const int cap = raw_opts(&cro_wire_compute, argv, &co);
    static cro_compute_result cr;
    static cro_compute_sm sms[CRO_COMPUTE_MAX_SMS];
    cro_compute_fault *faults = (cro_compute_fault *)calloc(cap > 0 ? (size_t)cap : 1, sizeof *faults);
    int n_sms = 0, got = 0;
    if (!faults) return 2;
    cro_probe_compute(ctx, idx, &co, &cr, sms, CRO_COMPUTE_MAX_SMS, &n_sms, faults, cap > 0 ? cap : 0, &got);
    return put_frame(&cro_wire_compute.frame, &cr, sms, (uint64_t)n_sms, faults, (uint64_t)got) ? 2 : end_frames(cr.status);
}

static int precision_raw(cro_ctx *ctx, int idx, char **argv) {
    static cro_precision_opts po;
    const int cap = raw_opts(&cro_wire_precision, argv, &po);
    static cro_precision_result pr;
    static cro_precision_sm sms[CRO_PRECISION_MAX_SMS];
    cro_precision_fault *faults = (cro_precision_fault *)calloc(cap > 0 ? (size_t)cap : 1, sizeof *faults);
    int n_sms = 0, got = 0;
    if (!faults) return 2;
    cro_probe_precision(ctx, idx, &po, &pr, sms, CRO_PRECISION_MAX_SMS, &n_sms, faults, cap > 0 ? cap : 0, &got);
    return put_frame(&cro_wire_precision.frame, &pr, sms, (uint64_t)n_sms, faults, (uint64_t)got) ? 2 : end_frames(pr.status);
}

static int sparse_raw(cro_ctx *ctx, int idx, char **argv) {
    static cro_sparse_opts so;
    const int cap = raw_opts(&cro_wire_sparse, argv, &so);
    static cro_sparse_result sr;
    static cro_sparse_sm sms[CRO_SPARSE_MAX_SMS];
    cro_sparse_fault *faults = (cro_sparse_fault *)calloc(cap > 0 ? (size_t)cap : 1, sizeof *faults);
    int n_sms = 0, got = 0;
    if (!faults) return 2;
    cro_probe_sparse(ctx, idx, &so, &sr, sms, CRO_SPARSE_MAX_SMS, &n_sms, faults, cap > 0 ? cap : 0, &got);
    return put_frame(&cro_wire_sparse.frame, &sr, sms, (uint64_t)n_sms, faults, (uint64_t)got) ? 2 : end_frames(sr.status);
}

static int warpmma_raw(cro_ctx *ctx, int idx, char **argv) {
    static cro_warpmma_opts wo;
    const int cap = raw_opts(&cro_wire_warpmma, argv, &wo);
    static cro_warpmma_result wr;
    static cro_warpmma_sm sms[CRO_WARPMMA_MAX_SMS];
    cro_warpmma_fault *faults = (cro_warpmma_fault *)calloc(cap > 0 ? (size_t)cap : 1, sizeof *faults);
    int n_sms = 0, got = 0;
    if (!faults) return 2;
    cro_probe_warpmma(ctx, idx, &wo, &wr, sms, CRO_WARPMMA_MAX_SMS, &n_sms, faults, cap > 0 ? cap : 0, &got);
    return put_frame(&cro_wire_warpmma.frame, &wr, sms, (uint64_t)n_sms, faults, (uint64_t)got) ? 2 : end_frames(wr.status);
}

static int l2_raw(cro_ctx *ctx, int idx, char **argv) {
    static cro_l2_opts lo;
    const int cap = raw_opts(&cro_wire_l2, argv, &lo);
    static cro_l2_result lr;
    static cro_l2_sm sms[CRO_L2_MAX_SMS];
    cro_l2_fault *faults = (cro_l2_fault *)calloc(cap > 0 ? (size_t)cap : 1, sizeof *faults);
    int n_sms = 0, got = 0;
    if (!faults) return 2;
    cro_probe_l2(ctx, idx, &lo, &lr, sms, CRO_L2_MAX_SMS, &n_sms, faults, cap > 0 ? cap : 0, &got);
    return put_frame(&cro_wire_l2.frame, &lr, sms, (uint64_t)n_sms, faults, (uint64_t)got) ? 2 : end_frames(lr.status);
}

static int regfile_raw(cro_ctx *ctx, int idx, char **argv) {
    static cro_regfile_opts ro;
    const int cap = raw_opts(&cro_wire_regfile, argv, &ro);
    static cro_regfile_result rr;
    static cro_regfile_sm sms[CRO_REGFILE_MAX_SMS];
    cro_regfile_fault *faults = (cro_regfile_fault *)calloc(cap > 0 ? (size_t)cap : 1, sizeof *faults);
    int n_sms = 0, got = 0;
    if (!faults) return 2;
    cro_probe_regfile(ctx, idx, &ro, &rr, sms, CRO_REGFILE_MAX_SMS, &n_sms, faults, cap > 0 ? cap : 0, &got);
    return put_frame(&cro_wire_regfile.frame, &rr, sms, (uint64_t)n_sms, faults, (uint64_t)got) ? 2 : end_frames(rr.status);
}

static int xlane_raw(cro_ctx *ctx, int idx, char **argv) {
    static cro_xlane_opts xo;
    const int cap = raw_opts(&cro_wire_xlane, argv, &xo);
    static cro_xlane_result xr;
    static cro_xlane_sm sms[CRO_XLANE_MAX_SMS];
    cro_xlane_fault *faults = (cro_xlane_fault *)calloc(cap > 0 ? (size_t)cap : 1, sizeof *faults);
    int n_sms = 0, got = 0;
    if (!faults) return 2;
    cro_probe_xlane(ctx, idx, &xo, &xr, sms, CRO_XLANE_MAX_SMS, &n_sms, faults, cap > 0 ? cap : 0, &got);
    return put_frame(&cro_wire_xlane.frame, &xr, sms, (uint64_t)n_sms, faults, (uint64_t)got) ? 2 : end_frames(xr.status);
}

static int alu_raw(cro_ctx *ctx, int idx, char **argv) {
    static cro_alu_opts ao;
    const int cap = raw_opts(&cro_wire_alu, argv, &ao);
    static cro_alu_result ar;
    static cro_alu_sm sms[CRO_ALU_MAX_SMS];
    cro_alu_fault *faults = (cro_alu_fault *)calloc(cap > 0 ? (size_t)cap : 1, sizeof *faults);
    int n_sms = 0, got = 0;
    if (!faults) return 2;
    cro_probe_alu(ctx, idx, &ao, &ar, sms, CRO_ALU_MAX_SMS, &n_sms, faults, cap > 0 ? cap : 0, &got);
    return put_frame(&cro_wire_alu.frame, &ar, sms, (uint64_t)n_sms, faults, (uint64_t)got) ? 2 : end_frames(ar.status);
}

static int barrier_raw(cro_ctx *ctx, int idx, char **argv) {
    static cro_barrier_opts bo;
    const int cap = raw_opts(&cro_wire_barrier, argv, &bo);
    static cro_barrier_result br;
    static cro_barrier_sm sms[CRO_BARRIER_MAX_SMS];
    cro_barrier_fault *faults = (cro_barrier_fault *)calloc(cap > 0 ? (size_t)cap : 1, sizeof *faults);
    int n_sms = 0, got = 0;
    if (!faults) return 2;
    cro_probe_barrier(ctx, idx, &bo, &br, sms, CRO_BARRIER_MAX_SMS, &n_sms, faults, cap > 0 ? cap : 0, &got);
    return put_frame(&cro_wire_barrier.frame, &br, sms, (uint64_t)n_sms, faults, (uint64_t)got) ? 2 : end_frames(br.status);
}

/* `scan`: the whole-HBM scan of the free memory (all of it but 1 GiB unless argv[3], in MiB, bounds it) as JSON. */
static int scan_json(cro_ctx *ctx, int idx, char **argv) {
    cro_scan_opts so;
    memset(&so, 0, sizeof so);
    if (argv[3]) so.max_bytes = (uint64_t)strtoull(argv[3], NULL, 10) << 20;
    static cro_scan_report sr;
    cro_fault_word *words = (cro_fault_word *)calloc(256, sizeof *words);
    int got = 0;
    size_t len = 0;
    if (!words) return 2;
    int rc = cro_scan_hbm(ctx, idx, &so, &sr, words, 256, &got);
    if (rc != CRO_OK && rc != CRO_ERR_CHECKSUM && rc != CRO_ERR_CUDA) return fail(ctx, "cro_scan_hbm", rc);
    if ((rc = cro_emit_scan_annotations_json(&sr, buf, sizeof buf, &len)) != CRO_OK) return fail(ctx, "emit", rc);
    printf("%s\n", buf);
    free(words);
    cro_probe_destroy(ctx);
    return sr.status == CRO_OK ? 0 : 1;
}

/* `health-raw`: cro_check_health, then its result and each check that ran as its own frame. */
static int health_raw(cro_ctx *ctx, int idx, char **argv) {
    static cro_health_opts ho;
    static cro_health_result hr;
    static cro_compute_sm csms[CRO_COMPUTE_MAX_SMS];
    static cro_precision_sm psms[CRO_PRECISION_MAX_SMS];
    static cro_sram_sm ssms[CRO_SRAM_MAX_SMS];
    static cro_l2_sm lsms[CRO_L2_MAX_SMS];
    ho.checks = (uint32_t)strtoul(argv[4], NULL, 10);
    int cap[CRO_HEALTH_CHECKS];
    for (int k = 0; k < CRO_HEALTH_CHECKS; ++k) {
        cap[k] = opts_at(cro_wire_health[k].wire, argv + cro_wire_health_at(k), (char *)&ho + cro_wire_health[k].opts_at);
        cap[k] = cap[k] > 0 ? cap[k] : 0;
    }
    cro_health_records rec;
    memset(&rec, 0, sizeof rec);
    rec.compute_sms = csms;
    rec.compute_sms_cap = CRO_COMPUTE_MAX_SMS;
    rec.precision_sms = psms;
    rec.precision_sms_cap = CRO_PRECISION_MAX_SMS;
    rec.sram_sms = ssms;
    rec.sram_sms_cap = CRO_SRAM_MAX_SMS;
    rec.l2_sms = lsms;
    rec.l2_sms_cap = CRO_L2_MAX_SMS;
    rec.compute_faults = calloc((size_t)cap[0] + 1, sizeof *rec.compute_faults);
    rec.precision_faults = calloc((size_t)cap[1] + 1, sizeof *rec.precision_faults);
    rec.sram_faults = calloc((size_t)cap[2] + 1, sizeof *rec.sram_faults);
    rec.l2_faults = calloc((size_t)cap[3] + 1, sizeof *rec.l2_faults);
    rec.link_faults = calloc((size_t)cap[4] + 1, sizeof *rec.link_faults);
    rec.scan_words = calloc((size_t)cap[5] + 1, sizeof *rec.scan_words);
    if (!rec.compute_faults || !rec.precision_faults || !rec.sram_faults || !rec.l2_faults || !rec.link_faults || !rec.scan_words)
        return 2;
    rec.compute_faults_cap = cap[0];
    rec.precision_faults_cap = cap[1];
    rec.sram_faults_cap = cap[2];
    rec.l2_faults_cap = cap[3];
    rec.link_faults_cap = cap[4];
    rec.scan_words_cap = cap[5];
    cro_check_health(ctx, idx, &ho, &hr, &rec);
    const void *sms[CRO_HEALTH_CHECKS] = {csms, psms, ssms, lsms, NULL, NULL};
    const int n_sms[CRO_HEALTH_CHECKS] = {rec.compute_sms_n, rec.precision_sms_n, rec.sram_sms_n, rec.l2_sms_n, 0, 0};
    const void *recs[CRO_HEALTH_CHECKS] = {rec.compute_faults, rec.precision_faults, rec.sram_faults,
                                           rec.l2_faults,      rec.link_faults,      rec.scan_words};
    const int n[CRO_HEALTH_CHECKS] = {rec.compute_faults_n, rec.precision_faults_n, rec.sram_faults_n,
                                      rec.l2_faults_n,      rec.link_faults_n,      rec.scan_words_n};
    if (fwrite(&hr, sizeof hr, 1, stdout) != 1) return 2;
    for (int k = 0; k < CRO_HEALTH_CHECKS; ++k)
        if ((hr.ran >> k & 1u) && put_frame(&cro_wire_health[k].wire->frame, (const char *)&hr + cro_wire_health[k].result_at, sms[k],
                                            (uint64_t)n_sms[k], recs[k], (uint64_t)n[k]))
            return 2;
    return end_frames(hr.status);
}

/* `health`: the health check with defaults; every check's annotations and the call's own as one JSON object. */
static int health_json(cro_ctx *ctx, int idx, char **argv) {
    static cro_health_result hr;
    size_t len = 0;
    (void)argv;
    int rc = cro_check_health(ctx, idx, NULL, &hr, NULL);
    if (rc == CRO_ERR_INVALID_ARG) return fail(ctx, "cro_check_health", rc);
    if ((rc = cro_emit_health_annotations_json(&hr, buf, sizeof buf, &len)) != CRO_OK) return fail(ctx, "emit", rc);
    printf("%s\n", buf);
    cro_probe_destroy(ctx);
    return hr.status == CRO_OK ? 0 : 1;
}

/* The commands that take a device (argv[2]): their name, or a raw command's argv and frame (helper_wire.h; NULL: argc at
 * least 3, the rest optional), cro_opts.flags and sweep region, and what runs once the device is found (NULL: main's own probe). */
static const struct command {
    const char *name;
    const cro_wire *wire;
    uint32_t flags;
    uint64_t sweep_mib;
    int (*run)(cro_ctx *ctx, int idx, char **argv);
} commands[] = {
    /* the hot-plug path: one device, identity from /proc (NVML's first call costs more than the probe), and a 1 GiB
     * first sweep unless argv[3] says otherwise — far beyond the L2, and it shortens everything before it */
    {"probe", NULL, CRO_F_LAZY_ALLOC | CRO_F_DEGRADE_ON_OOM | CRO_F_NO_NVML, 1024, NULL},
    {"probe-raw", NULL, CRO_F_LAZY_ALLOC | CRO_F_DEGRADE_ON_OOM | CRO_F_NO_NVML, 1024, NULL},
    {"cold", NULL, CRO_F_LAZY_ALLOC | CRO_F_DEGRADE_ON_OOM | CRO_F_NO_NVML, 1024, NULL},
    /* one check of one device by their own, not the HBM probe: no sweep region (the scan allocates its own chunks) and
     * NVML, whose DRAM / SRAM / L2 health record these read */
    {"scan", NULL, CRO_F_LAZY_ALLOC, 64, scan_json},
    {NULL, &cro_wire_scan, CRO_F_LAZY_ALLOC, 64, scan_raw},
    {NULL, &cro_wire_sram, CRO_F_LAZY_ALLOC, 64, sram_raw},
    {NULL, &cro_wire_l2, CRO_F_LAZY_ALLOC, 64, l2_raw},
    {NULL, &cro_wire_regfile, CRO_F_LAZY_ALLOC, 64, regfile_raw},
    {NULL, &cro_wire_xlane, CRO_F_LAZY_ALLOC, 64, xlane_raw},
    {NULL, &cro_wire_alu, CRO_F_LAZY_ALLOC, 64, alu_raw},
    {NULL, &cro_wire_barrier, CRO_F_LAZY_ALLOC, 64, barrier_raw},
    /* a region of exactly L, the link's bytes (the probe checks L <= S; no halving on a full GPU), and NVML for the
     * replay counters */
    {NULL, &cro_wire_link, CRO_F_LAZY_ALLOC, 256, link_raw},
    /* no health record to read, and NVML's first call is slow */
    {NULL, &cro_wire_compute, CRO_F_LAZY_ALLOC | CRO_F_NO_NVML, 64, compute_raw},
    {NULL, &cro_wire_precision, CRO_F_LAZY_ALLOC | CRO_F_NO_NVML, 64, precision_raw},
    {NULL, &cro_wire_sparse, CRO_F_LAZY_ALLOC | CRO_F_NO_NVML, 64, sparse_raw},
    {NULL, &cro_wire_warpmma, CRO_F_LAZY_ALLOC | CRO_F_NO_NVML, 64, warpmma_raw},
    /* every check of one device: the link check's region (exactly L when it is given) and NVML for the scan's, SRAM's and
     * L2's health records and the link's replay counters */
    {"health-raw", NULL, CRO_F_LAZY_ALLOC, 256, health_raw},
    {"health", NULL, CRO_F_LAZY_ALLOC, 256, health_json},
};

int main(int argc, char **argv) {
    if (argc < 2) {
        fprintf(stderr, "usage: croprobe-cli csv <query> | enumerate | probe <uuid|index> [sweep_MiB] | probe-raw <uuid> [sweep_MiB] | "
                        "cold <uuid|index> [sweep_MiB] [nvml] | scan <uuid|index> [max_MiB] | scan-raw <uuid> <max> <reserve> <seed> <chunk> "
                        "<first> <count> <and> <or> <cap> | sram-raw <uuid> <legs> <iterations> <cluster> <rounds> <leg> <sm> <element> <iteration> "
                        "<word> <mask> <cap> | link-raw <uuid> <seed_base> <bytes> <hops> <ctas> <check> <word> <mask> <cap> | "
                        "compute-raw <uuid> <seed_base> <iterations> <alu_iterations> <legs> <rounds> <leg> <sm> <iteration> <row> <col> "
                        "<mask> <cap> | precision-raw <uuid> <seed_base> <iterations> <alu_iterations> <legs> <rounds> <leg> <sm> <iteration> <row> "
                        "<col> <mask> <cap> | sparse-raw <uuid> <seed_base> <iterations> <legs> <rounds> <leg> <sm> <iteration> <row> <col> "
                        "<mask> <meta> <meta_leg> <meta_sm> <meta_iteration> <meta_row> <meta_group> <cap> | warpmma-raw <uuid> <seed_base> "
                        "<iterations> <legs> <rounds> <leg> <sm> <iteration> <row> <col> <mask> <addr> <addr_leg> <addr_sm> <addr_iteration> "
                        "<addr_row> <addr_kstep> <cap> | l2-raw <uuid> <seed_base> <bytes> <iterations> <a1> <a2> <leg> <sm> <element> <iteration> <word> <mask> <cap> | "
                        "regfile-raw <uuid> <seed_base> <iterations> <rounds> <sm> <warp> <lane> <slot> <element> <iteration> <mask> <cap> | "
                        "xlane-raw <uuid> <seed_base> <iterations> <legs> <rounds> <leg> <sm> <warp> <lane> <op> <iteration> <mask> <cap> | "
                        "alu-raw <uuid> <seed_base> <iterations> <legs> <rounds> <leg> <sm> <warp> <lane> <op> <iteration> <operand> <mask> "
                        "<cap> | "
                        "barrier-raw <uuid> <seed_base> <iterations> <legs> <rounds> <cluster> <leg> <sm> <warp> <lane> <op> <iteration> "
                        "<mask> <cap> | "
                        "health-raw <uuid> <seed_base> <checks> <compute-raw, precision-raw, sram-raw, l2-raw, link-raw, scan-raw options "
                        "and caps> | health <uuid|index>\n");
        return 64;
    }
    const double t_start = now_s();
    const char *cmd = argv[1];
    const struct command *c = NULL;
    for (size_t k = 0; k < sizeof commands / sizeof *commands; ++k)
        if (strcmp(cmd, commands[k].wire ? commands[k].wire->cmd : commands[k].name) == 0) c = &commands[k];
    const int want = !c ? 0 : c->wire ? cro_wire_argc(c->wire) : c->run == health_raw ? cro_wire_health_at(CRO_HEALTH_CHECKS) : 0;
    if (c && (argc < 3 || (want && argc != want))) return 64;
    const int cold = strcmp(cmd, "cold") == 0;
    cro_opts opts;
    memset(&opts, 0, sizeof opts);
    opts.abi_version = CRO_ABI_VERSION;
    opts.flags = CRO_F_LAZY_ALLOC | CRO_F_DEGRADE_ON_OOM;
    if (c) {
        opts.flags = c->flags;
        opts.sweep_bytes = c->sweep_mib << 20;
        if (c->wire ? c->wire->seeded : c->run == health_raw) opts.seed_base = (uint64_t)strtoull(argv[3], NULL, 10);
        if (!c->run && argc > 3) opts.sweep_bytes = (uint64_t)strtoull(argv[3], NULL, 10) << 20;    /* the probe's sweep_MiB */
        if (cold && argc > 4 && strcmp(argv[4], "nvml") == 0) opts.flags &= ~CRO_F_NO_NVML;
        /* L: the link's first option (the link is health-raw's fifth check) */
        const char *link_bytes = c->run == link_raw ? argv[4] : c->run == health_raw ? argv[cro_wire_health_at(4)] : "0";
        if (strtoull(link_bytes, NULL, 10)) opts.sweep_bytes = (uint64_t)strtoull(link_bytes, NULL, 10);
        if (strncmp(argv[2], "GPU-", 4) == 0) {
            /* before ANY CUDA call: this process's cuInit must enumerate that one GPU only (one primary context
             * instead of eight on a full box) */
            if (!getenv("CUDA_VISIBLE_DEVICES") || strcmp(getenv("CUDA_VISIBLE_DEVICES"), argv[2]) != 0)
                setenv("CUDA_VISIBLE_DEVICES", argv[2], 1);
        } else {
            opts.n_devices = 1;
            opts.devices[0] = atoi(argv[2]);
        }
    }

    const double t0 = now_s();
    cro_ctx *ctx = NULL;
    int rc = cro_probe_init(&opts, &ctx);
    if (rc == CRO_ERR_NO_DEVICE && strcmp(cmd, "csv") == 0) {   /* an empty box is not an error for enumeration */
        printf("No devices were found\n");
        return 0;
    }
    if (rc == CRO_ERR_NO_DEVICE && c && strncmp(argv[2], "GPU-", 4) == 0) {
        fprintf(stderr, "croprobe-cli: device '%s' is not visible\n", argv[2]);   /* found=0, like gpus.go:896-898 */
        return 3;
    }
    if (rc != CRO_OK) return fail(NULL, "cro_probe_init", rc);
    const double t_init = now_s() - t0;

    cro_dev_info devs[CRO_MAX_DEVICES];
    int n = 0;
    if ((rc = cro_enumerate(ctx, devs, CRO_MAX_DEVICES, &n)) != CRO_OK) return fail(ctx, "cro_enumerate", rc);
    size_t len = 0;

    if (strcmp(cmd, "csv") == 0) {
        if ((rc = cro_emit_csv(devs, n, argc > 2 ? argv[2] : "gpu_uuid", buf, sizeof buf, &len)) != CRO_OK) {
            fprintf(stdout, "%s\n", buf);   /* nvidia-smi prints its field error on stdout too */
            return 2;
        }
        fputs(buf, stdout);
    } else if (strcmp(cmd, "enumerate") == 0) {
        printf("[");
        for (int i = 0; i < n; ++i)
            printf("%s{\"index\":%d,\"device_minor\":%d,\"gpu_uuid\":\"%s\",\"pci.bus_id\":\"%s\",\"name\":\"%s\",\"in_process\":%s}", i ? "," : "",
                   devs[i].dev_index, devs[i].device_minor, devs[i].gpu_uuid, devs[i].pci_bus_id, devs[i].name,
                   (devs[i].flags & CRO_DEV_IN_PROCESS) ? "true" : "false");
        printf("]\n");
    } else if (c) {
        int idx = -1;
        for (int i = 0; i < n; ++i)
            if ((devs[i].flags & CRO_DEV_IN_PROCESS) && (strcmp(devs[i].gpu_uuid, argv[2]) == 0 || strncmp(argv[2], "GPU-", 4) != 0))
                idx = devs[i].dev_index;
        if (idx < 0) {
            fprintf(stderr, "croprobe-cli: device '%s' is not visible\n", argv[2]);
            cro_probe_destroy(ctx);
            return 3;
        }
        if (c->run) return c->run(ctx, idx, argv);
        cro_probe_result r;
        const double t1 = now_s();
        rc = cro_probe_device(ctx, idx, &r);
        const double t_cold = now_s() - t1;
        if (rc != CRO_OK && rc != CRO_ERR_CHECKSUM) return fail(ctx, "cro_probe_device", rc);
        if (cold) {
            const double t2 = now_s();
            cro_probe_result r2;
            int rc2 = cro_probe_device(ctx, idx, &r2);
            const double t_warm = now_s() - t2;
            const double total = now_s() - t_start - t_warm;     /* process start .. first verdict */
            printf("{\"gpu_uuid\":\"%s\",\"sweep_bytes\":%llu,\"init_s\":%.4f,\"cold_probe_s\":%.4f,\"warm_probe_s\":%.4f,"
                   "\"cold_total_s\":%.4f,\"cold_probes_per_s\":%.2f,\"warm_probes_per_s\":%.2f,\"nvml\":%s,\"status\":%d}\n",
                   r.gpu_uuid, (unsigned long long)r.sweep_bytes, t_init, t_cold, t_warm, total,
                   1.0 / total, 1.0 / t_warm, (opts.flags & CRO_F_NO_NVML) ? "false" : "true", rc2 ? rc2 : r.status);
        } else if (strcmp(cmd, "probe-raw") == 0) {
            return fwrite(&r, sizeof r, 1, stdout) != 1 ? 2 : end_frames(r.status);
        } else {
            if ((rc = cro_emit_probe_annotations_json(&r, buf, sizeof buf, &len)) != CRO_OK) return fail(ctx, "emit", rc);
            printf("%s\n", buf);
        }
        cro_probe_destroy(ctx);
        return r.status == CRO_OK ? 0 : 1;
    } else {
        fprintf(stderr, "croprobe-cli: unknown command '%s'\n", cmd);
        cro_probe_destroy(ctx);
        return 64;
    }
    cro_probe_destroy(ctx);
    return 0;
}
