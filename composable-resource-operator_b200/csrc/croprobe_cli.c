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
 *   croprobe-cli l2-raw <uuid> <seed_base> <bytes> <iterations> <a1_counters> <a2_counters> <inject_leg> <inject_sm>
 *                       <inject_element> <inject_iteration> <inject_word> <inject_mask> <cap>
 *                                                    the L2 probe with every cro_l2_opts field but the deadline, NVML on
 *                                                    for its health record; cro_l2_result, uint64_t n_sms and n,
 *                                                    CRO_L2_MAX_SMS cro_l2_sm entries (n_sms of them filled), then n
 *                                                    cro_l2_fault records (at most cap) on stdout
 *   link-raw, compute-raw, precision-raw and l2-raw take cro_opts.seed_base from argv (the device seed is seed_base | minor, as in process), so
 *   that the library can give every helper call fresh patterns and operands; their counts are the helper's own,
 *   because neither result says how many records follow.
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

/* A raw command's stdout, the result whatever its status (the library reads why from it): the result, n_counts counts
 * of the helper's own, the per-SM block and n records of rec_bytes each, the empty parts left out.  Then it exits 0 iff
 * the status is CRO_OK and 1 for any other, skipping the teardown (it costs as much as a probe): the process's buffers
 * and allocations go with it.  2 when stdout takes less. */
static int write_frame(const void *result, size_t result_bytes, const uint64_t *counts, size_t n_counts, const void *sms,
                       size_t sms_bytes, const void *records, size_t rec_bytes, int n, int status) {
    if (fwrite(result, result_bytes, 1, stdout) != 1 || (n_counts && fwrite(counts, sizeof *counts, n_counts, stdout) != n_counts) ||
        (sms_bytes && fwrite(sms, sms_bytes, 1, stdout) != 1) || (n > 0 && fwrite(records, rec_bytes, (size_t)n, stdout) != (size_t)n))
        return 2;
    fflush(stdout);
    _exit(status == CRO_OK ? 0 : 1);
}

/* The raw commands: each fills its probe's options from argv, runs the probe on device idx and writes its frame. */
static int scan_raw(cro_ctx *ctx, int idx, char **argv) {
    cro_scan_opts so;
    memset(&so, 0, sizeof so);
    uint64_t *f[] = {&so.max_bytes, &so.reserve_bytes, &so.seed, &so.test_chunk_bytes, &so.test_force_first,
                     &so.test_force_count, &so.test_force_and, &so.test_force_or};
    for (int k = 0; k < 8; ++k) *f[k] = (uint64_t)strtoull(argv[3 + k], NULL, 10);
    const int cap = atoi(argv[11]);
    static cro_scan_report sr;
    cro_fault_word *words = (cro_fault_word *)calloc(cap > 0 ? (size_t)cap : 1, sizeof *words);
    int got = 0;
    if (!words) return 2;
    cro_scan_hbm(ctx, idx, &so, &sr, words, cap, &got);
    return write_frame(&sr, sizeof sr, NULL, 0, NULL, 0, words, sizeof *words, got, sr.status);
}

static int sram_raw(cro_ctx *ctx, int idx, char **argv) {
    cro_sram_opts so;
    memset(&so, 0, sizeof so);
    so.legs = (uint32_t)strtoul(argv[3], NULL, 10);
    so.iterations = (uint32_t)strtoul(argv[4], NULL, 10);
    so.cluster = (uint32_t)strtoul(argv[5], NULL, 10);
    so.max_rounds = (uint32_t)strtoul(argv[6], NULL, 10);
    so.test_inject_leg = atoi(argv[7]);
    so.test_inject_sm = atoi(argv[8]);
    so.test_inject_element = (uint32_t)strtoul(argv[9], NULL, 10);
    so.test_inject_iteration = (uint32_t)strtoul(argv[10], NULL, 10);
    so.test_inject_word = atoi(argv[11]);
    so.test_inject_mask = (uint64_t)strtoull(argv[12], NULL, 10);
    const int cap = atoi(argv[13]);
    static cro_sram_result sr;
    static cro_sram_sm sms[CRO_SRAM_MAX_SMS];
    cro_sram_fault *faults = (cro_sram_fault *)calloc(cap > 0 ? (size_t)cap : 1, sizeof *faults);
    int n_sms = 0, got = 0;
    if (!faults) return 2;
    cro_probe_sram(ctx, idx, &so, &sr, sms, CRO_SRAM_MAX_SMS, &n_sms, faults, cap > 0 ? cap : 0, &got);
    return write_frame(&sr, sizeof sr, NULL, 0, sms, sizeof sms, faults, sizeof *faults, got, sr.status);
}

static int link_raw(cro_ctx *ctx, int idx, char **argv) {
    cro_link_opts lo;
    memset(&lo, 0, sizeof lo);
    lo.bytes = (uint64_t)strtoull(argv[4], NULL, 10);
    lo.hops = (uint32_t)strtoul(argv[5], NULL, 10);
    lo.ctas = (uint32_t)strtoul(argv[6], NULL, 10);
    lo.test_inject_check = atoi(argv[7]);
    lo.test_inject_word = (uint64_t)strtoull(argv[8], NULL, 10);
    lo.test_inject_mask = (uint64_t)strtoull(argv[9], NULL, 10);
    const int cap = atoi(argv[10]);
    static cro_link_result lr;
    cro_link_fault *faults = (cro_link_fault *)calloc(cap > 0 ? (size_t)cap : 1, sizeof *faults);
    int got = 0;
    if (!faults) return 2;
    cro_probe_host_link(ctx, idx, &lo, &lr, faults, cap > 0 ? cap : 0, &got);
    const uint64_t n_out = (uint64_t)got;
    return write_frame(&lr, sizeof lr, &n_out, 1, NULL, 0, faults, sizeof *faults, got, lr.status);
}

static int compute_raw(cro_ctx *ctx, int idx, char **argv) {
    cro_compute_opts co;
    memset(&co, 0, sizeof co);
    co.iterations = (uint32_t)strtoul(argv[4], NULL, 10);
    co.alu_iterations = (uint32_t)strtoul(argv[5], NULL, 10);
    co.legs = (uint32_t)strtoul(argv[6], NULL, 10);
    co.max_rounds = (uint32_t)strtoul(argv[7], NULL, 10);
    co.test_inject_leg = atoi(argv[8]);
    co.test_inject_sm = atoi(argv[9]);
    co.test_inject_iteration = (uint32_t)strtoul(argv[10], NULL, 10);
    co.test_inject_row = atoi(argv[11]);
    co.test_inject_col = atoi(argv[12]);
    co.test_inject_mask = (uint32_t)strtoul(argv[13], NULL, 10);
    const int cap = atoi(argv[14]);
    static cro_compute_result cr;
    static cro_compute_sm sms[CRO_COMPUTE_MAX_SMS];
    cro_compute_fault *faults = (cro_compute_fault *)calloc(cap > 0 ? (size_t)cap : 1, sizeof *faults);
    int n_sms = 0, got = 0;
    if (!faults) return 2;
    cro_probe_compute(ctx, idx, &co, &cr, sms, CRO_COMPUTE_MAX_SMS, &n_sms, faults, cap > 0 ? cap : 0, &got);
    const uint64_t counts[2] = {(uint64_t)n_sms, (uint64_t)got};
    return write_frame(&cr, sizeof cr, counts, 2, sms, sizeof sms, faults, sizeof *faults, got, cr.status);
}

static int precision_raw(cro_ctx *ctx, int idx, char **argv) {
    cro_precision_opts po;
    memset(&po, 0, sizeof po);
    po.iterations = (uint32_t)strtoul(argv[4], NULL, 10);
    po.alu_iterations = (uint32_t)strtoul(argv[5], NULL, 10);
    po.legs = (uint32_t)strtoul(argv[6], NULL, 10);
    po.max_rounds = (uint32_t)strtoul(argv[7], NULL, 10);
    po.test_inject_leg = atoi(argv[8]);
    po.test_inject_sm = atoi(argv[9]);
    po.test_inject_iteration = (uint32_t)strtoul(argv[10], NULL, 10);
    po.test_inject_row = atoi(argv[11]);
    po.test_inject_col = atoi(argv[12]);
    po.test_inject_mask = (uint64_t)strtoull(argv[13], NULL, 10);
    const int cap = atoi(argv[14]);
    static cro_precision_result pr;
    static cro_precision_sm sms[CRO_PRECISION_MAX_SMS];
    cro_precision_fault *faults = (cro_precision_fault *)calloc(cap > 0 ? (size_t)cap : 1, sizeof *faults);
    int n_sms = 0, got = 0;
    if (!faults) return 2;
    cro_probe_precision(ctx, idx, &po, &pr, sms, CRO_PRECISION_MAX_SMS, &n_sms, faults, cap > 0 ? cap : 0, &got);
    const uint64_t counts[2] = {(uint64_t)n_sms, (uint64_t)got};
    return write_frame(&pr, sizeof pr, counts, 2, sms, sizeof sms, faults, sizeof *faults, got, pr.status);
}

static int l2_raw(cro_ctx *ctx, int idx, char **argv) {
    cro_l2_opts lo;
    memset(&lo, 0, sizeof lo);
    lo.bytes = (uint64_t)strtoull(argv[4], NULL, 10);
    lo.iterations = (uint32_t)strtoul(argv[5], NULL, 10);
    lo.a1_counters = (uint32_t)strtoul(argv[6], NULL, 10);
    lo.a2_counters = (uint32_t)strtoul(argv[7], NULL, 10);
    lo.test_inject_leg = atoi(argv[8]);
    lo.test_inject_sm = atoi(argv[9]);
    lo.test_inject_element = atoi(argv[10]);
    lo.test_inject_iteration = (uint32_t)strtoul(argv[11], NULL, 10);
    lo.test_inject_word = (int64_t)strtoll(argv[12], NULL, 10);
    lo.test_inject_mask = (uint64_t)strtoull(argv[13], NULL, 10);
    const int cap = atoi(argv[14]);
    static cro_l2_result lr;
    static cro_l2_sm sms[CRO_L2_MAX_SMS];
    cro_l2_fault *faults = (cro_l2_fault *)calloc(cap > 0 ? (size_t)cap : 1, sizeof *faults);
    int n_sms = 0, got = 0;
    if (!faults) return 2;
    cro_probe_l2(ctx, idx, &lo, &lr, sms, CRO_L2_MAX_SMS, &n_sms, faults, cap > 0 ? cap : 0, &got);
    const uint64_t counts[2] = {(uint64_t)n_sms, (uint64_t)got};
    return write_frame(&lr, sizeof lr, counts, 2, sms, sizeof sms, faults, sizeof *faults, got, lr.status);
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

/* The commands that take a device (argv[2]): their argc (0: at least 3, the rest optional), cro_opts.flags and sweep
 * region, whether argv[3] is cro_opts.seed_base, and what runs once the device is found (NULL: main's own probe). */
static const struct command {
    const char *name;
    int argc;
    uint32_t flags;
    uint64_t sweep_mib;
    int seeded;
    int (*run)(cro_ctx *ctx, int idx, char **argv);
} commands[] = {
    /* the hot-plug path: one device, identity from /proc (NVML's first call costs more than the probe), and a 1 GiB
     * first sweep unless argv[3] says otherwise — far beyond the L2, and it shortens everything before it */
    {"probe", 0, CRO_F_LAZY_ALLOC | CRO_F_DEGRADE_ON_OOM | CRO_F_NO_NVML, 1024, 0, NULL},
    {"probe-raw", 0, CRO_F_LAZY_ALLOC | CRO_F_DEGRADE_ON_OOM | CRO_F_NO_NVML, 1024, 0, NULL},
    {"cold", 0, CRO_F_LAZY_ALLOC | CRO_F_DEGRADE_ON_OOM | CRO_F_NO_NVML, 1024, 0, NULL},
    /* one check of one device by their own, not the HBM probe: no sweep region (the scan allocates its own chunks) and
     * NVML, whose DRAM / SRAM / L2 health record these read */
    {"scan", 0, CRO_F_LAZY_ALLOC, 64, 0, scan_json},
    {"scan-raw", 12, CRO_F_LAZY_ALLOC, 64, 0, scan_raw},
    {"sram-raw", 14, CRO_F_LAZY_ALLOC, 64, 0, sram_raw},
    {"l2-raw", 15, CRO_F_LAZY_ALLOC, 64, 1, l2_raw},
    /* a region of exactly L, argv[4] (the probe checks L <= S; no halving on a full GPU), and NVML for the replay
     * counters */
    {"link-raw", 11, CRO_F_LAZY_ALLOC, 256, 1, link_raw},
    /* no health record to read, and NVML's first call is slow */
    {"compute-raw", 15, CRO_F_LAZY_ALLOC | CRO_F_NO_NVML, 64, 1, compute_raw},
    {"precision-raw", 15, CRO_F_LAZY_ALLOC | CRO_F_NO_NVML, 64, 1, precision_raw},
};

int main(int argc, char **argv) {
    if (argc < 2) {
        fprintf(stderr, "usage: croprobe-cli csv <query> | enumerate | probe <uuid|index> [sweep_MiB] | probe-raw <uuid> [sweep_MiB] | "
                        "cold <uuid|index> [sweep_MiB] [nvml] | scan <uuid|index> [max_MiB] | scan-raw <uuid> <max> <reserve> <seed> <chunk> "
                        "<first> <count> <and> <or> <cap> | sram-raw <uuid> <legs> <iterations> <cluster> <rounds> <leg> <sm> <element> <iteration> "
                        "<word> <mask> <cap> | link-raw <uuid> <seed_base> <bytes> <hops> <ctas> <check> <word> <mask> <cap> | "
                        "compute-raw <uuid> <seed_base> <iterations> <alu_iterations> <legs> <rounds> <leg> <sm> <iteration> <row> <col> "
                        "<mask> <cap> | precision-raw <uuid> <seed_base> <iterations> <alu_iterations> <legs> <rounds> <leg> <sm> <iteration> <row> "
                        "<col> <mask> <cap> | l2-raw <uuid> <seed_base> <bytes> <iterations> <a1> <a2> <leg> <sm> <element> <iteration> <word> <mask> <cap>\n");
        return 64;
    }
    const double t_start = now_s();
    const char *cmd = argv[1];
    const struct command *c = NULL;
    for (size_t k = 0; k < sizeof commands / sizeof *commands; ++k)
        if (strcmp(cmd, commands[k].name) == 0) c = &commands[k];
    if (c && (argc < 3 || (c->argc && argc != c->argc))) return 64;
    const int cold = strcmp(cmd, "cold") == 0;
    cro_opts opts;
    memset(&opts, 0, sizeof opts);
    opts.abi_version = CRO_ABI_VERSION;
    opts.flags = CRO_F_LAZY_ALLOC | CRO_F_DEGRADE_ON_OOM;
    if (c) {
        opts.flags = c->flags;
        opts.sweep_bytes = c->sweep_mib << 20;
        if (c->seeded) opts.seed_base = (uint64_t)strtoull(argv[3], NULL, 10);
        if (!c->run && argc > 3) opts.sweep_bytes = (uint64_t)strtoull(argv[3], NULL, 10) << 20;    /* the probe's sweep_MiB */
        if (cold && argc > 4 && strcmp(argv[4], "nvml") == 0) opts.flags &= ~CRO_F_NO_NVML;
        if (c->run == link_raw && strtoull(argv[4], NULL, 10)) opts.sweep_bytes = (uint64_t)strtoull(argv[4], NULL, 10);  /* L */
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
            return write_frame(&r, sizeof r, NULL, 0, NULL, 0, NULL, 0, 0, r.status);
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
