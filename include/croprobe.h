/*
 * croprobe.h — C ABI of libcroprobe, the H100-native post-attach device probe
 * and spec-emit path for the composable-resource operator.
 *
 * This header is the drop-in boundary (SURVEY.md §8b).  Everything here is
 * plain C: opaque context pointer, caller-allocated output buffers, integer
 * return codes.  No torch / C++ types cross it.  A Go host binds it with cgo
 * (see INTEGRATION.md and composable-resource-operator_b200/go/internal/cuda);
 * the tests and bench.py bind it with ctypes.
 *
 * Each entry point names the reference interface (path:line under the
 * reference tree) whose slot in the reconcile loop it fills or replaces.
 *
 * Threading: every entry point is re-entrant.  Calls that touch a device take
 * that device's mutex and call cudaSetDevice themselves, so they may be issued
 * from any OS thread (cgo migrates goroutines between threads).  No callbacks.
 * Ownership: cro_ctx is library-owned (cro_probe_destroy frees it); every
 * other buffer is caller-owned and is not retained after the call returns.
 */
#ifndef CROPROBE_H_
#define CROPROBE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CRO_ABI_VERSION 2u

/* ---- return codes (0 ok, <0 error; text via cro_strerror) ---------------- */
#define CRO_OK                  0
#define CRO_ERR_INVALID_ARG    -1
#define CRO_ERR_ABI_MISMATCH   -2
#define CRO_ERR_NO_DEVICE      -3   /* zero CUDA devices: not an error for enumerate (n=0) */
#define CRO_ERR_CUDA           -4   /* a CUDA runtime call failed; see cro_last_error */
#define CRO_ERR_OOM            -5   /* sweep buffer could not be allocated (device busy) */
#define CRO_ERR_CHECKSUM       -6   /* HBM sweep checksum differs from the closed form   */
#define CRO_ERR_BUFFER_SMALL   -7   /* caller buffer too small; *len holds the need      */
#define CRO_ERR_NCCL           -8
#define CRO_ERR_DEADLINE       -9
#define CRO_ERR_UNSUPPORTED   -10   /* e.g. unsupported field in a query string          */
#define CRO_ERR_PARSE         -11   /* malformed CSV / JSON handed to a parser           */
#define CRO_ERR_EXEC          -12   /* the enumerate command reported stderr / exec error */
#define CRO_ERR_P2P           -13
#define CRO_ERR_INTERNAL      -14

/* ---- option flags -------------------------------------------------------- */
#define CRO_F_SKIP_COPY       0x0001u  /* do not run the hbm_copy sweeps           */
#define CRO_F_SKIP_P2P        0x0002u  /* cro_probe_all: no NVLink rounds          */
#define CRO_F_SKIP_NCCL       0x0004u  /* cro_probe_all: host gather, no NCCL      */
#define CRO_F_NO_NVML         0x0008u  /* identity from /proc + CUDA runtime only  */
#define CRO_F_VERIFY_COPY     0x0010u  /* accepted, no effect: since ABI 2 every copy destination is re-read and
                                          compared inside the probe (copy_verified)                            */
#define CRO_F_LAZY_ALLOC      0x0020u  /* allocate sweep buffers at first probe    */
#define CRO_F_DEGRADE_ON_OOM  0x0040u  /* busy device: halve S (>= 64 MiB) instead of failing;
                                          the result's sweep_bytes says what was swept  */
#define CRO_F_SKIP_P2P_WRITE  0x0080u  /* cro_probe_all: peer reads only, no push leg */
#define CRO_F_TEST_INJECT     0x0100u  /* fault injection INSIDE the probe (tests of the device-side verdict): after sweep
                                          number test_inject_after (launch order: 0 = the fill, 1.. = copies, then reads)
                                          XOR test_inject_mask into 64-bit word test_inject_word of the region (half A is
                                          words [0, S/8), half B [S/8, 2S/8)) */

/* read-sweep kernel variants */
#define CRO_READ_AUTO   0u   /* by sweep size: 128-bit LDG up to 128 MiB, the TMA ring above (measured crossover) */
#define CRO_READ_LDG    1u   /* ld.global.nc.L1::no_allocate 128-bit, unrolled      */
#define CRO_READ_TMA    2u   /* cp.async.bulk (1-D TMA) smem ring + LDS.128 reduce  */
#define CRO_COPY_AUTO   0u
#define CRO_COPY_LDG    1u
#define CRO_COPY_TMA    2u   /* bulk load -> smem -> bulk store, no register pass   */
#define CRO_COPY_TMA_FUSED 3u /* the same, and consumer warps fold every tile out of shared memory: the sweep
                                yields the checksum of its source as read (the probe's default)          */
#define CRO_READ_LDG256 3u   /* 32-byte LDG flavour: two adjacent 128-bit loads, L2 evict_first */

#define CRO_MAX_DEVICES 16

typedef struct cro_ctx cro_ctx;

/* Options for cro_probe_init.  Zero means "default" for every field. */
typedef struct cro_opts {
    uint32_t abi_version;          /* must be CRO_ABI_VERSION                               */
    uint32_t flags;                /* CRO_F_*                                               */
    uint64_t sweep_bytes;          /* S, per-device sweep region; default 4 GiB             */
    uint64_t p2p_bytes;            /* S_p2p per directed pair; default 1 GiB (<= S)         */
    uint64_t seed_base;            /* default 0x00C0FFEE00000000; seed = base | minor       */
    uint32_t read_sweeps;          /* default 5                                             */
    uint32_t copy_sweeps;          /* default 5                                             */
    uint32_t latency_hops;         /* pointer-chase hops per directed pair; default 1024    */
    uint32_t read_variant;         /* CRO_READ_*                                            */
    uint32_t copy_variant;         /* CRO_COPY_*                                            */
    int32_t  deadline_ms;          /* per-call deadline, 0 = none (Go ctx cannot cross cgo) */
    int32_t  n_devices;            /* 0 = every visible CUDA device                         */
    int32_t  devices[CRO_MAX_DEVICES]; /* CUDA ordinals to manage                           */
    uint32_t rank_base;            /* one-process-per-GPU hosts: this process's first rank  */
    uint32_t world_override;       /* ... and the job's world size (0 = devices managed)    */
    uint32_t test_inject_after;    /* CRO_F_TEST_INJECT: see above                          */
    uint32_t reserved0;
    uint64_t test_inject_word;
    uint64_t test_inject_mask;
} cro_opts;

/*
 * Identity of one device in the spellings the reference consumes
 * (internal/utils/gpus.go:878-919 parses `nvidia-smi --query-gpu=...` CSV;
 * :1014-1089 parses /proc/driver/nvidia/gpus/<bus>/information).
 */
typedef struct cro_dev_info {
    int32_t  cuda_ordinal;
    int32_t  device_minor;         /* -1 if no source could supply it                       */
    char     gpu_uuid[48];         /* "GPU-xxxxxxxx-xxxx-xxxx-xxxx-xxxxxxxxxxxx", NUL padded */
    char     pci_bus_id[24];       /* nvidia-smi spelling "00000000:1F:00.0"                */
    char     name[64];
    uint64_t hbm_bytes_total;
    uint32_t sm_count;
    uint32_t cc_major, cc_minor;
    uint32_t identity_source;      /* 1 NVML, 2 /proc, 3 CUDA runtime only                  */
    uint32_t flags;                /* CRO_DEV_*                                             */
    int32_t  dev_index;            /* index for cro_probe_device / cro_hbm_*; -1: not in this process */
    uint32_t reserved[2];
} cro_dev_info;

/* The node's inventory is re-read on EVERY cro_enumerate (the reference execs a fresh nvidia-smi on every
 * reconcile, internal/utils/gpus.go:666-689); the devices a context can probe itself are fixed at cro_probe_init
 * because CUDA's device list is fixed at cuInit. */
#define CRO_DEV_IN_PROCESS    0x1u  /* managed by this context: probe it with cro_probe_device(dev_index)       */
#define CRO_DEV_NEEDS_HELPER  0x2u  /* on the node but attached after cro_probe_init: cro_probe_uuid probes it
                                       through a one-shot helper process (croprobe-cli) with its own cuInit     */

/*
 * Fixed-size, pointer-free, integer-only per-device result: the payload of the
 * single NCCL all-gather (SURVEY.md Appendix C).  512 bytes, little-endian.
 * Offsets 0..351 are Appendix C's; its reserved tail holds the rest.
 *
 * The struct is WRITTEN ON THE DEVICE (ABI 2): a one-CTA finalize kernel at the
 * end of the probe's CUDA graph compares every sweep with the closed form,
 * takes the sweep times from %globaltimer and fills the all-gather send buffer;
 * the host only copies it back.  Identity fields are staged once at init.
 *
 * Checksum of a sweep over 64-bit words w[0..n): xor = XOR of all words,
 * sum = wrapping sum, wsum = wrapping sum of w[i] * (2i + 1) — the last one
 * makes every word's POSITION matter.
 */
typedef struct cro_probe_result {
    uint32_t abi_version;          /*   0 */
    int32_t  status;               /*   4  CRO_OK or a CRO_ERR_* */
    int32_t  cuda_ordinal;         /*   8 */
    int32_t  device_minor;         /*  12 */
    char     gpu_uuid[48];         /*  16 */
    char     pci_bus_id[24];       /*  64 */
    uint64_t hbm_bytes_total;      /*  88 */
    uint64_t sweep_bytes;          /*  96 */
    uint64_t seed;                 /* 104  effective pattern seed of THIS probe:
                                           (seed_base | minor) + nonce * 0xD1B54A32D192ED03 */
    uint64_t checksum_xor;         /* 112  of read sweep 0 — or, when the first check that failed is a read sweep's
                                           (stale or wrong), of that read sweep */
    uint64_t checksum_sum;         /* 120 */
    uint64_t fill_ns;              /* 128  sweep times: %globaltimer, first CTA start .. last CTA end */
    uint64_t read_best_ns;         /* 136 */
    uint64_t read_median_ns;       /* 144 */
    uint64_t copy_best_ns;         /* 152 */
    uint64_t copy_median_ns;       /* 160 */
    uint32_t sm_count;             /* 168 */
    uint32_t sm_clock_mhz;         /* 172 */
    uint32_t mem_clock_mhz;        /* 176 */
    uint32_t ecc_errors;           /* 180  uncorrected volatile ECC errors (NVML), read at init, at
                                           cro_probe_all and after any failed probe */
    uint64_t p2p_read_ns[8];       /* 184  time to read p2p_bytes out of peer j's HBM over NVLink */
    uint64_t p2p_checksum_xor[8];  /* 248 */
    uint32_t p2p_latency_ns_x16[8];/* 312  mean hop latency x16 (fixed point): min(chase ns * 16 / hops, 2^32 - 1) */
    uint8_t  p2p_access[8];        /* 344  cudaDeviceCanAccessPeer                   */
    uint64_t p2p_bytes;            /* 352 */
    uint64_t expect_xor;           /* 360  closed-form checksum computed on the device
                                           by an independent generator kernel        */
    uint64_t expect_sum;           /* 368 */
    uint64_t expect_wsum;          /* 376 */
    uint64_t checksum_wsum;        /* 384 */
    uint64_t copy_checksum_xor;    /* 392  checksum of the LAST copy's destination (read back by the first read sweep);
                                           written only when the probe ran copy and read sweeps */
    uint64_t copy_checksum_sum;    /* 400 */
    uint64_t copy_checksum_wsum;   /* 408 */
    uint64_t total_ns;             /* 416  first CTA of the fill .. last CTA of any sweep (the latest t1 of the fill, copy
                                           and read slots, minus the fill's t0, modulo 2^64) */
    uint64_t p2p_write_ns[8];      /* 424  time to PUSH p2p_bytes into peer j's scratch half
                                           (posted NVLink writes; the peer re-reads and checks them) */
    uint32_t nonce;                /* 488  probe number on this device (0 = first probe of the context) */
    uint8_t  rank;                 /* 492  index in the minor-sorted device list      */
    uint8_t  world;                /* 493 */
    uint8_t  read_variant;         /* 494  CRO_READ_* actually used                  */
    uint8_t  copy_variant;         /* 495 */
    uint8_t  read_sweeps;          /* 496 */
    uint8_t  copy_sweeps;          /* 497 */
    uint8_t  copy_verified;        /* 498  copy sweeps whose destination was re-read and matched the closed form
                                           (sweep k+1 folds what sweep k wrote; the first read sweep folds the last).
                                           Counted per passing check, also after an earlier failure: every checksumming
                                           copy k >= 1 that passed, plus read sweep 0 if it passed and copies ran */
    uint8_t  fail_code;            /* 499  CRO_FAIL_*: which check failed first (0 = none), in the order: closed form,
                                           fill stamp, each copy sweep (stamp, then fold when it checksums), each read
                                           sweep (stamp, then fold); p2p_finalize adds its peer checks after all of them */
    uint8_t  fail_index;           /* 500  CRO_FAIL_STALE: the sweep's number in launch order (0 fill, 1.. copies, then
                                           reads); CRO_FAIL_COPY_SRC / CRO_FAIL_READ: the copy / read sweep's own index;
                                           CRO_FAIL_EXPECT: 0, or the peer whose prefix slot is stale; peer checks: the peer */
    uint8_t  p2p_ok;               /* 501  bit j: NVLink read of, push into and chase through peer j all verified */
    uint8_t  reserved8[2];         /* 502 */
    uint64_t t_start_ns;           /* 504  %globaltimer when the probe's first CTA started */
} cro_probe_result;

#define CRO_FAIL_NONE        0
#define CRO_FAIL_EXPECT      1   /* the closed-form slot is stale or short: the generator kernel did not run */
#define CRO_FAIL_COPY_SRC    2   /* copy sweep fail_index read something else than the pattern */
#define CRO_FAIL_READ        3   /* read sweep fail_index */
#define CRO_FAIL_P2P_READ    4   /* NVLink read of peer fail_index */
#define CRO_FAIL_P2P_PUSH    5   /* what peer fail_index pushed did not land here intact */
#define CRO_FAIL_P2P_CHASE   6   /* pointer chase through peer fail_index ended on the wrong slot */
#define CRO_FAIL_STALE       7   /* a sweep slot carries another probe's nonce: that kernel did not run */

/* CUDA-event times of the sweeps of the device's most recent probe, in launch order
 * (fill, copy sweeps, read sweeps).  kind: 0 fill, 1 copy, 2 read. */
typedef struct cro_sweep_time {
    uint32_t kind;
    uint32_t index;
    uint64_t bytes;                /* algorithmic bytes of the sweep (S, or 2S for a copy) */
    uint64_t event_ns;             /* CUDA events on the launching stream                 */
    uint64_t timer_ns;             /* %globaltimer window the kernel itself recorded      */
} cro_sweep_time;

/* One directed NVLink pair of the most recent cro_probe_all, in full (the 512-byte struct keeps a digest). */
typedef struct cro_p2p_detail {
    uint64_t read_ns, push_ns, reread_ns;
    uint64_t read_xor, read_sum, read_wsum;        /* what this device folded out of the peer's HBM   */
    uint64_t landed_xor, landed_sum, landed_wsum;  /* what the PEER found in its scratch half after this device's push */
    uint64_t expect_xor, expect_sum, expect_wsum;  /* closed form of the peer's first p2p_bytes       */
    uint64_t chase_ns;
    uint32_t chase_end, chase_expect, hops, access;
} cro_p2p_detail;

/* Result of one timed sweep (bench / parity entry points). */
typedef struct cro_sweep_result {
    uint64_t bytes;                /* algorithmic bytes of the sweep (S, or 2S for copy) */
    uint64_t ns;                   /* CUDA-event duration of the kernel launch(es)       */
    uint64_t checksum_xor;
    uint64_t checksum_sum;
    uint32_t variant;
    uint32_t launches;             /* kernels launched by this call                      */
    uint64_t checksum_wsum;        /* position-weighted sum: wrapping sum of w[i] * (2i + 1) */
    uint64_t timer_ns;             /* %globaltimer window the (last) kernel recorded itself */
} cro_sweep_result;

/* ---- lifecycle ----------------------------------------------------------- */

/* Creates the long-lived probe context (CUDA primary contexts, sweep buffers,
 * streams, events).  The reference has no counterpart: it re-execs nvidia-smi
 * every reconcile (internal/utils/gpus.go:886).  A warm context is what makes
 * the storm / churn configs meaningful (SURVEY.md §7 "cold-start cost"). */
int  cro_probe_init(const cro_opts *opts, cro_ctx **out);
void cro_probe_destroy(cro_ctx *ctx);

/* ---- enumeration: replaces the exec of nvidia-smi ------------------------ */

/* Replaces `nvidia-smi --query-gpu=gpu_uuid` run for its side effect by
 * utils.RunNvidiaSmi (internal/utils/gpus.go:666-689). */
int  cro_device_count(cro_ctx *ctx, int *n);

/* Replaces getGPUInfoFromNvidiaPod / getGPUInfoFromCroNodeAgentPod /
 * getGPUInfoFromProcInCroNodeAgentPod (internal/utils/gpus.go:878-919,
 * 921-962, 1014-1089).  Rows are in nvidia-smi order.  The answer is FRESH on every call: the driver's
 * registry under /proc/driver/nvidia/gpus is re-read (and NVML re-initialised when that shows a change), so a GPU
 * composed after cro_probe_init is listed (CRO_DEV_NEEDS_HELPER) and a GPU drained off the bus is not. */
int  cro_enumerate(cro_ctx *ctx, cro_dev_info *out, int cap, int *n);

/* The same merge without a context (ctx-free, no CUDA call): what cro_enumerate answers for a context managing
 * `in_process` on a node whose /proc is mounted at proc_root (NULL = "/proc").  Only /proc is consulted. */
int  cro_node_inventory(const char *proc_root, const cro_dev_info *in_process, int n_in_process,
                        cro_dev_info *out, int cap, int *n);

/* Probe by UUID — the form the reconcile step uses (Status.DeviceID is a UUID,
 * internal/controller/composableresource_controller.go:231-233).  In-process devices: cro_probe_device.  Devices
 * that reached the node after cro_probe_init: a helper process (`croprobe-cli probe-raw`, CUDA_VISIBLE_DEVICES=<uuid>,
 * deadline CRO_HELPER_TIMEOUT_MS).  A UUID the node does not list: CRO_ERR_NO_DEVICE — the reference's
 * "found = false", not an error of the probe.  ctx may be NULL (every device then goes through the helper). */
int  cro_probe_uuid(cro_ctx *ctx, const char *gpu_uuid, cro_probe_result *out);

/* Text that `nvidia-smi --query-gpu=<query> --format=csv,noheader,nounits`
 * would print for these devices, so the unchanged Go parser at
 * internal/utils/gpus.go:903-916 can consume it.  n == 0 emits
 * "No devices were found\n" (gpus.go:896).  query fields: device_minor,
 * gpu_uuid, pci.bus_id, name, index, memory.total. */
int  cro_emit_csv(const cro_dev_info *devs, int n, const char *query,
                  char *buf, size_t cap, size_t *len);

/* The reference's CSV parse rule (internal/utils/gpus.go:896-916), kept
 * quirk-for-quirk.  Output: Go encoding/json of the []map[string]string the
 * reference would build.  exec_err NULL means a nil error.  Returns
 * CRO_ERR_EXEC with the reference's formatted message in buf on the error
 * path, CRO_ERR_PARSE where the reference would panic (short row). */
int  cro_parse_gpu_csv(const char *std_out, const char *std_err, const char *exec_err,
                       const char *query, char *buf, size_t cap, size_t *len);

/* /proc flavour (internal/utils/gpus.go:1045-1089): input is the script's
 * "minor,uuid,bus" lines. */
int  cro_parse_proc_csv(const char *std_out, const char *std_err, const char *exec_err,
                        const char *query, char *buf, size_t cap, size_t *len);

/* Turns one /proc/driver/nvidia/gpus/<bus>/information text into the
 * "minor,uuid,bus" line of the awk script at gpus.go:1017-1037 ("" if any
 * of the three keys is missing). */
int  cro_proc_information_to_line(const char *information_text,
                                  char *buf, size_t cap, size_t *len);

/* Membership decision of utils.CheckGPUVisible, DEVICE_PLUGIN branch
 * (internal/utils/gpus.go:73-84): is device_id among the enumerated UUIDs. */
int  cro_check_gpu_visible(const cro_dev_info *devs, int n, const char *device_id,
                           int *visible);

/* Bus-id / device-path spellings the reference derives
 * (internal/utils/gpus.go:218,326,406,567,238,480).  kind:
 * 0 upper(trim), 1 lower(trim), 2 TrimPrefix("0000") of upper,
 * 3 "/dev/nvidia"+minor, 4 "/run/nvidia/driver/dev/nvidia"+minor. */
int  cro_normalize(int kind, const char *in, char *buf, size_t cap, size_t *len);

/* ---- the probe: new work in the slot of RunNvidiaSmi + CheckGPUVisible --- */

/* Full per-device probe (fill, read sweeps, copy sweeps, closed-form check).
 * Sits at internal/controller/composableresource_controller.go:259 and feeds
 * the decision at :275.  dev_index indexes the cro_enumerate order. */
int  cro_probe_device(cro_ctx *ctx, int dev_index, cro_probe_result *out);

/* Asynchronous form of cro_probe_device: begin enqueues the whole probe on the
 * device's stream and returns at once; end waits for the OLDEST probe begun on
 * the device and hands out its result.  One host thread (the reference's single
 * reconcile worker, MaxConcurrentReconciles=1) can keep every attached GPU busy
 * this way.  Up to TWO probes per device may be in flight: the second one's
 * kernels are queued behind the first's on the device, so the GPU does not idle
 * while the host collects a result and starts the next attach's probe.  A third
 * begin is a no-op; end without begin probes synchronously. */
int  cro_probe_begin(cro_ctx *ctx, int dev_index);
int  cro_probe_end(cro_ctx *ctx, int dev_index, cro_probe_result *out);

/* Concurrent probe of every managed device, NVLink P2P rounds, then ONE
 * ncclAllGather of the 512-byte result structs.  out[] receives the gathered
 * array as rank 0 holds it (asserted byte-identical on every rank).
 * NCCL is dlopen'ed at the first call: the copy the host process already carries if there is one, else
 * $CRO_NCCL_PATH, else libnccl.so.2 — never with RTLD_GLOBAL.  CRO_NCCL_PATH=off, or no usable library: the structs
 * come back per device over pinned memory instead and cro_fullbox_time.gather reports CRO_GATHER_DEGRADED. */
int  cro_probe_all(cro_ctx *ctx, cro_probe_result *out, int cap, int *n);

/* Device address of this device's result struct (the all-gather send buffer),
 * for hosts that run their own collective (bench.py under torchrun). */
int  cro_result_device_ptr(cro_ctx *ctx, int dev_index, uint64_t *dptr);

/* Single sweeps, timed with CUDA events on the launching stream. */
int  cro_hbm_fill(cro_ctx *ctx, int dev_index, cro_sweep_result *out);
int  cro_hbm_read_checksum(cro_ctx *ctx, int dev_index, uint32_t variant, cro_sweep_result *out);
int  cro_hbm_copy(cro_ctx *ctx, int dev_index, uint32_t variant, cro_sweep_result *out);
/* Checksum of the copy destination region (same kernel, other half). */
int  cro_hbm_read_checksum_dst(cro_ctx *ctx, int dev_index, uint32_t variant, cro_sweep_result *out);
/* Closed-form expected checksum computed on the device without touching HBM. */
int  cro_hbm_expected_checksum(cro_ctx *ctx, int dev_index, cro_sweep_result *out);
/* Fault injection for tests: XOR `mask` into the 64-bit word at word_index. */
int  cro_inject_fault(cro_ctx *ctx, int dev_index, uint64_t word_index, uint64_t mask);
/* Copies [word_first, word_first+n_words) of the sweep region to host memory. */
int  cro_read_words(cro_ctx *ctx, int dev_index, uint64_t word_first, uint64_t n_words, uint64_t *out);
/* Repeats the read sweep `iters` times back to back under one event pair. */
int  cro_hbm_read_loop(cro_ctx *ctx, int dev_index, uint32_t variant, uint32_t iters, cro_sweep_result *out);
int  cro_hbm_copy_loop(cro_ctx *ctx, int dev_index, uint32_t variant, uint32_t iters, cro_sweep_result *out);
int  cro_hbm_fill_loop(cro_ctx *ctx, int dev_index, uint32_t iters, cro_sweep_result *out);
/* Seed of the pattern the device's region holds now: (seed_base | minor) + nonce * 0xD1B54A32D192ED03, where
 * nonce counts the probes this context has run on the device (every probe writes a fresh pattern, so a fill or
 * copy that silently did nothing cannot pass on the previous probe's bytes). */
int  cro_device_seed(cro_ctx *ctx, int dev_index, uint64_t *seed);
/* CUDA-event and %globaltimer times of every sweep of the device's most recent probe, in launch order. */
int  cro_probe_sweep_times(cro_ctx *ctx, int dev_index, cro_sweep_time *out, int cap, int *n);
/* One directed NVLink pair (dev_index -> peer_index) of the most recent cro_probe_all. */
int  cro_p2p_detail_get(cro_ctx *ctx, int dev_index, int peer_index, cro_p2p_detail *out);
/* Phases of the most recent cro_probe_all. */
typedef struct cro_fullbox_time {
    uint64_t enqueue_ns;           /* host time spent enqueueing (no waits inside)                      */
    uint64_t wall_ns;              /* host wall clock of the call                                       */
    uint64_t hbm_ns;               /* slowest device's HBM probe (%globaltimer)                         */
    uint64_t p2p_ns;               /* slowest device's NVLink bandwidth rounds, first kernel .. last    */
    uint64_t chase_ns;             /* slowest pointer chase                                             */
    uint64_t gather_ns;            /* the all-gather, CUDA events on rank 0's stream                    */
    uint32_t rounds;               /* NVLink rounds (n-1 for even n)                                    */
    uint32_t host_syncs;           /* stream synchronisations the call made (one per device)            */
    uint32_t gather;               /* CRO_GATHER_*: how the result structs were brought together        */
    uint32_t reserved;
} cro_fullbox_time;
#define CRO_GATHER_HOST      0u    /* copied back per device, assembled on the host (one device, or CRO_F_SKIP_NCCL) */
#define CRO_GATHER_NCCL      1u    /* ncclAllGather on the devices' streams, every rank holds the same array         */
#define CRO_GATHER_DEGRADED  2u    /* NCCL was asked for but no usable libnccl is in reach: host-side gather over
                                      pinned memory instead — "replicas only" (SURVEY.md §8e); cro_last_error says why */
int  cro_fullbox_times(cro_ctx *ctx, cro_fullbox_time *out);
/* The reply structs the fabric decoders walk ("FMScaleUpResponse", "FMGetMachineResponse", "CMMachineData"), as
 * JSON: {"type","struct","fields":[{"json","of":{...}}]} in declaration order — so that a test can hold them against
 * the declarations in the reference's Go source (the .go files of internal/cdi/fti/fm/api, and internal/cdi/fti/cm/api/machine.go). */
int  cro_describe_wire_type(const char *name, char *buf, size_t cap, size_t *len);
/* Prometheus text exposition (counters and per-GPU gauges of the last probe) for the operator's metrics registry
 * (cmd/main.go:66,119-125 wires controller-runtime's registry; a Go collector forwards these lines):
 * cro_probe_total, cro_probe_failures_total, cro_fullbox_probe_total, cro_helper_probe_total,
 * cro_inventory_rescans_total, cro_kernel_launches_total, cro_probe_status{gpu_uuid,minor},
 * cro_probe_hbm_{read,copy,fill}_bytes_per_second{..}, cro_probe_copies_verified{..}, cro_probe_ecc_uncorrected{..}. */
int  cro_metrics_text(cro_ctx *ctx, char *buf, size_t cap, size_t *len);
/* Pointer-chase length of the following cro_probe_all calls (1 .. 16777216 hops per directed pair). */
int  cro_set_latency_hops(cro_ctx *ctx, uint32_t hops);
/* Where `hops` steps from slot 0 of the latency permutation of the directed pair (minor_src chases through
 * minor_dst's memory) end: Sattolo cycle over 65536 slots, mt19937_64 seeded with minor_src * 8 + minor_dst
 * (SURVEY.md §8d config 3).  Host arithmetic only. */
int  cro_chase_end(int minor_src, int minor_dst, uint32_t hops, uint32_t *end);
/* The CRO_* environment knobs are validated like the reference validates its own
 * (internal/controller/composableresource_adapter.go:42-45): an illegal value fails cro_probe_init with
 * "the env variable <NAME> has an invalid value: '<v>'".  This checks one (name, value) pair — or, with
 * name == NULL, the process environment as cro_probe_init would — without needing a GPU.  It is a check only:
 * a context keeps the values it was created with, whatever the environment says later. */
int  cro_validate_env(const char *name, const char *value, char *err_buf, size_t err_cap);
/* Kernel launches issued by this context so far (bench "gpu_launches"). */
uint64_t cro_launch_count(cro_ctx *ctx);

/* ---- fault locator: where a failed probe's bad words are ------------------- */

/*
 * After a probe failed (typically CRO_ERR_CHECKSUM), names the words behind it.  Nothing of the probe changes: the
 * locator runs only when called.  It takes the device's mutex and lets probes still in flight finish first (their
 * results stay collectable with cro_probe_end).
 *
 * Pass 0 (post-mortem) compares each half of the sweep region, as the last operation left it, with the pattern the
 * context knows that half holds; it writes nothing.  A half that holds no known pattern is skipped (after
 * cro_probe_all with the NVLink push leg half B holds a peer's prefix; a probe without copy sweeps leaves half B as it
 * was).  With CRO_LOCATE_RETEST two more passes follow: pass 1 fills both halves with a fresh pattern (retest seed: the
 * device seed + 2^63, a seed no probe nonce reaches) and compares, pass 2 does the same with the bitwise complement.
 * Every bit cell is then written and read back as 0 and as 1, so a stuck-at bit mismatches in exactly one of passes
 * 1 and 2.  The retest consumes no probe nonce; afterwards both halves hold no known pattern and the single-sweep
 * entry points refill half A first.
 *
 * Word indices are the region's, as for cro_inject_fault / cro_read_words: [0, S/8) half A, [S/8, S/4) half B.
 * Word i of either half is expected to hold pattern_word(seed, i) (XOR all ones in pass 2).
 */
#define CRO_LOCATE_RETEST        0x1u
#define CRO_LOCATE_RECORDS       4096     /* word records the device keeps per pass; counts stay exact beyond */
#define CRO_LOCATE_PASSES        3
#define CRO_LOCATE_GRANULE_BYTES (2u << 20)

#define CRO_FAULTS_NONE           0u      /* no pass found a mismatch                                          */
#define CRO_FAULTS_UNCLASSIFIED   1u      /* pass 0 found mismatches and no retest ran                          */
#define CRO_FAULTS_NOT_REPRODUCED 2u      /* pass 0 found mismatches, the retest found none: a transient error, or
                                             a write that went wrong once                                        */
#define CRO_FAULTS_PERSISTENT     3u      /* a retest pass found a mismatch: cells that do not hold what is written */

typedef struct cro_locate_opts {
    uint32_t flags;                /* CRO_LOCATE_*                                                          */
    uint32_t reserved0;
    /* test only: after each retest fill, word = (word & test_force_and) | test_force_or for the region words
       [test_force_first, test_force_first + test_force_count) — a stand-in for stuck cells or a fault storm */
    uint64_t test_force_first;
    uint64_t test_force_count;
    uint64_t test_force_and;
    uint64_t test_force_or;
} cro_locate_opts;

typedef struct cro_fault_word {
    uint64_t word_index;           /* region index                                                          */
    uint64_t expected;             /* from the first pass that saw the word                                 */
    uint64_t actual;
    uint32_t passes;               /* bit p: pass p found the word wrong                                    */
    uint32_t reserved;
} cro_fault_word;

typedef struct cro_locate_pass {
    uint32_t halves;               /*   0  bit h: half h (0 = A, 1 = B) was compared                        */
    uint32_t skipped;              /*   4  bit h: half h was not compared, it holds no known pattern          */
    uint64_t seed[2];              /*   8  seed half h was compared against (0 = not compared)                */
    uint64_t invert;               /*  24  XOR on the pattern: 0, all ones in pass 2                          */
    uint64_t words_scanned;        /*  32 */
    uint64_t mismatches;           /*  40  exact                                                             */
    uint64_t recorded;             /*  48  mismatches the device recorded (<= CRO_LOCATE_RECORDS)            */
    uint64_t granules;             /*  56  CRO_LOCATE_GRANULE_BYTES granules of the region with a mismatch     */
    uint64_t scan_ns;              /*  64  %globaltimer windows of the pass's compare sweeps, summed          */
    uint64_t fold_xor[2];          /*  72  checksum of half h as read (xor, sum, wsum as for a read sweep)    */
    uint64_t fold_sum[2];          /*  88 */
    uint64_t fold_wsum[2];         /* 104 */
} cro_locate_pass;                 /* 120 bytes */

typedef struct cro_fault_report {
    int32_t  status;               /*   0  the return value: CRO_OK when nothing mismatched, else CRO_ERR_CHECKSUM */
    uint32_t verdict;              /*   4  CRO_FAULTS_*                                                      */
    uint32_t n_passes;             /*   8  1, or 3 with CRO_LOCATE_RETEST                                     */
    uint32_t complete;             /*  12  1: every mismatch of every pass is in the caller's list, and for each
                                              compared half the located words' deltas reproduce the difference
                                              between its folded checksum and the half's closed form (xor, sum and
                                              weighted sum) — the compare path missed nothing the checksum saw     */
    uint64_t sweep_bytes;          /*  16  S                                                                 */
    uint64_t retest_seed;          /*  24  0 without CRO_LOCATE_RETEST                                        */
    uint64_t located;              /*  32  distinct words the device recorded over all passes                 */
    uint64_t recorded;             /*  40  words written to the caller's list (*n)                             */
    uint64_t flip_or;              /*  48  OR of every mismatch's actual ^ expected                            */
    uint64_t bit_flips[64];        /*  56  mismatches (over all passes) with bit b flipped                     */
    cro_locate_pass pass[CRO_LOCATE_PASSES];   /* 568 */
} cro_fault_report;                /* 928 bytes */

/* words[0 .. cap) receives the located words sorted by word_index, *n how many were written.  Devices probed through
 * the helper process (cro_probe_uuid of a GPU attached after init) cannot be located: dev_index is an in-process
 * device.  opts may be NULL (pass 0 only). */
int  cro_locate_faults(cro_ctx *ctx, int dev_index, const cro_locate_opts *opts,
                       cro_fault_report *out, cro_fault_word *words, int cap, int *n);

/* ---- host link: the PCIe path between the host and a composed GPU ------------ */

/*
 * The PCIe path a fabric composes is the one part of an attached GPU the HBM probe never exercises.  The link probe
 * moves a fresh pattern across it in both directions, with the copy engines and with the SMs (loads and stores to
 * mapped pinned host memory), each direction alone and both at once, checks every byte that crossed, times a
 * dependent pointer chase through host memory, and reads the link's trained speed and width, and those of every hop
 * above it, from sysfs.  It runs only when called and changes nothing of the probe.
 *
 * The call takes the device's mutex and lets probes still in flight finish first (their results stay collectable with
 * cro_probe_end).  It uses the first L bytes of the sweep region's half A and half B and allocates no device memory
 * beyond a few small result buffers; on its first call it allocates two pinned host buffers H0, H1 of L bytes (grown
 * when a later call asks for more) and an 8 MiB chase table, placed on the device's NUMA node when sysfs names one.
 * Afterwards neither half holds a known pattern: the next single sweep refills half A, and cro_locate_faults' pass 0
 * skips both halves.
 *
 * Three fresh patterns per call (P1, P2, P3 of seed[]), and each step's bytes are checked by a later step:
 *   leg CE_D2H          copy engine A -> H0 (A filled with P1)          checked by check 0
 *   leg SM_H2D          SMs read H0 over the link                        = check 0 (H0 against P1)
 *   leg CE_H2D          copy engine H0 -> B                              check 1 (B[0, L) against P1)
 *   leg SM_D2H          SMs write P2 into H1                             check 2
 *   legs SM_DUPLEX_*    one launch: SMs read H1 (= check 2, against P2) and write P3 into H0 at once
 *   legs CE_DUPLEX_*    copy engines H0 -> B and A -> H1 at once         check 3 (B against P3), check 4 (H1 against P1)
 *   leg  latency        chase through the host-resident table            check 5 (end slot)
 * An injected fault (test_inject_*) of check 0 sits in H0 and therefore also reaches check 1 (B is copied from H0);
 * one of checks 1 to 4 reaches only that check.
 */
#define CRO_LINK_LEG_CE_D2H         0
#define CRO_LINK_LEG_SM_H2D         1
#define CRO_LINK_LEG_CE_H2D         2
#define CRO_LINK_LEG_SM_D2H         3
#define CRO_LINK_LEG_SM_DUPLEX_H2D  4
#define CRO_LINK_LEG_SM_DUPLEX_D2H  5
#define CRO_LINK_LEG_CE_DUPLEX_H2D  6
#define CRO_LINK_LEG_CE_DUPLEX_D2H  7
#define CRO_LINK_LEGS               8

#define CRO_LINK_CHECK_D2H_COPY        0   /* H0 (CE copy of A) read by the SMs, against P1              */
#define CRO_LINK_CHECK_H2D_COPY        1   /* B[0, L) (CE copy of H0) against P1                         */
#define CRO_LINK_CHECK_SM_WRITE        2   /* H1 (SM stores) read by the duplex launch, against P2       */
#define CRO_LINK_CHECK_DUPLEX_WRITE    3   /* B[0, L) (duplex SM stores to H0, then CE H0 -> B) against P3 */
#define CRO_LINK_CHECK_DUPLEX_D2H_COPY 4   /* H1 (CE copy of A during the CE duplex) read by the SMs, P1 */
#define CRO_LINK_CHECK_CHASE           5   /* the chase ended on the slot the host walk names            */
#define CRO_LINK_CHECKS                6
#define CRO_LINK_WORD_CHECKS           5   /* checks 0..4 compare words                                  */
#define CRO_LINK_NO_FAIL               0xFFFFFFFFu
#define CRO_LINK_RECORDS               CRO_LOCATE_RECORDS   /* word records the device keeps per check     */

/* degraded: reported, never changes the status */
#define CRO_LINK_DEGRADED_SPEED       0x1u  /* the GPU's link runs below its max speed                    */
#define CRO_LINK_DEGRADED_WIDTH       0x2u  /* the GPU's link runs below its max width                    */
#define CRO_LINK_DEGRADED_PATH        0x4u  /* a hop above the GPU runs below its own max speed or width  */
#define CRO_LINK_DEGRADED_BOTTLENECK  0x8u  /* a hop above the GPU is slower (speed x width) than its link */

#define CRO_PCI_MAX_HOPS 8

typedef struct cro_pci_hop {
    char     bdf[16];              /*   0  sysfs spelling "0000:1f:00.0"                                    */
    uint32_t cur_speed;            /*  16  tenths of a GT/s (320 = 32.0 GT/s); 0: "Unknown" or no file       */
    uint32_t cur_width;            /*  20  lanes; 0: no file                                                */
    uint32_t max_speed;            /*  24 */
    uint32_t max_width;            /*  28 */
} cro_pci_hop;                     /* 32 bytes */

typedef struct cro_pci_path {
    int32_t  numa_node;            /*   0  the device's numa_node (-1: none, or no file)                     */
    uint32_t n_hops;               /*   4  entries of hop[]: the device, then each ancestor that is a PCI
                                              function with link files, up to the root bus                     */
    uint32_t bottleneck;           /*   8  index in hop[] of the least cur_speed * cur_width among hops whose
                                              speed and width are known (the lowest such index on a tie; 0 when
                                              none is known)                                                  */
    uint32_t truncated;            /*  12  1: the path had more than CRO_PCI_MAX_HOPS hops                     */
    cro_pci_hop hop[CRO_PCI_MAX_HOPS];   /* 16 */
} cro_pci_path;                    /* 272 bytes */

typedef struct cro_link_opts {
    uint64_t bytes;                /*   0  L: 0 = min(256 MiB, S); else a multiple of 16 with 16 <= L <= S     */
    uint32_t hops;                 /*   8  chase length: 0 = 1024, at most 2^24                                */
    uint32_t ctas;                 /*  12  grid of the SM legs: 0 = the default (DESIGN.md "host link")        */
    /* test only: with test_inject_mask != 0, word test_inject_word of the buffer check test_inject_check (0..4)
       verifies is XORed with the mask after that check's leg and before the check runs */
    int32_t  test_inject_check;    /*  16 */
    uint32_t reserved0;            /*  20 */
    uint64_t test_inject_word;     /*  24 */
    uint64_t test_inject_mask;     /*  32 */
} cro_link_opts;                   /* 40 bytes */

typedef struct cro_link_fault {
    uint32_t check;                /*   0  CRO_LINK_CHECK_*                                                  */
    uint32_t reserved;             /*   4 */
    uint64_t word_index;           /*   8  index in the buffer the check verified (word 0 = its first word)   */
    uint64_t expected;             /*  16 */
    uint64_t actual;               /*  24 */
    uint64_t host_value;           /*  32  word_index of the host buffer involved (see cro_probe_host_link)   */
} cro_link_fault;                  /* 40 bytes */

typedef struct cro_link_leg {
    uint64_t bytes;                /*   0  bytes the leg moved (L)                                           */
    uint64_t ns;                   /*   8  CUDA events around the leg (both duplex SM legs: the one launch)    */
    uint64_t timer_ns;             /*  16  SM legs: the role's own %globaltimer window; 0 for copy engines     */
} cro_link_leg;                    /* 24 bytes */

typedef struct cro_link_check {
    uint64_t words;                /*   0  words compared (L / 8)                                            */
    uint64_t mismatches;           /*   8  exact                                                            */
    uint64_t recorded;             /*  16  mismatches the device recorded (<= CRO_LINK_RECORDS)              */
    uint64_t seed;                 /*  24  pattern the buffer must hold: word i = pattern_word(seed, i)       */
    uint64_t fold_xor;             /*  32  the buffer as read: xor, sum, weighted sum as for a read sweep     */
    uint64_t fold_sum;             /*  40 */
    uint64_t fold_wsum;            /*  48 */
    uint64_t expect_xor;           /*  56  closed form of the pattern over the same words                    */
    uint64_t expect_sum;           /*  64 */
    uint64_t expect_wsum;          /*  72 */
} cro_link_check;                  /* 80 bytes */

typedef struct cro_link_result {
    int32_t  status;               /*   0  the return value                                                  */
    uint32_t first_fail;           /*   4  lowest failing CRO_LINK_CHECK_*, or CRO_LINK_NO_FAIL               */
    uint64_t bytes;                /*   8  L                                                                 */
    uint64_t seed[3];              /*  16  P1, P2, P3: seed_dev + 2^62 + (3k + j) * 0xD1B54A32D192ED03         */
    uint64_t call;                 /*  40  k: the call's number on this device, from 0                       */
    cro_link_leg leg[CRO_LINK_LEGS];   /* 48  CRO_LINK_LEG_*                                                */
    uint64_t ce_duplex_span_ns;    /* 240  first CE duplex start .. last CE duplex end (CUDA events)          */
    cro_link_check check[CRO_LINK_WORD_CHECKS];   /* 248 */
    uint32_t chase_hops;           /* 648 */
    uint32_t chase_end;            /* 652  slot the chase ended on                                         */
    uint32_t chase_expect;         /* 656  slot the host walk of the same permutation ends on               */
    uint32_t chase_minor;          /* 660  the table is the self pair (minor, minor) of cro_chase_end        */
    uint64_t chase_ns;             /* 664  the chase kernel's %globaltimer window                           */
    int32_t  dev_numa;             /* 672  path.numa_node                                                   */
    int32_t  host_numa[3];         /* 676  node the pages of H0, H1, the chase table landed on (first page;
                                              -1: unknown, e.g. a seccomp profile refuses get_mempolicy)       */
    uint32_t no_nvml;              /* 688  1: replay counters not read (CRO_F_NO_NVML, or NVML / the symbol is
                                              missing, or the device refused)                                  */
    uint32_t degraded;             /* 692  CRO_LINK_DEGRADED_*, from path                                     */
    uint64_t replays_before;       /* 696  nvmlDeviceGetPcieReplayCounter before the legs and after them       */
    uint64_t replays_after;        /* 704 */
    cro_pci_path path;             /* 712  sampled while the CE duplex leg was in flight (an idle GPU lowers its
                                              link speed)                                                      */
} cro_link_result;                 /* 984 bytes */

/* faults[0 .. cap) receives the mismatching words (by check, then word index), *n how many were written.
 * host_value is the same index of the host buffer the check involved (H0 for checks 0, 1, 3; H1 for checks 2, 4),
 * read by the CPU once the check ran and before any later leg rewrote that buffer: equal to actual, the corruption
 * reached host memory; equal to expected, it happened on the device side of the transfer.
 * CRO_OK: every check passed; CRO_ERR_CHECKSUM: a check mismatched (a chase that ended on the wrong slot included).
 * dev_index must be an in-process device (as for cro_locate_faults).  opts may be NULL: defaults. */
int  cro_probe_host_link(cro_ctx *ctx, int dev_index, const cro_link_opts *opts,
                         cro_link_result *out, cro_link_fault *faults, int cap, int *n);

/* The same probe of any GPU on the node, run by `croprobe-cli link-raw` (a fresh cuInit that sees only that GPU): the
 * form an operator calls (INTEGRATION.md §2).  It reaches GPUs attached after cro_probe_init, and an uncorrectable error
 * in the memory it uses costs the helper, not the caller's context.  The helper's sweep region is L (256 MiB when
 * opts->bytes is 0, the in-process default of a 4 GiB region), so L <= S always holds; every other option is checked as
 * in process, before any helper starts.  ctx may be NULL; a UUID the node does not list, or one the helper cannot see, is
 * CRO_ERR_NO_DEVICE; a GPU that is also an in-process device of ctx is held under that device's mutex while the helper
 * runs (probes in flight finish first and stay collectable; its sweep region is not touched, so the fault locator's
 * pass 0 still compares both halves).  deadline_ms 0: CRO_HELPER_TIMEOUT_MS; a helper past it is killed
 * (CRO_ERR_DEADLINE).  *helper_ns (may be NULL): the helper's spawn to exit.  The result and faults are what the
 * in-process call on that GPU writes; the seeds come from a base drawn per helper call (ctx's seed_base + (h << 8) for
 * its h-th such call, from 1, or one from the clock without ctx), and call is 0.  Malformed output or a crash:
 * CRO_ERR_EXEC. */
int  cro_probe_host_link_uuid(cro_ctx *ctx, const char *gpu_uuid, const cro_link_opts *opts, int deadline_ms,
                              cro_link_result *out, cro_link_fault *faults, int cap, int *n, uint64_t *helper_ns);

/* The PCIe path of pci_bus_id ("00000000:1F:00.0" or "0000:1f:00.0") under sys_root (NULL: "/sys"), from
 * <sys_root>/bus/pci/devices/<bdf>: current / max link speed and width and numa_node of the device and of every
 * ancestor on its real path that has link files.  Reads sysfs only; no context, no CUDA.  CRO_ERR_INVALID_ARG: a bus
 * id that parses as neither spelling; CRO_ERR_NO_DEVICE: no such device under sys_root. */
int  cro_pci_link_path(const char *sys_root, const char *pci_bus_id, cro_pci_path *out);

/* ---- SM compute: every SM's tensor cores and ALUs against an exact answer ----- */

/*
 * The HBM probe and the host link probe check memory and the PCIe path; nothing there checks that the SMs compute right
 * answers.  The compute probe has every SM compute one answer tile D = A * B (M x N x K below) many times, with its
 * tensor cores (wgmma: s8, bf16, e4m3) and with its CUDA cores (an FFMA chain and an IMAD chain), and compares what it
 * got with the answer the library computed on the host.  A wrong answer is attributed to the SM (%smid) that produced
 * it.  It runs only when called and changes nothing of the probe: it takes the device's mutex, lets probes still in
 * flight finish first (their results stay collectable with cro_probe_end), and never touches the sweep region, so the
 * fault locator's pass 0 still compares both halves afterwards.  It allocates only its own small buffers (the two
 * expected tiles, the per-CTA records and the fault records) and frees them before returning.
 *
 * Operands of call k on a device: seed = seed_dev + 2^61 + k * 0xD1B54A32D192ED03 (seed_dev = seed_base | minor).
 * Element e is byte (e mod 8) of pattern_word(seed, e / 8) (little-endian: byte b is bits 8b..8b+7), with
 *   e = m * 256 + k           for A[m][k]    (0 <= m < M, 0 <= k < K)
 *   e = 32768 + k * 256 + n   for B[k][n]    (0 <= n < N)
 * and two readings of that byte:
 *   s8         the byte as int8_t                                   (legs S8, IMAD:  the "s8 answer")
 *   small-int  (byte & 7) - 4, an integer in -4 .. 3                 (legs BF16, E4M3, FFMA: the "small-int answer")
 * The answer is D[m][n] = sum over k of A[m][k] * B[k][n], exact in any order of accumulation (DESIGN.md "The compute
 * probe"); float legs are compared after cvt.rni.s32.f32.
 *
 * Every CTA (one per SM, 256 threads: two warpgroups of 64 rows each) computes the whole tile `iterations` times.
 * Thread t holds 128 accumulator values, value j (0 <= j < 128) being the element
 *   row = 64 * (t / 128) + 16 * ((t / 32) % 4) + (t % 32) / 4 + 8 * ((j / 2) % 2),   col = 8 * (j / 4) + 2 * (t % 4) + j % 2
 * (the wgmma m64n256 accumulator fragment; the ALU legs use the same mapping).  After each iteration the thread adds
 * fold = sum over j of value_j * (2j + 1) (mod 2^64, values as int32) to a running sum, and at the end compares it with
 * iterations * fold(expected values): a mismatch counts as a fold mismatch.  The last iteration's values are compared
 * element by element with the expected tile: mismatches are counted exactly and recorded while there is room.
 */
#define CRO_COMPUTE_M             128
#define CRO_COMPUTE_N             256
#define CRO_COMPUTE_K             256
#define CRO_COMPUTE_LEG_S8        0       /* wgmma .s32.s8.s8 (IGMMA), s8 answer                      */
#define CRO_COMPUTE_LEG_BF16      1       /* wgmma .f32.bf16.bf16 (HGMMA), small-int answer            */
#define CRO_COMPUTE_LEG_E4M3      2       /* wgmma .f32.e4m3.e4m3 (QGMMA), small-int answer            */
#define CRO_COMPUTE_LEG_FFMA      3       /* FP32 FFMA chain on the CUDA cores, small-int answer        */
#define CRO_COMPUTE_LEG_IMAD      4       /* INT32 IMAD chain on the CUDA cores, s8 answer              */
#define CRO_COMPUTE_LEGS          5
#define CRO_COMPUTE_ALL_LEGS      0x1Fu   /* bit l: leg l                                              */
#define CRO_COMPUTE_ANSWER_S8     0
#define CRO_COMPUTE_ANSWER_SMALL  1
#define CRO_COMPUTE_RECORDS       4096    /* element records the device keeps per leg; counts stay exact beyond */
#define CRO_COMPUTE_MAX_SMS       256     /* SM ids the coverage bitmaps hold; a larger %nsmid fails the call    */
#define CRO_COMPUTE_MAX_ITERATIONS      65536
#define CRO_COMPUTE_MAX_ALU_ITERATIONS  1024
#define CRO_COMPUTE_MAX_ROUNDS    64

#define CRO_COMPUTE_NONE          0u      /* no SM failed                                               */
#define CRO_COMPUTE_SM            1u      /* a strict subset of the covered SMs failed: act on those SMs  */
#define CRO_COMPUTE_ALL           2u      /* every covered SM failed some leg, or a launched CTA did not publish:
                                             a common cause (operands, expected answer, launch), not one SM */

#define CRO_COMPUTE_PERSISTENT    1u      /* cro_compute_sm_leg.mark: the last iteration's answer was wrong */
#define CRO_COMPUTE_INTERMITTENT  2u      /* only the fold was wrong: an earlier iteration, right again by the last */

typedef struct cro_compute_opts {
    uint32_t iterations;           /*   0  tensor legs: 0 = the default (DESIGN.md), at most CRO_COMPUTE_MAX_ITERATIONS  */
    uint32_t alu_iterations;       /*   4  FFMA / IMAD legs: 0 = 4, at most CRO_COMPUTE_MAX_ALU_ITERATIONS              */
    uint32_t legs;                 /*   8  CRO_COMPUTE_ALL_LEGS bits; 0 = all                                            */
    uint32_t max_rounds;           /*  12  launches per leg while fewer than sm_count SMs were seen: 0 = 4               */
    /* test only: with test_inject_mask != 0, in each CTA of leg test_inject_leg whose %smid is test_inject_sm (-1: every
       SM), the mask is XORed into accumulator element (test_inject_row, test_inject_col) (-1: every row / column) after
       iteration test_inject_iteration's answer is complete and before its fold — a software stand-in for a wrong answer */
    int32_t  test_inject_leg;      /*  16 */
    int32_t  test_inject_sm;       /*  20 */
    uint32_t test_inject_iteration;/*  24 */
    int32_t  test_inject_row;      /*  28 */
    int32_t  test_inject_col;      /*  32 */
    uint32_t test_inject_mask;     /*  36 */
} cro_compute_opts;                /*  40 bytes */

typedef struct cro_compute_leg {
    uint32_t iterations;           /*   0  per CTA                                                              */
    uint32_t rounds;               /*   4  launches                                                             */
    uint64_t ops;                  /*   8  2 * M * N * K * iterations per CTA launched, summed                  */
    uint64_t ns;                   /*  16  CUDA events around the launches, summed over rounds                 */
    uint64_t timer_ns;             /*  24  %globaltimer: first CTA start .. last CTA end, summed over rounds    */
    uint32_t sms_covered;          /*  32  distinct SMs that ran a CTA of the leg                              */
    uint32_t complete;             /*  36  1: sms_covered == sm_count                                           */
    uint64_t mismatches;           /*  40  elements of the last iteration's answer that differ, exact          */
    uint64_t fold_mismatches;      /*  48  threads whose running fold differs                                   */
    uint64_t recorded;             /*  56  mismatches the device recorded (<= CRO_COMPUTE_RECORDS)              */
    uint32_t failed_sms;           /*  64  distinct SMs with a mismatch or a fold mismatch                       */
    uint32_t unpublished;          /*  68  CTAs launched that published no record                              */
    uint32_t ctas;                 /*  72  CTAs launched, over all rounds                                      */
    uint32_t slowest_sm;           /*  76  the SM with the most %clock64 cycles per iteration (cycles summed over
                                              its CTAs / (CTAs * iterations), integer division); on a tie the
                                              lowest SM id                                                     */
    uint32_t slow_permille;        /*  80  its cycles per iteration over the median SM's, x 1000, integer division,
                                              capped at 2^32 - 1 (report only).  The median of n SMs is the
                                              (n / 2)-th of their values sorted ascending, from 0: the upper one for
                                              an even n.  0 when the median is 0                               */
    uint32_t reserved;             /*  84 */
    uint64_t fold;                 /*  88  running fold summed over the threads of the CTA on the lowest SM id
                                              (the first such CTA to publish, by round and then by CTA index) */
    uint64_t expect_fold;          /*  96  iterations * the same sum over the expected answer                    */
} cro_compute_leg;                 /* 104 bytes */

typedef struct cro_compute_result {
    int32_t  status;               /*   0  the return value: CRO_OK, or CRO_ERR_CHECKSUM on any mismatch or missing publish */
    uint32_t verdict;              /*   4  CRO_COMPUTE_NONE / _SM / _ALL                                        */
    uint64_t seed;                 /*   8  operand seed of this call                                           */
    uint64_t call;                 /*  16  k: the call's number on this device, from 0                         */
    uint32_t sm_count;             /*  24  multiprocessors the device reports                                   */
    uint32_t legs;                 /*  28  legs run (CRO_COMPUTE_ALL_LEGS bits)                                 */
    uint64_t host_ref_ns;          /*  32  host time to compute both expected answers                          */
    uint32_t nsmid;                /*  40  %nsmid as the kernels read it                                       */
    uint32_t bad_sms;              /*  44  distinct SMs that failed any leg                                     */
    uint16_t bad_sm[16];           /*  48  the first 16 of them, ascending                                     */
    cro_compute_leg leg[CRO_COMPUTE_LEGS];   /*  80 */
} cro_compute_result;              /* 600 bytes */

typedef struct cro_compute_sm_leg {
    uint64_t mismatches;           /*   0 */
    uint64_t fold_mismatches;      /*   8 */
    uint64_t ns;                   /*  16  %globaltimer windows of the leg's CTAs on this SM, summed           */
    uint64_t cycles;               /*  24  %clock64 cycles of the same CTAs, summed                            */
    uint32_t ctas;                 /*  32  CTAs of the leg that ran on this SM (0: not seen in this leg)       */
    uint32_t mark;                 /*  36  0, CRO_COMPUTE_PERSISTENT or CRO_COMPUTE_INTERMITTENT                */
} cro_compute_sm_leg;              /*  40 bytes */

typedef struct cro_compute_sm {
    uint32_t smid;                 /*   0 */
    uint32_t reserved;             /*   4 */
    cro_compute_sm_leg leg[CRO_COMPUTE_LEGS];   /* 8 */
} cro_compute_sm;                  /* 208 bytes */

typedef struct cro_compute_fault {
    uint32_t leg;                  /*   0  CRO_COMPUTE_LEG_*                                                    */
    uint32_t smid;                 /*   4 */
    uint32_t row;                  /*   8 */
    uint32_t col;                  /*  12 */
    int32_t  expected;             /*  16 */
    int32_t  actual;               /*  20  as compared: float legs after cvt.rni.s32.f32                        */
} cro_compute_fault;               /*  24 bytes */

/* sms[0 .. sms_cap) receives one entry per SM seen, by SM id (*n_sms how many were written); faults[0 .. cap) the
 * element records sorted by (leg, smid, row, col) (*n how many).  dev_index must be an in-process device (as for
 * cro_locate_faults).  opts may be NULL: defaults.  Incomplete coverage never changes the status. */
int  cro_probe_compute(cro_ctx *ctx, int dev_index, const cro_compute_opts *opts, cro_compute_result *out,
                       cro_compute_sm *sms, int sms_cap, int *n_sms, cro_compute_fault *faults, int cap, int *n);

/* The same probe of any GPU on the node, run by `croprobe-cli compute-raw` (a fresh cuInit that sees only that GPU):
 * the form an operator calls (INTEGRATION.md §2).  Options are checked as in process, before any helper starts; ctx,
 * deadline_ms, *helper_ns, the seed base and the return codes are as for cro_probe_host_link_uuid (a failed launch:
 * CRO_ERR_CUDA, the helper's status). */
int  cro_probe_compute_uuid(cro_ctx *ctx, const char *gpu_uuid, const cro_compute_opts *opts, int deadline_ms,
                            cro_compute_result *out, cro_compute_sm *sms, int sms_cap, int *n_sms,
                            cro_compute_fault *faults, int cap, int *n, uint64_t *helper_ns);

/* The expected answer the call uploads: answer CRO_COMPUTE_ANSWER_S8 or _SMALL of the operands of `seed`, as
 * CRO_COMPUTE_M * CRO_COMPUTE_N int32 values, row-major.  Host arithmetic only; no context. */
int  cro_compute_expected(int answer, uint64_t seed, int32_t *out);

/* ---- SM precision: every SM's FP64, TF32, FP16 and E5M2 arithmetic against an exact answer, bit for bit ---- */

/*
 * The compute probe checks s8, bf16 and e4m3 tensor cores and FP32 / INT32 CUDA cores, and compares float answers after
 * rounding them to int32.  The precision probe checks the formats it leaves out, one leg each, on every SM: the FP64
 * tensor cores (DMMA) and CUDA cores (DFMA), TF32 and FP16 tensor cores with f32 accumulation, FP16 tensor cores with
 * f16 accumulation, E5M2 tensor cores, and the FP16 CUDA cores (HFMA2).  It is shaped like the compute probe (one CTA
 * per SM, one launch per leg, the same verdicts, marks, coverage rounds and slowest-SM report, and the same guarantees:
 * the device's mutex, probes in flight finish first, the sweep region untouched) but compares tighter: every value
 * must be IEEE-equal to the exact answer encoded in the leg's own type, and the fold adds the value's bit pattern, so
 * a flipped fraction bit fails even where it is worth far less than 0.5.
 *
 * Operands of call k on a device: seed = seed_dev + 2^58 + k * 0xD1B54A32D192ED03.  With the leg's M, N and K, element
 *   e = m * K + k             for A[m][k]
 *   e = M * K + k * N + n     for B[k][n]
 * is read one of three ways:
 *   small-int  (byte & 7) - 4 in -4 .. 3, byte = byte (e mod 8) of pattern_word(seed, e / 8)      (TF32, F16, E5M2)
 *   narrow     (byte & 3) - 2 in -2 .. 1, the same byte                                             (F16ACC, HFMA2)
 *   wide       the low 20 bits of pattern_word(seed, e), sign-extended: -2^19 .. 2^19 - 1          (F64, DFMA)
 * Each answer D[m][n] = sum over k of A[m][k] * B[k][n] is exact in any order of accumulation (DESIGN.md "The precision
 * probe"): small-int partial sums stay within 16 K <= 4096 (exact with 13 significant bits; every operand is exact in
 * tf32, f16 and e5m2), narrow ones within 4 * 256 = 1024 (exact in f16's 11), wide ones within 2^38 * 128 = 2^45
 * (exact in f64's 53).
 *
 * Legs (M x N x K; every CTA has 256 threads and holds the whole tile in shared memory):
 *   F64     mma.sync m16n8k16 .f64 (DMMA)        128 x  64 x 128   wide answer; warp w owns rows 16w .. 16w + 15
 *   DFMA    DFMA chains, the F64 fragment        128 x  64 x 128   wide answer
 *   TF32    wgmma m64n256k8 .f32.tf32 (HGMMA)    128 x 256 x 128   small-int answer at K = 128
 *   F16     wgmma m64n256k16 .f32.f16 (HGMMA)    128 x 256 x 256   small-int answer
 *   F16ACC  wgmma m64n256k16 .f16.f16 (HGMMA)    128 x 256 x 256   narrow answer, f16 accumulators
 *   E5M2    wgmma m64n256k32 .f32.e5m2 (QGMMA)   128 x 256 x 256   small-int answer
 *   HFMA2   HFMA2 chains, f16 accumulators       128 x 256 x 256   narrow answer; (col, col + 1) pairs packed
 * Thread t holds V values (V = 32 for F64 / DFMA, 128 otherwise); value j is the element
 *   row = r0(t) + 8 * ((j / 2) % 2),   col = 8 * (j / 4) + 2 * (t % 4) + j % 2
 * with r0(t) = 16 * (t / 32) + (t % 32) / 4 for F64 / DFMA and 64 * (t / 128) + 16 * ((t / 32) % 4) + (t % 32) / 4
 * otherwise (the mma / wgmma accumulator fragments; the CUDA-core legs use the same mapping).
 *
 * Compare: a value is right when it is IEEE-equal to its expected integer converted to the leg's type (exact for these
 * bounds, so -0 equals 0 and any fraction fails).  Fold: after every iteration the thread adds canon(v) * (2e + 1)
 * (mod 2^64) over its values, with canon(v) the value's bit pattern (64, 32 or 16 bits, zero-extended; -0 taken as 0)
 * and e = row * N + col; at the end it compares the running sum with iterations * the same sum over the expected
 * values.  The fold of a whole CTA is layout-free: the sum over every element of the tile.
 */
#define CRO_PRECISION_LEG_F64       0
#define CRO_PRECISION_LEG_DFMA      1
#define CRO_PRECISION_LEG_TF32      2
#define CRO_PRECISION_LEG_F16       3
#define CRO_PRECISION_LEG_F16ACC    4
#define CRO_PRECISION_LEG_E5M2      5
#define CRO_PRECISION_LEG_HFMA2     6
#define CRO_PRECISION_LEGS          7
#define CRO_PRECISION_ALL_LEGS      0x7Fu   /* bit l: leg l */
#define CRO_PRECISION_ANSWER_WIDE   0       /* 128 x 64, K = 128: F64, DFMA      */
#define CRO_PRECISION_ANSWER_SMALL128 1     /* 128 x 256, K = 128: TF32          */
#define CRO_PRECISION_ANSWER_SMALL  2       /* 128 x 256, K = 256: F16, E5M2     */
#define CRO_PRECISION_ANSWER_NARROW 3       /* 128 x 256, K = 256: F16ACC, HFMA2 */
#define CRO_PRECISION_ANSWERS       4
#define CRO_PRECISION_M             128
#define CRO_PRECISION_N             256     /* F64 / DFMA: CRO_PRECISION_F64_N */
#define CRO_PRECISION_K             256     /* F64 / DFMA / TF32: 128           */
#define CRO_PRECISION_F64_N         64
#define CRO_PRECISION_F64_K         128
#define CRO_PRECISION_TF32_K        128
#define CRO_PRECISION_RECORDS       4096    /* element records the device keeps per leg; counts stay exact beyond */
#define CRO_PRECISION_MAX_SMS       256
#define CRO_PRECISION_MAX_ITERATIONS      65536
#define CRO_PRECISION_MAX_ALU_ITERATIONS  4096
#define CRO_PRECISION_MAX_ROUNDS    64
/* verdicts: CRO_COMPUTE_NONE / _SM / _ALL; marks: CRO_COMPUTE_PERSISTENT / _INTERMITTENT */

typedef struct cro_precision_opts {
    uint32_t iterations;           /*   0  F64, TF32, F16, F16ACC, E5M2: 0 = the default, at most CRO_PRECISION_MAX_ITERATIONS */
    uint32_t alu_iterations;       /*   4  DFMA, HFMA2: 0 = the default, at most CRO_PRECISION_MAX_ALU_ITERATIONS             */
    uint32_t legs;                 /*   8  CRO_PRECISION_ALL_LEGS bits; 0 = all                                                */
    uint32_t max_rounds;           /*  12  launches per leg while fewer than sm_count SMs were seen: 0 = 4                     */
    /* test only: as cro_compute_opts, the mask XORed into the element's own bits (64 for F64 / DFMA, 32 for the f32
       accumulators, 16 for F16ACC / HFMA2; a mask wider than the leg's element is refused) */
    int32_t  test_inject_leg;      /*  16 */
    int32_t  test_inject_sm;       /*  20 */
    uint32_t test_inject_iteration;/*  24 */
    int32_t  test_inject_row;      /*  28 */
    int32_t  test_inject_col;      /*  32 */
    uint32_t reserved;             /*  36 */
    uint64_t test_inject_mask;     /*  40 */
} cro_precision_opts;              /*  48 bytes */

typedef struct cro_precision_result {
    int32_t  status;               /*   0  CRO_OK, or CRO_ERR_CHECKSUM on any mismatch or missing publish       */
    uint32_t verdict;              /*   4  CRO_COMPUTE_NONE / _SM / _ALL                                        */
    uint64_t seed;                 /*   8  operand seed of this call                                           */
    uint64_t call;                 /*  16  k: the call's number on this device, from 0                         */
    uint32_t sm_count;             /*  24 */
    uint32_t legs;                 /*  28  legs run (CRO_PRECISION_ALL_LEGS bits)                               */
    uint64_t host_ref_ns;          /*  32  host time to compute the four expected answers                       */
    uint32_t nsmid;                /*  40 */
    uint32_t bad_sms;              /*  44 */
    uint16_t bad_sm[16];           /*  48 */
    cro_compute_leg leg[CRO_PRECISION_LEGS];   /*  80  ops: 2 * M * N * K * iterations per CTA, the leg's own shape */
} cro_precision_result;            /* 808 bytes */

typedef struct cro_precision_sm {
    uint32_t smid;                 /*   0 */
    uint32_t reserved;             /*   4 */
    cro_compute_sm_leg leg[CRO_PRECISION_LEGS];   /* 8 */
} cro_precision_sm;                /* 288 bytes */

typedef struct cro_precision_fault {
    uint32_t leg;                  /*   0  CRO_PRECISION_LEG_*                                                  */
    uint32_t smid;                 /*   4 */
    uint32_t row;                  /*   8 */
    uint32_t col;                  /*  12 */
    int64_t  expected;             /*  16  the exact answer                                                     */
    uint64_t actual_bits;          /*  24  the accumulator's raw bits (64, 32 or 16 of them, zero-extended)      */
} cro_precision_fault;             /*  32 bytes */

/* As cro_probe_compute: sms one entry per SM seen, faults sorted by (leg, smid, row, col). */
int  cro_probe_precision(cro_ctx *ctx, int dev_index, const cro_precision_opts *opts, cro_precision_result *out,
                         cro_precision_sm *sms, int sms_cap, int *n_sms, cro_precision_fault *faults, int cap, int *n);

/* The same probe of any GPU on the node, run by `croprobe-cli precision-raw`; as cro_probe_compute_uuid. */
int  cro_probe_precision_uuid(cro_ctx *ctx, const char *gpu_uuid, const cro_precision_opts *opts, int deadline_ms,
                              cro_precision_result *out, cro_precision_sm *sms, int sms_cap, int *n_sms,
                              cro_precision_fault *faults, int cap, int *n, uint64_t *helper_ns);

/* The expected answer a call uploads: answer CRO_PRECISION_ANSWER_* of the operands of `seed`, as M * N int64 values
 * (128 x 64 for _WIDE, 128 x 256 otherwise), row-major.  Host arithmetic only; no context. */
int  cro_precision_expected(int answer, uint64_t seed, int64_t *out);

/* ---- whole-HBM scan: every free byte of a GPU's memory, and its DRAM health record ---- */

/*
 * The probe sweeps 2·S bytes (8 GiB by default); the scan tests the memory nobody holds.  It allocates cudaMalloc
 * chunks of CRO_SCAN_CHUNK_BYTES (the last one ragged) until it covers min(max_bytes, free - reserve_bytes) or an
 * allocation fails, runs four elements over ALL chunks each before the next element starts
 *   E0 fill P     E1 compare with P     E2 fill ~P     E3 compare with ~P
 * and frees the chunks on every way out.  Every bit cell is written and read back as 0 and as 1, so a stuck-at bit
 * mismatches in exactly one of the two compare passes (pass 0 = E1, pass 1 = E3), and a write that lands in the wrong
 * place anywhere is seen by the compare that follows.  Reading every location also turns latent weak cells into the
 * ECC and row-remapping events the scan reads from NVML before E0 and after E3.
 *
 * Scan word index: the chunks concatenated in allocation order; chunk k starts at word chunk[k].word0.  Word j holds
 * pattern_word(seed, j) after E0 and its complement after E2.  The seed is opts->seed, or (0) one derived from the
 * clock and reported, so no two calls share a pattern.
 *
 * Two forms.  cro_scan_hbm_uuid is the one an operator calls (INTEGRATION.md "The HBM scan"): the helper process
 * (`croprobe-cli scan-raw`, a fresh cuInit that sees only that GPU) reaches GPUs attached after cro_probe_init, can
 * take nearly all free memory and returns it by exiting, and an uncorrectable ECC error that takes down the CUDA
 * context which touched the memory costs the helper, not the caller's context.  cro_scan_hbm scans beside what this
 * process already holds; it takes the device's mutex and lets probes still in flight finish first (their results
 * stay collectable with cro_probe_end), and never touches the sweep region.
 *
 * status: CRO_ERR_CHECKSUM when a compare pass found a mismatch; CRO_ERR_CUDA when a CUDA call failed during the
 * elements (cuda_error holds the cudaError_t, e.g. cudaErrorECCUncorrectable: the memory faulted; the NVML "after"
 * read still happens and the report is filled as far as the scan got); CRO_ERR_OOM when not one chunk could be
 * allocated (nothing is then allocated at all).  The health bits never change the status: what counts as unhealthy
 * is the caller's call.
 */
#define CRO_SCAN_CHUNK_BYTES      (2ull << 30)
#define CRO_SCAN_RESERVE_BYTES    (1ull << 30)   /* default reserve_bytes                                        */
#define CRO_SCAN_MAX_CHUNKS       128            /* allocation also ends after this many chunks (256 GiB by default) */
#define CRO_SCAN_PASSES           2              /* compare passes: 0 = E1 (pattern), 1 = E3 (complement)          */
#define CRO_SCAN_ELEMENTS         4

/* cro_scan_report.health: reported, never changes the status */
#define CRO_SCAN_HEALTH_ECC_CORRECTED_DURING    0x1u   /* the volatile DRAM corrected count rose during the scan    */
#define CRO_SCAN_HEALTH_ECC_UNCORRECTED_DURING  0x2u   /* the volatile DRAM uncorrected count rose during the scan  */
#define CRO_SCAN_HEALTH_REMAP_PENDING           0x4u   /* a row remap waits for a GPU reset to take effect          */
#define CRO_SCAN_HEALTH_REMAP_FAILURE           0x8u   /* a remap failed: a bank has no spare rows left             */

/* cro_hbm_health.nvml: which reads NVML answered (a field NVML refused stays 0) */
#define CRO_HBM_NVML_ECC_CORRECTED    0x1u   /* nvmlDeviceGetMemoryErrorCounter, corrected, volatile, DRAM      */
#define CRO_HBM_NVML_ECC_UNCORRECTED  0x2u   /* ... uncorrected                                                */
#define CRO_HBM_NVML_REMAP            0x4u   /* nvmlDeviceGetRemappedRows                                       */
#define CRO_HBM_NVML_HISTOGRAM        0x8u   /* nvmlDeviceGetRowRemapperHistogram                               */

typedef struct cro_scan_opts {
    uint64_t max_bytes;            /*   0  0: all free memory but reserve_bytes                                  */
    uint64_t reserve_bytes;        /*   8  free memory left alone: 0 = CRO_SCAN_RESERVE_BYTES                     */
    uint64_t seed;                 /*  16  0: derived from the clock (reported)                                   */
    int32_t  deadline_ms;          /*  24  cro_scan_hbm_uuid: the helper's deadline; 0 = CRO_HELPER_TIMEOUT_MS     */
    uint32_t reserved0;            /*  28  0 */
    /* test only: chunk size (0 = CRO_SCAN_CHUNK_BYTES; a multiple of 16), so a small scan has several chunks */
    uint64_t test_chunk_bytes;     /*  32 */
    /* test only: after E0 and after E2, word = (word & test_force_and) | test_force_or for the scan words
       [test_force_first, test_force_first + test_force_count), split per chunk — a stand-in for stuck cells */
    uint64_t test_force_first;     /*  40 */
    uint64_t test_force_count;     /*  48 */
    uint64_t test_force_and;       /*  56 */
    uint64_t test_force_or;        /*  64 */
} cro_scan_opts;                   /*  72 bytes */

typedef struct cro_hbm_health {
    uint32_t nvml;                 /*   0  CRO_HBM_NVML_* of the reads NVML answered                              */
    uint32_t remap_corrected;      /*   4  rows remapped for corrected errors                                    */
    uint32_t remap_uncorrected;    /*   8  rows remapped for uncorrected errors                                  */
    uint32_t remap_pending;        /*  12  1: a remap waits for a GPU reset                                      */
    uint32_t remap_failure;        /*  16  1: a remap failed                                                     */
    uint32_t histogram[5];         /*  20  banks with max, high, partial, low, no spare rows left (after E3 only) */
    uint64_t ecc_corrected;        /*  40  volatile DRAM ECC counts                                              */
    uint64_t ecc_uncorrected;      /*  48 */
} cro_hbm_health;                  /*  56 bytes */

typedef struct cro_scan_pass {
    uint64_t invert;               /*   0  0 for pass 0 (E1), all ones for pass 1 (E3)                           */
    uint64_t words_scanned;        /*   8 */
    uint64_t mismatches;           /*  16  exact                                                                 */
    uint64_t recorded;             /*  24  mismatches the device recorded (<= CRO_LOCATE_RECORDS)                */
    uint64_t granules;             /*  32  CRO_LOCATE_GRANULE_BYTES granules of the scan with a mismatch          */
    uint64_t bit_flips[64];        /*  40  mismatches with bit b flipped                                         */
} cro_scan_pass;                   /* 552 bytes */

typedef struct cro_scan_chunk {
    uint64_t word0;                /*   0  scan index of the chunk's first word                                  */
    uint64_t bytes;                /*   8 */
    uint64_t fold_xor[2];          /*  16  the chunk as compare pass p read it (xor, sum, wsum as for a read
                                              sweep of pattern seed + word0: weights count from the chunk's start) */
    uint64_t fold_sum[2];          /*  32 */
    uint64_t fold_wsum[2];         /*  48 */
    uint64_t expect_xor;           /*  64  closed form of pattern_word(seed + word0, i) over the chunk (pass 0's;
                                              pass 1 compares against its complement)                           */
    uint64_t expect_sum;           /*  72 */
    uint64_t expect_wsum;          /*  80 */
} cro_scan_chunk;                  /*  88 bytes */

typedef struct cro_scan_report {
    int32_t  status;               /*    0  the return value                                                     */
    int32_t  cuda_error;           /*    4  cudaError_t of the CUDA call that failed during the elements; 0: none  */
    uint32_t health;               /*    8  CRO_SCAN_HEALTH_*                                                    */
    uint32_t complete;             /*   12  1: every mismatch of both passes is in the caller's list, and for each
                                               chunk the listed deltas reproduce its fold minus its closed form    */
    uint64_t seed;                 /*   16 */
    uint64_t total_bytes;          /*   24  the device's memory                                                   */
    uint64_t free_bytes;           /*   32  free when the call started                                            */
    uint64_t held_bytes;           /*   40  this context's sweep region on the device (0 in the helper)           */
    uint64_t covered_bytes;        /*   48  bytes scanned: the chunks' sum                                        */
    uint32_t n_chunks;             /*   56 */
    uint32_t elements_done;        /*   60  elements that completed: 4 for a whole scan                          */
    uint64_t located;              /*   64  distinct words the device recorded over both passes                  */
    uint64_t recorded;             /*   72  words written to the caller's list (*n)                              */
    uint64_t flip_or;              /*   80  OR of every mismatch's actual ^ expected                             */
    uint64_t element_ns[CRO_SCAN_ELEMENTS];   /*   88  CUDA events around each element                       */
    uint64_t alloc_ns;             /*  120  host time to allocate the chunks (and free them)                      */
    uint64_t nvml_ns;              /*  128  host time of both NVML reads                                          */
    uint64_t wall_ns;              /*  136  the whole scan call                                                  */
    uint64_t helper_ns;            /*  144  cro_scan_hbm_uuid: spawn of the helper to its exit; 0 in process      */
    cro_hbm_health before;         /*  152  read before E0 (no histogram)                                       */
    cro_hbm_health after;          /*  208  read after E3, or after the element that failed                      */
    cro_scan_pass pass[CRO_SCAN_PASSES];      /*  264 */
    cro_scan_chunk chunk[CRO_SCAN_MAX_CHUNKS]; /* 1368 */
} cro_scan_report;                 /* 12632 bytes */

/* words[0 .. cap) receives the mismatching words merged by scan index (*n how many): word_index is the scan index,
 * passes bit p that compare pass p saw it, and `reserved` the word's chunk number k (its offset in the chunk is
 * word_index - chunk[k].word0).  Device addresses mean nothing outside the call and are not reported.  opts may be NULL
 * (defaults).  cro_scan_hbm: dev_index is an in-process device.  cro_scan_hbm_uuid: ctx may be NULL; a UUID the node
 * does not list is CRO_ERR_NO_DEVICE; a GPU that is also an in-process device of ctx is held under that device's mutex
 * while the helper runs, so no probe of it runs beside the scan. */
int  cro_scan_hbm(cro_ctx *ctx, int dev_index, const cro_scan_opts *opts,
                  cro_scan_report *out, cro_fault_word *words, int cap, int *n);
int  cro_scan_hbm_uuid(cro_ctx *ctx, const char *gpu_uuid, const cro_scan_opts *opts,
                       cro_scan_report *out, cro_fault_word *words, int cap, int *n);

/* The device's DRAM health record from NVML, as the scan reads it after E3 (with the histogram): no context, no CUDA.
 * CRO_OK whatever NVML answered (out->nvml says which reads it did); CRO_ERR_INVALID_ARG for a NULL argument. */
int  cro_read_hbm_health(const char *gpu_uuid, cro_hbm_health *out);

/* ---- SRAM: every SM's shared memory and the SM-to-SM network, and the SRAM ECC record ---- */

/*
 * The probe, the scan and the compute probe keep operands in shared memory, but only as pseudo-random bytes: a bad cell
 * shows as a wrong fold or a wrong tile, and the compute probe cannot tell a bad SM's arithmetic from its memory.  The
 * SRAM probe writes every shared-memory word it can reach as 0 and as 1, reads it back and names the SM it belongs to.
 *
 * Local leg (CRO_SRAM_SMEM): one CTA per SM with the device's opt-in maximum of dynamic shared memory (bytes_per_sm,
 * 64-bit words w = 0 .. n - 1; thread t of T owns words t, t + T, ...).  Each iteration runs March C- with P(w) =
 * pattern_word(seed, w) and Q(w) = ~P(w):
 *   M0 write P;  M1 ascending: read P, write Q;  M2 ascending: read Q, write P;
 *   M3 descending: read P, write Q;  M4 descending: read Q, write P;  M5 read P
 * with a CTA barrier between elements.  The order holds per word and per thread; between words of different threads
 * it is not enforced.  Every read is compared (mismatches counted exactly per element, recorded while there is room);
 * M5's reads are also folded (xor, sum, sum of v * (2w + 1), over every iteration: xor of the iterations' folds, sums
 * summed) and the library compares each CTA's fold with the closed form.
 *
 * Network leg (CRO_SRAM_DSMEM): clusters of `cluster` CTAs (2, 4 or 8), as many as the device places at once, each CTA
 * with the local leg's shared memory.  The CTA of cluster rank r owns P_r(w) = pattern_word(seed + r * 0xD1B54A32D192ED03,
 * w), so a word read from the wrong peer mismatches.  Each iteration:
 *   D0 write P_r locally;  D1 read every peer's words over the network (mapa + ld.shared::cluster) against its P;
 *   D2 write Q of peer (r + 1) mod C into that peer (st.shared::cluster);  D3 read the own words locally against Q_r
 * with a cluster barrier between elements.  A D1 mismatch is a remote-read fault of (reader, owner); a D3 mismatch a
 * remote-write fault of (writer, owner).  Whether the network path carries ECC or parity is not documented: the
 * compare is end to end either way.
 *
 * Seeds: call k on a device uses seed = seed_dev + 2^60 + 8 * k * 0xD1B54A32D192ED03 (rank r adds r times the
 * stride), so no call passes on what an earlier call left in shared memory.  Each leg is relaunched while fewer than
 * sm_count SMs took part, up to max_rounds launches; short coverage is reported (complete = 0), never an error.  It
 * runs only when called: it takes the device's mutex, lets probes in flight finish first (their results stay
 * collectable) and never touches the sweep region.
 *
 * status: CRO_ERR_CHECKSUM on any mismatch, fold mismatch or CTA that did not publish; CRO_ERR_CUDA when a launch
 * failed (cuda_error holds the cudaError_t, e.g. 214 for an uncorrectable ECC error); CRO_ERR_UNSUPPORTED when the
 * device cannot place one cluster of the asked size.  The NVML SRAM health read before the first leg and after the
 * last never changes the status.
 */
#define CRO_SRAM_SMEM             0       /* leg index: the local march                                     */
#define CRO_SRAM_DSMEM            1       /* leg index: the SM-to-SM network                                */
#define CRO_SRAM_LEGS             2
#define CRO_SRAM_LEG_SMEM         0x1u    /* cro_sram_opts.legs bits                                        */
#define CRO_SRAM_LEG_DSMEM        0x2u
#define CRO_SRAM_ALL_LEGS         0x3u
#define CRO_SRAM_ELEMENTS         6       /* per-element counts: M0 .. M5 (local), D0 .. D3 (network)       */
#define CRO_SRAM_RECORDS          4096    /* word records the device keeps per leg; counts stay exact beyond */
#define CRO_SRAM_MAX_SMS          256     /* SM ids the results hold; a larger %nsmid fails the call         */
#define CRO_SRAM_MAX_ITERATIONS   4096
#define CRO_SRAM_MAX_ROUNDS       64
#define CRO_SRAM_MAX_PAIRS        8       /* network pairs listed in the result                             */

#define CRO_SRAM_NONE             0u      /* nothing failed                                                  */
#define CRO_SRAM_SM               1u      /* a strict subset of the covered SMs failed the local leg          */
#define CRO_SRAM_LINK             2u      /* network faults between SMs that both passed the local leg        */
#define CRO_SRAM_ALL              3u      /* every covered SM failed a leg, or a launched CTA did not publish  */

#define CRO_SRAM_PERSISTENT       1u      /* cro_sram_sm_leg.mark: the last iteration's compare failed         */
#define CRO_SRAM_INTERMITTENT     2u      /* an earlier iteration failed, or only the fold did                 */

#define CRO_SRAM_DIR_LOCAL        0u      /* cro_sram_fault.direction */
#define CRO_SRAM_DIR_READ         1u      /* D1: smid read peer_smid's words */
#define CRO_SRAM_DIR_WRITE        2u      /* D3: peer_smid wrote smid's words */

/* cro_sram_result.health: reported, never changes the status */
#define CRO_SRAM_HEALTH_CORRECTED_DURING    0x1u   /* the volatile SRAM corrected count rose during the call       */
#define CRO_SRAM_HEALTH_UNCORRECTED_DURING  0x2u   /* the volatile SRAM uncorrected count rose during the call     */
#define CRO_SRAM_HEALTH_THRESHOLD_EXCEEDED  0x4u   /* NVML's SRAM error status: the field-diag threshold is exceeded */

/* cro_sram_health.nvml: which reads NVML answered (a field NVML refused stays 0) */
#define CRO_SRAM_NVML_ECC_CORRECTED    0x1u   /* nvmlDeviceGetMemoryErrorCounter, corrected, volatile, SRAM       */
#define CRO_SRAM_NVML_ECC_UNCORRECTED  0x2u   /* ... uncorrected                                                  */
#define CRO_SRAM_NVML_STATUS           0x4u   /* nvmlDeviceGetSramEccErrorStatus (absent from older drivers)       */

typedef struct cro_sram_opts {
    uint32_t legs;                 /*   0  CRO_SRAM_LEG_* bits; 0 = both                                          */
    uint32_t iterations;           /*   4  per CTA, both legs: 0 = the default (DESIGN.md), at most MAX_ITERATIONS */
    uint32_t cluster;              /*   8  network leg: CTAs per cluster, 2, 4 or 8; 0 = 2                        */
    uint32_t max_rounds;           /*  12  launches per leg while fewer than sm_count SMs took part: 0 = 4         */
    int32_t  deadline_ms;          /*  16  cro_probe_sram_uuid: the helper's deadline; 0 = CRO_HELPER_TIMEOUT_MS   */
    /* test only: with test_inject_mask != 0, in each CTA of leg test_inject_leg (CRO_SRAM_SMEM / _DSMEM) whose %smid
       is test_inject_sm (-1: every SM), the mask is XORed into the word test_inject_word (-1: every word) of element
       test_inject_element in iteration test_inject_iteration: local leg, elements 1 .. 5, into the value read before
       the compare; network leg, element 1 into the value D1 read, element 2 into the value D2 writes.  A software
       stand-in for a bad cell: nothing is provoked in the hardware. */
    int32_t  test_inject_leg;      /*  20 */
    int32_t  test_inject_sm;       /*  24 */
    uint32_t test_inject_element;  /*  28 */
    uint32_t test_inject_iteration;/*  32 */
    int32_t  test_inject_word;     /*  36 */
    uint64_t test_inject_mask;     /*  40 */
} cro_sram_opts;                   /*  48 bytes */

typedef struct cro_sram_health {
    uint32_t nvml;                 /*   0  CRO_SRAM_NVML_* of the reads NVML answered                              */
    uint32_t threshold_exceeded;   /*   4  nvmlEccSramErrorStatus_t.bThresholdExceeded (after the last leg only)   */
    uint64_t ecc_corrected;        /*   8  volatile SRAM ECC counts                                               */
    uint64_t ecc_uncorrected;      /*  16 */
} cro_sram_health;                 /*  24 bytes */

typedef struct cro_sram_pair {
    uint16_t from;                 /*   0  the reader (CRO_SRAM_DIR_READ) or the writer (CRO_SRAM_DIR_WRITE)       */
    uint16_t owner;                /*   2  the SM whose shared memory holds the words                             */
    uint32_t direction;            /*   4  CRO_SRAM_DIR_READ / _WRITE                                            */
} cro_sram_pair;                   /*   8 bytes */

typedef struct cro_sram_leg {
    uint32_t iterations;           /*   0  per CTA                                                               */
    uint32_t rounds;               /*   4  launches                                                              */
    uint64_t bytes;                /*   8  shared-memory bytes read and written by the CTAs launched (reads over the
                                              network included)                                                 */
    uint64_t ns;                   /*  16  CUDA events around the launches, summed over rounds                  */
    uint64_t timer_ns;             /*  24  %globaltimer: first CTA start .. last CTA end, summed over rounds     */
    uint32_t sms_covered;          /*  32  distinct SMs that ran a CTA of the leg (network: took part in a cluster) */
    uint32_t complete;             /*  36  1: sms_covered == sm_count                                            */
    uint64_t mismatches[CRO_SRAM_ELEMENTS];   /*  40  per element, exact (local M1 .. M5; network D1, D3)         */
    uint64_t fold_mismatches;      /*  88  local: CTAs whose M5 fold differs from the closed form               */
    uint64_t recorded;             /*  96  mismatches the device recorded (<= CRO_SRAM_RECORDS)                  */
    uint32_t failed_sms;           /* 104  distinct SMs with a mark                                             */
    uint32_t unpublished;          /* 108  CTAs launched that published no record                              */
    uint32_t ctas;                 /* 112  CTAs launched, over all rounds                                       */
    uint32_t cluster;              /* 116  network: CTAs per cluster; 0 for the local leg                      */
    uint64_t fold_xor;             /* 120  local: M5 fold of the CTA on the lowest SM id (the first such CTA to
                                              publish, by round and then by CTA index)                          */
    uint64_t fold_sum;             /* 128 */
    uint64_t fold_wsum;            /* 136 */
    uint64_t expect_xor;           /* 144  local: the closed form every CTA's fold must equal                    */
    uint64_t expect_sum;           /* 152 */
    uint64_t expect_wsum;          /* 160 */
} cro_sram_leg;                    /* 168 bytes */

typedef struct cro_sram_result {
    int32_t  status;               /*   0  the return value                                                      */
    uint32_t verdict;              /*   4  CRO_SRAM_NONE / _SM / _LINK / _ALL                                     */
    uint64_t seed;                 /*   8  seed of this call (rank 0's)                                          */
    uint64_t call;                 /*  16  k: the call's number on this device, from 0                          */
    uint32_t sm_count;             /*  24  multiprocessors the device reports                                    */
    uint32_t legs;                 /*  28  legs run (CRO_SRAM_LEG_* bits)                                        */
    uint32_t nsmid;                /*  32  %nsmid as the kernels read it                                        */
    int32_t  cuda_error;           /*  36  cudaError_t of the launch that failed; 0: none                        */
    uint64_t bytes_per_sm;         /*  40  shared-memory bytes each CTA marches                                  */
    uint32_t health;               /*  48  CRO_SRAM_HEALTH_*                                                    */
    uint32_t bad_sms;              /*  52  distinct SMs that failed the local leg                                */
    uint16_t bad_sm[16];           /*  56  the first 16 of them, ascending                                      */
    uint32_t bad_pairs;            /*  88  distinct network pairs recorded whose SMs both passed the local leg   */
    uint32_t sms_listed;           /*  92  entries written to the caller's per-SM list                          */
    cro_sram_pair bad_pair[CRO_SRAM_MAX_PAIRS];   /*  96  the first of them, by (direction, from, owner)          */
    uint64_t recorded;             /* 160  word records written to the caller's list (*n)                       */
    uint64_t wall_ns;              /* 168  the whole call                                                       */
    uint64_t helper_ns;            /* 176  cro_probe_sram_uuid: spawn of the helper to its exit; 0 in process   */
    cro_sram_health before;        /* 184  read before the first leg                                            */
    cro_sram_health after;         /* 208  read after the last leg (with the threshold flag)                    */
    cro_sram_leg leg[CRO_SRAM_LEGS];         /* 232 */
} cro_sram_result;                 /* 568 bytes */

typedef struct cro_sram_sm_leg {
    uint64_t mismatches[CRO_SRAM_ELEMENTS];   /*   0  compares of this SM's CTAs that failed, per element          */
    uint64_t fold_mismatches;      /*  48 */
    uint64_t ns;                   /*  56  %globaltimer windows of the leg's CTAs on this SM, summed            */
    uint64_t cycles;               /*  64  %clock64 cycles of the same CTAs, summed                             */
    uint32_t ctas;                 /*  72  CTAs of the leg that ran on this SM (0: not seen in this leg)        */
    uint32_t mark;                 /*  76  0, CRO_SRAM_PERSISTENT or CRO_SRAM_INTERMITTENT                      */
} cro_sram_sm_leg;                 /*  80 bytes */

typedef struct cro_sram_sm {
    uint32_t smid;                 /*   0 */
    uint32_t reserved;             /*   4 */
    cro_sram_sm_leg leg[CRO_SRAM_LEGS];      /*   8 */
} cro_sram_sm;                     /* 168 bytes */

typedef struct cro_sram_fault {
    uint32_t leg;                  /*   0  CRO_SRAM_SMEM / _DSMEM                                               */
    uint32_t element;              /*   4  local 1 .. 5 (M1 .. M5); network 1 (D1) or 3 (D3)                     */
    uint32_t iteration;            /*   8 */
    uint32_t smid;                 /*  12  the SM whose compare failed: the local SM, the D1 reader, the D3 owner  */
    uint32_t peer_smid;            /*  16  network: the D1 owner or the D3 writer (from the CTAs' own records);
                                              local: smid                                                      */
    uint32_t direction;            /*  20  CRO_SRAM_DIR_*                                                       */
    uint32_t word;                 /*  24  word offset in the owner's shared memory                             */
    uint32_t reserved;             /*  28 */
    uint64_t expected;             /*  32 */
    uint64_t actual;               /*  40 */
} cro_sram_fault;                  /*  48 bytes */

/* sms[0 .. sms_cap) receives one entry per SM seen, by SM id (*n_sms how many); faults[0 .. cap) the word records
 * sorted by (leg, element, smid, iteration, word) (*n how many).  opts may be NULL: defaults.  cro_probe_sram:
 * dev_index is an in-process device.  cro_probe_sram_uuid runs `croprobe-cli sram-raw` (a fresh cuInit that sees only
 * that GPU): it reaches GPUs attached after cro_probe_init, and an uncorrectable SRAM error, which takes down the CUDA
 * context that hit it, costs the helper, not the caller's context (INTEGRATION.md "The SRAM probe").  ctx may be NULL;
 * a UUID the node does not list is CRO_ERR_NO_DEVICE; a GPU that is also an in-process device of ctx is held under
 * that device's mutex while the helper runs. */
int  cro_probe_sram(cro_ctx *ctx, int dev_index, const cro_sram_opts *opts, cro_sram_result *out,
                    cro_sram_sm *sms, int sms_cap, int *n_sms, cro_sram_fault *faults, int cap, int *n);
int  cro_probe_sram_uuid(cro_ctx *ctx, const char *gpu_uuid, const cro_sram_opts *opts, cro_sram_result *out,
                         cro_sram_sm *sms, int sms_cap, int *n_sms, cro_sram_fault *faults, int cap, int *n);

/* The device's SRAM health record from NVML, as the probe reads it after the last leg (with the threshold flag): no
 * context, no CUDA.  CRO_OK whatever NVML answered (out->nvml says which reads it did); CRO_ERR_INVALID_ARG for a
 * NULL argument. */
int  cro_read_sram_health(const char *gpu_uuid, cro_sram_health *out);

/* ---- L2: the L2 cache, the crossbar between the SMs and its slices, and the L2 atomic units ---- */

/*
 * The probe's sweeps stream through the L2 once under evict-first hints, and no kernel reads back on purpose what
 * another SM wrote, so an L2 or crossbar fault either shows as an HBM fault or not at all.  The L2 probe keeps a buffer
 * of `bytes` (W) resident in the L2 and marches it from SM to SM, then checks the L2's atomic units against answers
 * computed without atomics.
 *
 * March: one CTA per SM (G = sm_count CTAs, forced by the kernel's shared-memory request) over the buffer's 64-bit
 * words, cut into blocks of CRO_L2_BLOCK_BYTES.  Each iteration runs March C- with P(w) = pattern_word(seed, w) and
 * Q(w) = ~P(w):
 *   M0 write P;  M1 ascending: read P, write Q;  M2 ascending: read Q, write P;
 *   M3 descending: read P, write Q;  M4 descending: read Q, write P;  M5 read P
 * and each element is its own launch: the stream orders the elements, no kernel waits for another CTA.  Block b is
 * handled in element e by CTA (b + e * delta) mod G, with delta chosen so that M1 .. M5 of one word run on five
 * different CTAs: every word is written by one CTA and read back by another, through the L2 and the crossbar.  Every
 * access is a 128-bit ld/st.relaxed.gpu with an L2::evict_last cache policy: L1 is bypassed, the persisting-L2
 * set-aside is not touched.  Every read is compared (mismatches counted exactly per element and per CTA, recorded up to
 * CRO_L2_RECORDS a call with the reader's %smid and the CTA that wrote the word); M5's reads are also folded (xor, sum,
 * sum of v * (2w + 1) by global word index) and the CTAs' folds, combined, must equal the closed form once per
 * iteration.  Each CTA publishes a record per launch (the call number, %smid, %globaltimer window, counts); a CTA that
 * did not publish fails the call.
 *
 * Atomics: A1, every CTA j adds (red.add.u64) and xors (red.xor.b64) pattern_word(seed_atomic, j * n + i) into
 * counter i < a1_counters; a checker kernel without atomics recomputes every counter's sum and xor.  A2, for each of
 * a2_counters counters on its own 128-byte line, one warp of every CTA takes atom.add.u32 tickets and stores what it
 * got back; the checker marks each ticket present and counts holes (a duplicate or wrong ticket leaves one), and
 * checks the final value is 32 * G.
 *
 * Seeds: call k on a device uses seed = seed_dev + 2^59 + 2k * 0xD1B54A32D192ED03 for the march and the next stride
 * for the atomics.  Runs only when called: it takes the device's mutex, lets probes in flight finish first (their
 * results stay collectable), allocates its buffers per call and never touches the sweep region.
 *
 * Verdict: a word seen wrong by two or more reader SMs is a line fault (the storage at that offset: the L2 line or the
 * HBM behind it, which the probe cannot tell apart); a word seen wrong by one SM is that reader's fault.  CRO_L2_ALL
 * when a CTA did not publish, every SM that read in an element where a read went wrong saw a wrong word, or the
 * fold failed with every compare passing;
 * else CRO_L2_LINE when there are line faults; else CRO_L2_SM; else CRO_L2_ATOMIC when only A1 or A2 failed.  When
 * more mismatches happened than were recorded (overflow), the line / SM split rests on the records kept; the counts
 * stay exact.  status: CRO_ERR_CHECKSUM for any verdict but CRO_L2_NONE; CRO_ERR_CUDA when a launch failed
 * (cuda_error holds the cudaError_t).  The NVML health read before and after never changes the status.
 */
#define CRO_L2_BLOCK_BYTES        16384u  /* W is a multiple of this                                         */
#define CRO_L2_MIN_BYTES          (1u << 20)
#define CRO_L2_MAX_L2_MULTIPLE    8       /* W is at most 8 times cudaDevAttrL2CacheSize                     */
#define CRO_L2_ELEMENTS           6       /* per-element counts: M0 .. M5                                     */
#define CRO_L2_RECORDS            4096    /* word records a call keeps; counts stay exact beyond             */
#define CRO_L2_MAX_SMS            256     /* SM ids the results hold; a larger %nsmid fails the call          */
#define CRO_L2_MAX_ITERATIONS     256
#define CRO_L2_MAX_A1_COUNTERS    (1u << 20)
#define CRO_L2_MAX_A2_COUNTERS    8192
#define CRO_L2_MAX_LINES          8       /* line offsets listed in the result                               */
#define CRO_L2_MAX_COUNTERS       8       /* bad counters listed per atomic leg                              */

#define CRO_L2_MARCH              0       /* cro_l2_opts.test_inject_leg */
#define CRO_L2_A1                 1
#define CRO_L2_A2                 2

#define CRO_L2_NONE               0u      /* nothing failed                                                  */
#define CRO_L2_SM                 1u      /* a strict subset of the covered SMs read words wrong, no line fault */
#define CRO_L2_LINE               2u      /* words seen wrong by two or more SMs                              */
#define CRO_L2_ATOMIC             3u      /* only A1 or A2 failed                                             */
#define CRO_L2_ALL                4u      /* a CTA did not publish, every reader of a failing element failed, or only the fold did */

#define CRO_L2_PERSISTENT         1u      /* cro_l2_sm.mark: the SM's compares failed in the last iteration    */
#define CRO_L2_INTERMITTENT       2u      /* ... only in an earlier one                                        */

/* cro_l2_result.health: reported, never changes the status */
#define CRO_L2_HEALTH_SRAM_CORRECTED_DURING    0x1u   /* volatile SRAM corrected count rose during the call          */
#define CRO_L2_HEALTH_SRAM_UNCORRECTED_DURING  0x2u
#define CRO_L2_HEALTH_L2_CORRECTED_DURING      0x4u   /* volatile L2 corrected count rose (NVML may never answer)    */
#define CRO_L2_HEALTH_L2_UNCORRECTED_DURING    0x8u
#define CRO_L2_HEALTH_THRESHOLD_EXCEEDED       0x10u  /* NVML's SRAM error status: the field-diag threshold           */
#define CRO_L2_HEALTH_L2_BUCKET                0x20u  /* ... and its aggregate uncorrectable L2 bucket is not 0       */

/* cro_l2_health.nvml: which reads NVML answered (a field NVML refused stays 0) */
#define CRO_L2_NVML_SRAM_CORRECTED    0x1u    /* nvmlDeviceGetMemoryErrorCounter, volatile, SRAM (location 7)     */
#define CRO_L2_NVML_SRAM_UNCORRECTED  0x2u
#define CRO_L2_NVML_L2_CORRECTED      0x4u    /* ... L2 cache (location 1)                                        */
#define CRO_L2_NVML_L2_UNCORRECTED    0x8u
#define CRO_L2_NVML_STATUS            0x10u   /* nvmlDeviceGetSramEccErrorStatus (absent from older drivers)       */

typedef struct cro_l2_opts {
    uint64_t bytes;                /*   0  W: 0 = the default (DESIGN.md), else a multiple of CRO_L2_BLOCK_BYTES in
                                              [CRO_L2_MIN_BYTES, 8 * the device's L2 size]                       */
    uint32_t iterations;           /*   8  0 = the default, at most CRO_L2_MAX_ITERATIONS                          */
    uint32_t a1_counters;          /*  12  0 = 65536, at most CRO_L2_MAX_A1_COUNTERS                               */
    uint32_t a2_counters;          /*  16  0 = 1024, at most CRO_L2_MAX_A2_COUNTERS                                */
    int32_t  deadline_ms;          /*  20  cro_probe_l2_uuid: the helper's deadline; 0 = CRO_HELPER_TIMEOUT_MS.
                                              cro_probe_l2 waits for the stream as every in-process probe does
                                              (cro_opts.deadline_ms) and refuses a value other than 0          */
    /* test only: with test_inject_mask != 0.  Leg CRO_L2_MARCH: in each CTA whose %smid is test_inject_sm (-1: every
       SM), the mask is XORed into the value read of word test_inject_word (-1: every word) in element
       test_inject_element (1 .. 5; -1: every reading element) of iteration test_inject_iteration.  CRO_L2_A1: CTA 0's
       contribution to counter test_inject_word is XORed with the mask.  CRO_L2_A2: the ticket lane 0 of CTA 0 stores
       for counter test_inject_word is XORed with the mask's low 32 bits (a mask whose low 32 bits are 0 is refused).
       A software stand-in: nothing is provoked in the hardware. */
    int32_t  test_inject_leg;      /*  24 */
    int32_t  test_inject_sm;       /*  28 */
    int32_t  test_inject_element;  /*  32 */
    uint32_t test_inject_iteration;/*  36 */
    int64_t  test_inject_word;     /*  40 */
    uint64_t test_inject_mask;     /*  48 */
} cro_l2_opts;                     /*  56 bytes */

typedef struct cro_l2_health {
    uint32_t nvml;                 /*   0  CRO_L2_NVML_* of the reads NVML answered                               */
    uint32_t threshold_exceeded;   /*   4  nvmlEccSramErrorStatus_t.bThresholdExceeded (after the call only)       */
    uint64_t sram_corrected;       /*   8  volatile SRAM ECC counts                                               */
    uint64_t sram_uncorrected;     /*  16 */
    uint64_t l2_corrected;         /*  24  volatile L2 ECC counts                                                 */
    uint64_t l2_uncorrected;       /*  32 */
    uint64_t unc_bucket_l2;        /*  40  nvmlEccSramErrorStatus_t.aggregateUncBucketL2 (after the call only)     */
} cro_l2_health;                   /*  48 bytes */

typedef struct cro_l2_result {
    int32_t  status;               /*   0  the return value                                                      */
    uint32_t verdict;              /*   4  CRO_L2_NONE / _SM / _LINE / _ATOMIC / _ALL                            */
    uint64_t seed;                 /*   8  the march's seed                                                      */
    uint64_t seed_atomic;          /*  16  A1's seed                                                             */
    uint64_t call;                 /*  24  k: the call's number on this device, from 0                          */
    uint64_t bytes;                /*  32  W                                                                     */
    uint32_t sm_count;             /*  40  multiprocessors the device reports                                    */
    uint32_t nsmid;                /*  44  %nsmid as the kernels read it                                        */
    uint32_t ctas;                 /*  48  G: CTAs per launch                                                    */
    uint32_t blocks;               /*  52  W / CRO_L2_BLOCK_BYTES                                                */
    uint32_t delta;                /*  56  the rotation step between elements                                    */
    uint32_t iterations;           /*  60 */
    int32_t  cuda_error;           /*  64  cudaError_t of the launch that failed; 0: none                        */
    uint32_t health;               /*  68  CRO_L2_HEALTH_*                                                      */
    uint32_t sms_covered;          /*  72  distinct SMs that read words of the buffer (a CTA that owns no block in
                                              an element reads nothing there)                                  */
    uint32_t unpublished;          /*  76  march CTAs (over all launches) and checker CTAs that published nothing */
    uint64_t mismatches[CRO_L2_ELEMENTS];    /*  80  per element, exact                                         */
    uint64_t recorded;             /* 128  word records written to the caller's list (*n)                       */
    uint32_t overflow;             /* 136  1: more mismatches than the device kept records of                   */
    uint32_t sms_listed;           /* 140  entries written to the caller's per-SM list                          */
    uint32_t bad_sms;              /* 144  distinct SMs with a word only they saw wrong                         */
    uint32_t bad_lines;            /* 148  distinct words seen wrong by two or more SMs                          */
    uint16_t bad_sm[16];           /* 152  the first 16 bad SMs, ascending                                      */
    uint64_t bad_line[CRO_L2_MAX_LINES];     /* 184  byte offsets of the first line faults in this call's buffer   */
    uint64_t fold_xor;             /* 248  M5 fold of every CTA over every iteration                             */
    uint64_t fold_sum;             /* 256 */
    uint64_t fold_wsum;            /* 264 */
    uint64_t expect_xor;           /* 272  iterations x the closed form of pattern_word(seed, 0 .. W / 8)         */
    uint64_t expect_sum;           /* 280 */
    uint64_t expect_wsum;          /* 288 */
    uint32_t fold_ok;              /* 296  1: the fold equals the closed form                                   */
    uint32_t a1_counters;          /* 300 */
    uint32_t a2_counters;          /* 304 */
    uint32_t a2_tickets;           /* 308  32 * G: what every A2 counter must end at                             */
    uint64_t a1_bad;               /* 312  A1 counters whose sum or xor differs                                  */
    uint64_t a2_holes;             /* 320  tickets missing over all A2 counters                                  */
    uint64_t a2_bad;               /* 328  A2 counters with a hole or a wrong final value                        */
    uint32_t a1_bad_counter[CRO_L2_MAX_COUNTERS];   /* 336  the first of them, ascending                          */
    uint32_t a2_bad_counter[CRO_L2_MAX_COUNTERS];   /* 368 */
    uint64_t element_ns[CRO_L2_ELEMENTS];    /* 400  %globaltimer: first CTA start .. last CTA end, per element,
                                                       summed over iterations                                 */
    uint64_t march_ns;             /* 448  CUDA events around the march's launches                               */
    uint64_t march_bytes;          /* 456  bytes read and written by the march                                   */
    uint64_t a1_ns;                /* 464  CUDA events: A1's kernel, its checker, A2's kernel, its checker         */
    uint64_t a1_check_ns;          /* 472 */
    uint64_t a2_ns;                /* 480 */
    uint64_t a2_check_ns;          /* 488 */
    uint64_t l2_bytes;             /* 496  cudaDevAttrL2CacheSize                                                */
    uint64_t wall_ns;              /* 504  the whole call                                                       */
    uint64_t helper_ns;            /* 512  0 in process                                                         */
    cro_l2_health before;          /* 520  read before the first launch                                         */
    cro_l2_health after;           /* 568  read after the last (with the SRAM error status)                      */
} cro_l2_result;                   /* 616 bytes */

typedef struct cro_l2_sm {
    uint32_t smid;                 /*   0 */
    uint32_t mark;                 /*   4  0, CRO_L2_PERSISTENT or CRO_L2_INTERMITTENT (bad SMs only)           */
    uint32_t launches;             /*   8  march CTAs that ran on this SM                                       */
    uint32_t reserved;             /*  12 */
    uint64_t mismatches[CRO_L2_ELEMENTS];    /*  16  reads this SM saw wrong, per element                       */
    uint64_t last;                 /*  64  ... of them in the last iteration                                    */
    uint64_t words_read[CRO_L2_ELEMENTS];    /*  72  words this SM read, per element, by the rotation              */
    uint64_t ns;                   /* 120  %globaltimer windows of its CTAs, summed                             */
} cro_l2_sm;                       /* 128 bytes */

typedef struct cro_l2_fault {
    uint32_t element;              /*   0  1 .. 5 */
    uint32_t iteration;            /*   4 */
    uint32_t smid;                 /*   8  the reader                                                           */
    uint32_t cta;                  /*  12  the reader's CTA                                                      */
    uint32_t writer_cta;           /*  16  the CTA that wrote the word in the element before                     */
    uint32_t writer_smid;          /*  20  its SM, from its published record (0xFFFFFFFF: it did not publish)    */
    uint64_t word;                 /*  24  word index in this call's buffer (byte offset / 8)                    */
    uint64_t expected;             /*  32 */
    uint64_t actual;               /*  40 */
    uint32_t line;                 /*  48  1: the word was seen wrong by two or more SMs                         */
    uint32_t reserved;             /*  52 */
} cro_l2_fault;                    /*  56 bytes */

/* sms[0 .. sms_cap) receives one entry per SM seen, by SM id (*n_sms how many); faults[0 .. cap) the word records
 * sorted by (word, iteration, element) (*n how many).  opts may be NULL: defaults.  cro_probe_l2: dev_index is an
 * in-process device.  cro_probe_l2_uuid runs `croprobe-cli l2-raw` (a fresh cuInit that sees only that GPU), so it
 * reaches GPUs attached after cro_probe_init; ctx may be NULL; a UUID the node does not list is CRO_ERR_NO_DEVICE; a
 * GPU that is also an in-process device of ctx is held under that device's mutex while the helper runs.  Every helper
 * call gets a fresh cro_opts.seed_base (the context's seed_base + (h << 8) for its h-th helper call, or one from the
 * clock without a context), so its call 0 uses seeds no earlier call used.  Options are refused before any spawn with
 * the in-process error text, all but W's upper bound, which needs the device and which the helper checks. */
int  cro_probe_l2(cro_ctx *ctx, int dev_index, const cro_l2_opts *opts, cro_l2_result *out,
                  cro_l2_sm *sms, int sms_cap, int *n_sms, cro_l2_fault *faults, int cap, int *n);
int  cro_probe_l2_uuid(cro_ctx *ctx, const char *gpu_uuid, const cro_l2_opts *opts, cro_l2_result *out,
                       cro_l2_sm *sms, int sms_cap, int *n_sms, cro_l2_fault *faults, int cap, int *n);

/* The device's SRAM and L2 health record from NVML, as the probe reads it after the call (with the SRAM error
 * status): no context, no CUDA.  CRO_OK whatever NVML answered; CRO_ERR_INVALID_ARG for a NULL argument. */
int  cro_read_l2_health(const char *gpu_uuid, cro_l2_health *out);

/* Test hook: the probe's classification, a pure function.  Reads from *r unpublished, fold_ok, mismatches[5], a1_bad
 * and a2_bad; from sms[] smid, mismatches, last and words_read; and
 * the records faults[0 .. n) (element, iteration, smid, word).  Writes r's verdict, status, bad_sms, bad_sm,
 * bad_lines and bad_line, each sms[].mark and each faults[].line, as cro_probe_l2 does. */
int  cro_selftest_l2_classify(cro_l2_result *r, cro_l2_sm *sms, int n_sms, cro_l2_fault *faults, int n);

/* What one CTA of a compute or precision leg publishes at the end of a round. */
typedef struct cro_sm_cta {
    uint64_t stamp;                /*   0  the call number k; any other value: the CTA did not publish            */
    uint64_t t0, t1;               /*   8  %globaltimer around the iterations                                     */
    uint64_t cycles;               /*  24  %clock64 around the iterations                                         */
    uint64_t mismatches;           /*  32  elements of the last iteration that differ                             */
    uint64_t fold_mismatches;      /*  40  threads whose running fold differs                                     */
    uint64_t fold;                 /*  48  every thread's running fold, summed                                    */
    uint32_t smid;                 /*  56 */
    uint32_t nsmid;                /*  60 */
} cro_sm_cta;                      /*  64 bytes */

#define CRO_SM_LEGS_COMPUTE       0   /* cro_selftest_sm_legs_classify: the compute probe   */
#define CRO_SM_LEGS_PRECISION     1   /* ... the precision probe                           */

/* Test hook: the compute (probe CRO_SM_LEGS_COMPUTE: out a cro_compute_result, sms cro_compute_sm, records and faults
 * cro_compute_fault) or precision probe's (CRO_SM_LEGS_PRECISION: the cro_precision_* types) classification of call
 * `call` on a device of `grid` SMs, from caller-given rounds instead of launches.  legs: the legs that ran (0: all).
 * Per leg l of them: iterations[l] (>= 1) per CTA, rounds[l] rounds, each of `grid` records of ctas and of the
 * CRO_COMPUTE_MAX_SMS / 64 words of sm_bits (the leg's coverage bitmap after that round), and claims[l] record claims,
 * of which the first min(claims[l], CRO_COMPUTE_RECORDS) are in `records`; ctas, sm_bits and records run in leg order.
 * Every array is indexed by leg (CRO_COMPUTE_LEGS or CRO_PRECISION_LEGS entries).  Writes out, sms[0 .. sms_cap) and
 * faults[0 .. cap) (*n_sms, *n how many) exactly as the in-process call does, all but what needs the device: seed,
 * host_ref_ns, ns and expect_fold stay 0, and rounds is rounds[l].  Returns out->status (CRO_ERR_UNSUPPORTED with a
 * blanked result for a %nsmid above CRO_COMPUTE_MAX_SMS), or CRO_ERR_INVALID_ARG for a NULL array it needs, a negative
 * cap, grid 0, an unknown probe or leg, or a leg of 0 iterations. */
int  cro_selftest_sm_legs_classify(int probe, uint32_t legs, const uint32_t *iterations, uint32_t grid, uint64_t call,
                                   const uint32_t *rounds, const cro_sm_cta *ctas, const uint64_t *sm_bits,
                                   const uint64_t *claims, const void *records, void *out, void *sms, int sms_cap,
                                   int *n_sms, void *faults, int cap, int *n);

/* What one CTA of an SRAM leg publishes at the end of a round, and one word record of a leg. */
typedef struct cro_sram_cta {
    uint64_t stamp;                /*   0  the call number k; any other value: the CTA did not publish            */
    uint64_t t0, t1;               /*   8  %globaltimer around the iterations                                     */
    uint64_t cycles;               /*  24  %clock64 around the iterations                                         */
    uint64_t count[CRO_SRAM_ELEMENTS];   /*  32  compares that failed, per element                              */
    uint64_t last;                 /*  80  ... of them in the last iteration                                      */
    uint64_t fold_x, fold_s, fold_w;     /*  88  local: the M5 fold over every iteration                        */
    uint32_t smid;                 /* 112 */
    uint32_t nsmid;                /* 116 */
    uint32_t rank;                 /* 120  rank in the cluster (0 for the local leg)                              */
    uint32_t block;                /* 124  blockIdx.x                                                             */
} cro_sram_cta;                    /* 128 bytes */

typedef struct cro_sram_record {
    uint32_t element;              /*   0  local 1 .. 5; network 1 (D1) or 3 (D3)                                 */
    uint32_t iteration;            /*   4 */
    uint32_t smid;                 /*   8  the CTA whose compare failed                                           */
    uint32_t peer_block;           /*  12  network: blockIdx.x of the owner (D1) or the writer (D3)               */
    uint32_t round;                /*  16  the launch's round, whose CTA records resolve peer_block               */
    uint32_t word;                 /*  20 */
    uint64_t expected;             /*  24 */
    uint64_t actual;               /*  32 */
} cro_sram_record;                 /*  40 bytes */

/* Test hook: the SRAM probe's classification of call `call` (seed `seed`, n_words words per CTA, `iterations` per CTA,
 * network clusters of `cluster`) on a device of sm_count SMs, from caller-given rounds instead of launches.  legs: the
 * CRO_SRAM_LEG_* bits that ran (0: both).  Per leg l of them: rounds[l] rounds of sm_count (local) or net_grid
 * (network) records of ctas, and claims[l] record claims, of which the first min(claims[l], CRO_SRAM_RECORDS) are in
 * `records`; ctas and records run in leg order.  The local fold is checked against the library's own closed form.
 * Writes out, sms[0 .. sms_cap) and faults[0 .. cap) (*n_sms, *n, out->sms_listed, out->recorded) exactly as
 * cro_probe_sram does, all but what needs the device: ns, wall_ns, health, before and after stay 0, and rounds is
 * rounds[l].  Returns out->status (CRO_ERR_UNSUPPORTED with a blanked result for a %nsmid above CRO_SRAM_MAX_SMS), or
 * CRO_ERR_INVALID_ARG for a NULL array it needs, a negative cap, sm_count 0, a network leg of grid 0 or a grid that is
 * not whole clusters, legs outside CRO_SRAM_ALL_LEGS, a cluster other than 2, 4 or 8, or iterations 0 or above
 * CRO_SRAM_MAX_ITERATIONS. */
int  cro_selftest_sram_classify(uint32_t legs, uint32_t iterations, uint32_t n_words, uint64_t seed, uint32_t cluster,
                                uint32_t sm_count, uint32_t net_grid, uint64_t call, const uint32_t *rounds,
                                const cro_sram_cta *ctas, const uint64_t *claims, const cro_sram_record *records,
                                cro_sram_result *out, cro_sram_sm *sms, int sms_cap, int *n_sms, cro_sram_fault *faults,
                                int cap, int *n);

/* ---- emit: encoding/json-compatible writers ------------------------------ */

/* ComposableResourceStatus (api/v1alpha1/composableresource_types.go:36-41):
 * {"state":..,"error":..,"device_id":..,"cdi_device_id":..} with Go omitempty
 * rules; bytes identical to json.Marshal. */
int  cro_emit_status_json(const char *state, const char *error, const char *device_id,
                          const char *cdi_device_id, char *buf, size_t cap, size_t *len);

/* ScalarResourceStatus (api/v1alpha1/composabilityrequest_types.go:74-80). */
int  cro_emit_scalar_status_json(const char *state, const char *device_id,
                                 const char *cdi_device_id, const char *node_name,
                                 const char *error, char *buf, size_t cap, size_t *len);

/* FM ScaleUpBody / ScaleDownBody (internal/cdi/fti/fm/api/scale_up.go:19-41,
 * scale_down.go:19-41; built at fti/fm/client.go:115-144, :240-271). */
int  cro_emit_fm_scale_up(const char *tenant_uuid, const char *mach_uuid, const char *res_type,
                          const char *model, char *buf, size_t cap, size_t *len);
int  cro_emit_fm_scale_down(const char *tenant_uuid, const char *mach_uuid, const char *res_type,
                            const char *res_uuid, char *buf, size_t cap, size_t *len);
/* CM resize bodies (internal/cdi/fti/cm/client.go:62-79, :133-139, :211-218). */
int  cro_emit_cm_scale_up(const char *spec_uuid, int device_count,
                          char *buf, size_t cap, size_t *len);
int  cro_emit_cm_scale_down(const char *spec_uuid, int device_count, const char *device_id,
                            char *buf, size_t cap, size_t *len);
/* Sunfish CompositionRequest (internal/cdi/sunfish/client.go:48-61, :78). */
int  cro_emit_sunfish_request(const char *name, long long count, const char *proc_type,
                              const char *model, char *buf, size_t cap, size_t *len);

/* Additive probe annotations (cohdi.io/probe-*), a Go-marshalled
 * map[string]string (keys sorted).  Never mixed into the status bytes. */
int  cro_emit_probe_annotations_json(const cro_probe_result *r, char *buf, size_t cap, size_t *len);

/* Additive fault annotations (cohdi.io/probe-fault-*) of a cro_locate_faults report, the same Go-marshalled map:
 * -verdict ("none" | "unclassified" | "not-reproduced" | "persistent", from the report's per-pass counts),
 * -mismatches and -granules ("<pass>:<count>" per pass run, comma-separated), -bits (flipped bit positions,
 * ascending; only when a bit flipped) and -words (the first 8 of words[0 .. n) as "<index hex>:<flip mask hex16>";
 * only when n > 0). */
int  cro_emit_fault_annotations_json(const cro_fault_report *report, const cro_fault_word *words, int n,
                                     char *buf, size_t cap, size_t *len);

/* Additive host-link annotations (cohdi.io/probe-link-*) of a cro_probe_host_link result, the same Go-marshalled map,
 * integers and fixed spellings only (MB/s = bytes * 1000 / ns, integer division; 0 when ns is 0):
 * -verdict ("ok" | "corrupt:<check>" with <check> one of d2h-copy, h2d-copy, sm-write, duplex-write, duplex-d2h-copy,
 * chase | "error" for a call that failed otherwise), -h2d-mbps and -d2h-mbps (copy-engine legs), -duplex-mbps (both
 * copy-engine duplex legs' bytes over their span), -sm-h2d-mbps and -sm-d2h-mbps, -latency-ns (chase ns / hops),
 * -link ("<cur speed> x<cur width> / <max speed> x<max width>" of the GPU, a speed as "32.0GT/s" or "unknown"),
 * and only when they apply: -bottleneck ("<bdf> <speed> x<width>", with CRO_LINK_DEGRADED_BOTTLENECK), -degraded (the
 * flags' names speed, width, path, bottleneck, comma-separated) and -replays (the counter delta, when NVML answered). */
int  cro_emit_link_annotations_json(const cro_link_result *r, char *buf, size_t cap, size_t *len);

/* Additive compute annotations (cohdi.io/probe-compute-*) of a cro_probe_compute result, the same Go-marshalled map,
 * integers and fixed spellings only: -verdict ("ok" for CRO_OK; "sm" or "all" for CRO_ERR_CHECKSUM with that verdict;
 * "error" otherwise), -sms ("<covered>/<sm_count>", the least sms_covered over the legs run), -bad-sms (bad_sm[0 ..
 * min(bad_sms, 16)) ascending, comma-separated; only when bad_sms > 0), -failed-legs (s8, bf16, e4m3, ffma, imad of
 * the legs with a mismatch, a fold mismatch or an unpublished CTA, comma-separated; only when there are any),
 * -s8-gops, -bf16-gflops, -e4m3-gflops (ops / ns, integer division; 0 when ns is 0) and -slowest-sm ("<id>
 * <permille>" of the leg run with the largest slow_permille, the lowest leg on a tie). */
int  cro_emit_compute_annotations_json(const cro_compute_result *r, char *buf, size_t cap, size_t *len);

/* Additive precision annotations (cohdi.io/probe-precision-*) of a cro_probe_precision result, spelled as the compute
 * probe's: -verdict, -sms, -bad-sms, -failed-legs (f64, dfma, tf32, f16, f16acc, e5m2, hfma2), -f64-gflops,
 * -tf32-gflops, -f16-gflops, -f16acc-gflops, -e5m2-gflops (ops / ns, integer division; 0 when ns is 0) and -slowest-sm. */
int  cro_emit_precision_annotations_json(const cro_precision_result *r, char *buf, size_t cap, size_t *len);

/* Additive HBM scan annotations (cohdi.io/hbm-scan-*) of a cro_scan_hbm / cro_scan_hbm_uuid report, the same
 * Go-marshalled map, integers and fixed spellings only: -verdict ("ok" for CRO_OK, "corrupt" for CRO_ERR_CHECKSUM,
 * "cuda-error:<cuda_error>" for CRO_ERR_CUDA, "error" otherwise), -covered-bytes, -free-bytes, -seed (hex16),
 * -mismatches ("<pass 0>,<pass 1>") and -granules (the same), -gbs (4 * covered_bytes over the elements' summed ns, in
 * GB/s, integer division; 0 when that is 0), -bits (flipped bit positions, ascending; only when a bit flipped),
 * -health (the flags' names ecc-corrected, ecc-uncorrected, remap-pending, remap-failure, comma-separated; only when
 * any is set), and only when NVML answered the read: -ecc-corrected and -ecc-uncorrected (the deltas, after -
 * before, when both reads answered), -remapped ("<corrected>,<uncorrected>" rows after E3) and -remap-histogram ("max,
 * high, partial, low, none" without spaces). */
int  cro_emit_scan_annotations_json(const cro_scan_report *r, char *buf, size_t cap, size_t *len);

/* Additive SRAM annotations (cohdi.io/probe-sram-*) of a cro_probe_sram / cro_probe_sram_uuid result, the same
 * Go-marshalled map, integers and fixed spellings only: -verdict ("ok" for CRO_OK; "sm", "link" or "all" for
 * CRO_ERR_CHECKSUM with that verdict; "cuda-error:<cuda_error>" for CRO_ERR_CUDA; "error" otherwise), -sms
 * ("<covered>/<sm_count>", the least sms_covered over the legs run), -bad-sms (bad_sm[0 .. min(bad_sms, 16)),
 * comma-separated; only when bad_sms > 0), -bad-pairs (bad_pair[0 .. min(bad_pairs, 8)) as "<from>-<owner>:<r|w>",
 * comma-separated; only when bad_pairs > 0), -bytes-per-sm, -health (the flags' names corrected, uncorrected,
 * threshold-exceeded, comma-separated; only when any is set), and -ecc-corrected and -ecc-uncorrected (the deltas,
 * after - before; only when both reads answered). */
int  cro_emit_sram_annotations_json(const cro_sram_result *r, char *buf, size_t cap, size_t *len);

/* Additive L2 annotations (cohdi.io/probe-l2-*) of a cro_probe_l2 result, the same Go-marshalled map, integers and
 * fixed spellings only: -verdict ("ok" for CRO_OK; "sm", "line", "atomic" or "all" for CRO_ERR_CHECKSUM with that
 * verdict; "cuda-error:<cuda_error>" for CRO_ERR_CUDA; "error" otherwise), -sms ("<sms_covered>/<sm_count>"), -bytes,
 * -iterations, -march-gbs (march_bytes / march_ns, integer division; 0 when march_ns is 0), and only when they apply:
 * -bad-sms (bad_sm[0 .. min(bad_sms, 16)), comma-separated), -bad-lines (bad_line[0 .. min(bad_lines, 8)), decimal
 * byte offsets, comma-separated), -a1-bad-counters and -a2-bad-counters (the listed counters, at most 8, comma-
 * separated; when a1_bad / a2_bad > 0), -a2-holes (when a2_holes > 0), -overflow ("1"), -health (the flags' names
 * sram-corrected, sram-uncorrected, l2-corrected, l2-uncorrected, threshold-exceeded, l2-bucket, comma-separated). */
int  cro_emit_l2_annotations_json(const cro_l2_result *r, char *buf, size_t cap, size_t *len);

/* (deviceID, CDIDeviceID) from an FM ScaleUpResponse body, with the
 * res_op_status gate of internal/cdi/fti/fm/client.go:184-213.  On the error
 * branches the reference's message is written to err_buf. */
int  cro_fm_parse_scale_up_response(const char *body, const char *resource_name,
                                    const char *res_type, const char *model,
                                    char *device_id, size_t device_id_cap,
                                    char *cdi_device_id, size_t cdi_cap,
                                    char *err_buf, size_t err_cap);

/* CM flavour of the ID production: checkAddingResources
 * (internal/cdi/fti/cm/client.go:432-459,485-509) over the GET-machine JSON.
 * existing_device_ids: '\n'-joined Status.DeviceID of every ComposableResource.
 * Outputs: spec_uuid + *device_count for the resize request, or the unused
 * device's (device_id, cdi_device_id).  Returns CRO_ERR_PARSE with the
 * reference's message in err_buf on the ADD_FAILED / malformed branches (the
 * ids are still filled, as the reference returns them with the error). */
int  cro_cm_check_adding_resources(const char *machine_body, const char *existing_device_ids,
                                   const char *res_type, const char *model,
                                   char *spec_uuid, size_t spec_cap, int *device_count,
                                   char *device_id, size_t device_id_cap,
                                   char *cdi_device_id, size_t cdi_cap,
                                   char *err_buf, size_t err_cap);

/* ---- reconcile step: the caller of the hot path -------------------------- */

/*
 * One Reconcile pass of ComposableResourceReconciler for the state in
 * status.state: "" (handleNoneState :176-198), "Attaching" (handleAttachingState
 * :200-287, the hot path, with the CUDA probe in the RunNvidiaSmi /
 * CheckGPUVisible slots), "Online" (:289-318), "Detaching" (:320-407)
 * (all in internal/controller/composableresource_controller.go).
 *
 * in_json:  {"name":..,"spec":{type,model,target_node,force_detach},"labels":{..},
 *            "status":{state,error,device_id,cdi_device_id},
 *            "deleting":bool,
 *            "device_resource_type":"DEVICE_PLUGIN"|"DRA",
 *            "probe":bool,
 *            "provider":{"device_id","cdi_device_id","error","waiting",          AddResource
 *                        "fm_response_body" | "cm_machine_body"+"existing_device_ids",
 *                        "check_resource_error" | "fm_machine_body" | "cm_check_body",   CheckResource
 *                        "remove":{"waiting","error"}},                                   RemoveResource
 *            what the node would have answered, when there is no live context:
 *            "enumeration":{"stdout","stderr","exec_err"}, "enumeration_after_remove":{..},
 *            "resource_slices":[..], "resource_slices_after_remove":[..],
 *            "driver_pod_missing":bool, "daemonset_errors":{"ns/name":"error"},
 *            "load_check":{"stdout","stderr","exec_err","pod_name","driver_enabled"},
 *            "drain":{"error" | "fd_scan":{"stdout","stderr","exec_err"},"rke2":bool},
 *            "create_taint_error","delete_taint_error",
 *            "status_update_failures":{"after":N,"error":".."}   (the API server refuses Status().Update from attempt
 *                   N+1 on: the handler stops where the reference stops; out_json then carries "failed_status_updates"),
 *            an error text that starts "runtime error: " is a Go panic: no status write, reconcile error
 *            "panic: <text> [recovered]" (what controller-runtime's Reconcile wrapper makes of it),
 *            the DaemonSet restart rule (internal/utils/nodes.go:35-76) instead of canned errors:
 *            "daemonsets":{"ns/name":{"desired","ready","current","unavailable","misscheduled",
 *                                     "restarted_at":"<RFC3339>"}}, "now":"<RFC3339>",
 *            the real FM / CM / Sunfish client (csrc/provider.hpp) instead of "provider":
 *            "env":{"DEVICE_RESOURCE_TYPE","CDI_PROVIDER_TYPE","FTI_CDI_API_TYPE",
 *                   "FTI_CDI_TENANT_ID","FTI_CDI_CLUSTER_ID"}   (adapter selection,
 *                   internal/controller/composableresource_adapter.go:39-72),
 *            "fabric":{"http":[{"method","path"|"path_contains","status","body"}..],
 *                      "transport_error","token_error",
 *                      "objects":{"nodes":{name:{"annotations","provider_id"}},
 *                                 "metal3machines":{"ns/name":{"annotations"}},
 *                                 "baremetalhosts":{"ns/name":{"annotations"}},
 *                                 "composable_resource_device_ids":[..],"status_update_error"}}}
 * out_json: {"status":{...},"requeue_after_s":N,"delete_requested":bool,"error":"..",
 *            "status_updates":[...],"probe":{...},
 *            "daemonset_restarts":["ns/name@<stamp>"..], "fabric_requests":[{method,path,query,body}..]}
 * The status object inside out_json is byte-identical to json.Marshal of the
 * reference's ComposableResourceStatus after the same step.
 */
int  cro_reconcile_attach(cro_ctx *ctx, const char *in_json,
                          char *buf, size_t cap, size_t *len);

/* ---- fabric wire codec (response side) ------------------------------------ */

/* CdiProvider.CheckResource decision over the GET-machine body.  kind "fm":
 * internal/cdi/fti/fm/client.go:314-359; kind "cm": internal/cdi/fti/cm/client.go:262-304.
 * CRO_OK = healthy; CRO_ERR_EXEC = the reference's error text in err_buf. */
int  cro_fabric_check_resource(const char *kind, const char *machine_body, const char *res_type,
                               const char *model, const char *device_id, char *err_buf, size_t err_cap);
/* CdiProvider.GetResources decode for one node's machine (fm/client.go:385-410,
 * cm/client.go:335-343): JSON array of cdi.DeviceInfo
 * {"node_name","machine_uuid","device_type","model","device_id","cdi_device_id"}. */
int  cro_fabric_get_resources(const char *kind, const char *machine_body, const char *node_name,
                              const char *machine_uuid, char *buf, size_t cap, size_t *len);
/* CdiProvider.GetResources of the whole FM / CM client (internal/cdi/fti/fm/client.go:361-413,
 * internal/cdi/fti/cm/client.go:306-346) over a scripted fabric: request_json =
 * {"env": {"CDI_PROVIDER_TYPE","FTI_CDI_API_TYPE","DEVICE_RESOURCE_TYPE","FTI_CDI_TENANT_ID","FTI_CDI_CLUSTER_ID"},
 *  "fabric": {"http": [...], "objects": {...}, "token_error": "" | "token": {...}}} (the same "fabric" object
 * cro_reconcile_attach takes).  Reply: {"devices": [DeviceInfo...], "error": "", "fabric_requests": [...]};
 * the FM flavour skips nodes that fail, the CM flavour aborts with the first error. */
int  cro_fabric_list_devices(const char *request_json, char *buf, size_t cap, size_t *len);
/* What CachedToken.Token makes of the id_manager's answer (internal/cdi/fti/token.go:96-175): reply_json =
 * {"secret_error": "", "transport_error": "", "status": 200, "body": "<reply body>"}; writes
 * {"error": "<text, without the 'unable to rotate token: ' prefix GetToken adds>", "expiry": <exp claim, unix s>}.
 * The same object under "fabric"."token" makes cro_reconcile_attach / cro_fabric_list_devices run the
 * token cache (reuse while expiry - 30 s > "now") in front of every fabric request; they then also report
 * "token_fetches". */
int  cro_token_from_reply(const char *reply_json, char *buf, size_t cap, size_t *len);

/* ---- detach-side pre-flight (the step on the other side of the path) ------ */

/* Parse + decision of utils.CheckNoGPULoads (internal/utils/gpus.go:145-186)
 * over the output of `nvidia-smi --query-compute-apps=gpu_uuid,process_name`.
 * driver_enabled != 0: OCP branch (any load on the node); 0: RKE2 branch (only
 * loads on target_uuid).  CRO_OK = no load; CRO_ERR_EXEC = the reference's
 * error text in err_buf. */
int  cro_check_no_gpu_loads(const char *std_out, const char *std_err, const char *exec_err,
                            const char *pod_name, const char *node_name, const char *target_uuid,
                            int driver_enabled, char *err_buf, size_t err_cap);
/* checkGPUDrainStatus (internal/utils/gpus.go:964-1012) over `nvidia-smi drain -p <bus> -q`. */
int  cro_check_gpu_drain_status(const char *std_out, const char *std_err, const char *exec_err,
                                const char *node_name, const char *bus_id, int *draining,
                                char *err_buf, size_t err_cap);
/* Decision after the open-file scan (gpus.go:468-473, :629-634; RKE2 flavour :286-291). */
int  cro_check_device_file_scan(const char *std_out, const char *std_err, const char *exec_err, int rke2,
                                char *err_buf, size_t err_cap);
/* Native replacement of the fd-scan shell scripts (gpus.go:236-260, 441-457):
 * prints what the script would print for `target` (e.g. "/dev/nvidia0").
 * proc_root NULL = "/proc". */
int  cro_scan_device_file_holders(const char *proc_root, const char *target, int rke2,
                                  char *buf, size_t cap, size_t *len);

/* ---- the caller of the hot path: both reconcilers over an in-memory API --- */

/*
 * In-memory cluster (nodes, ComposabilityRequests, ComposableResources with
 * Kubernetes finalizer / deletionTimestamp semantics) driven by restatements of
 * ComposabilityRequestReconciler (internal/controller/composabilityrequest_controller.go:72-625)
 * and ComposableResourceReconciler (internal/controller/composableresource_controller.go:73-441).
 * Drives BASELINE configs 4 (reconcile storm) and 5 (attach/detach churn);
 * every attach runs the CUDA probe when config.probe is true.
 * config_json: {"nodes":["worker-0",...] | [{"name","cpu","memory","ephemeral_storage","pods"}],
 *               "device_resource_type":"DEVICE_PLUGIN"|"DRA","probe":bool,"seed":N,"uuids":[...]}
 */
typedef struct cro_sim cro_sim;
int  cro_sim_create(cro_ctx *ctx /* may be NULL when probe is false */, const char *config_json, cro_sim **out);
void cro_sim_destroy(cro_sim *sim);
/* kubectl apply: {"name":..,"resource":{type,model,size,force_detach,allocation_policy,target_node,other_spec}} */
int  cro_sim_apply(cro_sim *sim, const char *request_json, char *err_buf, size_t err_cap);
int  cro_sim_delete(cro_sim *sim, const char *request_name);
/* test hook: place an object in a given state ({"kind":"ComposabilityRequest"|"ComposableResource",...}) */
int  cro_sim_plant(cro_sim *sim, const char *object_json, char *err_buf, size_t err_cap);
/* run both controllers until quiescent (or max_reconciles); stats JSON out */
int  cro_sim_run(cro_sim *sim, long long max_reconciles, char *buf, size_t cap, size_t *len);
/* exactly one Reconcile of the request controller (how the reference's tests drive it) */
int  cro_sim_reconcile_request(cro_sim *sim, const char *name, char *err_buf, size_t err_cap);
int  cro_sim_reconcile_resource(cro_sim *sim, const char *name, char *err_buf, size_t err_cap);
/* One tick of the UpstreamSyncer (internal/controller/upstreamsyncer_controller.go:77-159) at time
 * now_s.  devices_json: [{"node_name","machine_uuid","device_type","model","device_id","cdi_device_id"}]
 * (cdi.DeviceInfo, internal/cdi/client.go:25-32) — from the fabric, or from the gathered probe
 * results: a device the node can probe but no ComposableResource owns is the drift it repairs. */
int  cro_sim_sync_upstream(cro_sim *sim, const char *devices_json, long long now_s, char *err_buf, size_t err_cap);
int  cro_sim_dump(cro_sim *sim, char *buf, size_t cap, size_t *len);

/* ---- node-side operations run ON the node ---------------------------------- */

/*
 * One of the node-side operations of internal/utils/gpus.go, executed locally instead of through pod
 * execs: scans are native /proc walks, `nvidia-smi --query-gpu=...` is answered from ctx's enumeration
 * (ctx may be NULL: then nvidia-smi is spawned), every other command is spawned.
 * request_json: {"op": "check_no_gpu_loads" (gpus.go:88-186) | "run_nvidia_smi" (:666-689) |
 *                      "check_gpu_visible" (:54-86) | "drain" (:188-664),
 *                "node": "...", "device_id": "GPU-...", "device_resource_type": "DEVICE_PLUGIN"|"DRA",
 *                "driver_container": bool   (true: the gpu-operator flavour; false: the RKE2 / host-driver flavour),
 *                "allow_mutation": bool     (false = dry run: persistence-mode / drain / rm / modprobe / sysfs
 *                                            writes are logged as skipped and succeed),
 *                "proc_root": "/proc"}
 * Reply: {"error": "<the reference's error text or empty>", "visible": bool,
 *         "exec_log": [{"kind","argv","how": "native"|"spawned"|"skipped (dry run)","failed"}..]}
 */
int  cro_local_node_op(cro_ctx *ctx, const char *request_json, char *buf, size_t cap, size_t *len);
/* One command through the same local executor cro_local_node_op uses, for hosts that drive the flows themselves:
 * request_json = {"argv": [...], "allow_mutation": bool, "exec_deadline_ms": N}.  While allow_mutation is false only
 * the argv shapes known to READ are executed (nvidia-smi --query-gpu / --query-compute-apps, `nvidia-smi drain -p <bus>
 * -q`, lsmod, each optionally behind `/bin/chroot /host-root`); everything else is reported "skipped (dry run)".  A
 * child that outlives exec_deadline_ms (default 60 s) is killed and reaped: "context deadline exceeded".
 * The detach side's nvidia-smi invocations — --query-compute-apps=gpu_uuid,process_name (gpus.go:125,134), drain -p <bus>
 * -q (:970), and with allow_mutation: -i <uuid> -pm 0|1 (:267), drain -p <bus> -m 0|1 (:269), drain -p <bus> -r (:311) —
 * are answered through NVML inside this process when libnvidia-ml is there ("how": "native": no child process, no
 * second NVML init), with nvidia-smi's stdout and exit code (the two queries are pinned byte for byte against the real
 * nvidia-smi on a GPU box; the three mutating texts are not — the reference never parses them).  "native_nvml": false
 * spawns instead; "nvml_lib": "<path>" names another libnvidia-ml (tests).  Both keys work in cro_local_node_op too.
 * Reply: {"how": "spawned"|"skipped (dry run)"|"native", "failed": bool, "exec_err", "stdout", "stderr"}. */
int  cro_local_exec(const char *request_json, char *buf, size_t cap, size_t *len);
/* The cmdline scan of checkResetGPUCommandStillRunning (gpus.go:1182-1226), natively:
 * *found = 1 if another process's command line mentions `needle`. */
int  cro_scan_cmdline_for(const char *proc_root, const char *needle, int *found);

/* ---- diagnostics --------------------------------------------------------- */
const char *cro_strerror(int code);
/* Last error text recorded on this context by the calling thread's most
 * recent failing call (thread-safe copy-out).  ctx == NULL: the text of the
 * calling thread's last failed cro_probe_init (which returns no context), e.g.
 * the cudaMalloc that could not be satisfied. */
int  cro_last_error(cro_ctx *ctx, char *buf, size_t cap);
/* No C++ exception crosses this ABI: every entry point catches, returns CRO_ERR_OOM (std::bad_alloc) or
 * CRO_ERR_INTERNAL (anything else) and keeps the text for cro_last_error(NULL, ...).  This self-test throws on purpose
 * behind the same barrier — kind 0: std::runtime_error, 1: std::bad_alloc, 2: a non-std exception — and returns what the
 * barrier made of it; any other kind returns CRO_OK without throwing. */
int  cro_selftest_exception_barrier(int kind);
const char *cro_version(void);

/* ---- test hooks: the verdict kernels on caller-given inputs ---------------- */
/* Test-only: nothing on the probe path calls these.  Each takes the device's mutex, lets any probe still in flight on
 * it finish first, runs one kernel on buffers of its own (never a probe's slots or result struct) and frees them before
 * returning. */

/* One sweep's result slot as the kernels write it into a device's slot array: 64 bytes. */
typedef struct cro_sweep_slot {
    uint64_t x, s, w;              /* checksum triple of what the sweep folded (zero for the fill and the plain copies) */
    uint64_t t0, t1;               /* %globaltimer window: first CTA start, last CTA end                                */
    uint64_t stamp;                /* nonce of the probe whose kernel wrote the slot                                     */
    uint64_t n_words;              /* 64-bit words the sweep covered                                                     */
    uint64_t pad;
} cro_sweep_slot;

/* Slot map of one device's slot array. */
#define CRO_SLOT_FILL           0
#define CRO_SLOT_SWEEP0         1   /* copy sweeps first, then read sweeps: 1 .. 1 + C + R                   */
#define CRO_MAX_SWEEPS_EACH    30   /* at most this many copy sweeps and this many read sweeps               */
#define CRO_SLOT_EXPECT        62   /* closed form of the whole region                                       */
#define CRO_SLOT_PREFIX        63   /* closed form of the first p2p_bytes (what the peers must read)         */
#define CRO_SLOT_P2P0          64   /* per peer j: 64 + 3j + {0 read of j, 1 push into j, 2 re-read of j's push} */
#define CRO_SLOT_SCRATCH       (CRO_SLOT_P2P0 + 3 * CRO_MAX_DEVICES)   /* the single-sweep entry points       */
#define CRO_SLOT_COUNT         (CRO_SLOT_SCRATCH + 4)

/* Runs probe_finalize_kernel on device dev_index over tmpl (the identity template), slots[CRO_SLOT_COUNT] and the probe
 * parameters given, and writes the 512 bytes it produced to *out.  copy_variant is the resolved CRO_COPY_* of the copy
 * sweeps; read_sweeps and copy_sweeps are at most CRO_MAX_SWEEPS_EACH. */
int  cro_selftest_probe_finalize(cro_ctx *ctx, int dev_index, const cro_probe_result *tmpl, const cro_sweep_slot *slots,
                                 uint64_t seed, uint64_t nonce, uint64_t sweep_bytes, uint32_t read_sweeps,
                                 uint32_t copy_sweeps, uint32_t read_variant, uint32_t copy_variant, cro_probe_result *out);
/* Runs p2p_finalize_kernel on device dev_index: *result (what probe_finalize wrote) is updated in place.
 * slots[CRO_SLOT_COUNT] is this device's slot array; peer_slots[j] points at peer j's (CRO_SLOT_COUNT slots) or is NULL
 * for no such peer; peer_stamp, chase_expect: CRO_MAX_DEVICES entries; chase_out: 2 * CRO_MAX_DEVICES words
 * ([2j] end slot, [2j+1] ns).  n <= CRO_MAX_DEVICES, self < n. */
int  cro_selftest_p2p_finalize(cro_ctx *ctx, int dev_index, cro_probe_result *result, const cro_sweep_slot *slots,
                               const cro_sweep_slot *const *peer_slots, const uint64_t *peer_stamp,
                               const uint64_t *chase_out, const uint32_t *chase_expect, uint32_t n, uint32_t self,
                               uint32_t hops, uint32_t have_push, uint32_t push_folded, uint64_t p2p_bytes, uint64_t stamp);
/* Builds, on device dev_index, the latency permutation of the directed pair (minor_src[j], minor_dst[j]) for each of
 * n <= CRO_MAX_DEVICES rows (a row with minor_src[j] < 0 gets no table), arms the chase output as the probe does, runs
 * chase_kernel for `hops` hops and copies the 2 * n output words to out ([2j] end slot, [2j+1] ns). */
int  cro_selftest_chase(cro_ctx *ctx, int dev_index, const int32_t *minor_src, const int32_t *minor_dst, uint32_t n,
                        uint32_t hops, uint64_t *out);

/* Kernels cro_selftest_sweep runs (cro_selftest_sweep_opts.kernel). */
#define CRO_SELFTEST_SWEEP_FILL         1   /* the pattern of seed, or its complement (invert), over the other one   */
#define CRO_SELFTEST_SWEEP_COPY_LDG     2   /* copies: the source holds the pattern of seed, the destination its     */
                                            /* complement                                                            */
#define CRO_SELFTEST_SWEEP_COPY_TMA     3
#define CRO_SELFTEST_SWEEP_COPY_FUSED   4
#define CRO_SELFTEST_SWEEP_READ_LDG     5   /* reads and locate: the interior holds the pattern of seed (^ invert)    */
#define CRO_SELFTEST_SWEEP_READ_TMA     6
#define CRO_SELFTEST_SWEEP_READ_LDG256  7
#define CRO_SELFTEST_SWEEP_LOCATE       8   /* compared with pattern_word(seed, i) ^ invert, recorded as word0 + i    */
#define CRO_SELFTEST_SWEEP_FORCE_WORDS  9   /* force range 0 of an interior holding the pattern of seed              */
#define CRO_SELFTEST_SWEEP_LINK_READ   10   /* link_stream's read role over a host interior holding the pattern     */
#define CRO_SELFTEST_SWEEP_LINK_WRITE  11   /* link_stream's write role: the pattern of seed into a host interior    */
                                            /* holding its complement                                                */
/* Where a copy's two interiors lie (cro_selftest_sweep_opts.layout; 0 for every other kernel). */
#define CRO_SELFTEST_LAYOUT_SRC_DST     1   /* [guard | src | dst | guard]: the probe's A -> B                       */
#define CRO_SELFTEST_LAYOUT_DST_SRC     2   /* [guard | dst | src | guard]: the probe's B -> A                       */
#define CRO_SELFTEST_LAYOUT_APART       3   /* [guard | src | guard | dst | guard]                                    */
#define CRO_SELFTEST_GUARD_BYTES  (2u << 20) /* the least a guard holds: more than any ring (tile * stages) a knob takes */
#define CRO_SELFTEST_F_INTERIORS        1u  /* copy the interiors back too, not only the guards                       */

typedef struct cro_selftest_sweep_opts {
    uint32_t kernel;               /*   0  CRO_SELFTEST_SWEEP_*                                                  */
    uint32_t layout;               /*   4  CRO_SELFTEST_LAYOUT_* of a copy, else 0                               */
    uint64_t offset;               /*   8  each interior starts this far past a 2 MiB boundary: a multiple of 16  */
    uint64_t bytes;                /*  16  of each interior: a multiple of 16, at least 16                       */
    uint64_t seed;                 /*  24  the interior's pattern                                               */
    uint64_t canary;               /*  32  the guards' pattern: word j of guard g (counted from the buffer's     */
                                   /*      start) holds pattern_word(canary, g * 2^32 + j)                      */
    uint64_t invert;               /*  40  fill, locate: XOR on the pattern (0 or all ones)                      */
    uint64_t word0;                /*  48  locate: scan index of the interior's first word; word0 + bytes / 8 <= 2^37 */
    uint64_t force_first[2];       /*  56  interior word ranges set to (word & and) | or once the interior is   */
    uint64_t force_count[2];       /*  72  prepared: locate only, both ranges; force_words: range 0 is the       */
    uint64_t force_and[2];         /*  88  kernel's own and range 1 stays empty; any other kernel: both empty    */
    uint64_t force_or[2];          /* 104  (count 0 = no range)                                                 */
    uint32_t flags;                /* 120  CRO_SELFTEST_F_*                                                      */
    uint32_t reserved;             /* 124  0                                                                     */
} cro_selftest_sweep_opts;

typedef struct cro_selftest_sweep_out {
    cro_sweep_result sweep;        /*   0  the kernel's slot: its fold (reads, fused copy, locate, link read),    */
                                   /*      window, bytes (2 * bytes for a copy) and variant (reads and copies)    */
    uint64_t buf_bytes;            /*  56  the buffer: guards and interiors                                     */
    uint64_t at[2];                /*  64  byte offset in it of interior 0 (a copy's source) and interior 1 (a   */
                                   /*      copy's destination; the one interior again for every other kernel)   */
    uint64_t after_xor[2];         /*  80  each interior's fold once the kernel is done, by the LDG read sweep   */
    uint64_t after_sum[2];         /*  96                                                                        */
    uint64_t after_wsum[2];        /* 112                                                                        */
    uint64_t mismatches;           /* 128  locate, link read: the kernel's exact count                          */
    uint64_t claims;               /* 136  ... and the record slots it claimed                                  */
    uint64_t granules;             /* 144  ... and the granule bits it set (the locator's CRO_LOCATE_GRANULE_BYTES) */
    uint64_t granule_min;          /* 152  lowest and highest granule set (0 when none)                         */
    uint64_t granule_max;          /* 160                                                                        */
} cro_selftest_sweep_out;

/* Runs one sweep kernel of device dev_index, through the launch plan the context's CRO_* knobs made, on a fresh buffer of
 * its own (device memory; mapped pinned host memory for the link rows) laid out as guards around the interior(s):
 * [guard | interior | guard], or a copy's layout.  A guard is at least CRO_SELFTEST_GUARD_BYTES, so a kernel that
 * strays past its interior by up to a ring lands in the hook's own allocation.  Before the kernel each guard is filled
 * with its canary words (opts->canary) and each interior is prepared as the kernel's row above says: what the kernel
 * writes starts as the complement of what it should write, so a word it misses shows.  The kernel runs once between the context's timing
 * events and is waited for with the context's deadline (CRO_ERR_DEADLINE).  Then each interior is folded by the LDG
 * read, the guards (and with CRO_SELFTEST_F_INTERIORS the interiors) are copied to buf at their buffer offsets, and
 * words[0 .. *n) gets the kernel's records (locate, link read), by word, at most cap of them.  A buffer shorter than
 * the layout (cap_bytes < out->buf_bytes) is CRO_ERR_BUFFER_SMALL with out->buf_bytes set, before anything runs.
 * Never touches the sweep region; everything it allocates is freed before it returns. */
int  cro_selftest_sweep(cro_ctx *ctx, int dev_index, const cro_selftest_sweep_opts *opts, cro_selftest_sweep_out *out,
                        void *buf, uint64_t cap_bytes, cro_fault_word *words, int cap, int *n);

#ifdef __cplusplus
}
#endif
#endif /* CROPROBE_H_ */
