/*
 * fake_nvml_l2.c — a stand-in libnvidia-ml for the CPU tests of the L2 health reader (identity.cpp NvmlL2Health,
 * cro_read_l2_health): the calls the L2 probe makes, answering crafted values.
 *
 * $FAKE_L2_HEALTH, read at every call, lists the devices, ';'-separated:
 *   <uuid> <sram corrected> <sram uncorrected> <l2 corrected> <l2 uncorrected> <threshold> <l2 bucket> <refuse mask>
 * refuse mask bit 0: corrected SRAM count, 1: uncorrected SRAM, 2: corrected L2, 3: uncorrected L2, 4: the SRAM error
 * status (NVML_ERROR_NOT_SUPPORTED).  Only the SRAM (7) and L2 (1) locations answer; any other, the L1 (0) and DRAM (2)
 * among them, is refused, so a reader that asks for the wrong location reads nothing.  Built with -DNO_SRAM_STATUS the
 * library lacks nvmlDeviceGetSramEccErrorStatus, as an older driver's does.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define NVML_SUCCESS 0
#define NVML_ERROR_INVALID_ARGUMENT 2
#define NVML_ERROR_NOT_SUPPORTED 3
#define NVML_ERROR_NOT_FOUND 6
#define NVML_ERROR_ARGUMENT_VERSION_MISMATCH 25

typedef struct {
    char uuid[96];
    unsigned long long sce, sue, lce, lue, bucket;
    unsigned threshold, refuse;
} Dev;

static Dev devs[8];

static int load(void) {
    const char *s = getenv("FAKE_L2_HEALTH");
    int n = 0;
    while (s && *s && n < 8) {
        Dev *d = &devs[n];
        memset(d, 0, sizeof *d);
        if (sscanf(s, "%95s %llu %llu %llu %llu %u %llu %u", d->uuid, &d->sce, &d->sue, &d->lce, &d->lue, &d->threshold,
                   &d->bucket, &d->refuse) != 8)
            break;
        ++n;
        s = strchr(s, ';');
        if (!s) break;
        ++s;
    }
    return n;
}

static Dev *dev_of(void *h) {
    const long i = (long)h - 1;
    return i >= 0 && i < load() ? &devs[i] : NULL;
}

int nvmlInit_v2(void) { return NVML_SUCCESS; }
int nvmlShutdown(void) { return NVML_SUCCESS; }

int nvmlDeviceGetHandleByUUID(const char *uuid, void **h) {
    const int n = load();
    for (int i = 0; i < n; ++i)
        if (strcmp(devs[i].uuid, uuid) == 0) {
            *h = (void *)(long)(i + 1);
            return NVML_SUCCESS;
        }
    return NVML_ERROR_NOT_FOUND;
}

int nvmlDeviceGetMemoryErrorCounter(void *h, int type, int counter, int location, unsigned long long *count) {
    Dev *d = dev_of(h);
    if (!d || counter != 0 /* volatile */ || (location != 7 && location != 1) || (type != 0 && type != 1))
        return NVML_ERROR_INVALID_ARGUMENT;
    const int bit = (location == 7 ? 0 : 2) + type;
    if (d->refuse & (1u << bit)) return NVML_ERROR_NOT_SUPPORTED;
    *count = location == 7 ? (type ? d->sue : d->sce) : (type ? d->lue : d->lce);
    return NVML_SUCCESS;
}

#ifndef NO_SRAM_STATUS
typedef struct {     /* nvmlEccSramErrorStatus_v1_t */
    unsigned version;
    unsigned long long counts[11];
    unsigned bThresholdExceeded;
} SramStatus;

int nvmlDeviceGetSramEccErrorStatus(void *h, SramStatus *st) {
    Dev *d = dev_of(h);
    if (!d) return NVML_ERROR_INVALID_ARGUMENT;
    if (st->version != ((unsigned)sizeof(SramStatus) | (1u << 24))) return NVML_ERROR_ARGUMENT_VERSION_MISMATCH;
    if (d->refuse & 16u) return NVML_ERROR_NOT_SUPPORTED;
    memset(st->counts, 0, sizeof st->counts);
    st->counts[6] = d->bucket;  /* aggregateUncBucketL2 */
    st->bThresholdExceeded = d->threshold;
    return NVML_SUCCESS;
}
#endif
