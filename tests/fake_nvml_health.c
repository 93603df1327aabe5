/*
 * fake_nvml_health.c — a stand-in libnvidia-ml for the CPU tests of the DRAM health readers (identity.cpp
 * NvmlHbmHealth, cro_read_hbm_health): the three calls the whole-HBM scan makes, answering crafted values.
 *
 * $FAKE_HBM_HEALTH, read at every call, lists the devices, ';'-separated:
 *   <uuid> <ecc corrected> <ecc uncorrected> <remap corrected> <remap uncorrected> <pending> <failure>
 *          <hist max> <hist high> <hist partial> <hist low> <hist none> <refuse mask>
 * refuse mask bit 0: corrected ECC count, 1: uncorrected, 2: remapped rows, 3: histogram (NVML_ERROR_NOT_SUPPORTED).
 * Built with -DNO_HISTOGRAM the library lacks nvmlDeviceGetRowRemapperHistogram, as an older driver's does.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define NVML_SUCCESS 0
#define NVML_ERROR_INVALID_ARGUMENT 2
#define NVML_ERROR_NOT_SUPPORTED 3
#define NVML_ERROR_NOT_FOUND 6

typedef struct {
    char uuid[96];
    unsigned long long ce, ue;
    unsigned rc, ru, pending, failure, hist[5], refuse;
} Dev;

static Dev devs[8];

static int load(void) {
    const char *s = getenv("FAKE_HBM_HEALTH");
    int n = 0;
    while (s && *s && n < 8) {
        Dev *d = &devs[n];
        memset(d, 0, sizeof *d);
        if (sscanf(s, "%95s %llu %llu %u %u %u %u %u %u %u %u %u %u", d->uuid, &d->ce, &d->ue, &d->rc, &d->ru, &d->pending,
                   &d->failure, &d->hist[0], &d->hist[1], &d->hist[2], &d->hist[3], &d->hist[4], &d->refuse) != 13)
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
    if (!d || counter != 0 /* volatile */ || location != 2 /* DRAM */ || (type != 0 && type != 1)) return NVML_ERROR_INVALID_ARGUMENT;
    if (d->refuse & (1u << type)) return NVML_ERROR_NOT_SUPPORTED;
    *count = type ? d->ue : d->ce;
    return NVML_SUCCESS;
}

int nvmlDeviceGetRemappedRows(void *h, unsigned *corr, unsigned *unc, unsigned *pending, unsigned *failure) {
    Dev *d = dev_of(h);
    if (!d) return NVML_ERROR_INVALID_ARGUMENT;
    if (d->refuse & 4u) return NVML_ERROR_NOT_SUPPORTED;
    *corr = d->rc;
    *unc = d->ru;
    *pending = d->pending;
    *failure = d->failure;
    return NVML_SUCCESS;
}

#ifndef NO_HISTOGRAM
int nvmlDeviceGetRowRemapperHistogram(void *h, unsigned *values /* max, high, partial, low, none */) {
    Dev *d = dev_of(h);
    if (!d) return NVML_ERROR_INVALID_ARGUMENT;
    if (d->refuse & 8u) return NVML_ERROR_NOT_SUPPORTED;
    memcpy(values, d->hist, sizeof d->hist);
    return NVML_SUCCESS;
}
#endif
