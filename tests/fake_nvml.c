/*
 * fake_nvml.c — a stand-in libnvidia-ml for the CPU tests of csrc/nvml_ops.cpp (this container has no NVML).
 *
 * State lives in the directory $FAKE_NVML_DIR, re-read on every call so a test can change it between calls:
 *   gpus    one line per GPU:      <uuid> <domain:bus:dev.fn> <persistence 0|1>
 *   procs   one line per process:  <uuid> <pid> <name or ->          ("-" = name lookup fails, like a foreign pid namespace)
 *   drain   one line per address:  <bus_id as NVML spells it> <0|1>
 *   fail    optional:              <function name> <nvmlReturn_t>    (that call fails with that code)
 *   calls   appended by this library: one line per state-changing call
 * Only the entry points nvml_ops.cpp binds exist.  Test infrastructure, never shipped.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

typedef struct { char busIdLegacy[16]; unsigned domain, bus, device, pciDeviceId, pciSubSystemId; char busId[32]; } PciInfo;
typedef struct { unsigned pid; unsigned long long usedGpuMemory; unsigned gpuInstanceId, computeInstanceId; } ProcessInfo;
typedef struct { char uuid[96]; char bus[40]; int persistence; } Gpu;

static Gpu g_gpus[16];
static int g_n;

static FILE *open_state(const char *name, const char *mode) {
    const char *dir = getenv("FAKE_NVML_DIR");
    char path[512];
    if (!dir) return NULL;
    snprintf(path, sizeof path, "%s/%s", dir, name);
    return fopen(path, mode);
}

static int forced_failure(const char *fn) {
    FILE *f = open_state("fail", "r");
    char name[128];
    int rc, out = 0;
    if (!f) return 0;
    while (fscanf(f, "%127s %d", name, &rc) == 2)
        if (strcmp(name, fn) == 0) out = rc;
    fclose(f);
    return out;
}

static void load_gpus(void) {
    FILE *f = open_state("gpus", "r");
    g_n = 0;
    if (!f) return;
    while (g_n < 16 && fscanf(f, "%95s %39s %d", g_gpus[g_n].uuid, g_gpus[g_n].bus, &g_gpus[g_n].persistence) == 3) ++g_n;
    fclose(f);
}

static void log_call(const char *text) {
    FILE *f = open_state("calls", "a");
    if (!f) return;
    fprintf(f, "%s\n", text);
    fclose(f);
}

int nvmlInit_v2(void) { return forced_failure("nvmlInit_v2"); }
int nvmlShutdown(void) { return 0; }
const char *nvmlErrorString(int rc) {
    switch (rc) {
        case 0: return "Success";
        case 2: return "Invalid Argument";
        case 3: return "Not Supported";
        case 4: return "Insufficient Permissions";
        case 6: return "Not Found";
        case 19: return "In use by another client";
        default: return "Unknown Error";
    }
}
int nvmlDeviceGetCount_v2(unsigned *n) {
    int rc = forced_failure("nvmlDeviceGetCount_v2");
    if (rc) return rc;
    load_gpus();
    *n = (unsigned)g_n;
    return 0;
}
/* a handle is index + 1 */
int nvmlDeviceGetHandleByIndex_v2(unsigned i, void **dev) {
    load_gpus();
    if ((int)i >= g_n) return 2;
    *dev = (void *)(size_t)(i + 1);
    return 0;
}
int nvmlDeviceGetHandleByUUID(const char *uuid, void **dev) {
    load_gpus();
    for (int i = 0; i < g_n; ++i)
        if (strcmp(g_gpus[i].uuid, uuid) == 0) { *dev = (void *)(size_t)(i + 1); return 0; }
    return 6;
}
int nvmlDeviceGetHandleByPciBusId_v2(const char *bus, void **dev) {
    load_gpus();
    for (int i = 0; i < g_n; ++i)
        if (strcasecmp(g_gpus[i].bus, bus) == 0) { *dev = (void *)(size_t)(i + 1); return 0; }
    return 6;
}
int nvmlDeviceGetUUID(void *dev, char *out, unsigned cap) {
    int i = (int)(size_t)dev - 1;
    if (i < 0 || i >= g_n) return 2;
    snprintf(out, cap, "%s", g_gpus[i].uuid);
    return 0;
}
int nvmlDeviceGetMinorNumber(void *dev, unsigned *minor) {
    int i = (int)(size_t)dev - 1;
    if (i < 0 || i >= g_n) return 2;
    *minor = (unsigned)i;
    return 0;
}
int nvmlDeviceGetName(void *dev, char *out, unsigned cap) {
    int i = (int)(size_t)dev - 1;
    if (i < 0 || i >= g_n) return 2;
    snprintf(out, cap, "NVIDIA B200");
    return 0;
}
int nvmlDeviceGetPciInfo_v3(void *dev, PciInfo *p) {
    int i = (int)(size_t)dev - 1, rc = forced_failure("nvmlDeviceGetPciInfo_v3");
    if (rc) return rc;
    if (i < 0 || i >= g_n) return 2;
    memset(p, 0, sizeof *p);
    snprintf(p->busId, sizeof p->busId, "%s", g_gpus[i].bus);
    sscanf(g_gpus[i].bus, "%x:%x:%x", &p->domain, &p->bus, &p->device);
    return 0;
}
int nvmlDeviceGetComputeRunningProcesses_v3(void *dev, unsigned *count, ProcessInfo *infos) {
    int i = (int)(size_t)dev - 1, rc = forced_failure("nvmlDeviceGetComputeRunningProcesses_v3");
    unsigned n = 0, cap = *count;
    char uuid[96], name[256];
    unsigned pid;
    FILE *f;
    if (rc) return rc;
    if (i < 0 || i >= g_n) return 2;
    f = open_state("procs", "r");
    if (f) {
        while (fscanf(f, "%95s %u %255s", uuid, &pid, name) == 3)
            if (strcmp(uuid, g_gpus[i].uuid) == 0) {
                if (n < cap && infos) { memset(&infos[n], 0, sizeof infos[n]); infos[n].pid = pid; }
                ++n;
            }
        fclose(f);
    }
    *count = n;
    return n > cap ? 7 : 0;          /* NVML_ERROR_INSUFFICIENT_SIZE, *count = what is needed */
}
int nvmlSystemGetProcessName(unsigned pid, char *out, unsigned cap) {
    char uuid[96], name[256];
    unsigned p;
    int rc = 6;
    FILE *f = open_state("procs", "r");
    if (!f) return 6;
    while (fscanf(f, "%95s %u %255s", uuid, &p, name) == 3)
        if (p == pid && strcmp(name, "-") != 0) { snprintf(out, cap, "%s", name); rc = 0; }
    fclose(f);
    return rc;
}
static int drain_lookup(const char *bus, int *state) {
    char b[64];
    int s, found = 0;
    FILE *f = open_state("drain", "r");
    if (!f) return 0;
    while (fscanf(f, "%63s %d", b, &s) == 2)
        if (strcmp(b, bus) == 0) { *state = s; found = 1; }      /* the last line wins */
    fclose(f);
    return found;
}
int nvmlDeviceQueryDrainState(PciInfo *p, int *state) {
    int rc = forced_failure("nvmlDeviceQueryDrainState");
    if (rc) return rc;
    return drain_lookup(p->busId, state) ? 0 : 6;
}
int nvmlDeviceModifyDrainState(PciInfo *p, int state) {
    char line[128];
    int rc = forced_failure("nvmlDeviceModifyDrainState"), cur;
    FILE *f;
    if (rc) return rc;
    if (!drain_lookup(p->busId, &cur)) return 6;
    f = open_state("drain", "a");
    if (f) { fprintf(f, "%s %d\n", p->busId, state); fclose(f); }
    snprintf(line, sizeof line, "modify_drain %s %d domain=%x bus=%x device=%x", p->busId, state, p->domain, p->bus, p->device);
    log_call(line);
    return 0;
}
int nvmlDeviceRemoveGpu_v2(PciInfo *p, int gpuState, int linkState) {
    char line[128];
    int rc = forced_failure("nvmlDeviceRemoveGpu_v2"), cur = 0;
    if (rc) return rc;
    if (!drain_lookup(p->busId, &cur)) return 6;
    if (!cur) return 19;             /* not draining: the driver refuses (NVML_ERROR_IN_USE) */
    snprintf(line, sizeof line, "remove_gpu %s gpu_state=%d link_state=%d", p->busId, gpuState, linkState);
    log_call(line);
    return 0;
}
int nvmlDeviceSetPersistenceMode(void *dev, int mode) {
    char line[160];
    int i = (int)(size_t)dev - 1, rc = forced_failure("nvmlDeviceSetPersistenceMode");
    if (rc) return rc;
    if (i < 0 || i >= g_n) return 2;
    snprintf(line, sizeof line, "set_persistence %s %d", g_gpus[i].uuid, mode);
    log_call(line);
    return 0;
}
