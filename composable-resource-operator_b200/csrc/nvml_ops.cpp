// nvml_ops.cpp — see nvml_ops.hpp.
#include "nvml_ops.hpp"

#include "identity.hpp"

#include <dlfcn.h>

#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>

namespace cro {
namespace nvml {

namespace {

using nvmlDevice_t = void*;
struct PciInfo {  // nvmlPciInfo_t, v3 layout
    char busIdLegacy[16];
    unsigned int domain, bus, device, pciDeviceId, pciSubSystemId;
    char busId[32];
};
struct ProcessInfo {  // nvmlProcessInfo_t as the _v3 entry points fill it
    unsigned int pid;
    unsigned long long usedGpuMemory;
    unsigned int gpuInstanceId, computeInstanceId;
};
static_assert(sizeof(PciInfo) == 68, "nvmlPciInfo_t");
static_assert(sizeof(ProcessInfo) == 24, "nvmlProcessInfo_t");

constexpr int kSuccess = 0, kInvalidArgument = 2, kNotFound = 6, kInsufficientSize = 7;

struct Session {
    bool ok = false;
    int (*count)(unsigned*) = nullptr;
    int (*byIndex)(unsigned, nvmlDevice_t*) = nullptr;
    int (*byUuid)(const char*, nvmlDevice_t*) = nullptr;
    int (*byBus)(const char*, nvmlDevice_t*) = nullptr;
    int (*uuid)(nvmlDevice_t, char*, unsigned) = nullptr;
    int (*pci)(nvmlDevice_t, PciInfo*) = nullptr;
    int (*procs)(nvmlDevice_t, unsigned*, ProcessInfo*) = nullptr;
    int (*procName)(unsigned, char*, unsigned) = nullptr;
    int (*queryDrain)(PciInfo*, int*) = nullptr;
    int (*modifyDrain)(PciInfo*, int) = nullptr;
    int (*removeGpu)(PciInfo*, int, int) = nullptr;
    int (*setPersistence)(nvmlDevice_t, int) = nullptr;
    int (*minor)(nvmlDevice_t, unsigned*) = nullptr;          // optional
    int (*name)(nvmlDevice_t, char*, unsigned) = nullptr;     // optional
    const char* (*errorString)(int) = nullptr;
};

// One session per library path for the life of the process (nvmlInit costs tens of ms and NVML dislikes being unloaded).
Session* session(const std::string& lib) {
    static std::mutex mu;
    static std::map<std::string, std::unique_ptr<Session>> sessions;
    std::lock_guard<std::mutex> g(mu);
    auto it = sessions.find(lib);
    if (it != sessions.end()) return it->second.get();
    std::unique_ptr<Session> s(new Session);
    if (void* h = dlopen(lib.empty() ? "libnvidia-ml.so.1" : lib.c_str(), RTLD_NOW | RTLD_LOCAL)) {
        auto sym = [&](const char* n) { return dlsym(h, n); };
        auto init = (int (*)())sym("nvmlInit_v2");
        s->count = (int (*)(unsigned*))sym("nvmlDeviceGetCount_v2");
        s->byIndex = (int (*)(unsigned, nvmlDevice_t*))sym("nvmlDeviceGetHandleByIndex_v2");
        s->byUuid = (int (*)(const char*, nvmlDevice_t*))sym("nvmlDeviceGetHandleByUUID");
        s->byBus = (int (*)(const char*, nvmlDevice_t*))sym("nvmlDeviceGetHandleByPciBusId_v2");
        s->uuid = (int (*)(nvmlDevice_t, char*, unsigned))sym("nvmlDeviceGetUUID");
        s->pci = (int (*)(nvmlDevice_t, PciInfo*))sym("nvmlDeviceGetPciInfo_v3");
        s->procs = (int (*)(nvmlDevice_t, unsigned*, ProcessInfo*))sym("nvmlDeviceGetComputeRunningProcesses_v3");
        s->procName = (int (*)(unsigned, char*, unsigned))sym("nvmlSystemGetProcessName");
        s->queryDrain = (int (*)(PciInfo*, int*))sym("nvmlDeviceQueryDrainState");
        s->modifyDrain = (int (*)(PciInfo*, int))sym("nvmlDeviceModifyDrainState");
        s->removeGpu = (int (*)(PciInfo*, int, int))sym("nvmlDeviceRemoveGpu_v2");
        s->setPersistence = (int (*)(nvmlDevice_t, int))sym("nvmlDeviceSetPersistenceMode");
        s->minor = (int (*)(nvmlDevice_t, unsigned*))sym("nvmlDeviceGetMinorNumber");
        s->name = (int (*)(nvmlDevice_t, char*, unsigned))sym("nvmlDeviceGetName");
        s->errorString = (const char* (*)(int))sym("nvmlErrorString");
        s->ok = init && s->count && s->byIndex && s->byUuid && s->uuid && s->pci && s->procs && s->procName && s->queryDrain &&
                s->modifyDrain && s->removeGpu && s->setPersistence && init() == kSuccess;
    }
    Session* raw = s.get();
    sessions[lib] = std::move(s);
    return raw;
}

std::string err_text(const Session* s, int rc) {
    if (s->errorString)
        if (const char* t = s->errorString(rc)) return t;
    return "NVML error " + std::to_string(rc);
}

bool hex_field(const std::string& s, unsigned* out) {
    if (s.empty() || s.size() > 8) return false;
    unsigned v = 0;
    for (char c : s) {
        unsigned d;
        if (c >= '0' && c <= '9') d = (unsigned)(c - '0');
        else if (c >= 'a' && c <= 'f') d = (unsigned)(c - 'a' + 10);
        else if (c >= 'A' && c <= 'F') d = (unsigned)(c - 'A' + 10);
        else return false;
        v = v * 16 + d;
    }
    *out = v;
    return true;
}

// nvidia-smi's spelling of a PCI address: 8-hex domain, upper case ("00000000:1F:00.0").
std::string smi_bus(unsigned domain, unsigned bus, unsigned device) {
    char b[40];
    snprintf(b, sizeof b, "%08X:%02X:%02X.0", domain, bus, device);
    return b;
}

bool fill_pci(const std::string& bus_id, PciInfo* p) {
    unsigned domain = 0, bus = 0, device = 0;
    if (!ParseBusId(bus_id, &domain, &bus, &device)) return false;
    const size_t first = bus_id.find(':'), second = first == std::string::npos ? first : bus_id.find(':', first + 1);
    if (second != std::string::npos && first > 4) return false;      // "00000000:40:00.0": nvidia-smi drain refuses it
    memset(p, 0, sizeof *p);
    p->domain = domain;
    p->bus = bus;
    p->device = device;
    snprintf(p->busId, sizeof p->busId, "%08X:%02X:%02X.0", domain, bus, device);
    snprintf(p->busIdLegacy, sizeof p->busIdLegacy, "%04X:%02X:%02X.0", domain & 0xffffu, bus, device);
    return true;
}

Reply unavailable() { return Reply(); }

// pinned on the box (driver 580): `drain -p junk -q` and `drain -p 00000000:40:00.0 -q` both print this and exit 2 —
// nvidia-smi's drain wants the 4-digit domain, which is why the reference trims "0000" first (gpus.go:406,567)
Reply bad_device(Reply r) {
    r.exit_code = kInvalidArgument;
    r.std_out = "Failed to parse device specified at the command-line\n";
    return r;
}

}  // namespace

bool ParseBusId(const std::string& text, unsigned* domain, unsigned* bus, unsigned* device) {
    // [domain:]bus:device[.function]
    std::vector<std::string> parts;
    size_t from = 0;
    for (;;) {
        const size_t c = text.find(':', from);
        parts.push_back(text.substr(from, c == std::string::npos ? std::string::npos : c - from));
        if (c == std::string::npos) break;
        from = c + 1;
    }
    if (parts.size() < 2 || parts.size() > 3) return false;
    std::string dev = parts.back();
    const size_t dot = dev.find('.');
    if (dot != std::string::npos) {
        unsigned fn = 0;
        if (!hex_field(dev.substr(dot + 1), &fn)) return false;
        dev = dev.substr(0, dot);
    }
    *domain = 0;
    if (parts.size() == 3 && !hex_field(parts[0], domain)) return false;
    if (!hex_field(parts[parts.size() - 2], bus) || *bus > 0xff) return false;
    if (!hex_field(dev, device) || *device > 0x1f) return false;
    return true;
}

Reply QueryGpu(const std::string& lib, const std::string& query) {
    Session* s = session(lib);
    if (!s->ok) return unavailable();
    Reply r;
    unsigned n = 0;
    if (s->count(&n) != kSuccess) return unavailable();
    std::vector<cro_dev_info> devs;
    for (unsigned i = 0; i < n; ++i) {
        nvmlDevice_t dev = nullptr;
        if (s->byIndex(i, &dev) != kSuccess) continue;           // e.g. a GPU that fell off the bus
        cro_dev_info d;
        memset(&d, 0, sizeof d);
        d.cuda_ordinal = -1;
        d.device_minor = -1;
        d.dev_index = -1;
        d.identity_source = 1;
        char uuid[96] = {0};
        if (s->uuid(dev, uuid, sizeof uuid) != kSuccess) continue;
        snprintf(d.gpu_uuid, sizeof d.gpu_uuid, "%.47s", uuid);
        PciInfo p;
        memset(&p, 0, sizeof p);
        // nvidia-smi spells a bus id NVML will not give (some virtualised hosts) "[N/A]"
        snprintf(d.pci_bus_id, sizeof d.pci_bus_id, "%.23s", s->pci(dev, &p) == kSuccess ? p.busId : "[N/A]");
        unsigned minor = 0;
        if (s->minor && s->minor(dev, &minor) == kSuccess) d.device_minor = (int)minor;
        char name[96] = {0};
        if (s->name && s->name(dev, name, sizeof name) == kSuccess) snprintf(d.name, sizeof d.name, "%.63s", name);
        devs.push_back(d);
    }
    std::string err;
    if (identity::EmitCsv(devs.data(), (int)devs.size(), query, &r.std_out, &err) != CRO_OK) return unavailable();   // a field only nvidia-smi knows
    r.available = true;
    return r;
}

Reply ComputeApps(const std::string& lib) {
    Session* s = session(lib);
    if (!s->ok) return unavailable();
    Reply r;
    r.available = true;
    unsigned n = 0;
    int rc = s->count(&n);
    if (rc != kSuccess) {
        r.exit_code = rc;
        r.std_out = "Failed to get device count: " + err_text(s, rc) + "\n";
        return r;
    }
    if (n == 0) {
        r.exit_code = kNotFound;                       // nvidia-smi: "No devices were found", exit 6
        r.std_out = "No devices were found\n";
        return r;
    }
    for (unsigned i = 0; i < n; ++i) {
        nvmlDevice_t dev = nullptr;
        if (s->byIndex(i, &dev) != kSuccess) continue;
        char uuid[96] = {0};
        if (s->uuid(dev, uuid, sizeof uuid) != kSuccess) continue;
        std::vector<ProcessInfo> infos(64);
        unsigned cnt = (unsigned)infos.size();
        rc = s->procs(dev, &cnt, infos.data());
        if (rc == kInsufficientSize) {                 // cnt now holds the size needed; leave room for newcomers
            infos.resize(cnt + 16);
            cnt = (unsigned)infos.size();
            rc = s->procs(dev, &cnt, infos.data());
        }
        if (rc != kSuccess) continue;                  // nvidia-smi prints no row for a device it cannot ask
        for (unsigned k = 0; k < cnt; ++k) {
            char name[256] = {0};
            // the path of the executable; a pid outside this pid namespace has none
            if (s->procName(infos[k].pid, name, sizeof name) != kSuccess) snprintf(name, sizeof name, "[Not Found]");
            r.std_out += std::string(uuid) + ", " + name + "\n";
        }
    }
    return r;
}

Reply DrainQuery(const std::string& lib, const std::string& bus_id) {
    Session* s = session(lib);
    if (!s->ok) return unavailable();
    Reply r;
    r.available = true;
    PciInfo p;
    if (!fill_pci(bus_id, &p)) return bad_device(r);
    int state = 0;
    const int rc = s->queryDrain(&p, &state);
    if (rc != kSuccess) {
        r.exit_code = 255;                             // pinned on the box: an address with no GPU behind it
        r.std_out = "Failed to query the GPU drain state.\n";
        return r;
    }
    r.std_out = "The current drain state of GPU " + smi_bus(p.domain, p.bus, p.device) + " is: " + (state ? "draining" : "not draining") + ".\n";
    return r;
}

Reply DrainModify(const std::string& lib, const std::string& bus_id, bool on) {
    Session* s = session(lib);
    if (!s->ok) return unavailable();
    Reply r;
    r.available = true;
    PciInfo p;
    if (!fill_pci(bus_id, &p)) return bad_device(r);
    const int rc = s->modifyDrain(&p, on ? 1 : 0);
    if (rc != kSuccess) {
        r.exit_code = 255;
        r.std_out = "Failed to set the GPU drain state: " + err_text(s, rc) + "\n";
        return r;
    }
    r.std_out = "Successfully set GPU " + smi_bus(p.domain, p.bus, p.device) + " drain state to: " + (on ? "draining" : "not draining") + ".\n";
    return r;
}

Reply DrainRemove(const std::string& lib, const std::string& bus_id) {
    Session* s = session(lib);
    if (!s->ok) return unavailable();
    Reply r;
    r.available = true;
    PciInfo p;
    if (!fill_pci(bus_id, &p)) return bad_device(r);
    // what `nvidia-smi drain -r` asks for: detach the GPU from the driver, leave the PCIe link as it is
    const int rc = s->removeGpu(&p, /*NVML_DETACH_GPU_REMOVE*/ 1, /*NVML_PCIE_LINK_KEEP*/ 0);
    if (rc != kSuccess) {
        r.exit_code = 255;
        r.std_out = "Failed to remove the GPU: " + err_text(s, rc) + "\n";
        return r;
    }
    r.std_out = "Successfully removed GPU " + smi_bus(p.domain, p.bus, p.device) + "\n";
    return r;
}

Reply SetPersistence(const std::string& lib, const std::string& gpu, bool on) {
    Session* s = session(lib);
    if (!s->ok) return unavailable();
    Reply r;
    r.available = true;
    nvmlDevice_t dev = nullptr;
    int rc;
    unsigned domain = 0, bus = 0, device = 0;
    if (gpu.compare(0, 4, "GPU-") == 0 || gpu.compare(0, 4, "MIG-") == 0) rc = s->byUuid(gpu.c_str(), &dev);
    else if (ParseBusId(gpu, &domain, &bus, &device) && s->byBus) rc = s->byBus(smi_bus(domain, bus, device).c_str(), &dev);
    else {
        unsigned idx = 0;
        bool digits = !gpu.empty() && gpu.size() < 6;
        for (char c : gpu) digits = digits && c >= '0' && c <= '9';
        if (!digits) rc = kInvalidArgument;
        else {
            for (char c : gpu) idx = idx * 10 + (unsigned)(c - '0');
            rc = s->byIndex(idx, &dev);
        }
    }
    if (rc != kSuccess) {
        r.exit_code = rc == kInvalidArgument ? kNotFound : rc;     // nvidia-smi -i <unknown>: "No devices were found", exit 6
        r.std_out = "No devices were found\n";
        return r;
    }
    PciInfo p;
    memset(&p, 0, sizeof p);
    s->pci(dev, &p);
    rc = s->setPersistence(dev, on ? 1 : 0);
    if (rc != kSuccess) {
        r.exit_code = rc;
        r.std_out = "Unable to set persistence mode for GPU " + std::string(p.busId) + ": " + err_text(s, rc) + "\n";
        return r;
    }
    r.std_out = std::string(on ? "Enabled" : "Disabled") + " persistence mode for GPU " + p.busId + ".\nAll done.\n";
    return r;
}

}  // namespace nvml
}  // namespace cro
