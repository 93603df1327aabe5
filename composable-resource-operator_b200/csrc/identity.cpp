// identity.cpp — see identity.hpp.
#include "identity.hpp"

#include <mutex>

#include <dirent.h>
#include <fcntl.h>
#include <dlfcn.h>
#include <sys/stat.h>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <sstream>

#include "gojson.hpp"

namespace cro {
namespace identity {

namespace {

// Go unicode.IsSpace over decoded runes.
bool is_space_rune(unsigned r) {
    switch (r) {
        case '\t': case '\n': case '\v': case '\f': case '\r': case ' ':
        case 0x85: case 0xA0: case 0x1680: case 0x2028: case 0x2029: case 0x202F: case 0x205F:
        case 0x3000:
            return true;
        default:
            return r >= 0x2000 && r <= 0x200A;
    }
}

// Decodes the rune starting at s[i]; returns its length (1 for invalid bytes,
// with rune = 0xFFFD, which is not a space).
size_t decode_at(const std::string& s, size_t i, unsigned* r) {
    const unsigned char c = (unsigned char)s[i];
    if (c < 0x80) { *r = c; return 1; }
    auto cb = [&](size_t k) { return i + k < s.size() && (((unsigned char)s[i + k]) & 0xC0) == 0x80; };
    if (c >= 0xC2 && c <= 0xDF && cb(1)) {
        *r = ((c & 0x1Fu) << 6) | ((unsigned char)s[i + 1] & 0x3Fu);
        return 2;
    }
    if (c >= 0xE0 && c <= 0xEF && cb(1) && cb(2)) {
        *r = ((c & 0x0Fu) << 12) | (((unsigned char)s[i + 1] & 0x3Fu) << 6) |
             ((unsigned char)s[i + 2] & 0x3Fu);
        if (*r >= 0x800 && !(*r >= 0xD800 && *r <= 0xDFFF)) return 3;
    }
    *r = 0xFFFD;
    return 1;
}

}  // namespace

std::string TrimSpace(const std::string& s) {
    size_t b = 0, e = s.size();
    while (b < e) {
        unsigned r;
        const size_t n = decode_at(s, b, &r);
        if (!is_space_rune(r)) break;
        b += n;
    }
    while (e > b) {
        // step back one rune: at most 3 bytes for anything that can be a space
        size_t k = e - 1;
        while (k > b && (((unsigned char)s[k]) & 0xC0) == 0x80 && e - k < 3) --k;
        unsigned r;
        const size_t n = decode_at(s, k, &r);
        if (k + n != e) {  // the tail is not one whole rune: last byte stands alone
            k = e - 1;
            decode_at(s, k, &r);
            if ((unsigned char)s[k] >= 0x80) r = 0xFFFD;
        }
        if (!is_space_rune(r)) break;
        e = k;
    }
    return s.substr(b, e - b);
}

std::vector<std::string> Split(const std::string& s, const std::string& sep) {
    std::vector<std::string> out;
    if (sep.empty()) {  // not used on this path; Go splits into runes
        out.push_back(s);
        return out;
    }
    size_t pos = 0;
    for (;;) {
        const size_t hit = s.find(sep, pos);
        if (hit == std::string::npos) {
            out.push_back(s.substr(pos));
            return out;
        }
        out.push_back(s.substr(pos, hit - pos));
        pos = hit + sep.size();
    }
}

std::string ToUpper(const std::string& s) {
    std::string o = s;
    for (char& c : o)
        if (c >= 'a' && c <= 'z') c = (char)(c - 'a' + 'A');
    return o;
}
std::string ToLower(const std::string& s) {
    std::string o = s;
    for (char& c : o)
        if (c >= 'A' && c <= 'Z') c = (char)(c - 'A' + 'a');
    return o;
}
std::string TrimPrefix(const std::string& s, const std::string& prefix) {
    if (s.size() >= prefix.size() && s.compare(0, prefix.size(), prefix) == 0)
        return s.substr(prefix.size());
    return s;
}

std::string FormatGpuUuid(const unsigned char b[16]) {
    char buf[48];
    snprintf(buf, sizeof buf,
             "GPU-%02x%02x%02x%02x-%02x%02x-%02x%02x-%02x%02x-%02x%02x%02x%02x%02x%02x", b[0], b[1],
             b[2], b[3], b[4], b[5], b[6], b[7], b[8], b[9], b[10], b[11], b[12], b[13], b[14],
             b[15]);
    return buf;
}

std::string FormatBusIdSmi(unsigned domain, unsigned bus, unsigned device, unsigned function) {
    char buf[32];
    snprintf(buf, sizeof buf, "%08X:%02X:%02X.%X", domain, bus, device, function);
    return buf;
}

static std::string go_err_text(const char* exec_err) { return exec_err ? exec_err : "<nil>"; }

GpuInfoResult getGPUInfoFromNvidiaSmiOutput(const std::string& stdOut, const std::string& stdErr,
                                            const char* exec_err, const std::string& queryArgs) {
    GpuInfoResult res;
    const std::vector<std::string> fieldNames = Split(queryArgs, ",");

    // gpus.go:896 — tested on stdout first, wins over stderr / exec error
    if (TrimSpace(stdOut) == "No devices were found") {
        res.nil_slice = false;  // []map[string]string{}
        return res;
    }
    if (!stdErr.empty() || exec_err != nullptr) {
        res.code = CRO_ERR_EXEC;
        res.error = "get gpu info command failed: err: '" + go_err_text(exec_err) + "', stderr: '" +
                    stdErr + "', stdout: '" + stdOut + "'";
        return res;
    }
    for (const std::string& line : Split(TrimSpace(stdOut), "\n")) {
        if (line.empty()) continue;
        const std::vector<std::string> parts = Split(line, ",");
        GpuInfo info;
        for (size_t i = 0; i < fieldNames.size(); ++i) {
            if (i >= parts.size()) {  // gpus.go:913 indexes parts[i] unguarded: Go panics
                res.code = CRO_ERR_PARSE;
                res.error = "runtime error: index out of range [" + std::to_string(i) +
                            "] with length " + std::to_string(parts.size());
                res.infos.clear();
                return res;
            }
            info[fieldNames[i]] = TrimSpace(parts[i]);
        }
        res.infos.push_back(std::move(info));
        res.nil_slice = false;
    }
    return res;
}

GpuInfoResult getGPUInfoFromProcOutput(const std::string& stdOut, const std::string& stdErr,
                                       const char* exec_err, const std::string& queryArgs) {
    GpuInfoResult res;
    const std::vector<std::string> fieldNames = Split(queryArgs, ",");
    if (!stdErr.empty() || exec_err != nullptr) {
        res.code = CRO_ERR_EXEC;
        res.error = "get gpu info command failed: err: '" + go_err_text(exec_err) + "', stderr: '" +
                    stdErr + "', stdout: '" + stdOut + "'";
        return res;
    }
    const std::string trimmed = TrimSpace(stdOut);
    if (trimmed.empty()) {
        res.nil_slice = false;
        return res;
    }
    for (const std::string& line : Split(trimmed, "\n")) {
        if (line.empty()) continue;
        const std::vector<std::string> parts = Split(line, ",");
        if (parts.size() < 3) {
            res.code = CRO_ERR_PARSE;
            res.error = "unexpected GPU information format: '" + line + "'";
            res.infos.clear();
            return res;
        }
        const GpuInfo values = {{"device_minor", TrimSpace(parts[0])},
                                {"gpu_uuid", TrimSpace(parts[1])},
                                {"pci.bus_id", TrimSpace(parts[2])}};
        GpuInfo info;
        for (const std::string& fieldName : fieldNames) {
            const std::string name = TrimSpace(fieldName);
            auto it = values.find(name);
            if (it == values.end()) {
                res.code = CRO_ERR_UNSUPPORTED;
                res.error = "unsupported field '" + name + "' requested in queryArgs";
                res.infos.clear();
                return res;
            }
            info[name] = it->second;
        }
        res.infos.push_back(std::move(info));
        res.nil_slice = false;
    }
    return res;
}

std::string GpuInfosToJson(const GpuInfoResult& r) {
    if (r.nil_slice && r.infos.empty()) return "null";
    gojson::Writer w;
    w.begin_array();
    for (const GpuInfo& g : r.infos) w.string_map(g);
    w.end_array();
    return w.take();
}

// awk default field splitting: runs of blanks/tabs/newlines; $3 of the first
// line matching ^<key>.
static std::string awk_third_field(const std::string& text, const std::string& key) {
    std::istringstream in(text);
    std::string line;
    while (std::getline(in, line)) {
        if (line.compare(0, key.size(), key) != 0) continue;
        std::vector<std::string> f;
        size_t i = 0;
        while (i < line.size()) {
            while (i < line.size() && (line[i] == ' ' || line[i] == '\t' || line[i] == '\n')) ++i;
            size_t j = i;
            while (j < line.size() && !(line[j] == ' ' || line[j] == '\t' || line[j] == '\n')) ++j;
            if (j > i) f.push_back(line.substr(i, j - i));
            i = j;
        }
        return f.size() >= 3 ? f[2] : std::string();  // "exit" after the first match
    }
    return std::string();
}

std::string ProcInformationToLine(const std::string& text) {
    const std::string minor = awk_third_field(text, "Device Minor:");
    const std::string uuid = awk_third_field(text, "GPU UUID:");
    const std::string bus = awk_third_field(text, "Bus Location:");
    if (minor.empty() || uuid.empty() || bus.empty()) return std::string();
    return minor + "," + uuid + "," + bus + "\n";
}

int EmitCsv(const cro_dev_info* devs, int n, const std::string& query, std::string* out,
            std::string* err) {
    out->clear();
    if (n <= 0) {
        *out = "No devices were found\n";
        return CRO_OK;
    }
    const std::vector<std::string> fields = Split(query, ",");
    for (int d = 0; d < n; ++d) {
        std::string row;
        for (size_t f = 0; f < fields.size(); ++f) {
            const std::string name = TrimSpace(fields[f]);
            std::string v;
            if (name == "gpu_uuid" || name == "uuid") v = devs[d].gpu_uuid;
            else if (name == "device_minor" || name == "minor_number")
                v = devs[d].device_minor >= 0 ? std::to_string(devs[d].device_minor) : "[N/A]";
            else if (name == "pci.bus_id" || name == "gpu_bus_id") v = devs[d].pci_bus_id;
            else if (name == "name" || name == "gpu_name") v = devs[d].name;
            else if (name == "index") v = std::to_string(d);
            else {
                if (err) *err = "Field \"" + name + "\" is not a valid field to query.";
                out->clear();
                return CRO_ERR_UNSUPPORTED;
            }
            if (f) row += ", ";
            row += v;
        }
        *out += row;
        out->push_back('\n');
    }
    return CRO_OK;
}

bool CheckGPUVisible(const cro_dev_info* devs, int n, const std::string& deviceID) {
    for (int i = 0; i < n; ++i) {
        const std::string u(devs[i].gpu_uuid, strnlen(devs[i].gpu_uuid, sizeof devs[i].gpu_uuid));
        if (u == deviceID) return true;  // gpus.go:79
    }
    return false;
}

int Normalize(int kind, const std::string& in, std::string* out) {
    switch (kind) {
        case 0: *out = ToUpper(TrimSpace(in)); return CRO_OK;                       // gpus.go:218
        case 1: *out = ToLower(TrimSpace(in)); return CRO_OK;                       // gpus.go:326
        case 2: *out = TrimPrefix(ToUpper(TrimSpace(in)), "0000"); return CRO_OK;   // gpus.go:406,567
        case 3: *out = "/dev/nvidia" + in; return CRO_OK;                           // gpus.go:238
        case 4: *out = "/run/nvidia/driver/dev/nvidia" + in; return CRO_OK;         // gpus.go:480
        default: return CRO_ERR_INVALID_ARG;
    }
}

std::vector<ProcGpu> ScanProc(const std::string& proc_root) {
    std::vector<ProcGpu> out;
    const std::string base = (proc_root.empty() ? std::string("/proc") : proc_root) + "/driver/nvidia/gpus";
    DIR* d = opendir(base.c_str());
    if (!d) return out;
    std::vector<std::string> names;
    while (dirent* e = readdir(d)) {
        if (e->d_name[0] == '.') continue;
        names.push_back(e->d_name);
    }
    closedir(d);
    std::sort(names.begin(), names.end());  // the shell glob at gpus.go:1022 expands sorted
    for (const std::string& name : names) {
        const std::string path = base + "/" + name + "/information";
        std::ifstream f(path);
        if (!f) continue;
        std::stringstream ss;
        ss << f.rdbuf();
        const std::string text = ss.str();
        ProcGpu g;
        g.dir = name;
        g.minor = awk_third_field(text, "Device Minor:");
        g.uuid = awk_third_field(text, "GPU UUID:");
        g.bus = awk_third_field(text, "Bus Location:");
        if (!g.minor.empty() && !g.uuid.empty() && !g.bus.empty()) out.push_back(g);
    }
    return out;
}

// ---- NVML through dlopen (the image ships only a stub library) -------------
namespace {
struct NvmlPciInfo {  // nvmlPciInfo_t (v3 layout)
    char busIdLegacy[16];
    unsigned int domain, bus, device, pciDeviceId, pciSubSystemId;
    char busId[32];
};
using nvmlDevice_t = void*;
}  // namespace

std::string ProcRegistryListing(const std::string& proc_root) {
    const std::string base = (proc_root.empty() ? std::string("/proc") : proc_root) + "/driver/nvidia/gpus";
    DIR* d = opendir(base.c_str());
    if (!d) return std::string();
    std::vector<std::string> names;
    while (dirent* e = readdir(d)) {
        if (e->d_name[0] == '.') continue;
        // name : inode : change time.  procfs hands a re-created entry the lowest free inode NUMBER — usually the one
        // it had — but a new inode object, whose times are the moment it was made.
        struct stat st;
        std::string tag = std::string(e->d_name) + ":" + std::to_string((unsigned long long)e->d_ino);
        if (fstatat(dirfd(d), e->d_name, &st, AT_SYMLINK_NOFOLLOW) == 0)
            tag += ":" + std::to_string((long long)st.st_ctim.tv_sec) + "." + std::to_string((long)st.st_ctim.tv_nsec);
        names.push_back(tag);
    }
    closedir(d);
    std::sort(names.begin(), names.end());
    std::string out = "P";
    for (const std::string& n : names) out += "|" + n;
    return out;
}

bool ScanNvml(std::vector<NvmlGpu>* out, std::string* err) {
    void* h = dlopen("libnvidia-ml.so.1", RTLD_NOW | RTLD_LOCAL);
    if (!h) {
        if (err) *err = "dlopen libnvidia-ml.so.1 failed";
        return false;
    }
    auto sym = [&](const char* n) { return dlsym(h, n); };
    auto init = (int (*)())sym("nvmlInit_v2");
    auto shutdown = (int (*)())sym("nvmlShutdown");
    auto count = (int (*)(unsigned*))sym("nvmlDeviceGetCount_v2");
    auto byIndex = (int (*)(unsigned, nvmlDevice_t*))sym("nvmlDeviceGetHandleByIndex_v2");
    auto getUuid = (int (*)(nvmlDevice_t, char*, unsigned))sym("nvmlDeviceGetUUID");
    auto getMinor = (int (*)(nvmlDevice_t, unsigned*))sym("nvmlDeviceGetMinorNumber");
    auto getPci = (int (*)(nvmlDevice_t, NvmlPciInfo*))sym("nvmlDeviceGetPciInfo_v3");
    auto getClock = (int (*)(nvmlDevice_t, int, unsigned*))sym("nvmlDeviceGetClockInfo");
    if (!init || !shutdown || !count || !byIndex || !getUuid || !getMinor || !getPci) {
        if (err) *err = "libnvidia-ml.so.1 lacks a required symbol";
        dlclose(h);
        return false;
    }
    if (init() != 0) {
        if (err) *err = "nvmlInit_v2 failed";
        dlclose(h);
        return false;
    }
    unsigned n = 0;
    bool ok = count(&n) == 0;
    for (unsigned i = 0; ok && i < n; ++i) {
        nvmlDevice_t dev = nullptr;
        if (byIndex(i, &dev) != 0) continue;  // e.g. a GPU that fell off the bus
        NvmlGpu g;
        char uuid[96] = {0};
        unsigned minor = 0;
        NvmlPciInfo pci;
        memset(&pci, 0, sizeof pci);
        if (getUuid(dev, uuid, sizeof uuid) != 0) continue;
        g.uuid = uuid;
        if (getMinor(dev, &minor) == 0) g.minor = (int)minor;
        // a device whose PCI info NVML will not give (some virtualised hosts): nvidia-smi prints "[N/A]" for it
        g.bus_id = getPci(dev, &pci) == 0 ? std::string(pci.busId) : std::string("[N/A]");
        if (getClock) {
            unsigned c = 0;
            if (getClock(dev, /*NVML_CLOCK_SM*/ 1, &c) == 0) g.sm_clock_mhz = c;
            if (getClock(dev, /*NVML_CLOCK_MEM*/ 2, &c) == 0) g.mem_clock_mhz = c;
        }
        out->push_back(g);
    }
    shutdown();
    // the handle stays open: NVML dislikes being unloaded and re-loaded
    if (!ok && err) *err = "nvmlDeviceGetCount_v2 failed";
    return ok;
}

// One NVML session for the life of the process (init is reference-counted, so the init/shutdown pairs of ScanNvml
// still balance): the per-probe ECC read, the link probe's replay counter and the scan's and SRAM probe's memory health
// must not pay nvmlInit every time.  A reader whose symbol the library lacks answers false.
namespace {
struct NvmlRemapHistogram {  // nvmlRowRemapperHistogramValues_t
    unsigned max, high, partial, low, none;
};
struct NvmlSramStatus {  // nvmlEccSramErrorStatus_v1_t
    unsigned version;
    unsigned long long aggregateUncParity, aggregateUncSecDed, aggregateCor, volatileUncParity, volatileUncSecDed,
        volatileCor, aggregateUncBucketL2, aggregateUncBucketSm, aggregateUncBucketPcie, aggregateUncBucketMcu,
        aggregateUncBucketOther;
    unsigned bThresholdExceeded;
};
static_assert(sizeof(NvmlSramStatus) == 104, "nvmlEccSramErrorStatus_v1_t");
constexpr unsigned kNvmlSramStatusV1 = (unsigned)sizeof(NvmlSramStatus) | (1u << 24);   // NVML_STRUCT_VERSION(.., 1)
struct NvmlSession {
    int (*byUuid)(const char*, nvmlDevice_t*) = nullptr;
    int (*ecc)(nvmlDevice_t, int, int, unsigned long long*) = nullptr;
    int (*replays)(nvmlDevice_t, unsigned*) = nullptr;
    int (*memErrors)(nvmlDevice_t, int, int, int, unsigned long long*) = nullptr;
    int (*remapped)(nvmlDevice_t, unsigned*, unsigned*, unsigned*, unsigned*) = nullptr;
    int (*histogram)(nvmlDevice_t, NvmlRemapHistogram*) = nullptr;
    int (*sramStatus)(nvmlDevice_t, NvmlSramStatus*) = nullptr;
    bool ok = false;
};
const NvmlSession& nvml_session() {
    static NvmlSession s;
    static std::once_flag once;
    std::call_once(once, [] {
        void* h = dlopen("libnvidia-ml.so.1", RTLD_NOW | RTLD_LOCAL);
        if (!h) return;
        auto init = (int (*)())dlsym(h, "nvmlInit_v2");
        s.byUuid = (int (*)(const char*, nvmlDevice_t*))dlsym(h, "nvmlDeviceGetHandleByUUID");
        s.ecc = (int (*)(nvmlDevice_t, int, int, unsigned long long*))dlsym(h, "nvmlDeviceGetTotalEccErrors");
        s.replays = (int (*)(nvmlDevice_t, unsigned*))dlsym(h, "nvmlDeviceGetPcieReplayCounter");
        s.memErrors = (int (*)(nvmlDevice_t, int, int, int, unsigned long long*))dlsym(h, "nvmlDeviceGetMemoryErrorCounter");
        s.remapped = (int (*)(nvmlDevice_t, unsigned*, unsigned*, unsigned*, unsigned*))dlsym(h, "nvmlDeviceGetRemappedRows");
        s.histogram = (int (*)(nvmlDevice_t, NvmlRemapHistogram*))dlsym(h, "nvmlDeviceGetRowRemapperHistogram");
        s.sramStatus = (int (*)(nvmlDevice_t, NvmlSramStatus*))dlsym(h, "nvmlDeviceGetSramEccErrorStatus");
        s.ok = init && s.byUuid && init() == 0;
    });
    return s;
}
bool nvml_device(const NvmlSession& s, const std::string& gpu_uuid, nvmlDevice_t* dev) {
    return s.ok && s.byUuid(gpu_uuid.c_str(), dev) == 0;
}
}  // namespace

bool NvmlEccUncorrected(const std::string& gpu_uuid, unsigned long long* out) {
    const NvmlSession& s = nvml_session();
    nvmlDevice_t dev = nullptr;
    if (!s.ecc || !nvml_device(s, gpu_uuid, &dev)) return false;
    return s.ecc(dev, /*NVML_MEMORY_ERROR_TYPE_UNCORRECTED*/ 1, /*NVML_VOLATILE_ECC*/ 0, out) == 0;
}

bool NvmlPcieReplays(const std::string& gpu_uuid, unsigned long long* out) {
    const NvmlSession& s = nvml_session();
    nvmlDevice_t dev = nullptr;
    if (!s.replays || !nvml_device(s, gpu_uuid, &dev)) return false;
    unsigned v = 0;
    if (s.replays(dev, &v) != 0) return false;
    *out = v;
    return true;
}

void NvmlHbmHealth(const std::string& gpu_uuid, bool histogram, cro_hbm_health* out) {
    memset(out, 0, sizeof *out);
    const NvmlSession& s = nvml_session();
    nvmlDevice_t dev = nullptr;
    if (!nvml_device(s, gpu_uuid, &dev)) return;
    if (s.memErrors) {
        // NVML_MEMORY_ERROR_TYPE_CORRECTED 0 / _UNCORRECTED 1, NVML_VOLATILE_ECC 0, NVML_MEMORY_LOCATION_DRAM 2
        unsigned long long v = 0;
        if (s.memErrors(dev, 0, 0, 2, &v) == 0) { out->ecc_corrected = v; out->nvml |= CRO_HBM_NVML_ECC_CORRECTED; }
        v = 0;
        if (s.memErrors(dev, 1, 0, 2, &v) == 0) { out->ecc_uncorrected = v; out->nvml |= CRO_HBM_NVML_ECC_UNCORRECTED; }
    }
    unsigned corr = 0, unc = 0, pending = 0, failure = 0;
    if (s.remapped && s.remapped(dev, &corr, &unc, &pending, &failure) == 0) {
        out->remap_corrected = corr;
        out->remap_uncorrected = unc;
        out->remap_pending = pending ? 1u : 0u;
        out->remap_failure = failure ? 1u : 0u;
        out->nvml |= CRO_HBM_NVML_REMAP;
    }
    NvmlRemapHistogram h{};
    if (histogram && s.histogram && s.histogram(dev, &h) == 0) {
        const unsigned v[5] = {h.max, h.high, h.partial, h.low, h.none};
        memcpy(out->histogram, v, sizeof v);
        out->nvml |= CRO_HBM_NVML_HISTOGRAM;
    }
}

void NvmlSramHealth(const std::string& gpu_uuid, bool status, cro_sram_health* out) {
    memset(out, 0, sizeof *out);
    const NvmlSession& s = nvml_session();
    nvmlDevice_t dev = nullptr;
    if (!nvml_device(s, gpu_uuid, &dev)) return;
    if (s.memErrors) {
        // NVML_MEMORY_ERROR_TYPE_CORRECTED 0 / _UNCORRECTED 1, NVML_VOLATILE_ECC 0, NVML_MEMORY_LOCATION_SRAM 7
        unsigned long long v = 0;
        if (s.memErrors(dev, 0, 0, 7, &v) == 0) { out->ecc_corrected = v; out->nvml |= CRO_SRAM_NVML_ECC_CORRECTED; }
        v = 0;
        if (s.memErrors(dev, 1, 0, 7, &v) == 0) { out->ecc_uncorrected = v; out->nvml |= CRO_SRAM_NVML_ECC_UNCORRECTED; }
    }
    NvmlSramStatus st{};
    st.version = kNvmlSramStatusV1;
    if (status && s.sramStatus && s.sramStatus(dev, &st) == 0) {
        out->threshold_exceeded = st.bThresholdExceeded ? 1u : 0u;
        out->nvml |= CRO_SRAM_NVML_STATUS;
    }
}

void NvmlL2Health(const std::string& gpu_uuid, bool status, cro_l2_health* out) {
    memset(out, 0, sizeof *out);
    const NvmlSession& s = nvml_session();
    nvmlDevice_t dev = nullptr;
    if (!nvml_device(s, gpu_uuid, &dev)) return;
    if (s.memErrors) {
        // NVML_MEMORY_ERROR_TYPE_CORRECTED 0 / _UNCORRECTED 1, NVML_VOLATILE_ECC 0, NVML_MEMORY_LOCATION_SRAM 7 and
        // NVML_MEMORY_LOCATION_L2_CACHE 1 (which a Hopper driver may refuse: its L2 errors are counted as SRAM's)
        unsigned long long v = 0;
        if (s.memErrors(dev, 0, 0, 7, &v) == 0) { out->sram_corrected = v; out->nvml |= CRO_L2_NVML_SRAM_CORRECTED; }
        v = 0;
        if (s.memErrors(dev, 1, 0, 7, &v) == 0) { out->sram_uncorrected = v; out->nvml |= CRO_L2_NVML_SRAM_UNCORRECTED; }
        v = 0;
        if (s.memErrors(dev, 0, 0, 1, &v) == 0) { out->l2_corrected = v; out->nvml |= CRO_L2_NVML_L2_CORRECTED; }
        v = 0;
        if (s.memErrors(dev, 1, 0, 1, &v) == 0) { out->l2_uncorrected = v; out->nvml |= CRO_L2_NVML_L2_UNCORRECTED; }
    }
    NvmlSramStatus st{};
    st.version = kNvmlSramStatusV1;
    if (status && s.sramStatus && s.sramStatus(dev, &st) == 0) {
        out->threshold_exceeded = st.bThresholdExceeded ? 1u : 0u;
        out->unc_bucket_l2 = st.aggregateUncBucketL2;
        out->nvml |= CRO_L2_NVML_STATUS;
    }
}

}  // namespace identity
}  // namespace cro
