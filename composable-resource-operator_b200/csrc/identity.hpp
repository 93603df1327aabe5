// identity.hpp — device identity strings and the reference's text handling.
//
// Host-side mirror of the enumerate/parse/decide half of the hot path:
//   getGPUInfoFromNvidiaPod            internal/utils/gpus.go:878-919
//   getGPUInfoFromCroNodeAgentPod      internal/utils/gpus.go:921-962
//   getGPUInfoFromProcInCroNodeAgentPod internal/utils/gpus.go:1014-1089
//   CheckGPUVisible (DEVICE_PLUGIN)    internal/utils/gpus.go:73-84
//   bus-id / dev-path spellings        internal/utils/gpus.go:218,326,406,567,238,480
// Function names follow the reference's; behaviour (including the quirks in
// SURVEY.md Appendix A) is kept so the unchanged Go callers see the same data.
#pragma once
#include <map>
#include <string>
#include <vector>

#include "../../include/croprobe.h"

namespace cro {
namespace identity {

// Go strings.TrimSpace / Split / ToUpper / ToLower / TrimPrefix (ASCII case map).
std::string TrimSpace(const std::string& s);
std::vector<std::string> Split(const std::string& s, const std::string& sep);
std::string ToUpper(const std::string& s);
std::string ToLower(const std::string& s);
std::string TrimPrefix(const std::string& s, const std::string& prefix);

// "GPU-%02x*4-%02x*2-%02x*2-%02x*2-%02x*6" from cudaDeviceProp.uuid bytes.
std::string FormatGpuUuid(const unsigned char bytes[16]);
// nvidia-smi pci.bus_id spelling: 8-hex domain, upper case ("00000000:1F:00.0").
std::string FormatBusIdSmi(unsigned domain, unsigned bus, unsigned device, unsigned function);

using GpuInfo = std::map<std::string, std::string>;
struct GpuInfoResult {
    int code = CRO_OK;             // CRO_OK, CRO_ERR_EXEC, CRO_ERR_PARSE, CRO_ERR_UNSUPPORTED
    bool nil_slice = true;         // Go `var gpuInfos []map[string]string` never appended to
    std::vector<GpuInfo> infos;
    std::string error;             // the reference's error text (or the panic message)
};

// The parse rule of getGPUInfoFromNvidiaPod (gpus.go:896-916).  exec_err ==
// nullptr is a nil error.
GpuInfoResult getGPUInfoFromNvidiaSmiOutput(const std::string& stdOut, const std::string& stdErr,
                                            const char* exec_err, const std::string& queryArgs);
// The parse rule of getGPUInfoFromProcInCroNodeAgentPod (gpus.go:1045-1089).
GpuInfoResult getGPUInfoFromProcOutput(const std::string& stdOut, const std::string& stdErr,
                                       const char* exec_err, const std::string& queryArgs);
// json.Marshal of the []map[string]string.
std::string GpuInfosToJson(const GpuInfoResult& r);

// What the awk lines at gpus.go:1030-1034 print for one information file.
std::string ProcInformationToLine(const std::string& information_text);

// nvidia-smi CSV text for `--query-gpu=<query> --format=csv,noheader,nounits`.
int EmitCsv(const cro_dev_info* devs, int n, const std::string& query, std::string* out,
            std::string* err);

bool CheckGPUVisible(const cro_dev_info* devs, int n, const std::string& deviceID);

// kind: see cro_normalize in croprobe.h.
int Normalize(int kind, const std::string& in, std::string* out);

// ---- identity sources on the node -----------------------------------------
struct ProcGpu {
    std::string dir;       // directory name under /proc/driver/nvidia/gpus
    std::string minor, uuid, bus;
};
// Scans <root>/driver/nvidia/gpus/*/information (root defaults to /proc).
std::vector<ProcGpu> ScanProc(const std::string& proc_root);
// The registry's directory listing alone — "<name>:<inode>:<ctime>" per GPU, sorted, joined by '|' — without opening
// any `information` file: reading those goes through the driver and its locks (slow while
// nvidia-smi polls, and slower for a whole 8-GPU box), listing and stat-ing the directory does not.  A GPU that leaves or
// joins the bus changes the listing; a re-created entry is a new inode object with new times even when procfs hands it
// its old inode number.  Empty string: the registry directory does not exist.
std::string ProcRegistryListing(const std::string& proc_root);

struct NvmlGpu {
    std::string uuid;      // "GPU-..."
    std::string bus_id;    // nvmlPciInfo_t.busId, "00000000:1F:00.0"; "[N/A]", as nvidia-smi prints it, when NVML refuses
    int minor = -1;
    unsigned sm_clock_mhz = 0, mem_clock_mhz = 0;
};
// dlopen("libnvidia-ml.so.1"); false if the library or any call is missing.
bool ScanNvml(std::vector<NvmlGpu>* out, std::string* err);
// Uncorrected volatile ECC errors of the device since the driver was loaded
// (nvmlDeviceGetTotalEccErrors); false when NVML or ECC reporting is unavailable.
bool NvmlEccUncorrected(const std::string& gpu_uuid, unsigned long long* out);
// PCIe replays of the device's link since the driver was loaded (nvmlDeviceGetPcieReplayCounter); false when NVML or
// the symbol is missing or the device refuses.
bool NvmlPcieReplays(const std::string& gpu_uuid, unsigned long long* out);
// The device's DRAM health record: volatile DRAM ECC counts (nvmlDeviceGetMemoryErrorCounter), remapped rows
// (nvmlDeviceGetRemappedRows) and, with `histogram`, the row remapper's histogram.  out->nvml has a CRO_HBM_NVML_* bit
// per read NVML answered; a refused read leaves its fields 0.
void NvmlHbmHealth(const std::string& gpu_uuid, bool histogram, cro_hbm_health* out);
// The device's SRAM health record: volatile SRAM ECC counts (nvmlDeviceGetMemoryErrorCounter) and, with `status`, the
// field-diag threshold flag of nvmlDeviceGetSramEccErrorStatus (looked up by name: older drivers lack it).
// out->nvml has a CRO_SRAM_NVML_* bit per read NVML answered.
void NvmlSramHealth(const std::string& gpu_uuid, bool status, cro_sram_health* out);
// The record the L2 probe reads: volatile SRAM and L2 ECC counts (nvmlDeviceGetMemoryErrorCounter, locations 7 and 1)
// and, with `status`, nvmlDeviceGetSramEccErrorStatus's threshold flag and aggregate uncorrectable L2 bucket.
// out->nvml has a CRO_L2_NVML_* bit per read NVML answered.
void NvmlL2Health(const std::string& gpu_uuid, bool status, cro_l2_health* out);

}  // namespace identity
}  // namespace cro
