// inventory.hpp — what the node has NOW, as opposed to what CUDA saw at cuInit.
//
// The reference answers every visibility question from a FRESH enumeration: it execs nvidia-smi on each
// reconcile (internal/utils/gpus.go:666-689 RunNvidiaSmi, :878-919 getGPUInfoFromNvidiaPod, called from
// composableresource_controller.go:259,275,381).  A long-lived CUDA process cannot do the same through the CUDA
// runtime: its device list is fixed at cuInit.  So the probe context keeps two things apart:
//   * the devices it can probe IN PROCESS (its CUDA contexts, fixed at cro_probe_init), and
//   * the node's inventory, re-read on every enumeration / visibility query from the driver's own registry
//     (/proc/driver/nvidia/gpus/*/information — a directory walk — with NVML re-initialised only when
//     that walk shows a change).
// A GPU composed after init shows up in the inventory flagged CRO_DEV_NEEDS_HELPER and is probed by a one-shot helper
// process (croprobe-cli, which runs its own cuInit); a GPU drained / removed from the bus drops out of the inventory
// at once, so Detaching sees visible=false like the reference does.
#pragma once
#include <functional>
#include <string>
#include <vector>

#include "../../include/croprobe.h"
#include "identity.hpp"

namespace cro {
namespace inventory {

struct Seen {
    std::string uuid;
    std::string bus_id;     // nvidia-smi spelling, "00000000:1B:00.0"
    int minor = -1;
    int source = 2;         // 1 NVML, 2 /proc
};

// "0000:1b:00.0" (the /proc "Bus Location" spelling) -> "00000000:1B:00.0" (nvidia-smi's pci.bus_id).
std::string ProcBusToSmi(const std::string& bus);

// The node's GPUs from a /proc scan, in minor order (what nvidia-smi lists when NVML is not consulted).
std::vector<Seen> FromProc(const std::vector<identity::ProcGpu>& proc);

// Merges the in-process devices (in their enumeration order) with a fresh scan of the node.
//   have_scan == false: nothing on the node can be consulted — the in-process list is all there is.
//   otherwise the result lists exactly the scanned GPUs, in scan order: known ones keep their identity and get
//   CRO_DEV_IN_PROCESS + their dev_index; unknown ones get cuda_ordinal -1, dev_index -1 and CRO_DEV_NEEDS_HELPER;
//   in-process devices the scan no longer shows are dropped.
std::vector<cro_dev_info> Merge(const std::vector<cro_dev_info>& in_process, bool have_scan, const std::vector<Seen>& seen);

// True when <root>/driver/nvidia/gpus exists (an empty directory means "no GPU left", a missing one "no information").
bool ProcRegistryExists(const std::string& proc_root);

// Runs the probe helper for one GPU: `<helper> probe-raw <uuid> <sweep_MiB>` with CUDA_VISIBLE_DEVICES=<uuid>, reads the
// 512-byte result struct from its stdout, enforces deadline_ms (SIGKILL + reap on expiry).  helper_path empty: the
// croprobe-cli beside libcroprobe.so, or $CRO_HELPER_PATH.  Returns CRO_OK / the struct's status, CRO_ERR_NO_DEVICE
// when the helper reports the device invisible (exit 3), CRO_ERR_DEADLINE, CRO_ERR_EXEC with *err filled otherwise.
int RunHelper(const std::string& helper_path, const std::string& uuid, uint64_t sweep_bytes, int deadline_ms,
              cro_probe_result* out, std::string* err);

// What RunHelper and the check helpers share: `<helper> <args...>` with CUDA_VISIBLE_DEVICES=<uuid>, its stdout read
// into *out under deadline_ms (SIGKILL + reap on expiry).  The output is a head of `head` bytes followed by tail(out,
// size) more, at most max_tail (tail may be empty when there is none; it sees the output's first `size` >= head bytes
// and gives ~0 for a malformed one).  CRO_OK when the helper exited 0 or 1 with exactly that; CRO_ERR_NO_DEVICE (exit
// 3), CRO_ERR_DEADLINE, CRO_ERR_EXEC otherwise, *err naming `what` ("probe helper", "scan helper").
int RunHelperRaw(const std::string& helper_path, const std::string& what, const std::string& uuid,
                 const std::vector<std::string>& args, int deadline_ms, size_t head, size_t max_tail,
                 const std::function<uint64_t(const unsigned char* out, size_t size)>& tail, std::string* out,
                 std::string* err);

std::string DefaultHelperPath();

}  // namespace inventory
}  // namespace cro
