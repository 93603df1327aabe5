// pcilink.hpp — the PCIe path of a device as sysfs describes it (cro_pci_link_path), and the host-side helpers of the
// link probe that need no CUDA: NUMA-placed anonymous memory.
#pragma once
#include <stddef.h>

#include <string>

#include "../../include/croprobe.h"

namespace cro {
namespace pcilink {

// "00000000:1F:00.0" or "0000:1f:00.0" -> "0000:1f:00.0"; false when it parses as neither.
bool SysfsBdf(const std::string& bus_id, std::string* out);
// "32.0 GT/s PCIe", "8 GT/s", "2.5 GT/s" -> tenths of a GT/s; "Unknown", empty, anything else -> 0.
unsigned ParseSpeed(const std::string& text);
// cro_pci_link_path: CRO_OK, CRO_ERR_INVALID_ARG (bus id), CRO_ERR_NO_DEVICE (no such device under sys_root).
int ReadPath(const std::string& sys_root, const std::string& bus_id, cro_pci_path* out);
// CRO_LINK_DEGRADED_* of a path.
unsigned Degraded(const cro_pci_path& p);

// Anonymous memory of `bytes`, preferring NUMA node `node` (>= 0) with mbind(MPOL_PREFERRED) by syscall, then touched
// page by page so the pages are placed now.  nullptr when mmap fails; a refused mbind is not an error.
void* MapOnNode(size_t bytes, int node);
void Unmap(void* p, size_t bytes);
// Node of the page at p (get_mempolicy(MPOL_F_NODE | MPOL_F_ADDR)), -1 when the kernel will not say.
int NodeOf(const void* p);

}  // namespace pcilink
}  // namespace cro
