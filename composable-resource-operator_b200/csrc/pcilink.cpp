// pcilink.cpp — the PCIe path of a device from sysfs, and NUMA-placed host memory for the link probe.
//
// sysfs is only read, never written.  Under <sys_root>/bus/pci/devices/<bdf> (a symlink into
// <sys_root>/devices/pci<domain>:<bus>/...) each PCI function that has a link exposes current_link_speed,
// current_link_width, max_link_speed and max_link_width; the device's real path names every bridge above it up to
// the root bus, so walking its parent directories visits the whole path the host's traffic takes.
#include "pcilink.hpp"

#include <limits.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <cstdio>
#include <fstream>
#include <sstream>

namespace cro {
namespace pcilink {

namespace {

bool read_file(const std::string& path, std::string* out) {
    std::ifstream f(path);
    if (!f) return false;
    std::stringstream ss;
    ss << f.rdbuf();
    std::string s = ss.str();
    size_t b = s.find_first_not_of(" \t\r\n"), e = s.find_last_not_of(" \t\r\n");
    *out = b == std::string::npos ? std::string() : s.substr(b, e - b + 1);
    return true;
}

unsigned parse_width(const std::string& s) {
    if (s.empty() || s.size() > 4) return 0;
    unsigned v = 0;
    for (char ch : s) {
        if (ch < '0' || ch > '9') return 0;
        v = v * 10 + (unsigned)(ch - '0');
    }
    return v;
}

// dddd:bb:dd.f with a domain of four or more hex digits, lower case, as the kernel names a PCI function.
bool is_bdf(const std::string& name) {
    const size_t c1 = name.find(':');
    if (c1 == std::string::npos || c1 < 4) return false;
    if (name.size() != c1 + 8 || name[c1 + 3] != ':' || name[c1 + 6] != '.') return false;
    for (size_t i = 0; i < name.size(); ++i) {
        if (i == c1 || i == c1 + 3 || i == c1 + 6) continue;
        const char ch = name[i];
        if (!((ch >= '0' && ch <= '9') || (ch >= 'a' && ch <= 'f'))) return false;
    }
    return name[c1 + 7] >= '0' && name[c1 + 7] <= '7';
}

// Reads the four link files of dir into h; false when none of them exists.
bool read_hop(const std::string& dir, const std::string& bdf, cro_pci_hop* h) {
    memset(h, 0, sizeof *h);
    snprintf(h->bdf, sizeof h->bdf, "%s", bdf.c_str());
    std::string t;
    bool any = false;
    if (read_file(dir + "/current_link_speed", &t)) { any = true; h->cur_speed = ParseSpeed(t); }
    if (read_file(dir + "/current_link_width", &t)) { any = true; h->cur_width = parse_width(t); }
    if (read_file(dir + "/max_link_speed", &t)) { any = true; h->max_speed = ParseSpeed(t); }
    if (read_file(dir + "/max_link_width", &t)) { any = true; h->max_width = parse_width(t); }
    return any;
}

uint64_t rate(const cro_pci_hop& h) { return (uint64_t)h.cur_speed * h.cur_width; }

}  // namespace

bool SysfsBdf(const std::string& bus_id, std::string* out) {
    unsigned dom = 0, bus = 0, dev = 0, fn = 0;
    char tail = 0;
    if (bus_id.empty() || bus_id.size() > 16) return false;
    if (sscanf(bus_id.c_str(), "%x:%x:%x.%x%c", &dom, &bus, &dev, &fn, &tail) != 4) return false;
    if (bus > 0xff || dev > 0x1f || fn > 7) return false;
    char b[24];
    snprintf(b, sizeof b, "%04x:%02x:%02x.%x", dom, bus, dev, fn);
    *out = b;
    return true;
}

unsigned ParseSpeed(const std::string& text) {
    const char* p = text.c_str();
    if (*p < '0' || *p > '9') return 0;
    unsigned whole = 0, tenth = 0;
    while (*p >= '0' && *p <= '9') whole = whole * 10 + (unsigned)(*p++ - '0');
    if (*p == '.') {
        ++p;
        if (*p >= '0' && *p <= '9') tenth = (unsigned)(*p - '0');
        while (*p >= '0' && *p <= '9') ++p;
    }
    while (*p == ' ') ++p;
    if (strncmp(p, "GT/s", 4) != 0 || whole > 1000) return 0;
    return whole * 10 + tenth;
}

int ReadPath(const std::string& sys_root, const std::string& bus_id, cro_pci_path* out) {
    memset(out, 0, sizeof *out);
    out->numa_node = -1;
    std::string bdf;
    if (!SysfsBdf(bus_id, &bdf)) return CRO_ERR_INVALID_ARG;
    char real[PATH_MAX];
    if (!realpath((sys_root + "/bus/pci/devices/" + bdf).c_str(), real)) return CRO_ERR_NO_DEVICE;
    std::string dir = real;
    std::string t;
    if (read_file(dir + "/numa_node", &t)) {
        char* end = nullptr;
        const long v = strtol(t.c_str(), &end, 10);
        if (end && *end == 0 && !t.empty() && v >= -1 && v < 1024) out->numa_node = (int32_t)v;
    }
    read_hop(dir, bdf, &out->hop[0]);      // the device itself is hop 0 even when it has no link files
    out->n_hops = 1;
    for (;;) {
        const size_t slash = dir.rfind('/');
        if (slash == std::string::npos || slash == 0) break;
        dir = dir.substr(0, slash);
        const std::string name = dir.substr(dir.rfind('/') + 1);
        if (!is_bdf(name)) break;          // pci<domain>:<bus>: the root bus
        cro_pci_hop h;
        if (!read_hop(dir, name, &h)) continue;
        if (out->n_hops == CRO_PCI_MAX_HOPS) {
            out->truncated = 1;
            break;
        }
        out->hop[out->n_hops++] = h;
    }
    bool any = false;
    for (uint32_t i = 0; i < out->n_hops; ++i) {
        const cro_pci_hop& h = out->hop[i];
        if (!h.cur_speed || !h.cur_width) continue;
        if (!any || rate(h) < rate(out->hop[out->bottleneck])) out->bottleneck = i;
        any = true;
    }
    return CRO_OK;
}

unsigned Degraded(const cro_pci_path& p) {
    unsigned f = 0;
    if (p.n_hops == 0) return 0;
    const cro_pci_hop& g = p.hop[0];
    if (g.cur_speed && g.max_speed && g.cur_speed < g.max_speed) f |= CRO_LINK_DEGRADED_SPEED;
    if (g.cur_width && g.max_width && g.cur_width < g.max_width) f |= CRO_LINK_DEGRADED_WIDTH;
    for (uint32_t i = 1; i < p.n_hops && i < CRO_PCI_MAX_HOPS; ++i) {
        const cro_pci_hop& h = p.hop[i];
        if ((h.cur_speed && h.max_speed && h.cur_speed < h.max_speed) || (h.cur_width && h.max_width && h.cur_width < h.max_width))
            f |= CRO_LINK_DEGRADED_PATH;
    }
    if (rate(g) && p.bottleneck != 0 && p.bottleneck < CRO_PCI_MAX_HOPS && rate(p.hop[p.bottleneck]) < rate(g))
        f |= CRO_LINK_DEGRADED_BOTTLENECK;
    return f;
}

void* MapOnNode(size_t bytes, int node) {
    void* p = mmap(nullptr, bytes, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
    if (p == MAP_FAILED) return nullptr;
    if (node >= 0 && node < 1024) {
        unsigned long mask[1024 / (8 * sizeof(unsigned long))] = {};
        mask[(size_t)node / (8 * sizeof(unsigned long))] = 1ul << ((size_t)node % (8 * sizeof(unsigned long)));
        // MPOL_PREFERRED = 1.  Container seccomp profiles often refuse mbind (EPERM): the pages then land where the
        // kernel puts them, and the caller reports the node they landed on.
        syscall(SYS_mbind, p, bytes, 1, mask, (unsigned long)1024, 0u);
    }
    const long pg = sysconf(_SC_PAGESIZE);
    for (size_t off = 0; off < bytes; off += (size_t)(pg > 0 ? pg : 4096)) static_cast<volatile char*>(p)[off] = 0;
    return p;
}

void Unmap(void* p, size_t bytes) {
    if (p) munmap(p, bytes);
}

int NodeOf(const void* p) {
    int node = -1;
    // MPOL_F_NODE | MPOL_F_ADDR = 3: the node of the page at p
    if (syscall(SYS_get_mempolicy, &node, nullptr, 0ul, p, 3ul) != 0) return -1;
    return node;
}

}  // namespace pcilink
}  // namespace cro
