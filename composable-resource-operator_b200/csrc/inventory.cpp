// inventory.cpp — see inventory.hpp (reference behaviour being kept: a fresh enumeration per reconcile,
// internal/utils/gpus.go:666-689, :878-919).
#include "inventory.hpp"

#include <dirent.h>
#include <dlfcn.h>
#include <fcntl.h>
#include <poll.h>
#include <signal.h>
#include <spawn.h>
#include <sys/stat.h>
#include <sys/wait.h>
#include <unistd.h>

#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>

extern char** environ;

namespace cro {
namespace inventory {

std::string ProcBusToSmi(const std::string& bus) {
    // /proc prints the 4-hex-domain kernel spelling in lower case; nvidia-smi an 8-hex domain in upper case
    const std::string t = identity::ToUpper(identity::TrimSpace(bus));
    const size_t colon = t.find(':');
    if (colon == std::string::npos) return t;
    std::string dom = t.substr(0, colon);
    while (dom.size() < 8) dom = "0" + dom;
    return dom + t.substr(colon);
}

std::vector<Seen> FromProc(const std::vector<identity::ProcGpu>& proc) {
    std::vector<Seen> v;
    for (const identity::ProcGpu& g : proc) {
        Seen s;
        s.uuid = g.uuid;
        s.bus_id = ProcBusToSmi(g.bus);
        s.minor = atoi(g.minor.c_str());
        s.source = 2;
        v.push_back(s);
    }
    std::stable_sort(v.begin(), v.end(), [](const Seen& a, const Seen& b) { return a.minor < b.minor; });
    return v;
}

static void set_str(char* dst, size_t cap, const std::string& s) {
    memset(dst, 0, cap);
    memcpy(dst, s.data(), std::min(cap - 1, s.size()));
}

std::vector<cro_dev_info> Merge(const std::vector<cro_dev_info>& in_process, bool have_scan, const std::vector<Seen>& seen) {
    std::vector<cro_dev_info> out;
    if (!have_scan) {
        for (size_t i = 0; i < in_process.size(); ++i) {
            cro_dev_info d = in_process[i];
            d.flags = CRO_DEV_IN_PROCESS;
            d.dev_index = (int32_t)i;
            out.push_back(d);
        }
        return out;
    }
    for (const Seen& s : seen) {
        bool known = false;
        for (size_t i = 0; i < in_process.size(); ++i) {
            if (std::string(in_process[i].gpu_uuid, strnlen(in_process[i].gpu_uuid, sizeof in_process[i].gpu_uuid)) != s.uuid) continue;
            cro_dev_info d = in_process[i];
            d.flags = CRO_DEV_IN_PROCESS;
            d.dev_index = (int32_t)i;
            if (s.minor >= 0) d.device_minor = s.minor;      // a re-bound device may come back under another minor
            out.push_back(d);
            known = true;
            break;
        }
        if (known) continue;
        cro_dev_info d;
        memset(&d, 0, sizeof d);
        d.cuda_ordinal = -1;
        d.dev_index = -1;
        d.device_minor = s.minor;
        set_str(d.gpu_uuid, sizeof d.gpu_uuid, s.uuid);
        set_str(d.pci_bus_id, sizeof d.pci_bus_id, s.bus_id);
        d.identity_source = (uint32_t)s.source;
        d.flags = CRO_DEV_NEEDS_HELPER;
        out.push_back(d);
    }
    return out;
}

bool ProcRegistryExists(const std::string& proc_root) {
    struct stat st;
    const std::string base = (proc_root.empty() ? std::string("/proc") : proc_root) + "/driver/nvidia/gpus";
    return stat(base.c_str(), &st) == 0 && S_ISDIR(st.st_mode);
}

std::string DefaultHelperPath() {
    if (const char* p = getenv("CRO_HELPER_PATH"))
        if (*p) return p;
    Dl_info info;
    if (dladdr((const void*)&DefaultHelperPath, &info) && info.dli_fname) {
        std::string lib = info.dli_fname;
        const size_t slash = lib.rfind('/');
        return (slash == std::string::npos ? std::string(".") : lib.substr(0, slash)) + "/croprobe-cli";
    }
    return "croprobe-cli";
}

int RunHelperRaw(const std::string& helper_path, const std::string& what, const std::string& uuid,
                 const std::vector<std::string>& args, int deadline_ms, size_t head, size_t max_tail,
                 const std::function<uint64_t(const unsigned char* out, size_t size)>& tail, std::string* out,
                 std::string* err) {
    const std::string helper = helper_path.empty() ? DefaultHelperPath() : helper_path;
    if (access(helper.c_str(), X_OK) != 0) {
        if (err) *err = what + " '" + helper + "' is not executable";
        return CRO_ERR_EXEC;
    }
    int fds[2];
    if (pipe(fds) != 0) {
        if (err) *err = std::string("pipe: ") + strerror(errno);
        return CRO_ERR_EXEC;
    }
    // posix_spawn, not fork: the host process is multi-threaded (CUDA's own threads at least), and the child's
    // environment — CUDA_VISIBLE_DEVICES=<uuid>, so that the helper's cuInit sees this one GPU and nothing else — is
    // built here, before the spawn, instead of with setenv() in a forked child (not async-signal-safe).
    std::vector<std::string> env_store;
    for (char** e = environ; e && *e; ++e)
        if (strncmp(*e, "CUDA_VISIBLE_DEVICES=", 21) != 0) env_store.push_back(*e);
    env_store.push_back("CUDA_VISIBLE_DEVICES=" + uuid);
    std::vector<char*> envp;
    for (std::string& e : env_store) envp.push_back(const_cast<char*>(e.c_str()));
    envp.push_back(nullptr);
    std::vector<const char*> argv = {helper.c_str()};
    for (const std::string& a : args) argv.push_back(a.c_str());
    argv.push_back(nullptr);
    posix_spawn_file_actions_t fa;
    posix_spawn_file_actions_init(&fa);
    posix_spawn_file_actions_adddup2(&fa, fds[1], 1);
    posix_spawn_file_actions_addclose(&fa, fds[0]);
    posix_spawn_file_actions_addclose(&fa, fds[1]);
    pid_t pid = 0;
    const int src = posix_spawn(&pid, helper.c_str(), &fa, nullptr, const_cast<char* const*>(argv.data()), envp.data());
    posix_spawn_file_actions_destroy(&fa);
    if (src != 0) {
        close(fds[0]); close(fds[1]);
        if (err) *err = "posix_spawn of the " + what + ": " + strerror(src);
        return CRO_ERR_EXEC;
    }
    close(fds[1]);
    const size_t cap = head + max_tail;
    out->clear();
    bool timed_out = false;
    const auto until = std::chrono::steady_clock::now() + std::chrono::milliseconds(deadline_ms > 0 ? deadline_ms : 30000);
    for (;;) {
        const auto left = std::chrono::duration_cast<std::chrono::milliseconds>(until - std::chrono::steady_clock::now()).count();
        if (left <= 0) { timed_out = true; break; }
        struct pollfd pfd = {fds[0], POLLIN, 0};
        const int pr = poll(&pfd, 1, (int)std::min<long long>(left, 1000));
        if (pr < 0 && errno == EINTR) continue;
        if (pr < 0) break;
        if (pr == 0) continue;
        unsigned char tmp[4096];
        const ssize_t n = read(fds[0], tmp, sizeof tmp);
        if (n < 0 && errno == EINTR) continue;
        if (n <= 0) break;                                     // EOF: the helper is done
        out->append(reinterpret_cast<const char*>(tmp), std::min<size_t>((size_t)n, cap - out->size()));
    }
    close(fds[0]);
    int status = 0;
    if (timed_out) {
        kill(pid, SIGKILL);
        waitpid(pid, &status, 0);
        if (err) *err = what + " for " + uuid + " exceeded its deadline of " + std::to_string(deadline_ms) + " ms and was killed";
        return CRO_ERR_DEADLINE;
    }
    // the pipe is closed; give the process until the deadline to exit, then reap it
    for (;;) {
        const pid_t w = waitpid(pid, &status, WNOHANG);
        if (w == pid) break;
        if (w < 0 && errno != EINTR) break;
        if (std::chrono::steady_clock::now() > until) {
            kill(pid, SIGKILL);
            waitpid(pid, &status, 0);
            break;
        }
        usleep(1000);
    }
    const int code = WIFEXITED(status) ? WEXITSTATUS(status) : -1;
    if (code == 3) {
        if (err) *err = "device '" + uuid + "' is not visible to a fresh CUDA process";
        return CRO_ERR_NO_DEVICE;
    }
    const uint64_t n_tail = out->size() >= head && tail ? tail(reinterpret_cast<const unsigned char*>(out->data()), out->size()) : 0;
    if (out->size() < head || n_tail > max_tail || out->size() != head + n_tail || (code != 0 && code != 1)) {
        if (err) *err = what + " for " + uuid + " failed (exit " + std::to_string(code) + ", " + std::to_string(out->size()) + " result bytes)";
        return CRO_ERR_EXEC;
    }
    return CRO_OK;
}

int RunHelper(const std::string& helper_path, const std::string& uuid, uint64_t sweep_bytes, int deadline_ms,
              cro_probe_result* out, std::string* err) {
    const std::string mib = std::to_string(std::max<uint64_t>(1, sweep_bytes >> 20));
    std::string got;
    const int rc = RunHelperRaw(helper_path, "probe helper", uuid, {"probe-raw", uuid, mib}, deadline_ms, sizeof *out, 0, nullptr,
                                &got, err);
    if (rc != CRO_OK) return rc;
    memcpy(out, got.data(), sizeof *out);
    if (out->abi_version != CRO_ABI_VERSION) {
        if (err) *err = "probe helper speaks another ABI version";
        return CRO_ERR_ABI_MISMATCH;
    }
    return out->status;
}

}  // namespace inventory
}  // namespace cro
