// sm_holder.cu — test-only (tests/test_held_sms.py): keep k SMs of a device busy for a bounded window, the way another
// kernel of the same process would, so the per-SM probes can be checked on a GPU where some SMs are taken.
//
// hold() launches k CTAs of one kernel on a non-blocking stream of its own.  Each CTA asks for the device's whole
// opt-in shared memory (227 KiB on an H100; with the 1 KiB the SM reserves per CTA that is all of its 228 KiB), so no
// other CTA can share its SM while it runs.  Each CTA publishes its %smid in its own slot of mapped pinned memory (the
// resident count is the number of published slots), then thread 0 polls a mapped release flag and %globaltimer while
// the other threads wait at a barrier: the CTA exits at release() or at start + hold_ns, whichever comes first.  Not
// part of the library or its build; nothing here touches a device setting.
#include <cuda_runtime.h>

#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <thread>

namespace {

constexpr unsigned kPublished = 0x80000000u;   // a slot's mark: the CTA is resident and the low bits are its %smid
constexpr int kMaxCtas = 1024;

struct Holder {
    int device = -1;
    cudaStream_t stream = nullptr;
    volatile unsigned* slots = nullptr;        // mapped pinned: [kMaxCtas] SM slots, then the release flag
    unsigned* d_slots = nullptr;               // the same memory as the device sees it
    int k = 0;
    bool active = false;
    char error[512] = {0};
};
Holder g;

int fail(const char* what, cudaError_t e) {
    snprintf(g.error, sizeof g.error, "%s: %s", what, cudaGetErrorString(e));
    return -1;
}

__global__ void __launch_bounds__(128) hold_sm(unsigned* slots, unsigned long long hold_ns) {
    extern __shared__ unsigned char smem[];     // never touched: asking for it is what holds the SM
    if (threadIdx.x == 0) {
        unsigned smid;
        unsigned long long t0, t;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
        *(volatile unsigned*)(slots + blockIdx.x) = kPublished | smid;
        __threadfence_system();
        const volatile unsigned* release = slots + kMaxCtas;
        do {
            __nanosleep(2000);
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        } while (!*release && t - t0 < hold_ns);
    }
    __syncthreads();
}

}  // namespace

extern "C" {

const char* holder_error() { return g.error; }

// Opt-in shared memory per block of `device` (what each holding CTA asks for), or -1.
int holder_smem_bytes(int device) {
    int v = 0;
    cudaError_t e = cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
    return e == cudaSuccess ? v : fail("cudaDeviceGetAttribute", e);
}

// Holds k SMs of `device` for at most hold_ns.  Returns 0 once all k CTAs are resident, with their %smid in
// smids[0 .. k); -1 (holder_error() says why) on a CUDA error or when they are not all resident within 2 s, in which
// case the CTAs that did start are released before it returns.
int holder_hold(int device, int k, unsigned long long hold_ns, unsigned* smids) {
    if (g.active) { snprintf(g.error, sizeof g.error, "a hold is already active"); return -1; }
    if (k < 1 || k > kMaxCtas) { snprintf(g.error, sizeof g.error, "k = %d is out of range", k); return -1; }
    cudaError_t e;
    if ((e = cudaSetDevice(device))) return fail("cudaSetDevice", e);
    if (g.device != device) {
        if (g.device >= 0) { snprintf(g.error, sizeof g.error, "the holder is bound to device %d", g.device); return -1; }
        unsigned* h = nullptr;
        if ((e = cudaHostAlloc((void**)&h, (kMaxCtas + 1) * sizeof(unsigned), cudaHostAllocMapped))) return fail("cudaHostAlloc", e);
        g.slots = h;
        if ((e = cudaHostGetDevicePointer((void**)&g.d_slots, h, 0))) return fail("cudaHostGetDevicePointer", e);
        if ((e = cudaStreamCreateWithFlags(&g.stream, cudaStreamNonBlocking))) return fail("cudaStreamCreateWithFlags", e);
        g.device = device;
    }
    const int smem = holder_smem_bytes(device);
    if (smem <= 0) return -1;
    if ((e = cudaFuncSetAttribute(hold_sm, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)))
        return fail("cudaFuncSetAttribute", e);
    memset((void*)g.slots, 0, (kMaxCtas + 1) * sizeof(unsigned));
    hold_sm<<<k, 128, (size_t)smem, g.stream>>>(g.d_slots, hold_ns);
    if ((e = cudaGetLastError())) return fail("hold_sm launch", e);
    g.k = k;
    g.active = true;
    const auto until = std::chrono::steady_clock::now() + std::chrono::seconds(2);
    for (;;) {
        int n = 0;
        for (int i = 0; i < k; ++i) n += (g.slots[i] & kPublished) ? 1 : 0;
        if (n == k) break;
        if (std::chrono::steady_clock::now() > until) {
            snprintf(g.error, sizeof g.error, "only %d of %d holding CTAs were resident after 2 s", n, k);
            g.slots[kMaxCtas] = 1;
            cudaStreamSynchronize(g.stream);
            g.active = false;
            return -1;
        }
        std::this_thread::sleep_for(std::chrono::microseconds(20));
    }
    for (int i = 0; i < k; ++i) smids[i] = g.slots[i] & ~kPublished;
    return 0;
}

// Ends the hold (a no-op when none is active) and waits for its CTAs to exit.
int holder_release() {
    if (!g.active) return 0;
    g.slots[kMaxCtas] = 1;
    g.active = false;
    cudaError_t e = cudaStreamSynchronize(g.stream);
    return e ? fail("cudaStreamSynchronize", e) : 0;
}

}  // extern "C"
