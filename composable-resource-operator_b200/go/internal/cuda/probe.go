// Package cuda is the thin cgo shim over libcroprobe (include/croprobe.h).
//
// UNCOMPILED IN THIS REPOSITORY'S BUILD IMAGE: there is no Go toolchain there
// (`go version`: command not found).  Every behaviour claimed for this file is
// exercised through the same C entry points by the ctypes tests in tests/.
//
// It is a new sibling of internal/utils (SURVEY.md §1, layer L1c) and is called
// from handleAttachingState at the two slots the reference fills with
// utils.RunNvidiaSmi (internal/controller/composableresource_controller.go:259)
// and utils.CheckGPUVisible (:275).
package cuda

/*
#cgo CFLAGS: -I${SRCDIR}/../../../../include
#cgo LDFLAGS: -lcroprobe -ldl -lpthread
#include <stdlib.h>
#include "croprobe.h"
*/
import "C"

import (
	"fmt"
	"runtime"
	"sync"
	"unsafe"
)

// ProbeResult mirrors cro_probe_result (512 bytes, integer-only).
type ProbeResult struct {
	Status       int32
	CudaOrdinal  int32
	DeviceMinor  int32
	GPUUUID      string
	PCIBusID     string
	SweepBytes   uint64
	ChecksumXor  uint64
	ChecksumSum  uint64
	ChecksumWsum uint64 // position-weighted sum: every word's place matters
	Nonce        uint32 // probe number on this device; every probe writes a fresh pattern
	CopyVerified uint8  // copy sweeps whose destination was re-read and matched the closed form
	FailCode     uint8  // CRO_FAIL_*: which device-side check failed first
	FailIndex    uint8
	P2POk        uint8 // bit j: NVLink read / push / chase through peer j verified
	FillNs       uint64
	ReadBestNs   uint64
	CopyBestNs   uint64
	P2PReadNs    [8]uint64
	P2PWriteNs   [8]uint64
	P2PLatencyNs [8]uint32
	EccErrors    uint32 // uncorrected volatile ECC errors (NVML), read at init / full-box probe / failed probe
	Annotations  string // Go-marshalled map[string]string of cohdi.io/probe-* keys
}

// OK mirrors `probe.OK` in SURVEY.md §3.3.
func (r ProbeResult) OK() bool { return r.Status == C.CRO_OK }

// Options are the env-style knobs (SURVEY.md §5: env vars with validated values).
type Options struct {
	SweepBytes uint64 // 0 = 4 GiB
	DeadlineMs int32  // a Go ctx cannot cross cgo; pass its remaining time here
	Flags      uint32
}

// Context is the long-lived probe context.  Create it once per manager
// process; it is safe for concurrent use (per-device mutexes inside the
// library, cudaSetDevice in every entry point, so goroutine migration between
// OS threads is harmless).
type Context struct {
	mu sync.Mutex
	h  *C.cro_ctx
}

func errorOf(h *C.cro_ctx, rc C.int) error {
	if rc == C.CRO_OK {
		return nil
	}
	buf := (*C.char)(C.malloc(1024))
	defer C.free(unsafe.Pointer(buf))
	detail := ""
	if h != nil && C.cro_last_error(h, buf, 1024) == C.CRO_OK {
		detail = ": " + C.GoString(buf)
	}
	// stable prefix, surfaced verbatim into Status.Error by requeueOnErr
	// (internal/controller/composableresource_controller.go:423-433)
	return fmt.Errorf("cuda probe failed: %s%s", C.GoString(C.cro_strerror(rc)), detail)
}

// NewContext wraps cro_probe_init.
func NewContext(o Options) (*Context, error) {
	var opts C.cro_opts
	opts.abi_version = C.CRO_ABI_VERSION
	opts.sweep_bytes = C.uint64_t(o.SweepBytes)
	opts.deadline_ms = C.int32_t(o.DeadlineMs)
	opts.flags = C.uint32_t(o.Flags)
	c := &Context{}
	if rc := C.cro_probe_init(&opts, &c.h); rc != C.CRO_OK {
		return nil, errorOf(nil, rc)
	}
	runtime.SetFinalizer(c, func(c *Context) { c.Close() })
	return c, nil
}

// Close wraps cro_probe_destroy.
func (c *Context) Close() {
	c.mu.Lock()
	defer c.mu.Unlock()
	if c.h != nil {
		C.cro_probe_destroy(c.h)
		c.h = nil
	}
}

// EnumerateCSV returns the text `nvidia-smi --query-gpu=<query>
// --format=csv,noheader,nounits` would print, so the UNCHANGED parser at
// internal/utils/gpus.go:903-916 can consume it ("No devices were found" for
// an empty box, gpus.go:896).
func (c *Context) EnumerateCSV(query string) (string, error) {
	var devs [C.CRO_MAX_DEVICES]C.cro_dev_info
	var n C.int
	if rc := C.cro_enumerate(c.h, &devs[0], C.CRO_MAX_DEVICES, &n); rc != C.CRO_OK {
		return "", errorOf(c.h, rc)
	}
	q := C.CString(query)
	defer C.free(unsafe.Pointer(q))
	buf := (*C.char)(C.malloc(8192)) // caller-allocated; C does not retain it
	defer C.free(unsafe.Pointer(buf))
	var ln C.size_t
	if rc := C.cro_emit_csv(&devs[0], n, q, buf, 8192, &ln); rc != C.CRO_OK {
		return "", errorOf(c.h, rc)
	}
	return C.GoStringN(buf, C.int(ln)), nil
}

func convert(r *C.cro_probe_result) ProbeResult {
	out := ProbeResult{
		Status: int32(r.status), CudaOrdinal: int32(r.cuda_ordinal), DeviceMinor: int32(r.device_minor),
		GPUUUID: C.GoString(&r.gpu_uuid[0]), PCIBusID: C.GoString(&r.pci_bus_id[0]),
		SweepBytes: uint64(r.sweep_bytes), ChecksumXor: uint64(r.checksum_xor), ChecksumSum: uint64(r.checksum_sum),
		ChecksumWsum: uint64(r.checksum_wsum), Nonce: uint32(r.nonce), CopyVerified: uint8(r.copy_verified),
		FailCode: uint8(r.fail_code), FailIndex: uint8(r.fail_index), P2POk: uint8(r.p2p_ok),
		FillNs: uint64(r.fill_ns), ReadBestNs: uint64(r.read_best_ns), CopyBestNs: uint64(r.copy_best_ns),
		EccErrors: uint32(r.ecc_errors),
	}
	for j := 0; j < 8; j++ {
		out.P2PReadNs[j] = uint64(r.p2p_read_ns[j])
		out.P2PWriteNs[j] = uint64(r.p2p_write_ns[j])
		out.P2PLatencyNs[j] = uint32(r.p2p_latency_ns_x16[j]) / 16
	}
	buf := (*C.char)(C.malloc(4096))
	defer C.free(unsafe.Pointer(buf))
	var ln C.size_t
	if C.cro_emit_probe_annotations_json(r, buf, 4096, &ln) == C.CRO_OK {
		out.Annotations = C.GoStringN(buf, C.int(ln))
	}
	return out
}

// ProbeAll wraps cro_probe_all: concurrent probe of every attached GPU, NVLink
// rounds, one NCCL all-gather of the result structs.
func (c *Context) ProbeAll() ([]ProbeResult, error) {
	var res [C.CRO_MAX_DEVICES]C.cro_probe_result
	var n C.int
	rc := C.cro_probe_all(c.h, &res[0], C.CRO_MAX_DEVICES, &n)
	if rc != C.CRO_OK && rc != C.CRO_ERR_CHECKSUM {
		return nil, errorOf(c.h, rc)
	}
	out := make([]ProbeResult, 0, int(n))
	for i := 0; i < int(n); i++ {
		out = append(out, convert(&res[i]))
	}
	return out, nil
}

// ProbeUUID probes the one device whose UUID is deviceID (Status.DeviceID,
// internal/controller/composableresource_controller.go:231-233).  The library
// re-reads the node's inventory on every call (the reference execs a fresh
// nvidia-smi per reconcile, internal/utils/gpus.go:666-689): a device this
// context holds is probed in process, a device that reached the node AFTER
// cro_probe_init — which no running CUDA process can see — is probed by a
// one-shot helper process with its own cuInit.  found=false (CRO_ERR_NO_DEVICE)
// mirrors the reference's "not yet visible" (false, nil) + RequeueAfter 30 s.
func (c *Context) ProbeUUID(deviceID string) (r ProbeResult, found bool, err error) {
	id := C.CString(deviceID)
	defer C.free(unsafe.Pointer(id))
	var res C.cro_probe_result
	rc := C.cro_probe_uuid(c.h, id, &res)
	if rc == C.CRO_ERR_NO_DEVICE {
		return r, false, nil
	}
	if rc != C.CRO_OK {
		return convert(&res), true, errorOf(c.h, rc)
	}
	return convert(&res), true, nil
}

// FaultReport is the summary of cro_fault_report an operator acts on: detach,
// retry, or flag the GPU for RMA.
type FaultReport struct {
	Verdict     uint32    // CRO_FAULTS_*
	Complete    bool      // every mismatch is listed and explains the checksums exactly
	Mismatches  [3]uint64 // per pass: 0 post-mortem, 1 fresh pattern, 2 its complement
	Granules    [3]uint64 // 2 MiB granules with a mismatch, per pass
	FlipOr      uint64    // OR of every mismatch's flipped bits
	RetestSeed  uint64
	Words       []FaultWord
	Annotations string // Go-marshalled map[string]string of cohdi.io/probe-fault-* keys
}

// FaultWord is one located word (cro_fault_word).
type FaultWord struct {
	Index    uint64 // region word index: half A first, then half B
	Expected uint64
	Actual   uint64
	Passes   uint32 // bit p: pass p saw it
}

// LocateFaults runs cro_locate_faults on the in-process device whose UUID is
// deviceID, typically right after its probe failed with CRO_ERR_CHECKSUM.
// retest adds the fresh-pattern and complement passes that tell a stuck cell
// from a one-off error.  A device probed through the helper process has no
// resident region here and is an error.
func (c *Context) LocateFaults(deviceID string, retest bool) (FaultReport, error) {
	var devs [C.CRO_MAX_DEVICES]C.cro_dev_info
	var n C.int
	if rc := C.cro_enumerate(c.h, &devs[0], C.CRO_MAX_DEVICES, &n); rc != C.CRO_OK {
		return FaultReport{}, errorOf(c.h, rc)
	}
	idx := C.int(-1)
	for i := 0; i < int(n); i++ {
		if C.GoString(&devs[i].gpu_uuid[0]) == deviceID && devs[i].flags&C.CRO_DEV_IN_PROCESS != 0 {
			idx = C.int(devs[i].dev_index)
		}
	}
	if idx < 0 {
		return FaultReport{}, fmt.Errorf("cuda fault locator: %s is not a device of this context", deviceID)
	}
	var opts C.cro_locate_opts
	if retest {
		opts.flags = C.CRO_LOCATE_RETEST
	}
	var rep C.cro_fault_report
	var words [256]C.cro_fault_word
	var got C.int
	rc := C.cro_locate_faults(c.h, idx, &opts, &rep, &words[0], 256, &got)
	if rc != C.CRO_OK && rc != C.CRO_ERR_CHECKSUM {
		return FaultReport{}, errorOf(c.h, rc)
	}
	out := FaultReport{Verdict: uint32(rep.verdict), Complete: rep.complete != 0, FlipOr: uint64(rep.flip_or),
		RetestSeed: uint64(rep.retest_seed)}
	for p := 0; p < 3; p++ {
		out.Mismatches[p] = uint64(rep.pass[p].mismatches)
		out.Granules[p] = uint64(rep.pass[p].granules)
	}
	for i := 0; i < int(got); i++ {
		w := words[i]
		out.Words = append(out.Words, FaultWord{uint64(w.word_index), uint64(w.expected), uint64(w.actual), uint32(w.passes)})
	}
	buf := (*C.char)(C.malloc(4096))
	defer C.free(unsafe.Pointer(buf))
	var ln C.size_t
	if C.cro_emit_fault_annotations_json(&rep, &words[0], got, buf, 4096, &ln) == C.CRO_OK {
		out.Annotations = C.GoStringN(buf, C.int(ln))
	}
	return out, nil
}

// LinkResult is the summary of cro_link_result an operator reads after
// composing a GPU: whether every byte crossed the PCIe link intact, at what
// rates, and how the link trained.
type LinkResult struct {
	OK          bool
	FirstFail   uint32            // CRO_LINK_CHECK_*, CRO_LINK_NO_FAIL when every check passed
	Bytes       uint64            // L
	LegBytes    [8]uint64         // per CRO_LINK_LEG_*
	LegNs       [8]uint64         // CUDA events around each leg
	DuplexNs    uint64            // span of the copy-engine duplex leg
	ChaseNs     uint64            // chase through host memory, all hops
	ChaseHops   uint32
	Degraded    uint32            // CRO_LINK_DEGRADED_*
	Faults      []LinkFault
	Annotations string // Go-marshalled map[string]string of cohdi.io/probe-link-* keys
}

// LinkFault is one mismatching word (cro_link_fault).
type LinkFault struct {
	Check     uint32
	Index     uint64 // word index in the buffer the check verified
	Expected  uint64
	Actual    uint64
	HostValue uint64 // the host buffer's word: equal to Actual, the corruption reached host memory
}

func linkResult(res *C.cro_link_result, faults []C.cro_link_fault, got C.int) LinkResult {
	out := LinkResult{OK: res.status == C.CRO_OK, FirstFail: uint32(res.first_fail), Bytes: uint64(res.bytes),
		DuplexNs: uint64(res.ce_duplex_span_ns), ChaseNs: uint64(res.chase_ns), ChaseHops: uint32(res.chase_hops),
		Degraded: uint32(res.degraded)}
	for g := 0; g < int(C.CRO_LINK_LEGS); g++ {
		out.LegBytes[g] = uint64(res.leg[g].bytes)
		out.LegNs[g] = uint64(res.leg[g].ns)
	}
	for i := 0; i < int(got); i++ {
		f := faults[i]
		out.Faults = append(out.Faults, LinkFault{uint32(f.check), uint64(f.word_index), uint64(f.expected), uint64(f.actual),
			uint64(f.host_value)})
	}
	buf := (*C.char)(C.malloc(4096))
	defer C.free(unsafe.Pointer(buf))
	var ln C.size_t
	if C.cro_emit_link_annotations_json(res, buf, 4096, &ln) == C.CRO_OK {
		out.Annotations = C.GoStringN(buf, C.int(ln))
	}
	return out
}

// ProbeHostLinkByUUID runs cro_probe_host_link_uuid with its defaults: the host
// link probe of any GPU on the node through the helper process, the form an
// operator calls once after a passing HBM probe of a freshly composed GPU
// (INTEGRATION.md §2).  A mismatch is a result, not an error; found is false
// when the node does not list the GPU.
func (c *Context) ProbeHostLinkByUUID(deviceID string) (r LinkResult, found bool, err error) {
	id := C.CString(deviceID)
	defer C.free(unsafe.Pointer(id))
	var res C.cro_link_result
	var faults [256]C.cro_link_fault
	var got C.int
	rc := C.cro_probe_host_link_uuid(c.h, id, nil, 0, &res, &faults[0], 256, &got, nil)
	if rc == C.CRO_ERR_NO_DEVICE {
		return r, false, nil
	}
	if rc != C.CRO_OK && rc != C.CRO_ERR_CHECKSUM {
		return r, true, errorOf(c.h, rc)
	}
	return linkResult(&res, faults[:], got), true, nil
}

// ProbeHostLink runs cro_probe_host_link with its defaults on the in-process
// device whose UUID is deviceID.  ProbeHostLinkByUUID is the form an operator
// should call: it also reaches a GPU composed after the manager started.
func (c *Context) ProbeHostLink(deviceID string) (LinkResult, error) {
	var devs [C.CRO_MAX_DEVICES]C.cro_dev_info
	var n C.int
	if rc := C.cro_enumerate(c.h, &devs[0], C.CRO_MAX_DEVICES, &n); rc != C.CRO_OK {
		return LinkResult{}, errorOf(c.h, rc)
	}
	idx := C.int(-1)
	for i := 0; i < int(n); i++ {
		if C.GoString(&devs[i].gpu_uuid[0]) == deviceID && devs[i].flags&C.CRO_DEV_IN_PROCESS != 0 {
			idx = C.int(devs[i].dev_index)
		}
	}
	if idx < 0 {
		return LinkResult{}, fmt.Errorf("cuda host link probe: %s is not a device of this context", deviceID)
	}
	var res C.cro_link_result
	var faults [256]C.cro_link_fault
	var got C.int
	rc := C.cro_probe_host_link(c.h, idx, nil, &res, &faults[0], 256, &got)
	if rc != C.CRO_OK && rc != C.CRO_ERR_CHECKSUM {
		return LinkResult{}, errorOf(c.h, rc)
	}
	return linkResult(&res, faults[:], got), nil
}

// ComputeResult is the summary of cro_compute_result an operator reads: whether
// every SM computed the exact answer on its tensor cores and CUDA cores, and
// which SMs did not.
type ComputeResult struct {
	OK          bool
	Verdict     uint32            // CRO_COMPUTE_NONE / _SM / _ALL
	SMCount     uint32
	Covered     [5]uint32         // SMs seen per CRO_COMPUTE_LEG_*
	Mismatches  [5]uint64         // wrong elements of the last iteration, per leg
	BadSMs      []uint32          // SMs that failed any leg, ascending
	Faults      []ComputeFault
	Annotations string // Go-marshalled map[string]string of cohdi.io/probe-compute-* keys
}

// ComputeFault is one wrong element (cro_compute_fault).
type ComputeFault struct {
	Leg, SM, Row, Col uint32
	Expected, Actual  int32
}

func computeResult(res *C.cro_compute_result, sms []C.cro_compute_sm, nSMs C.int, faults []C.cro_compute_fault,
	got C.int) ComputeResult {
	out := ComputeResult{OK: res.status == C.CRO_OK, Verdict: uint32(res.verdict), SMCount: uint32(res.sm_count)}
	for l := 0; l < int(C.CRO_COMPUTE_LEGS); l++ {
		out.Covered[l] = uint32(res.leg[l].sms_covered)
		out.Mismatches[l] = uint64(res.leg[l].mismatches)
	}
	for i := 0; i < int(nSMs); i++ {
		for l := 0; l < int(C.CRO_COMPUTE_LEGS); l++ {
			if sms[i].leg[l].mark != 0 {
				out.BadSMs = append(out.BadSMs, uint32(sms[i].smid))
				break
			}
		}
	}
	for i := 0; i < int(got); i++ {
		f := faults[i]
		out.Faults = append(out.Faults, ComputeFault{uint32(f.leg), uint32(f.smid), uint32(f.row), uint32(f.col),
			int32(f.expected), int32(f.actual)})
	}
	buf := (*C.char)(C.malloc(4096))
	defer C.free(unsafe.Pointer(buf))
	var ln C.size_t
	if C.cro_emit_compute_annotations_json(res, buf, 4096, &ln) == C.CRO_OK {
		out.Annotations = C.GoStringN(buf, C.int(ln))
	}
	return out
}

// ProbeComputeByUUID runs cro_probe_compute_uuid with its defaults: the compute
// probe of any GPU on the node through the helper process, the form an operator
// calls after a passing HBM probe of a freshly composed GPU and after a locator
// verdict of not-reproduced (INTEGRATION.md §2).  A mismatch or a failed launch
// (CRO_ERR_CUDA) is a result, not an error; found is false when the node does
// not list the GPU.
func (c *Context) ProbeComputeByUUID(deviceID string) (r ComputeResult, found bool, err error) {
	id := C.CString(deviceID)
	defer C.free(unsafe.Pointer(id))
	var res C.cro_compute_result
	sms := make([]C.cro_compute_sm, C.CRO_COMPUTE_MAX_SMS)
	var faults [256]C.cro_compute_fault
	var nSMs, got C.int
	rc := C.cro_probe_compute_uuid(c.h, id, nil, 0, &res, &sms[0], C.CRO_COMPUTE_MAX_SMS, &nSMs, &faults[0], 256, &got, nil)
	if rc == C.CRO_ERR_NO_DEVICE {
		return r, false, nil
	}
	if rc != C.CRO_OK && rc != C.CRO_ERR_CHECKSUM && rc != C.CRO_ERR_CUDA {
		return r, true, errorOf(c.h, rc)
	}
	return computeResult(&res, sms, nSMs, faults[:], got), true, nil
}

// ProbeCompute runs cro_probe_compute with its defaults on the in-process
// device whose UUID is deviceID.  ProbeComputeByUUID is the form an operator
// should call: it also reaches a GPU composed after the manager started.
func (c *Context) ProbeCompute(deviceID string) (ComputeResult, error) {
	var devs [C.CRO_MAX_DEVICES]C.cro_dev_info
	var n C.int
	if rc := C.cro_enumerate(c.h, &devs[0], C.CRO_MAX_DEVICES, &n); rc != C.CRO_OK {
		return ComputeResult{}, errorOf(c.h, rc)
	}
	idx := C.int(-1)
	for i := 0; i < int(n); i++ {
		if C.GoString(&devs[i].gpu_uuid[0]) == deviceID && devs[i].flags&C.CRO_DEV_IN_PROCESS != 0 {
			idx = C.int(devs[i].dev_index)
		}
	}
	if idx < 0 {
		return ComputeResult{}, fmt.Errorf("cuda compute probe: %s is not a device of this context", deviceID)
	}
	var res C.cro_compute_result
	sms := make([]C.cro_compute_sm, C.CRO_COMPUTE_MAX_SMS)
	var faults [256]C.cro_compute_fault
	var nSMs, got C.int
	rc := C.cro_probe_compute(c.h, idx, nil, &res, &sms[0], C.CRO_COMPUTE_MAX_SMS, &nSMs, &faults[0], 256, &got)
	if rc != C.CRO_OK && rc != C.CRO_ERR_CHECKSUM {
		return ComputeResult{}, errorOf(c.h, rc)
	}
	return computeResult(&res, sms, nSMs, faults[:], got), nil
}

// PrecisionResult is the summary of cro_precision_result an operator reads:
// whether every SM computed the exact answer, bit for bit, in FP64 (DMMA,
// DFMA), TF32, FP16 (f32 and f16 accumulation, HFMA2) and E5M2, and which SMs
// did not.
type PrecisionResult struct {
	OK          bool
	Verdict     uint32            // CRO_COMPUTE_NONE / _SM / _ALL
	SMCount     uint32
	Covered     [7]uint32         // SMs seen per CRO_PRECISION_LEG_*
	Mismatches  [7]uint64         // wrong elements of the last iteration, per leg
	BadSMs      []uint32          // SMs that failed any leg, ascending
	Faults      []PrecisionFault
	Annotations string // Go-marshalled map[string]string of cohdi.io/probe-precision-* keys
}

// PrecisionFault is one wrong element (cro_precision_fault): the exact answer
// and the accumulator's raw bits.
type PrecisionFault struct {
	Leg, SM, Row, Col uint32
	Expected          int64
	ActualBits        uint64
}

func precisionResult(res *C.cro_precision_result, sms []C.cro_precision_sm, nSMs C.int, faults []C.cro_precision_fault,
	got C.int) PrecisionResult {
	out := PrecisionResult{OK: res.status == C.CRO_OK, Verdict: uint32(res.verdict), SMCount: uint32(res.sm_count)}
	for l := 0; l < int(C.CRO_PRECISION_LEGS); l++ {
		out.Covered[l] = uint32(res.leg[l].sms_covered)
		out.Mismatches[l] = uint64(res.leg[l].mismatches)
	}
	for i := 0; i < int(nSMs); i++ {
		for l := 0; l < int(C.CRO_PRECISION_LEGS); l++ {
			if sms[i].leg[l].mark != 0 {
				out.BadSMs = append(out.BadSMs, uint32(sms[i].smid))
				break
			}
		}
	}
	for i := 0; i < int(got); i++ {
		f := faults[i]
		out.Faults = append(out.Faults, PrecisionFault{uint32(f.leg), uint32(f.smid), uint32(f.row), uint32(f.col),
			int64(f.expected), uint64(f.actual_bits)})
	}
	buf := (*C.char)(C.malloc(4096))
	defer C.free(unsafe.Pointer(buf))
	var ln C.size_t
	if C.cro_emit_precision_annotations_json(res, buf, 4096, &ln) == C.CRO_OK {
		out.Annotations = C.GoStringN(buf, C.int(ln))
	}
	return out
}

// ProbePrecisionByUUID runs cro_probe_precision_uuid with its defaults: the
// precision probe of any GPU on the node through the helper process, the form
// an operator calls next to the compute probe, after a passing HBM probe of a
// freshly composed GPU and before it goes to an FP64 or FP16 tenant
// (INTEGRATION.md §2f).  A mismatch or a failed launch (CRO_ERR_CUDA) is a
// result, not an error; found is false when the node does not list the GPU.
func (c *Context) ProbePrecisionByUUID(deviceID string) (r PrecisionResult, found bool, err error) {
	id := C.CString(deviceID)
	defer C.free(unsafe.Pointer(id))
	var res C.cro_precision_result
	sms := make([]C.cro_precision_sm, C.CRO_PRECISION_MAX_SMS)
	var faults [256]C.cro_precision_fault
	var nSMs, got C.int
	rc := C.cro_probe_precision_uuid(c.h, id, nil, 0, &res, &sms[0], C.CRO_PRECISION_MAX_SMS, &nSMs, &faults[0], 256, &got, nil)
	if rc == C.CRO_ERR_NO_DEVICE {
		return r, false, nil
	}
	if rc != C.CRO_OK && rc != C.CRO_ERR_CHECKSUM && rc != C.CRO_ERR_CUDA {
		return r, true, errorOf(c.h, rc)
	}
	return precisionResult(&res, sms, nSMs, faults[:], got), true, nil
}

// ProbePrecision runs cro_probe_precision with its defaults on the in-process
// device whose UUID is deviceID.  ProbePrecisionByUUID is the form an operator
// should call: it also reaches a GPU composed after the manager started.
func (c *Context) ProbePrecision(deviceID string) (PrecisionResult, error) {
	var devs [C.CRO_MAX_DEVICES]C.cro_dev_info
	var n C.int
	if rc := C.cro_enumerate(c.h, &devs[0], C.CRO_MAX_DEVICES, &n); rc != C.CRO_OK {
		return PrecisionResult{}, errorOf(c.h, rc)
	}
	idx := C.int(-1)
	for i := 0; i < int(n); i++ {
		if C.GoString(&devs[i].gpu_uuid[0]) == deviceID && devs[i].flags&C.CRO_DEV_IN_PROCESS != 0 {
			idx = C.int(devs[i].dev_index)
		}
	}
	if idx < 0 {
		return PrecisionResult{}, fmt.Errorf("cuda precision probe: %s is not a device of this context", deviceID)
	}
	var res C.cro_precision_result
	sms := make([]C.cro_precision_sm, C.CRO_PRECISION_MAX_SMS)
	var faults [256]C.cro_precision_fault
	var nSMs, got C.int
	rc := C.cro_probe_precision(c.h, idx, nil, &res, &sms[0], C.CRO_PRECISION_MAX_SMS, &nSMs, &faults[0], 256, &got)
	if rc != C.CRO_OK && rc != C.CRO_ERR_CHECKSUM {
		return PrecisionResult{}, errorOf(c.h, rc)
	}
	return precisionResult(&res, sms, nSMs, faults[:], got), nil
}

// SparseResult is the summary of cro_sparse_result an operator reads: whether
// every SM computed the exact answer with 2:4 structured-sparsity wgmma in s8,
// E4M3, E5M2, BF16, F16 and TF32 (1:2), and which SMs did not.
type SparseResult struct {
	OK          bool
	Verdict     uint32            // CRO_COMPUTE_NONE / _SM / _ALL
	SMCount     uint32
	Covered     [6]uint32         // SMs seen per CRO_SPARSE_LEG_*
	Mismatches  [6]uint64         // wrong elements of the last iteration, per leg
	BadSMs      []uint32          // SMs that failed any leg, ascending
	Faults      []SparseFault
	Annotations string // Go-marshalled map[string]string of cohdi.io/probe-sparse-* keys
}

// SparseFault is one wrong element (cro_sparse_fault): the exact answer and
// the accumulator's raw 32 bits (int32 for S8, f32 otherwise).
type SparseFault struct {
	Leg, SM, Row, Col uint32
	Expected          int32
	ActualBits        uint32
}

// ProbeSparseByUUID runs cro_probe_sparse_uuid with its defaults: the sparse
// probe of any GPU on the node through the helper process, the form an
// operator calls next to the compute and precision probes, before a freshly
// composed GPU goes to a tenant running 2:4-pruned inference (INTEGRATION.md
// §2h).  A mismatch or a failed launch (CRO_ERR_CUDA) is a result, not an
// error; found is false when the node does not list the GPU.
func (c *Context) ProbeSparseByUUID(deviceID string) (r SparseResult, found bool, err error) {
	id := C.CString(deviceID)
	defer C.free(unsafe.Pointer(id))
	var res C.cro_sparse_result
	sms := make([]C.cro_sparse_sm, C.CRO_SPARSE_MAX_SMS)
	var faults [256]C.cro_sparse_fault
	var nSMs, got C.int
	rc := C.cro_probe_sparse_uuid(c.h, id, nil, 0, &res, &sms[0], C.CRO_SPARSE_MAX_SMS, &nSMs, &faults[0], 256, &got, nil)
	if rc == C.CRO_ERR_NO_DEVICE {
		return r, false, nil
	}
	if rc != C.CRO_OK && rc != C.CRO_ERR_CHECKSUM && rc != C.CRO_ERR_CUDA {
		return r, true, errorOf(c.h, rc)
	}
	r = SparseResult{OK: res.status == C.CRO_OK, Verdict: uint32(res.verdict), SMCount: uint32(res.sm_count)}
	for l := 0; l < int(C.CRO_SPARSE_LEGS); l++ {
		r.Covered[l] = uint32(res.leg[l].sms_covered)
		r.Mismatches[l] = uint64(res.leg[l].mismatches)
	}
	for i := 0; i < int(nSMs); i++ {
		for l := 0; l < int(C.CRO_SPARSE_LEGS); l++ {
			if sms[i].leg[l].mark != 0 {
				r.BadSMs = append(r.BadSMs, uint32(sms[i].smid))
				break
			}
		}
	}
	for i := 0; i < int(got); i++ {
		f := faults[i]
		r.Faults = append(r.Faults, SparseFault{uint32(f.leg), uint32(f.smid), uint32(f.row), uint32(f.col),
			int32(f.expected), uint32(f.actual_bits)})
	}
	buf := (*C.char)(C.malloc(4096))
	defer C.free(unsafe.Pointer(buf))
	var ln C.size_t
	if C.cro_emit_sparse_annotations_json(&res, buf, 4096, &ln) == C.CRO_OK {
		r.Annotations = C.GoStringN(buf, C.int(ln))
	}
	return r, true, nil
}

// WarpMMAResult is the summary of cro_warpmma_result an operator reads:
// whether every SM computed the exact answer with warp-synchronous mma.sync in
// s8, F16, BF16, TF32 and F16 accumulation from ldmatrix fragments, and moved
// a tile through ldmatrix, movmatrix and stmatrix intact, and which SMs did not.
type WarpMMAResult struct {
	OK          bool
	Verdict     uint32    // CRO_COMPUTE_NONE / _SM / _ALL
	SMCount     uint32
	Covered     [6]uint32 // SMs seen per CRO_WARPMMA_LEG_*
	Mismatches  [6]uint64 // wrong elements of the last iteration, per leg
	BadSMs      []uint32  // SMs that failed any leg, ascending
	Faults      []WarpMMAFault
	Annotations string // Go-marshalled map[string]string of cohdi.io/probe-warpmma-* keys
}

// WarpMMAFault is one wrong element (cro_warpmma_fault): the exact answer and
// the value's raw bits (int32 for S8, f32 for F16 / BF16 / TF32, f16 for
// F16ACC, the 16-bit word for MOVE).
type WarpMMAFault struct {
	Leg, SM, Row, Col uint32
	Expected          int32
	ActualBits        uint32
}

// ProbeWarpMMAByUUID runs cro_probe_warpmma_uuid with its defaults: the
// warp-MMA probe of any GPU on the node through the helper process, the form
// an operator calls next to the compute, precision and sparse probes, before a
// freshly composed GPU goes to a tenant whose kernels drive the tensor cores
// with mma.sync, such as FlashAttention-2 (INTEGRATION.md §2j).  A mismatch or
// a failed launch (CRO_ERR_CUDA) is a result, not an error; found is false
// when the node does not list the GPU.
func (c *Context) ProbeWarpMMAByUUID(deviceID string) (r WarpMMAResult, found bool, err error) {
	id := C.CString(deviceID)
	defer C.free(unsafe.Pointer(id))
	var res C.cro_warpmma_result
	sms := make([]C.cro_warpmma_sm, C.CRO_WARPMMA_MAX_SMS)
	var faults [256]C.cro_warpmma_fault
	var nSMs, got C.int
	rc := C.cro_probe_warpmma_uuid(c.h, id, nil, 0, &res, &sms[0], C.CRO_WARPMMA_MAX_SMS, &nSMs, &faults[0], 256, &got, nil)
	if rc == C.CRO_ERR_NO_DEVICE {
		return r, false, nil
	}
	if rc != C.CRO_OK && rc != C.CRO_ERR_CHECKSUM && rc != C.CRO_ERR_CUDA {
		return r, true, errorOf(c.h, rc)
	}
	r = WarpMMAResult{OK: res.status == C.CRO_OK, Verdict: uint32(res.verdict), SMCount: uint32(res.sm_count)}
	for l := 0; l < int(C.CRO_WARPMMA_LEGS); l++ {
		r.Covered[l] = uint32(res.leg[l].sms_covered)
		r.Mismatches[l] = uint64(res.leg[l].mismatches)
	}
	for i := 0; i < int(nSMs); i++ {
		for l := 0; l < int(C.CRO_WARPMMA_LEGS); l++ {
			if sms[i].leg[l].mark != 0 {
				r.BadSMs = append(r.BadSMs, uint32(sms[i].smid))
				break
			}
		}
	}
	for i := 0; i < int(got); i++ {
		f := faults[i]
		r.Faults = append(r.Faults, WarpMMAFault{uint32(f.leg), uint32(f.smid), uint32(f.row), uint32(f.col),
			int32(f.expected), uint32(f.actual_bits)})
	}
	buf := (*C.char)(C.malloc(4096))
	defer C.free(unsafe.Pointer(buf))
	var ln C.size_t
	if C.cro_emit_warpmma_annotations_json(&res, buf, 4096, &ln) == C.CRO_OK {
		r.Annotations = C.GoStringN(buf, C.int(ln))
	}
	return r, true, nil
}

// ScanResult is the summary of cro_scan_report an operator reads: whether every
// free byte of the GPU's memory held what was written, how much was covered,
// and the memory's own health record from NVML.
type ScanResult struct {
	Status       int32     // CRO_OK, CRO_ERR_CHECKSUM or CRO_ERR_CUDA
	CudaError    int32     // cudaError_t of a failed element (CRO_ERR_CUDA)
	Health       uint32    // CRO_SCAN_HEALTH_* bits; never change Status
	Seed         uint64
	CoveredBytes uint64
	FreeBytes    uint64
	Mismatches   [2]uint64 // per compare pass: 0 against the pattern, 1 against its complement
	Words        []ScanWord
	Annotations  string // Go-marshalled map[string]string of cohdi.io/hbm-scan-* keys
}

// ScanWord is one mismatching scan word (cro_fault_word of a scan).
type ScanWord struct {
	Index    uint64 // scan word index
	Expected uint64
	Actual   uint64
	Passes   uint32 // bit p: compare pass p saw it
	Chunk    uint32
	Offset   uint64 // word offset in the chunk
}

func scanResult(rep *C.cro_scan_report, words []C.cro_fault_word, got C.int) ScanResult {
	out := ScanResult{Status: int32(rep.status), CudaError: int32(rep.cuda_error), Health: uint32(rep.health),
		Seed: uint64(rep.seed), CoveredBytes: uint64(rep.covered_bytes), FreeBytes: uint64(rep.free_bytes)}
	for p := 0; p < 2; p++ {
		out.Mismatches[p] = uint64(rep.pass[p].mismatches)
	}
	for i := 0; i < int(got); i++ {
		w := words[i]
		k := uint32(w.reserved)
		out.Words = append(out.Words, ScanWord{uint64(w.word_index), uint64(w.expected), uint64(w.actual), uint32(w.passes), k,
			uint64(w.word_index) - uint64(rep.chunk[k].word0)})
	}
	buf := (*C.char)(C.malloc(4096))
	defer C.free(unsafe.Pointer(buf))
	var ln C.size_t
	if C.cro_emit_scan_annotations_json(rep, buf, 4096, &ln) == C.CRO_OK {
		out.Annotations = C.GoStringN(buf, C.int(ln))
	}
	return out
}

// ScanHBMByUUID runs cro_scan_hbm_uuid: the whole-HBM scan of any GPU on the
// node through the helper process, the form to call before handing a freshly
// composed GPU to a tenant.  maxBytes 0 scans all free memory but 1 GiB.  A
// memory fault (CRO_ERR_CUDA) or a mismatch is a result, not an error; found is
// false when the node does not list the GPU.
func (c *Context) ScanHBMByUUID(deviceID string, maxBytes uint64) (r ScanResult, found bool, err error) {
	id := C.CString(deviceID)
	defer C.free(unsafe.Pointer(id))
	var opts C.cro_scan_opts
	opts.max_bytes = C.uint64_t(maxBytes)
	rep := (*C.cro_scan_report)(C.malloc(C.size_t(unsafe.Sizeof(C.cro_scan_report{}))))
	defer C.free(unsafe.Pointer(rep))
	var words [256]C.cro_fault_word
	var got C.int
	rc := C.cro_scan_hbm_uuid(c.h, id, &opts, rep, &words[0], 256, &got)
	if rc == C.CRO_ERR_NO_DEVICE {
		return r, false, nil
	}
	if rc != C.CRO_OK && rc != C.CRO_ERR_CHECKSUM && rc != C.CRO_ERR_CUDA {
		return r, true, errorOf(c.h, rc)
	}
	return scanResult(rep, words[:], got), true, nil
}

// ScanHBM runs cro_scan_hbm on the in-process device whose UUID is deviceID:
// the memory this process can allocate beside what it holds.  ScanHBMByUUID is
// the form an operator should call (INTEGRATION.md "The HBM scan").
func (c *Context) ScanHBM(deviceID string, maxBytes uint64) (ScanResult, error) {
	var devs [C.CRO_MAX_DEVICES]C.cro_dev_info
	var n C.int
	if rc := C.cro_enumerate(c.h, &devs[0], C.CRO_MAX_DEVICES, &n); rc != C.CRO_OK {
		return ScanResult{}, errorOf(c.h, rc)
	}
	idx := C.int(-1)
	for i := 0; i < int(n); i++ {
		if C.GoString(&devs[i].gpu_uuid[0]) == deviceID && devs[i].flags&C.CRO_DEV_IN_PROCESS != 0 {
			idx = C.int(devs[i].dev_index)
		}
	}
	if idx < 0 {
		return ScanResult{}, fmt.Errorf("cuda hbm scan: %s is not a device of this context", deviceID)
	}
	var opts C.cro_scan_opts
	opts.max_bytes = C.uint64_t(maxBytes)
	rep := (*C.cro_scan_report)(C.malloc(C.size_t(unsafe.Sizeof(C.cro_scan_report{}))))
	defer C.free(unsafe.Pointer(rep))
	var words [256]C.cro_fault_word
	var got C.int
	rc := C.cro_scan_hbm(c.h, idx, &opts, rep, &words[0], 256, &got)
	if rc != C.CRO_OK && rc != C.CRO_ERR_CHECKSUM && rc != C.CRO_ERR_CUDA {
		return ScanResult{}, errorOf(c.h, rc)
	}
	return scanResult(rep, words[:], got), nil
}

// SRAMResult is the summary of cro_sram_result an operator reads: whether every
// SM's shared memory and the SM-to-SM network held what was written, which SMs
// or pairs did not, and the SRAM ECC record from NVML.
type SRAMResult struct {
	Status      int32     // CRO_OK, CRO_ERR_CHECKSUM or CRO_ERR_CUDA
	CudaError   int32     // cudaError_t of a failed launch (CRO_ERR_CUDA)
	Verdict     uint32    // CRO_SRAM_NONE / _SM / _LINK / _ALL
	Health      uint32    // CRO_SRAM_HEALTH_* bits; never change Status
	SMCount     uint32
	Covered     [2]uint32 // SMs seen per leg: CRO_SRAM_SMEM, CRO_SRAM_DSMEM
	BytesPerSM  uint64
	BadSMs      []uint32   // SMs that failed the local leg, ascending (at most 16)
	BadPairs    []SRAMPair // network pairs whose SMs both passed the local leg (at most 8)
	Faults      []SRAMFault
	Annotations string // Go-marshalled map[string]string of cohdi.io/probe-sram-* keys
}

// SRAMPair is a failed network pair: From read (Direction CRO_SRAM_DIR_READ)
// or wrote (CRO_SRAM_DIR_WRITE) Owner's shared memory.
type SRAMPair struct {
	From, Owner, Direction uint32
}

// SRAMFault is one failed compare (cro_sram_fault).
type SRAMFault struct {
	Leg, Element, Iteration, SM, PeerSM, Direction, Word uint32
	Expected, Actual                                     uint64
}

func sramResult(res *C.cro_sram_result, faults []C.cro_sram_fault, got C.int) SRAMResult {
	out := SRAMResult{Status: int32(res.status), CudaError: int32(res.cuda_error), Verdict: uint32(res.verdict),
		Health: uint32(res.health), SMCount: uint32(res.sm_count), BytesPerSM: uint64(res.bytes_per_sm)}
	for l := 0; l < 2; l++ {
		out.Covered[l] = uint32(res.leg[l].sms_covered)
	}
	for i := 0; i < int(res.bad_sms) && i < 16; i++ {
		out.BadSMs = append(out.BadSMs, uint32(res.bad_sm[i]))
	}
	for i := 0; i < int(res.bad_pairs) && i < int(C.CRO_SRAM_MAX_PAIRS); i++ {
		p := res.bad_pair[i]
		out.BadPairs = append(out.BadPairs, SRAMPair{uint32(p.from), uint32(p.owner), uint32(p.direction)})
	}
	for i := 0; i < int(got); i++ {
		f := faults[i]
		out.Faults = append(out.Faults, SRAMFault{uint32(f.leg), uint32(f.element), uint32(f.iteration), uint32(f.smid),
			uint32(f.peer_smid), uint32(f.direction), uint32(f.word), uint64(f.expected), uint64(f.actual)})
	}
	buf := (*C.char)(C.malloc(4096))
	defer C.free(unsafe.Pointer(buf))
	var ln C.size_t
	if C.cro_emit_sram_annotations_json(res, buf, 4096, &ln) == C.CRO_OK {
		out.Annotations = C.GoStringN(buf, C.int(ln))
	}
	return out
}

// ProbeSRAMByUUID runs cro_probe_sram_uuid with its defaults: the SRAM probe of
// any GPU on the node through the helper process, the form to call on a freshly
// composed GPU (INTEGRATION.md "The SRAM probe").  A mismatch or a fault
// (CRO_ERR_CUDA) is a result, not an error; found is false when the node does
// not list the GPU.
func (c *Context) ProbeSRAMByUUID(deviceID string) (r SRAMResult, found bool, err error) {
	id := C.CString(deviceID)
	defer C.free(unsafe.Pointer(id))
	var res C.cro_sram_result
	sms := make([]C.cro_sram_sm, C.CRO_SRAM_MAX_SMS)
	var faults [256]C.cro_sram_fault
	var nSMs, got C.int
	rc := C.cro_probe_sram_uuid(c.h, id, nil, &res, &sms[0], C.CRO_SRAM_MAX_SMS, &nSMs, &faults[0], 256, &got)
	if rc == C.CRO_ERR_NO_DEVICE {
		return r, false, nil
	}
	if rc != C.CRO_OK && rc != C.CRO_ERR_CHECKSUM && rc != C.CRO_ERR_CUDA {
		return r, true, errorOf(c.h, rc)
	}
	return sramResult(&res, faults[:], got), true, nil
}

// ProbeSRAM runs cro_probe_sram with its defaults on the in-process device whose
// UUID is deviceID.  ProbeSRAMByUUID is the form an operator should call.
func (c *Context) ProbeSRAM(deviceID string) (SRAMResult, error) {
	var devs [C.CRO_MAX_DEVICES]C.cro_dev_info
	var n C.int
	if rc := C.cro_enumerate(c.h, &devs[0], C.CRO_MAX_DEVICES, &n); rc != C.CRO_OK {
		return SRAMResult{}, errorOf(c.h, rc)
	}
	idx := C.int(-1)
	for i := 0; i < int(n); i++ {
		if C.GoString(&devs[i].gpu_uuid[0]) == deviceID && devs[i].flags&C.CRO_DEV_IN_PROCESS != 0 {
			idx = C.int(devs[i].dev_index)
		}
	}
	if idx < 0 {
		return SRAMResult{}, fmt.Errorf("cuda sram probe: %s is not a device of this context", deviceID)
	}
	var res C.cro_sram_result
	sms := make([]C.cro_sram_sm, C.CRO_SRAM_MAX_SMS)
	var faults [256]C.cro_sram_fault
	var nSMs, got C.int
	rc := C.cro_probe_sram(c.h, idx, nil, &res, &sms[0], C.CRO_SRAM_MAX_SMS, &nSMs, &faults[0], 256, &got)
	if rc != C.CRO_OK && rc != C.CRO_ERR_CHECKSUM && rc != C.CRO_ERR_CUDA {
		return SRAMResult{}, errorOf(c.h, rc)
	}
	return sramResult(&res, faults[:], got), nil
}

// RegfileResult is the summary of cro_regfile_result an operator reads: whether
// every SM's registers held the pattern written into them, which SMs did not,
// and the SRAM ECC record from NVML.
type RegfileResult struct {
	Status      int32  // CRO_OK, CRO_ERR_CHECKSUM or CRO_ERR_CUDA
	CudaError   int32  // cudaError_t of a failed launch (CRO_ERR_CUDA)
	Verdict     uint32 // CRO_REGFILE_NONE / _SM / _ALL
	Health      uint32 // CRO_SRAM_HEALTH_* bits; never change Status
	SMCount     uint32
	Covered     uint32
	RegsHeld    uint32 // registers per SM that held a pattern word (K * T)
	RegsPerSM   uint32
	BadSMs      []uint32 // SMs that failed, ascending (at most 16)
	Faults      []RegfileFault
	Annotations string // Go-marshalled map[string]string of cohdi.io/probe-regfile-* keys
}

// RegfileFault is one failed compare (cro_regfile_fault).
type RegfileFault struct {
	Element, Iteration, SM, Warp, Lane, Slot, Expected, Actual uint32
}

// ProbeRegfileByUUID runs cro_probe_regfile_uuid with its defaults: the
// register-file probe of any GPU on the node through the helper process
// (INTEGRATION.md "The register-file probe").  A mismatch or a fault
// (CRO_ERR_CUDA) is a result, not an error; found is false when the node does
// not list the GPU.
func (c *Context) ProbeRegfileByUUID(deviceID string) (r RegfileResult, found bool, err error) {
	id := C.CString(deviceID)
	defer C.free(unsafe.Pointer(id))
	var res C.cro_regfile_result
	sms := make([]C.cro_regfile_sm, C.CRO_REGFILE_MAX_SMS)
	var faults [256]C.cro_regfile_fault
	var nSMs, got C.int
	rc := C.cro_probe_regfile_uuid(c.h, id, nil, &res, &sms[0], C.CRO_REGFILE_MAX_SMS, &nSMs, &faults[0], 256, &got)
	if rc == C.CRO_ERR_NO_DEVICE {
		return r, false, nil
	}
	if rc != C.CRO_OK && rc != C.CRO_ERR_CHECKSUM && rc != C.CRO_ERR_CUDA {
		return r, true, errorOf(c.h, rc)
	}
	r = RegfileResult{Status: int32(res.status), CudaError: int32(res.cuda_error), Verdict: uint32(res.verdict),
		Health: uint32(res.health), SMCount: uint32(res.sm_count), Covered: uint32(res.sms_covered),
		RegsHeld: uint32(res.slots) * uint32(res.threads), RegsPerSM: uint32(res.regs_per_sm)}
	for i := 0; i < int(res.bad_sms) && i < 16; i++ {
		r.BadSMs = append(r.BadSMs, uint32(res.bad_sm[i]))
	}
	for i := 0; i < int(got); i++ {
		f := faults[i]
		r.Faults = append(r.Faults, RegfileFault{uint32(f.element), uint32(f.iteration), uint32(f.smid), uint32(f.warp),
			uint32(f.lane), uint32(f.slot), uint32(f.expected), uint32(f.actual)})
	}
	buf := (*C.char)(C.malloc(4096))
	defer C.free(unsafe.Pointer(buf))
	var ln C.size_t
	if C.cro_emit_regfile_annotations_json(&res, buf, 4096, &ln) == C.CRO_OK {
		r.Annotations = C.GoStringN(buf, C.int(ln))
	}
	return r, true, nil
}

// XlaneResult is the summary of cro_xlane_result an operator reads: whether
// every SM's shuffle, vote, match, warp-reduce and shared-atomic units gave the
// right answer on every lane, and which SMs and legs did not.
type XlaneResult struct {
	Status      int32  // CRO_OK, CRO_ERR_CHECKSUM or CRO_ERR_CUDA
	CudaError   int32  // cudaError_t of a failed launch (CRO_ERR_CUDA)
	Verdict     uint32 // CRO_XLANE_NONE / _SM / _ALL
	FailedLegs  uint32 // bit per CRO_XLANE_LEG_* that failed
	SMCount     uint32
	Covered     uint32
	BadSMs      []uint32 // SMs that failed, ascending (at most 16)
	Faults      []XlaneFault
	Annotations string // Go-marshalled map[string]string of cohdi.io/probe-xlane-* keys
}

// XlaneFault is one failed compare (cro_xlane_fault).
type XlaneFault struct {
	Leg, Op, Iteration, SM, Warp, Lane, Peer uint32
	Expected, Actual                         uint64
}

// ProbeXlaneByUUID runs cro_probe_xlane_uuid with its defaults: the cross-lane
// probe of any GPU on the node through the helper process (INTEGRATION.md
// "The cross-lane probe").  A mismatch or a fault (CRO_ERR_CUDA) is a result,
// not an error; found is false when the node does not list the GPU.
func (c *Context) ProbeXlaneByUUID(deviceID string) (r XlaneResult, found bool, err error) {
	id := C.CString(deviceID)
	defer C.free(unsafe.Pointer(id))
	var res C.cro_xlane_result
	sms := make([]C.cro_xlane_sm, C.CRO_XLANE_MAX_SMS)
	var faults [256]C.cro_xlane_fault
	var nSMs, got C.int
	rc := C.cro_probe_xlane_uuid(c.h, id, nil, &res, &sms[0], C.CRO_XLANE_MAX_SMS, &nSMs, &faults[0], 256, &got)
	if rc == C.CRO_ERR_NO_DEVICE {
		return r, false, nil
	}
	if rc != C.CRO_OK && rc != C.CRO_ERR_CHECKSUM && rc != C.CRO_ERR_CUDA {
		return r, true, errorOf(c.h, rc)
	}
	r = XlaneResult{Status: int32(res.status), CudaError: int32(res.cuda_error), Verdict: uint32(res.verdict),
		FailedLegs: uint32(res.failed_legs), SMCount: uint32(res.sm_count), Covered: uint32(res.sms_covered)}
	for i := 0; i < int(res.bad_sms) && i < 16; i++ {
		r.BadSMs = append(r.BadSMs, uint32(res.bad_sm[i]))
	}
	for i := 0; i < int(got); i++ {
		f := faults[i]
		r.Faults = append(r.Faults, XlaneFault{uint32(f.leg), uint32(f.op), uint32(f.iteration), uint32(f.smid), uint32(f.warp),
			uint32(f.lane), uint32(f.peer), uint64(f.expected), uint64(f.actual)})
	}
	buf := (*C.char)(C.malloc(4096))
	defer C.free(unsafe.Pointer(buf))
	var ln C.size_t
	if C.cro_emit_xlane_annotations_json(&res, buf, 4096, &ln) == C.CRO_OK {
		r.Annotations = C.GoStringN(buf, C.int(ln))
	}
	return r, true, nil
}

// AluResult is the summary of cro_alu_result an operator reads: whether every
// SM's integer, bit-manipulation, DPX and directed-rounding floating-point
// instructions gave the exact answer on every lane, and which SMs and legs did not.
type AluResult struct {
	Status      int32  // CRO_OK, CRO_ERR_CHECKSUM or CRO_ERR_CUDA
	CudaError   int32  // cudaError_t of a failed launch (CRO_ERR_CUDA)
	Verdict     uint32 // CRO_ALU_NONE / _SM / _ALL
	FailedLegs  uint32 // bit per CRO_ALU_LEG_* that failed
	SMCount     uint32
	Covered     uint32
	BadSMs      []uint32 // SMs that failed, ascending (at most 16)
	Faults      []AluFault
	Annotations string // Go-marshalled map[string]string of cohdi.io/probe-alu-* keys
}

// AluFault is one failed compare (cro_alu_fault): the op, where it ran, its
// operands as the table holds them, and the expected and actual result words.
type AluFault struct {
	Leg, Op, Iteration, SM, Warp, Lane uint32
	In                                 [4]uint64
	Expected, Actual                   [3]uint64
}

// ProbeAluByUUID runs cro_probe_alu_uuid with its defaults: the ALU probe of
// any GPU on the node through the helper process (INTEGRATION.md "The ALU
// probe").  A mismatch or a fault (CRO_ERR_CUDA) is a result, not an error;
// found is false when the node does not list the GPU.
func (c *Context) ProbeAluByUUID(deviceID string) (r AluResult, found bool, err error) {
	id := C.CString(deviceID)
	defer C.free(unsafe.Pointer(id))
	var res C.cro_alu_result
	sms := make([]C.cro_alu_sm, C.CRO_ALU_MAX_SMS)
	var faults [256]C.cro_alu_fault
	var nSMs, got C.int
	rc := C.cro_probe_alu_uuid(c.h, id, nil, &res, &sms[0], C.CRO_ALU_MAX_SMS, &nSMs, &faults[0], 256, &got)
	if rc == C.CRO_ERR_NO_DEVICE {
		return r, false, nil
	}
	if rc != C.CRO_OK && rc != C.CRO_ERR_CHECKSUM && rc != C.CRO_ERR_CUDA {
		return r, true, errorOf(c.h, rc)
	}
	r = AluResult{Status: int32(res.status), CudaError: int32(res.cuda_error), Verdict: uint32(res.verdict),
		FailedLegs: uint32(res.failed_legs), SMCount: uint32(res.sm_count), Covered: uint32(res.sms_covered)}
	for i := 0; i < int(res.bad_sms) && i < 16; i++ {
		r.BadSMs = append(r.BadSMs, uint32(res.bad_sm[i]))
	}
	for i := 0; i < int(got); i++ {
		f := faults[i]
		a := AluFault{Leg: uint32(f.leg), Op: uint32(f.op), Iteration: uint32(f.iteration), SM: uint32(f.smid),
			Warp: uint32(f.warp), Lane: uint32(f.lane)}
		for k := 0; k < 4; k++ {
			a.In[k] = uint64(f.in[k])
		}
		for k := 0; k < 3; k++ {
			a.Expected[k], a.Actual[k] = uint64(f.expected[k]), uint64(f.actual[k])
		}
		r.Faults = append(r.Faults, a)
	}
	buf := (*C.char)(C.malloc(4096))
	defer C.free(unsafe.Pointer(buf))
	var ln C.size_t
	if C.cro_emit_alu_annotations_json(&res, buf, 4096, &ln) == C.CRO_OK {
		r.Annotations = C.GoStringN(buf, C.int(ln))
	}
	return r, true, nil
}

// BarrierResult is the summary of cro_barrier_result an operator reads: whether
// every SM's named barriers, mbarrier phases and transaction counts, and cluster
// barriers with async remote stores behaved exactly, and which SMs, legs and
// (SM, peer SM) pairs did not.
type BarrierResult struct {
	Status      int32  // CRO_OK, CRO_ERR_CHECKSUM or CRO_ERR_CUDA
	CudaError   int32  // cudaError_t of a failed launch (CRO_ERR_CUDA)
	Verdict     uint32 // CRO_BARRIER_NONE / _SM / _ALL / _LINK
	FailedLegs  uint32 // bit per CRO_BARRIER_LEG_* that failed
	SMCount     uint32
	Covered     uint32
	Timeouts    uint64      // mbarrier waits that ran out, among the kept records
	BadSMs      []uint32    // SMs that failed, ascending (at most 16)
	BadPairs    [][2]uint32 // (SM, peer SM) of the failed CLUSTER records (at most 16)
	Faults      []BarrierFault
	Annotations string // Go-marshalled map[string]string of cohdi.io/probe-barrier-* keys
}

// BarrierFault is one failed check (cro_barrier_fault): the leg and row, where
// it ran, its kind, barrier id or form, phase and slot, and the expected and
// actual values.
type BarrierFault struct {
	Leg, Op, Iteration, SM, Warp, Lane, Kind, Bar, Phase, Slot, PeerSM uint32
	Expected, Actual                                                   uint64
}

// ProbeBarrierByUUID runs cro_probe_barrier_uuid with its defaults: the
// barrier probe of any GPU on the node through the helper process, whose
// deadline contains a barrier that never releases (INTEGRATION.md "The barrier
// probe").  A mismatch or a fault (CRO_ERR_CUDA) is a result, not an error;
// found is false when the node does not list the GPU.
func (c *Context) ProbeBarrierByUUID(deviceID string) (r BarrierResult, found bool, err error) {
	id := C.CString(deviceID)
	defer C.free(unsafe.Pointer(id))
	var res C.cro_barrier_result
	sms := make([]C.cro_barrier_sm, C.CRO_BARRIER_MAX_SMS)
	var faults [256]C.cro_barrier_fault
	var nSMs, got C.int
	rc := C.cro_probe_barrier_uuid(c.h, id, nil, &res, &sms[0], C.CRO_BARRIER_MAX_SMS, &nSMs, &faults[0], 256, &got)
	if rc == C.CRO_ERR_NO_DEVICE {
		return r, false, nil
	}
	if rc != C.CRO_OK && rc != C.CRO_ERR_CHECKSUM && rc != C.CRO_ERR_CUDA {
		return r, true, errorOf(c.h, rc)
	}
	r = BarrierResult{Status: int32(res.status), CudaError: int32(res.cuda_error), Verdict: uint32(res.verdict),
		FailedLegs: uint32(res.failed_legs), SMCount: uint32(res.sm_count), Covered: uint32(res.sms_covered),
		Timeouts: uint64(res.timeouts)}
	for i := 0; i < int(res.bad_sms) && i < 16; i++ {
		r.BadSMs = append(r.BadSMs, uint32(res.bad_sm[i]))
	}
	for i := 0; i < int(res.bad_pairs) && i < 16; i++ {
		r.BadPairs = append(r.BadPairs, [2]uint32{uint32(res.bad_pair[i].smid), uint32(res.bad_pair[i].peer_smid)})
	}
	for i := 0; i < int(got); i++ {
		f := faults[i]
		r.Faults = append(r.Faults, BarrierFault{Leg: uint32(f.leg), Op: uint32(f.op), Iteration: uint32(f.iteration),
			SM: uint32(f.smid), Warp: uint32(f.warp), Lane: uint32(f.lane), Kind: uint32(f.kind), Bar: uint32(f.bar),
			Phase: uint32(f.phase), Slot: uint32(f.slot), PeerSM: uint32(f.peer_smid), Expected: uint64(f.expected),
			Actual: uint64(f.actual)})
	}
	buf := (*C.char)(C.malloc(4096))
	defer C.free(unsafe.Pointer(buf))
	var ln C.size_t
	if C.cro_emit_barrier_annotations_json(&res, buf, 4096, &ln) == C.CRO_OK {
		r.Annotations = C.GoStringN(buf, C.int(ln))
	}
	return r, true, nil
}

// L2Result is the summary of cro_l2_result an operator reads: whether the
// L2-resident buffer held what each SM wrote when another SM read it back,
// whether the L2 atomic units gave the right answers, which SMs, buffer offsets
// or counters did not, and the SRAM / L2 ECC record from NVML.
type L2Result struct {
	Status        int32  // CRO_OK, CRO_ERR_CHECKSUM or CRO_ERR_CUDA
	CudaError     int32  // cudaError_t of a failed launch (CRO_ERR_CUDA)
	Verdict       uint32 // CRO_L2_NONE / _SM / _LINE / _ATOMIC / _ALL
	Health        uint32 // CRO_L2_HEALTH_* bits; never change Status
	SMCount       uint32
	Covered       uint32 // SMs that read words of the buffer
	Bytes         uint64 // W
	Overflow      bool   // more mismatches than records kept; counts stay exact
	BadSMs        []uint32
	BadLines      []uint64 // byte offsets into the call's buffer (at most 8)
	A1BadCounters []uint32
	A2BadCounters []uint32
	A2Holes       uint64
	Faults        []L2Fault
	Annotations   string // Go-marshalled map[string]string of cohdi.io/probe-l2-* keys
}

// L2Fault is one failed compare (cro_l2_fault).
type L2Fault struct {
	Element, Iteration, SM, CTA, WriterCTA, WriterSM uint32
	Word, Expected, Actual                           uint64
	Line                                             bool
}

func l2Result(res *C.cro_l2_result, faults []C.cro_l2_fault, got C.int) L2Result {
	out := L2Result{Status: int32(res.status), CudaError: int32(res.cuda_error), Verdict: uint32(res.verdict),
		Health: uint32(res.health), SMCount: uint32(res.sm_count), Covered: uint32(res.sms_covered),
		Bytes: uint64(res.bytes), Overflow: res.overflow != 0, A2Holes: uint64(res.a2_holes)}
	for i := 0; i < int(res.bad_sms) && i < 16; i++ {
		out.BadSMs = append(out.BadSMs, uint32(res.bad_sm[i]))
	}
	for i := 0; i < int(res.bad_lines) && i < int(C.CRO_L2_MAX_LINES); i++ {
		out.BadLines = append(out.BadLines, uint64(res.bad_line[i]))
	}
	for i := 0; i < int(res.a1_bad) && i < int(C.CRO_L2_MAX_COUNTERS); i++ {
		out.A1BadCounters = append(out.A1BadCounters, uint32(res.a1_bad_counter[i]))
	}
	for i := 0; i < int(res.a2_bad) && i < int(C.CRO_L2_MAX_COUNTERS); i++ {
		out.A2BadCounters = append(out.A2BadCounters, uint32(res.a2_bad_counter[i]))
	}
	for i := 0; i < int(got); i++ {
		f := faults[i]
		out.Faults = append(out.Faults, L2Fault{uint32(f.element), uint32(f.iteration), uint32(f.smid), uint32(f.cta),
			uint32(f.writer_cta), uint32(f.writer_smid), uint64(f.word), uint64(f.expected), uint64(f.actual), f.line != 0})
	}
	buf := (*C.char)(C.malloc(4096))
	defer C.free(unsafe.Pointer(buf))
	var ln C.size_t
	if C.cro_emit_l2_annotations_json(res, buf, 4096, &ln) == C.CRO_OK {
		out.Annotations = C.GoStringN(buf, C.int(ln))
	}
	return out
}

// ProbeL2ByUUID runs cro_probe_l2_uuid with its defaults: the L2 probe of any
// GPU on the node through the helper process, the form to call on a freshly
// composed GPU (INTEGRATION.md "The L2 probe").  A mismatch or a fault
// (CRO_ERR_CUDA) is a result, not an error; found is false when the node does
// not list the GPU.
func (c *Context) ProbeL2ByUUID(deviceID string) (r L2Result, found bool, err error) {
	id := C.CString(deviceID)
	defer C.free(unsafe.Pointer(id))
	var res C.cro_l2_result
	sms := make([]C.cro_l2_sm, C.CRO_L2_MAX_SMS)
	var faults [256]C.cro_l2_fault
	var nSMs, got C.int
	rc := C.cro_probe_l2_uuid(c.h, id, nil, &res, &sms[0], C.CRO_L2_MAX_SMS, &nSMs, &faults[0], 256, &got)
	if rc == C.CRO_ERR_NO_DEVICE {
		return r, false, nil
	}
	if rc != C.CRO_OK && rc != C.CRO_ERR_CHECKSUM && rc != C.CRO_ERR_CUDA {
		return r, true, errorOf(c.h, rc)
	}
	return l2Result(&res, faults[:], got), true, nil
}

// ProbeL2 runs cro_probe_l2 with its defaults on the in-process device whose
// UUID is deviceID.  ProbeL2ByUUID is the form an operator should call.
func (c *Context) ProbeL2(deviceID string) (L2Result, error) {
	var devs [C.CRO_MAX_DEVICES]C.cro_dev_info
	var n C.int
	if rc := C.cro_enumerate(c.h, &devs[0], C.CRO_MAX_DEVICES, &n); rc != C.CRO_OK {
		return L2Result{}, errorOf(c.h, rc)
	}
	idx := C.int(-1)
	for i := 0; i < int(n); i++ {
		if C.GoString(&devs[i].gpu_uuid[0]) == deviceID && devs[i].flags&C.CRO_DEV_IN_PROCESS != 0 {
			idx = C.int(devs[i].dev_index)
		}
	}
	if idx < 0 {
		return L2Result{}, fmt.Errorf("cuda l2 probe: %s is not a device of this context", deviceID)
	}
	var res C.cro_l2_result
	sms := make([]C.cro_l2_sm, C.CRO_L2_MAX_SMS)
	var faults [256]C.cro_l2_fault
	var nSMs, got C.int
	rc := C.cro_probe_l2(c.h, idx, nil, &res, &sms[0], C.CRO_L2_MAX_SMS, &nSMs, &faults[0], 256, &got)
	if rc != C.CRO_OK && rc != C.CRO_ERR_CHECKSUM && rc != C.CRO_ERR_CUDA {
		return L2Result{}, errorOf(c.h, rc)
	}
	return l2Result(&res, faults[:], got), nil
}

// HealthResult is the summary of cro_health_result an operator reads: the
// call's status and which checks failed, errored, did not run or fell short of
// every SM, each check that ran as its own Go result, and every annotation.
type HealthResult struct {
	Status      int32  // CRO_OK, CRO_ERR_CHECKSUM, or the first other status a check returned
	Ran         uint32 // CRO_HEALTH_* bits
	Failed      uint32 // ... that returned CRO_ERR_CHECKSUM
	Errored     uint32 // ... that returned another status but CRO_OK
	NotRun      uint32 // selected, but after a check that returned CRO_ERR_CUDA
	Incomplete  uint32 // ran on fewer SMs than the device has; never changes Status
	HelperNs    uint64 // the helper's spawn to exit
	Compute     ComputeResult
	Precision   PrecisionResult
	SRAM        SRAMResult
	L2          L2Result
	Link        LinkResult
	Scan        ScanResult
	Annotations string // Go-marshalled map[string]string: every ran check's keys and cohdi.io/probe-health-*
}

// CheckHealthByUUID runs cro_check_health_uuid: the selected checks (checks 0:
// all six) of any GPU on the node in one helper process, each with its defaults,
// the form to call once after the first passing HBM probe of a freshly composed
// GPU (INTEGRATION.md §2g).  A failed check is a result, not an error; found is
// false when the node does not list the GPU.
func (c *Context) CheckHealthByUUID(deviceID string, checks uint32) (r HealthResult, found bool, err error) {
	id := C.CString(deviceID)
	defer C.free(unsafe.Pointer(id))
	var opts C.cro_health_opts
	opts.checks = C.uint32_t(checks)
	// the result and the record arrays live in C memory: the records struct the call takes holds pointers to them
	res := (*C.cro_health_result)(C.malloc(C.size_t(unsafe.Sizeof(C.cro_health_result{}))))
	defer C.free(unsafe.Pointer(res))
	rec := (*C.cro_health_records)(C.malloc(C.size_t(unsafe.Sizeof(C.cro_health_records{}))))
	defer C.free(unsafe.Pointer(rec))
	*rec = C.cro_health_records{} // the SRAM and L2 per-SM lists stay NULL with cap 0
	alloc := func(n int, size uintptr) unsafe.Pointer { return C.malloc(C.size_t(n) * C.size_t(size)) }
	rec.compute_sms = (*C.cro_compute_sm)(alloc(int(C.CRO_COMPUTE_MAX_SMS), unsafe.Sizeof(C.cro_compute_sm{})))
	rec.compute_sms_cap = C.CRO_COMPUTE_MAX_SMS
	rec.compute_faults = (*C.cro_compute_fault)(alloc(256, unsafe.Sizeof(C.cro_compute_fault{})))
	rec.compute_faults_cap = 256
	rec.precision_sms = (*C.cro_precision_sm)(alloc(int(C.CRO_PRECISION_MAX_SMS), unsafe.Sizeof(C.cro_precision_sm{})))
	rec.precision_sms_cap = C.CRO_PRECISION_MAX_SMS
	rec.precision_faults = (*C.cro_precision_fault)(alloc(256, unsafe.Sizeof(C.cro_precision_fault{})))
	rec.precision_faults_cap = 256
	rec.sram_faults = (*C.cro_sram_fault)(alloc(256, unsafe.Sizeof(C.cro_sram_fault{})))
	rec.sram_faults_cap = 256
	rec.l2_faults = (*C.cro_l2_fault)(alloc(256, unsafe.Sizeof(C.cro_l2_fault{})))
	rec.l2_faults_cap = 256
	rec.link_faults = (*C.cro_link_fault)(alloc(256, unsafe.Sizeof(C.cro_link_fault{})))
	rec.link_faults_cap = 256
	rec.scan_words = (*C.cro_fault_word)(alloc(256, unsafe.Sizeof(C.cro_fault_word{})))
	rec.scan_words_cap = 256
	for _, p := range []unsafe.Pointer{unsafe.Pointer(rec.compute_sms), unsafe.Pointer(rec.compute_faults),
		unsafe.Pointer(rec.precision_sms), unsafe.Pointer(rec.precision_faults), unsafe.Pointer(rec.sram_faults),
		unsafe.Pointer(rec.l2_faults), unsafe.Pointer(rec.link_faults), unsafe.Pointer(rec.scan_words)} {
		defer C.free(p)
	}
	rc := C.cro_check_health_uuid(c.h, id, &opts, 0, res, rec, nil)
	if rc == C.CRO_ERR_NO_DEVICE {
		return r, false, nil
	}
	if rc != C.CRO_OK && res.ran == 0 {
		return r, true, errorOf(c.h, rc)
	}
	r = HealthResult{Status: int32(res.status), Ran: uint32(res.ran), Failed: uint32(res.failed), Errored: uint32(res.errored),
		NotRun: uint32(res.not_run), Incomplete: uint32(res.incomplete), HelperNs: uint64(res.helper_ns)}
	if r.Ran&C.CRO_HEALTH_COMPUTE != 0 {
		r.Compute = computeResult(&res.compute, unsafe.Slice(rec.compute_sms, C.CRO_COMPUTE_MAX_SMS), rec.compute_sms_n,
			unsafe.Slice(rec.compute_faults, 256), rec.compute_faults_n)
	}
	if r.Ran&C.CRO_HEALTH_PRECISION != 0 {
		r.Precision = precisionResult(&res.precision, unsafe.Slice(rec.precision_sms, C.CRO_PRECISION_MAX_SMS), rec.precision_sms_n,
			unsafe.Slice(rec.precision_faults, 256), rec.precision_faults_n)
	}
	if r.Ran&C.CRO_HEALTH_SRAM != 0 {
		r.SRAM = sramResult(&res.sram, unsafe.Slice(rec.sram_faults, 256), rec.sram_faults_n)
	}
	if r.Ran&C.CRO_HEALTH_L2 != 0 {
		r.L2 = l2Result(&res.l2, unsafe.Slice(rec.l2_faults, 256), rec.l2_faults_n)
	}
	if r.Ran&C.CRO_HEALTH_LINK != 0 {
		r.Link = linkResult(&res.link, unsafe.Slice(rec.link_faults, 256), rec.link_faults_n)
	}
	if r.Ran&C.CRO_HEALTH_SCAN != 0 {
		r.Scan = scanResult(&res.scan, unsafe.Slice(rec.scan_words, 256), rec.scan_words_n)
	}
	buf := (*C.char)(C.malloc(65536))
	defer C.free(unsafe.Pointer(buf))
	var ln C.size_t
	if C.cro_emit_health_annotations_json(res, buf, 65536, &ln) == C.CRO_OK {
		r.Annotations = C.GoStringN(buf, C.int(ln))
	}
	return r, true, nil
}

// MetricsText is the Prometheus text exposition of the context's counters and
// per-GPU gauges; a prometheus.Collector registered with
// sigs.k8s.io/controller-runtime/pkg/metrics.Registry (cmd/main.go:66,119-125
// wires that registry) forwards it.
func (c *Context) MetricsText() (string, error) {
	buf := (*C.char)(C.malloc(16384))
	defer C.free(unsafe.Pointer(buf))
	var ln C.size_t
	if rc := C.cro_metrics_text(c.h, buf, 16384, &ln); rc != C.CRO_OK {
		return "", errorOf(c.h, rc)
	}
	return C.GoStringN(buf, C.int(ln)), nil
}

// LocalNodeOp runs one node-side operation of internal/utils/gpus.go on the node
// itself (a cro-node-agent that links libcroprobe): request is
// {"op": "check_no_gpu_loads"|"run_nvidia_smi"|"check_gpu_visible"|"drain",
// "node", "device_id", "device_resource_type", "driver_container",
// "allow_mutation"}.  The flows, their exec sequence and their error strings are
// the reference's (CheckNoGPULoads :88-186, DrainGPU :188-664); the /proc scans
// are native and the nvidia-smi steps (compute apps, drain -q / -m 1 / -r,
// -pm 0) are NVML calls in this process, so a detach pre-flight is a handful of
// library calls instead of 3-8 SPDY execs.  The reply's "error" is what the
// reference would have returned ("" = nil); "exec_log" says how each step ran.
func (c *Context) LocalNodeOp(requestJSON string) (string, error) {
	req := C.CString(requestJSON)
	defer C.free(unsafe.Pointer(req))
	buf := (*C.char)(C.malloc(65536))
	defer C.free(unsafe.Pointer(buf))
	var ln C.size_t
	if rc := C.cro_local_node_op(c.h, req, buf, 65536, &ln); rc != C.CRO_OK {
		return "", errorOf(c.h, rc)
	}
	return C.GoStringN(buf, C.int(ln)), nil
}

// Visible is the decision of utils.CheckGPUVisible (internal/utils/gpus.go:73-84)
// strengthened: listed AND the probe reproduced the HBM pattern.
func Visible(results []ProbeResult, deviceID string) bool {
	for _, r := range results {
		if r.GPUUUID == deviceID {
			return r.OK()
		}
	}
	return false
}
