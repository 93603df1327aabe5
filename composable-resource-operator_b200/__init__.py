"""composable-resource-operator_b200 — H100-native post-attach probe + spec path.

Thin ctypes binding of ``libcroprobe.so`` (the C ABI in ``include/croprobe.h``),
the same entry points a Go host binds with cgo (INTEGRATION.md).  The package
name is not a Python identifier; import it with::

    import importlib
    cro = importlib.import_module("composable-resource-operator_b200")

There is no CPU fallback: if the shared library is missing the import raises,
and ``ProbeContext`` raises ``ProbeError`` when no CUDA device is usable.  The
host-side mirror of the reference interface (parse / decide / emit / attach
step) lives in the library too (``csrc/identity.cpp``, ``csrc/reconcile.cpp``);
this module only marshals arguments.

Reference slots (paths relative to the reference tree):
  enumerate / parse     internal/utils/gpus.go:878-919, 921-962, 1014-1089
  visibility decision   internal/utils/gpus.go:54-86
  attach step           internal/controller/composableresource_controller.go:200-287
  wire structs          internal/cdi/fti/fm/api/*.go, fti/cm/client.go:62-79,
                        sunfish/client.go:48-61, api/v1alpha1/*_types.go
"""
from __future__ import annotations

import ctypes
import json
import os
from typing import Dict, List, Optional, Tuple

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libcroprobe.so")

ABI_VERSION = 2
MAX_DEVICES = 16

OK = 0
ERR_INVALID_ARG, ERR_ABI_MISMATCH, ERR_NO_DEVICE, ERR_CUDA, ERR_OOM = -1, -2, -3, -4, -5
ERR_CHECKSUM, ERR_BUFFER_SMALL, ERR_NCCL, ERR_DEADLINE, ERR_UNSUPPORTED = -6, -7, -8, -9, -10
ERR_PARSE, ERR_EXEC, ERR_P2P, ERR_INTERNAL = -11, -12, -13, -14

F_SKIP_COPY, F_SKIP_P2P, F_SKIP_NCCL, F_NO_NVML, F_VERIFY_COPY, F_LAZY_ALLOC, F_DEGRADE_ON_OOM, F_SKIP_P2P_WRITE = 1, 2, 4, 8, 16, 32, 64, 128
F_TEST_INJECT = 256
READ_AUTO, READ_LDG, READ_TMA, READ_LDG256 = 0, 1, 2, 3
COPY_AUTO, COPY_LDG, COPY_TMA, COPY_TMA_FUSED = 0, 1, 2, 3
DEV_IN_PROCESS, DEV_NEEDS_HELPER = 1, 2
FAIL_NONE, FAIL_EXPECT, FAIL_COPY_SRC, FAIL_READ, FAIL_P2P_READ, FAIL_P2P_PUSH, FAIL_P2P_CHASE, FAIL_STALE = range(8)


class ProbeError(RuntimeError):
    def __init__(self, code: int, msg: str = "") -> None:
        self.code = code
        super().__init__("croprobe error %d (%s)%s" % (code, strerror(code), (": " + msg) if msg else ""))


class Opts(ctypes.Structure):
    _fields_ = [
        ("abi_version", ctypes.c_uint32), ("flags", ctypes.c_uint32),
        ("sweep_bytes", ctypes.c_uint64), ("p2p_bytes", ctypes.c_uint64), ("seed_base", ctypes.c_uint64),
        ("read_sweeps", ctypes.c_uint32), ("copy_sweeps", ctypes.c_uint32), ("latency_hops", ctypes.c_uint32),
        ("read_variant", ctypes.c_uint32), ("copy_variant", ctypes.c_uint32), ("deadline_ms", ctypes.c_int32),
        ("n_devices", ctypes.c_int32), ("devices", ctypes.c_int32 * MAX_DEVICES),
        ("rank_base", ctypes.c_uint32), ("world_override", ctypes.c_uint32),
        ("test_inject_after", ctypes.c_uint32), ("reserved0", ctypes.c_uint32),
        ("test_inject_word", ctypes.c_uint64), ("test_inject_mask", ctypes.c_uint64),
    ]


class DevInfo(ctypes.Structure):
    _fields_ = [
        ("cuda_ordinal", ctypes.c_int32), ("device_minor", ctypes.c_int32),
        ("gpu_uuid", ctypes.c_char * 48), ("pci_bus_id", ctypes.c_char * 24), ("name", ctypes.c_char * 64),
        ("hbm_bytes_total", ctypes.c_uint64), ("sm_count", ctypes.c_uint32),
        ("cc_major", ctypes.c_uint32), ("cc_minor", ctypes.c_uint32), ("identity_source", ctypes.c_uint32),
        ("flags", ctypes.c_uint32), ("dev_index", ctypes.c_int32), ("reserved", ctypes.c_uint32 * 2),
    ]


class ProbeResult(ctypes.Structure):
    """cro_probe_result (ABI 2): written on the device by the finalize kernel, 512 bytes."""
    _fields_ = [
        ("abi_version", ctypes.c_uint32), ("status", ctypes.c_int32),
        ("cuda_ordinal", ctypes.c_int32), ("device_minor", ctypes.c_int32),
        ("gpu_uuid", ctypes.c_char * 48), ("pci_bus_id", ctypes.c_char * 24),
        ("hbm_bytes_total", ctypes.c_uint64), ("sweep_bytes", ctypes.c_uint64), ("seed", ctypes.c_uint64),
        ("checksum_xor", ctypes.c_uint64), ("checksum_sum", ctypes.c_uint64),
        ("fill_ns", ctypes.c_uint64), ("read_best_ns", ctypes.c_uint64), ("read_median_ns", ctypes.c_uint64),
        ("copy_best_ns", ctypes.c_uint64), ("copy_median_ns", ctypes.c_uint64),
        ("sm_count", ctypes.c_uint32), ("sm_clock_mhz", ctypes.c_uint32), ("mem_clock_mhz", ctypes.c_uint32),
        ("ecc_errors", ctypes.c_uint32),
        ("p2p_read_ns", ctypes.c_uint64 * 8), ("p2p_checksum_xor", ctypes.c_uint64 * 8),
        ("p2p_latency_ns_x16", ctypes.c_uint32 * 8), ("p2p_access", ctypes.c_uint8 * 8),
        ("p2p_bytes", ctypes.c_uint64), ("expect_xor", ctypes.c_uint64), ("expect_sum", ctypes.c_uint64),
        ("expect_wsum", ctypes.c_uint64), ("checksum_wsum", ctypes.c_uint64),
        ("copy_checksum_xor", ctypes.c_uint64), ("copy_checksum_sum", ctypes.c_uint64), ("copy_checksum_wsum", ctypes.c_uint64),
        ("total_ns", ctypes.c_uint64), ("p2p_write_ns", ctypes.c_uint64 * 8),
        ("nonce", ctypes.c_uint32), ("rank", ctypes.c_uint8), ("world", ctypes.c_uint8),
        ("read_variant", ctypes.c_uint8), ("copy_variant", ctypes.c_uint8),
        ("read_sweeps", ctypes.c_uint8), ("copy_sweeps", ctypes.c_uint8), ("copy_verified", ctypes.c_uint8),
        ("fail_code", ctypes.c_uint8), ("fail_index", ctypes.c_uint8), ("p2p_ok", ctypes.c_uint8),
        ("reserved8", ctypes.c_uint8 * 2), ("t_start_ns", ctypes.c_uint64),
    ]

    @property
    def checksum(self) -> Tuple[int, int, int]:
        return (self.checksum_xor, self.checksum_sum, self.checksum_wsum)

    @property
    def expect(self) -> Tuple[int, int, int]:
        return (self.expect_xor, self.expect_sum, self.expect_wsum)

    @property
    def copy_checksum(self) -> Tuple[int, int, int]:
        return (self.copy_checksum_xor, self.copy_checksum_sum, self.copy_checksum_wsum)


class SweepResult(ctypes.Structure):
    _fields_ = [("bytes", ctypes.c_uint64), ("ns", ctypes.c_uint64), ("checksum_xor", ctypes.c_uint64),
                ("checksum_sum", ctypes.c_uint64), ("variant", ctypes.c_uint32), ("launches", ctypes.c_uint32),
                ("checksum_wsum", ctypes.c_uint64), ("timer_ns", ctypes.c_uint64)]

    @property
    def checksum(self) -> Tuple[int, int, int]:
        return (self.checksum_xor, self.checksum_sum, self.checksum_wsum)


class SweepTime(ctypes.Structure):
    _fields_ = [("kind", ctypes.c_uint32), ("index", ctypes.c_uint32), ("bytes", ctypes.c_uint64),
                ("event_ns", ctypes.c_uint64), ("timer_ns", ctypes.c_uint64)]


class P2PDetail(ctypes.Structure):
    _fields_ = [("read_ns", ctypes.c_uint64), ("push_ns", ctypes.c_uint64), ("reread_ns", ctypes.c_uint64),
                ("read_xor", ctypes.c_uint64), ("read_sum", ctypes.c_uint64), ("read_wsum", ctypes.c_uint64),
                ("landed_xor", ctypes.c_uint64), ("landed_sum", ctypes.c_uint64), ("landed_wsum", ctypes.c_uint64),
                ("expect_xor", ctypes.c_uint64), ("expect_sum", ctypes.c_uint64), ("expect_wsum", ctypes.c_uint64),
                ("chase_ns", ctypes.c_uint64),
                ("chase_end", ctypes.c_uint32), ("chase_expect", ctypes.c_uint32), ("hops", ctypes.c_uint32), ("access", ctypes.c_uint32)]


class FullBoxTime(ctypes.Structure):
    _fields_ = [("enqueue_ns", ctypes.c_uint64), ("wall_ns", ctypes.c_uint64), ("hbm_ns", ctypes.c_uint64),
                ("p2p_ns", ctypes.c_uint64), ("chase_ns", ctypes.c_uint64), ("gather_ns", ctypes.c_uint64),
                ("rounds", ctypes.c_uint32), ("host_syncs", ctypes.c_uint32), ("gather", ctypes.c_uint32),
                ("reserved", ctypes.c_uint32)]


GATHER_HOST, GATHER_NCCL, GATHER_DEGRADED = 0, 1, 2

# fault locator (cro_locate_faults)
LOCATE_RETEST = 1
LOCATE_RECORDS, LOCATE_PASSES, LOCATE_GRANULE_BYTES = 4096, 3, 2 << 20
FAULTS_NONE, FAULTS_UNCLASSIFIED, FAULTS_NOT_REPRODUCED, FAULTS_PERSISTENT = 0, 1, 2, 3


class LocateOpts(ctypes.Structure):
    _fields_ = [("flags", ctypes.c_uint32), ("reserved0", ctypes.c_uint32),
                ("test_force_first", ctypes.c_uint64), ("test_force_count", ctypes.c_uint64),
                ("test_force_and", ctypes.c_uint64), ("test_force_or", ctypes.c_uint64)]


class FaultWord(ctypes.Structure):
    """One located word: region index (half B starts at S / 8), expected and actual value, bit p = pass p saw it."""
    _fields_ = [("word_index", ctypes.c_uint64), ("expected", ctypes.c_uint64), ("actual", ctypes.c_uint64),
                ("passes", ctypes.c_uint32), ("reserved", ctypes.c_uint32)]


class LocatePass(ctypes.Structure):
    _fields_ = [("halves", ctypes.c_uint32), ("skipped", ctypes.c_uint32), ("seed", ctypes.c_uint64 * 2),
                ("invert", ctypes.c_uint64), ("words_scanned", ctypes.c_uint64), ("mismatches", ctypes.c_uint64),
                ("recorded", ctypes.c_uint64), ("granules", ctypes.c_uint64), ("scan_ns", ctypes.c_uint64),
                ("fold_xor", ctypes.c_uint64 * 2), ("fold_sum", ctypes.c_uint64 * 2), ("fold_wsum", ctypes.c_uint64 * 2)]

    def fold(self, h: int) -> Tuple[int, int, int]:
        """Checksum (xor, sum, weighted sum) of half h as the pass read it."""
        return (self.fold_xor[h], self.fold_sum[h], self.fold_wsum[h])


class FaultReport(ctypes.Structure):
    """cro_fault_report: what cro_locate_faults found, per pass and over all passes."""
    _fields_ = [("status", ctypes.c_int32), ("verdict", ctypes.c_uint32), ("n_passes", ctypes.c_uint32),
                ("complete", ctypes.c_uint32), ("sweep_bytes", ctypes.c_uint64), ("retest_seed", ctypes.c_uint64),
                ("located", ctypes.c_uint64), ("recorded", ctypes.c_uint64), ("flip_or", ctypes.c_uint64),
                ("bit_flips", ctypes.c_uint64 * 64), ("pass_", LocatePass * LOCATE_PASSES)]


# host link probe (cro_probe_host_link, cro_pci_link_path)
(LINK_LEG_CE_D2H, LINK_LEG_SM_H2D, LINK_LEG_CE_H2D, LINK_LEG_SM_D2H, LINK_LEG_SM_DUPLEX_H2D, LINK_LEG_SM_DUPLEX_D2H,
 LINK_LEG_CE_DUPLEX_H2D, LINK_LEG_CE_DUPLEX_D2H) = range(8)
LINK_LEGS = 8
(LINK_CHECK_D2H_COPY, LINK_CHECK_H2D_COPY, LINK_CHECK_SM_WRITE, LINK_CHECK_DUPLEX_WRITE, LINK_CHECK_DUPLEX_D2H_COPY,
 LINK_CHECK_CHASE) = range(6)
LINK_CHECKS, LINK_WORD_CHECKS, LINK_NO_FAIL, LINK_RECORDS = 6, 5, 0xFFFFFFFF, 4096
LINK_DEGRADED_SPEED, LINK_DEGRADED_WIDTH, LINK_DEGRADED_PATH, LINK_DEGRADED_BOTTLENECK = 1, 2, 4, 8
PCI_MAX_HOPS = 8


class PciHop(ctypes.Structure):
    """One PCI function on the path: sysfs bdf, current / max link speed (tenths of a GT/s, 0 unknown) and width."""
    _fields_ = [("bdf", ctypes.c_char * 16), ("cur_speed", ctypes.c_uint32), ("cur_width", ctypes.c_uint32),
                ("max_speed", ctypes.c_uint32), ("max_width", ctypes.c_uint32)]


class PciPath(ctypes.Structure):
    """cro_pci_path: hop[0] is the device, then each ancestor with link files up to the root bus."""
    _fields_ = [("numa_node", ctypes.c_int32), ("n_hops", ctypes.c_uint32), ("bottleneck", ctypes.c_uint32),
                ("truncated", ctypes.c_uint32), ("hop", PciHop * PCI_MAX_HOPS)]


class LinkOpts(ctypes.Structure):
    _fields_ = [("bytes", ctypes.c_uint64), ("hops", ctypes.c_uint32), ("ctas", ctypes.c_uint32),
                ("test_inject_check", ctypes.c_int32), ("reserved0", ctypes.c_uint32),
                ("test_inject_word", ctypes.c_uint64), ("test_inject_mask", ctypes.c_uint64)]


class LinkFault(ctypes.Structure):
    """One mismatching word: the check, its index in the buffer that check verified, expected, actual, and the same
    index of the host buffer involved (equal to actual: the corruption reached host memory)."""
    _fields_ = [("check", ctypes.c_uint32), ("reserved", ctypes.c_uint32), ("word_index", ctypes.c_uint64),
                ("expected", ctypes.c_uint64), ("actual", ctypes.c_uint64), ("host_value", ctypes.c_uint64)]


class LinkLeg(ctypes.Structure):
    _fields_ = [("bytes", ctypes.c_uint64), ("ns", ctypes.c_uint64), ("timer_ns", ctypes.c_uint64)]


class LinkCheck(ctypes.Structure):
    _fields_ = [("words", ctypes.c_uint64), ("mismatches", ctypes.c_uint64), ("recorded", ctypes.c_uint64),
                ("seed", ctypes.c_uint64), ("fold_xor", ctypes.c_uint64), ("fold_sum", ctypes.c_uint64),
                ("fold_wsum", ctypes.c_uint64), ("expect_xor", ctypes.c_uint64), ("expect_sum", ctypes.c_uint64),
                ("expect_wsum", ctypes.c_uint64)]

    @property
    def fold(self) -> Tuple[int, int, int]:
        return (self.fold_xor, self.fold_sum, self.fold_wsum)

    @property
    def expect(self) -> Tuple[int, int, int]:
        return (self.expect_xor, self.expect_sum, self.expect_wsum)


class LinkResult(ctypes.Structure):
    """cro_link_result: legs, checks, chase, path, NUMA placement and replay counters of one host link probe."""
    _fields_ = [("status", ctypes.c_int32), ("first_fail", ctypes.c_uint32), ("bytes", ctypes.c_uint64),
                ("seed", ctypes.c_uint64 * 3), ("call", ctypes.c_uint64), ("leg", LinkLeg * LINK_LEGS),
                ("ce_duplex_span_ns", ctypes.c_uint64), ("check", LinkCheck * LINK_WORD_CHECKS),
                ("chase_hops", ctypes.c_uint32), ("chase_end", ctypes.c_uint32), ("chase_expect", ctypes.c_uint32),
                ("chase_minor", ctypes.c_uint32), ("chase_ns", ctypes.c_uint64), ("dev_numa", ctypes.c_int32),
                ("host_numa", ctypes.c_int32 * 3), ("no_nvml", ctypes.c_uint32), ("degraded", ctypes.c_uint32),
                ("replays_before", ctypes.c_uint64), ("replays_after", ctypes.c_uint64), ("path", PciPath)]


# SM compute probe (cro_probe_compute, cro_compute_expected)
COMPUTE_M, COMPUTE_N, COMPUTE_K = 128, 256, 256
COMPUTE_LEG_S8, COMPUTE_LEG_BF16, COMPUTE_LEG_E4M3, COMPUTE_LEG_FFMA, COMPUTE_LEG_IMAD = range(5)
COMPUTE_LEGS, COMPUTE_ALL_LEGS = 5, 0x1F
COMPUTE_ANSWER_S8, COMPUTE_ANSWER_SMALL = 0, 1
COMPUTE_RECORDS, COMPUTE_MAX_SMS = 4096, 256
COMPUTE_MAX_ITERATIONS, COMPUTE_MAX_ALU_ITERATIONS, COMPUTE_MAX_ROUNDS = 65536, 1024, 64
COMPUTE_NONE, COMPUTE_SM, COMPUTE_ALL = 0, 1, 2
COMPUTE_PERSISTENT, COMPUTE_INTERMITTENT = 1, 2


class ComputeOpts(ctypes.Structure):
    _fields_ = [("iterations", ctypes.c_uint32), ("alu_iterations", ctypes.c_uint32), ("legs", ctypes.c_uint32),
                ("max_rounds", ctypes.c_uint32), ("test_inject_leg", ctypes.c_int32), ("test_inject_sm", ctypes.c_int32),
                ("test_inject_iteration", ctypes.c_uint32), ("test_inject_row", ctypes.c_int32),
                ("test_inject_col", ctypes.c_int32), ("test_inject_mask", ctypes.c_uint32)]


class ComputeLeg(ctypes.Structure):
    _fields_ = [("iterations", ctypes.c_uint32), ("rounds", ctypes.c_uint32), ("ops", ctypes.c_uint64),
                ("ns", ctypes.c_uint64), ("timer_ns", ctypes.c_uint64), ("sms_covered", ctypes.c_uint32),
                ("complete", ctypes.c_uint32), ("mismatches", ctypes.c_uint64), ("fold_mismatches", ctypes.c_uint64),
                ("recorded", ctypes.c_uint64), ("failed_sms", ctypes.c_uint32), ("unpublished", ctypes.c_uint32),
                ("ctas", ctypes.c_uint32), ("slowest_sm", ctypes.c_uint32), ("slow_permille", ctypes.c_uint32),
                ("reserved", ctypes.c_uint32), ("fold", ctypes.c_uint64), ("expect_fold", ctypes.c_uint64)]


class ComputeResult(ctypes.Structure):
    """cro_compute_result: status, verdict and per-leg counts, coverage and times of one compute probe call."""
    _fields_ = [("status", ctypes.c_int32), ("verdict", ctypes.c_uint32), ("seed", ctypes.c_uint64),
                ("call", ctypes.c_uint64), ("sm_count", ctypes.c_uint32), ("legs", ctypes.c_uint32),
                ("host_ref_ns", ctypes.c_uint64), ("nsmid", ctypes.c_uint32), ("bad_sms", ctypes.c_uint32),
                ("bad_sm", ctypes.c_uint16 * 16), ("leg", ComputeLeg * COMPUTE_LEGS)]


class ComputeSmLeg(ctypes.Structure):
    _fields_ = [("mismatches", ctypes.c_uint64), ("fold_mismatches", ctypes.c_uint64), ("ns", ctypes.c_uint64),
                ("cycles", ctypes.c_uint64), ("ctas", ctypes.c_uint32), ("mark", ctypes.c_uint32)]


class ComputeSm(ctypes.Structure):
    """One SM seen by a compute probe call, with its counts, times and COMPUTE_PERSISTENT / _INTERMITTENT mark per leg."""
    _fields_ = [("smid", ctypes.c_uint32), ("reserved", ctypes.c_uint32), ("leg", ComputeSmLeg * COMPUTE_LEGS)]


class ComputeFault(ctypes.Structure):
    """One wrong element of a last iteration's answer: leg, SM, row, column, expected and actual (float legs after
    rounding to int32)."""
    _fields_ = [("leg", ctypes.c_uint32), ("smid", ctypes.c_uint32), ("row", ctypes.c_uint32), ("col", ctypes.c_uint32),
                ("expected", ctypes.c_int32), ("actual", ctypes.c_int32)]


# SM precision probe (cro_probe_precision, cro_precision_expected); verdicts and marks are COMPUTE_*
PRECISION_LEG_F64, PRECISION_LEG_DFMA, PRECISION_LEG_TF32, PRECISION_LEG_F16, PRECISION_LEG_F16ACC, PRECISION_LEG_E5M2, \
    PRECISION_LEG_HFMA2 = range(7)
PRECISION_LEGS, PRECISION_ALL_LEGS = 7, 0x7F
PRECISION_ANSWER_WIDE, PRECISION_ANSWER_SMALL128, PRECISION_ANSWER_SMALL, PRECISION_ANSWER_NARROW = range(4)
PRECISION_ANSWERS = 4
PRECISION_M, PRECISION_N, PRECISION_K, PRECISION_F64_N, PRECISION_F64_K, PRECISION_TF32_K = 128, 256, 256, 64, 128, 128
PRECISION_RECORDS, PRECISION_MAX_SMS = 4096, 256
PRECISION_MAX_ITERATIONS, PRECISION_MAX_ALU_ITERATIONS, PRECISION_MAX_ROUNDS = 65536, 4096, 64


class PrecisionOpts(ctypes.Structure):
    _fields_ = [("iterations", ctypes.c_uint32), ("alu_iterations", ctypes.c_uint32), ("legs", ctypes.c_uint32),
                ("max_rounds", ctypes.c_uint32), ("test_inject_leg", ctypes.c_int32), ("test_inject_sm", ctypes.c_int32),
                ("test_inject_iteration", ctypes.c_uint32), ("test_inject_row", ctypes.c_int32),
                ("test_inject_col", ctypes.c_int32), ("reserved", ctypes.c_uint32), ("test_inject_mask", ctypes.c_uint64)]


class PrecisionResult(ctypes.Structure):
    """cro_precision_result: status, verdict and per-leg counts, coverage and times of one precision probe call."""
    _fields_ = [("status", ctypes.c_int32), ("verdict", ctypes.c_uint32), ("seed", ctypes.c_uint64),
                ("call", ctypes.c_uint64), ("sm_count", ctypes.c_uint32), ("legs", ctypes.c_uint32),
                ("host_ref_ns", ctypes.c_uint64), ("nsmid", ctypes.c_uint32), ("bad_sms", ctypes.c_uint32),
                ("bad_sm", ctypes.c_uint16 * 16), ("leg", ComputeLeg * PRECISION_LEGS)]


class PrecisionSm(ctypes.Structure):
    """One SM seen by a precision probe call, with its counts, times and COMPUTE_PERSISTENT / _INTERMITTENT mark per leg."""
    _fields_ = [("smid", ctypes.c_uint32), ("reserved", ctypes.c_uint32), ("leg", ComputeSmLeg * PRECISION_LEGS)]


class PrecisionFault(ctypes.Structure):
    """One wrong element of a last iteration's answer: leg, SM, row, column, the exact answer and the raw bits got."""
    _fields_ = [("leg", ctypes.c_uint32), ("smid", ctypes.c_uint32), ("row", ctypes.c_uint32), ("col", ctypes.c_uint32),
                ("expected", ctypes.c_int64), ("actual_bits", ctypes.c_uint64)]


# whole-HBM scan (cro_scan_hbm, cro_scan_hbm_uuid, cro_read_hbm_health)
SCAN_CHUNK_BYTES, SCAN_RESERVE_BYTES, SCAN_MAX_CHUNKS, SCAN_PASSES, SCAN_ELEMENTS = 2 << 30, 1 << 30, 128, 2, 4
(SCAN_HEALTH_ECC_CORRECTED_DURING, SCAN_HEALTH_ECC_UNCORRECTED_DURING, SCAN_HEALTH_REMAP_PENDING,
 SCAN_HEALTH_REMAP_FAILURE) = 1, 2, 4, 8
HBM_NVML_ECC_CORRECTED, HBM_NVML_ECC_UNCORRECTED, HBM_NVML_REMAP, HBM_NVML_HISTOGRAM = 1, 2, 4, 8


class ScanOpts(ctypes.Structure):
    _fields_ = [("max_bytes", ctypes.c_uint64), ("reserve_bytes", ctypes.c_uint64), ("seed", ctypes.c_uint64),
                ("deadline_ms", ctypes.c_int32), ("reserved0", ctypes.c_uint32), ("test_chunk_bytes", ctypes.c_uint64),
                ("test_force_first", ctypes.c_uint64), ("test_force_count", ctypes.c_uint64),
                ("test_force_and", ctypes.c_uint64), ("test_force_or", ctypes.c_uint64)]


class HbmHealth(ctypes.Structure):
    """cro_hbm_health: NVML's DRAM ECC counts and row-remapping state; `nvml` has a HBM_NVML_* bit per read answered."""
    _fields_ = [("nvml", ctypes.c_uint32), ("remap_corrected", ctypes.c_uint32), ("remap_uncorrected", ctypes.c_uint32),
                ("remap_pending", ctypes.c_uint32), ("remap_failure", ctypes.c_uint32), ("histogram", ctypes.c_uint32 * 5),
                ("ecc_corrected", ctypes.c_uint64), ("ecc_uncorrected", ctypes.c_uint64)]


class ScanPass(ctypes.Structure):
    _fields_ = [("invert", ctypes.c_uint64), ("words_scanned", ctypes.c_uint64), ("mismatches", ctypes.c_uint64),
                ("recorded", ctypes.c_uint64), ("granules", ctypes.c_uint64), ("bit_flips", ctypes.c_uint64 * 64)]


class ScanChunk(ctypes.Structure):
    _fields_ = [("word0", ctypes.c_uint64), ("bytes", ctypes.c_uint64), ("fold_xor", ctypes.c_uint64 * 2),
                ("fold_sum", ctypes.c_uint64 * 2), ("fold_wsum", ctypes.c_uint64 * 2), ("expect_xor", ctypes.c_uint64),
                ("expect_sum", ctypes.c_uint64), ("expect_wsum", ctypes.c_uint64)]

    def fold(self, p: int) -> Tuple[int, int, int]:
        """Checksum (xor, sum, weighted sum) of the chunk as compare pass p read it."""
        return (self.fold_xor[p], self.fold_sum[p], self.fold_wsum[p])

    @property
    def expect(self) -> Tuple[int, int, int]:
        return (self.expect_xor, self.expect_sum, self.expect_wsum)


class ScanReport(ctypes.Structure):
    """cro_scan_report: sizes, seed, per-pass counts, per-chunk folds, element times and NVML health of one scan."""
    _fields_ = [("status", ctypes.c_int32), ("cuda_error", ctypes.c_int32), ("health", ctypes.c_uint32),
                ("complete", ctypes.c_uint32), ("seed", ctypes.c_uint64), ("total_bytes", ctypes.c_uint64),
                ("free_bytes", ctypes.c_uint64), ("held_bytes", ctypes.c_uint64), ("covered_bytes", ctypes.c_uint64),
                ("n_chunks", ctypes.c_uint32), ("elements_done", ctypes.c_uint32), ("located", ctypes.c_uint64),
                ("recorded", ctypes.c_uint64), ("flip_or", ctypes.c_uint64), ("element_ns", ctypes.c_uint64 * SCAN_ELEMENTS),
                ("alloc_ns", ctypes.c_uint64), ("nvml_ns", ctypes.c_uint64), ("wall_ns", ctypes.c_uint64),
                ("helper_ns", ctypes.c_uint64), ("before", HbmHealth), ("after", HbmHealth),
                ("pass_", ScanPass * SCAN_PASSES), ("chunk", ScanChunk * SCAN_MAX_CHUNKS)]

    def place(self, w: "FaultWord") -> Tuple[int, int]:
        """(chunk number, word offset in the chunk) of a scan word."""
        return w.reserved, w.word_index - self.chunk[w.reserved].word0


# SRAM probe (cro_probe_sram, cro_probe_sram_uuid, cro_read_sram_health)
SRAM_SMEM, SRAM_DSMEM, SRAM_LEGS = 0, 1, 2
SRAM_LEG_SMEM, SRAM_LEG_DSMEM, SRAM_ALL_LEGS = 1, 2, 3
SRAM_ELEMENTS, SRAM_RECORDS, SRAM_MAX_SMS, SRAM_MAX_ITERATIONS, SRAM_MAX_ROUNDS, SRAM_MAX_PAIRS = 6, 4096, 256, 4096, 64, 8
SRAM_NONE, SRAM_SM, SRAM_LINK, SRAM_ALL = 0, 1, 2, 3
SRAM_PERSISTENT, SRAM_INTERMITTENT = 1, 2
SRAM_DIR_LOCAL, SRAM_DIR_READ, SRAM_DIR_WRITE = 0, 1, 2
SRAM_HEALTH_CORRECTED_DURING, SRAM_HEALTH_UNCORRECTED_DURING, SRAM_HEALTH_THRESHOLD_EXCEEDED = 1, 2, 4
SRAM_NVML_ECC_CORRECTED, SRAM_NVML_ECC_UNCORRECTED, SRAM_NVML_STATUS = 1, 2, 4


class SramOpts(ctypes.Structure):
    _fields_ = [("legs", ctypes.c_uint32), ("iterations", ctypes.c_uint32), ("cluster", ctypes.c_uint32),
                ("max_rounds", ctypes.c_uint32), ("deadline_ms", ctypes.c_int32), ("test_inject_leg", ctypes.c_int32),
                ("test_inject_sm", ctypes.c_int32), ("test_inject_element", ctypes.c_uint32),
                ("test_inject_iteration", ctypes.c_uint32), ("test_inject_word", ctypes.c_int32),
                ("test_inject_mask", ctypes.c_uint64)]


class SramHealth(ctypes.Structure):
    """cro_sram_health: NVML's volatile SRAM ECC counts and field-diag threshold flag; `nvml` has a SRAM_NVML_* bit per
    read answered."""
    _fields_ = [("nvml", ctypes.c_uint32), ("threshold_exceeded", ctypes.c_uint32), ("ecc_corrected", ctypes.c_uint64),
                ("ecc_uncorrected", ctypes.c_uint64)]


class SramPair(ctypes.Structure):
    """A network pair that failed: `from` (the reader or the writer, by `direction`) and the owner of the words."""
    _fields_ = [("from_", ctypes.c_uint16), ("owner", ctypes.c_uint16), ("direction", ctypes.c_uint32)]


class SramLeg(ctypes.Structure):
    _fields_ = [("iterations", ctypes.c_uint32), ("rounds", ctypes.c_uint32), ("bytes", ctypes.c_uint64),
                ("ns", ctypes.c_uint64), ("timer_ns", ctypes.c_uint64), ("sms_covered", ctypes.c_uint32),
                ("complete", ctypes.c_uint32), ("mismatches", ctypes.c_uint64 * SRAM_ELEMENTS),
                ("fold_mismatches", ctypes.c_uint64), ("recorded", ctypes.c_uint64), ("failed_sms", ctypes.c_uint32),
                ("unpublished", ctypes.c_uint32), ("ctas", ctypes.c_uint32), ("cluster", ctypes.c_uint32),
                ("fold_xor", ctypes.c_uint64), ("fold_sum", ctypes.c_uint64), ("fold_wsum", ctypes.c_uint64),
                ("expect_xor", ctypes.c_uint64), ("expect_sum", ctypes.c_uint64), ("expect_wsum", ctypes.c_uint64)]

    @property
    def fold(self) -> Tuple[int, int, int]:
        return (self.fold_xor, self.fold_sum, self.fold_wsum)

    @property
    def expect(self) -> Tuple[int, int, int]:
        return (self.expect_xor, self.expect_sum, self.expect_wsum)


class SramResult(ctypes.Structure):
    """cro_sram_result: status, verdict, bad SMs and pairs, per-leg counts, coverage and times, and NVML's SRAM health of
    one SRAM probe call."""
    _fields_ = [("status", ctypes.c_int32), ("verdict", ctypes.c_uint32), ("seed", ctypes.c_uint64),
                ("call", ctypes.c_uint64), ("sm_count", ctypes.c_uint32), ("legs", ctypes.c_uint32),
                ("nsmid", ctypes.c_uint32), ("cuda_error", ctypes.c_int32), ("bytes_per_sm", ctypes.c_uint64),
                ("health", ctypes.c_uint32), ("bad_sms", ctypes.c_uint32), ("bad_sm", ctypes.c_uint16 * 16),
                ("bad_pairs", ctypes.c_uint32), ("sms_listed", ctypes.c_uint32), ("bad_pair", SramPair * SRAM_MAX_PAIRS),
                ("recorded", ctypes.c_uint64), ("wall_ns", ctypes.c_uint64), ("helper_ns", ctypes.c_uint64),
                ("before", SramHealth), ("after", SramHealth), ("leg", SramLeg * SRAM_LEGS)]


class SramSmLeg(ctypes.Structure):
    _fields_ = [("mismatches", ctypes.c_uint64 * SRAM_ELEMENTS), ("fold_mismatches", ctypes.c_uint64),
                ("ns", ctypes.c_uint64), ("cycles", ctypes.c_uint64), ("ctas", ctypes.c_uint32), ("mark", ctypes.c_uint32)]


class SramSm(ctypes.Structure):
    """One SM seen by an SRAM probe call, with its per-element counts, times and SRAM_PERSISTENT / _INTERMITTENT mark
    per leg."""
    _fields_ = [("smid", ctypes.c_uint32), ("reserved", ctypes.c_uint32), ("leg", SramSmLeg * SRAM_LEGS)]


class SramFault(ctypes.Structure):
    """One failed compare: leg, element, iteration, the SM that compared, the other SM of a network pair, the direction,
    the word's offset, expected and actual."""
    _fields_ = [("leg", ctypes.c_uint32), ("element", ctypes.c_uint32), ("iteration", ctypes.c_uint32),
                ("smid", ctypes.c_uint32), ("peer_smid", ctypes.c_uint32), ("direction", ctypes.c_uint32),
                ("word", ctypes.c_uint32), ("reserved", ctypes.c_uint32), ("expected", ctypes.c_uint64),
                ("actual", ctypes.c_uint64)]


# L2 probe (cro_probe_l2, cro_read_l2_health, cro_selftest_l2_classify)
L2_BLOCK_BYTES, L2_MIN_BYTES, L2_MAX_L2_MULTIPLE, L2_ELEMENTS, L2_RECORDS, L2_MAX_SMS = 16384, 1 << 20, 8, 6, 4096, 256
L2_MAX_ITERATIONS, L2_MAX_A1_COUNTERS, L2_MAX_A2_COUNTERS, L2_MAX_LINES, L2_MAX_COUNTERS = 256, 1 << 20, 8192, 8, 8
L2_MARCH, L2_A1, L2_A2 = 0, 1, 2
L2_NONE, L2_SM, L2_LINE, L2_ATOMIC, L2_ALL = 0, 1, 2, 3, 4
L2_PERSISTENT, L2_INTERMITTENT = 1, 2
(L2_HEALTH_SRAM_CORRECTED_DURING, L2_HEALTH_SRAM_UNCORRECTED_DURING, L2_HEALTH_L2_CORRECTED_DURING,
 L2_HEALTH_L2_UNCORRECTED_DURING, L2_HEALTH_THRESHOLD_EXCEEDED, L2_HEALTH_L2_BUCKET) = 1, 2, 4, 8, 16, 32
L2_NVML_SRAM_CORRECTED, L2_NVML_SRAM_UNCORRECTED, L2_NVML_L2_CORRECTED, L2_NVML_L2_UNCORRECTED, L2_NVML_STATUS = 1, 2, 4, 8, 16


class L2Opts(ctypes.Structure):
    _fields_ = [("bytes", ctypes.c_uint64), ("iterations", ctypes.c_uint32), ("a1_counters", ctypes.c_uint32),
                ("a2_counters", ctypes.c_uint32), ("deadline_ms", ctypes.c_int32), ("test_inject_leg", ctypes.c_int32),
                ("test_inject_sm", ctypes.c_int32), ("test_inject_element", ctypes.c_int32),
                ("test_inject_iteration", ctypes.c_uint32), ("test_inject_word", ctypes.c_int64),
                ("test_inject_mask", ctypes.c_uint64)]


class L2Health(ctypes.Structure):
    """cro_l2_health: NVML's volatile SRAM and L2 ECC counts, and the SRAM error status's threshold flag and L2 bucket;
    `nvml` has an L2_NVML_* bit per read answered."""
    _fields_ = [("nvml", ctypes.c_uint32), ("threshold_exceeded", ctypes.c_uint32), ("sram_corrected", ctypes.c_uint64),
                ("sram_uncorrected", ctypes.c_uint64), ("l2_corrected", ctypes.c_uint64), ("l2_uncorrected", ctypes.c_uint64),
                ("unc_bucket_l2", ctypes.c_uint64)]


class L2Result(ctypes.Structure):
    """cro_l2_result: status, verdict, bad SMs, lines and counters, exact counts, the M5 fold against its closed form,
    times and NVML health of one L2 probe call."""
    _fields_ = [("status", ctypes.c_int32), ("verdict", ctypes.c_uint32), ("seed", ctypes.c_uint64),
                ("seed_atomic", ctypes.c_uint64), ("call", ctypes.c_uint64), ("bytes", ctypes.c_uint64),
                ("sm_count", ctypes.c_uint32), ("nsmid", ctypes.c_uint32), ("ctas", ctypes.c_uint32), ("blocks", ctypes.c_uint32),
                ("delta", ctypes.c_uint32), ("iterations", ctypes.c_uint32), ("cuda_error", ctypes.c_int32),
                ("health", ctypes.c_uint32), ("sms_covered", ctypes.c_uint32), ("unpublished", ctypes.c_uint32),
                ("mismatches", ctypes.c_uint64 * L2_ELEMENTS), ("recorded", ctypes.c_uint64), ("overflow", ctypes.c_uint32),
                ("sms_listed", ctypes.c_uint32), ("bad_sms", ctypes.c_uint32), ("bad_lines", ctypes.c_uint32),
                ("bad_sm", ctypes.c_uint16 * 16), ("bad_line", ctypes.c_uint64 * L2_MAX_LINES),
                ("fold_xor", ctypes.c_uint64), ("fold_sum", ctypes.c_uint64), ("fold_wsum", ctypes.c_uint64),
                ("expect_xor", ctypes.c_uint64), ("expect_sum", ctypes.c_uint64), ("expect_wsum", ctypes.c_uint64),
                ("fold_ok", ctypes.c_uint32), ("a1_counters", ctypes.c_uint32), ("a2_counters", ctypes.c_uint32),
                ("a2_tickets", ctypes.c_uint32), ("a1_bad", ctypes.c_uint64), ("a2_holes", ctypes.c_uint64),
                ("a2_bad", ctypes.c_uint64), ("a1_bad_counter", ctypes.c_uint32 * L2_MAX_COUNTERS),
                ("a2_bad_counter", ctypes.c_uint32 * L2_MAX_COUNTERS), ("element_ns", ctypes.c_uint64 * L2_ELEMENTS),
                ("march_ns", ctypes.c_uint64), ("march_bytes", ctypes.c_uint64), ("a1_ns", ctypes.c_uint64),
                ("a1_check_ns", ctypes.c_uint64), ("a2_ns", ctypes.c_uint64), ("a2_check_ns", ctypes.c_uint64),
                ("l2_bytes", ctypes.c_uint64), ("wall_ns", ctypes.c_uint64), ("helper_ns", ctypes.c_uint64),
                ("before", L2Health), ("after", L2Health)]

    @property
    def fold(self) -> Tuple[int, int, int]:
        return (self.fold_xor, self.fold_sum, self.fold_wsum)

    @property
    def expect(self) -> Tuple[int, int, int]:
        return (self.expect_xor, self.expect_sum, self.expect_wsum)


class L2Sm(ctypes.Structure):
    """One SM seen by an L2 probe call: its launches, the reads it saw wrong per element (and in the last iteration),
    the words it read per element and its L2_PERSISTENT / _INTERMITTENT mark."""
    _fields_ = [("smid", ctypes.c_uint32), ("mark", ctypes.c_uint32), ("launches", ctypes.c_uint32),
                ("reserved", ctypes.c_uint32), ("mismatches", ctypes.c_uint64 * L2_ELEMENTS), ("last", ctypes.c_uint64),
                ("words_read", ctypes.c_uint64 * L2_ELEMENTS), ("ns", ctypes.c_uint64)]


class L2Fault(ctypes.Structure):
    """One failed compare: element, iteration, the reader's SM and CTA, the writer's CTA and SM, the word, expected,
    actual and whether the word is a line fault."""
    _fields_ = [("element", ctypes.c_uint32), ("iteration", ctypes.c_uint32), ("smid", ctypes.c_uint32),
                ("cta", ctypes.c_uint32), ("writer_cta", ctypes.c_uint32), ("writer_smid", ctypes.c_uint32),
                ("word", ctypes.c_uint64), ("expected", ctypes.c_uint64), ("actual", ctypes.c_uint64),
                ("line", ctypes.c_uint32), ("reserved", ctypes.c_uint32)]


# test hooks: the compute, precision and SRAM probes' classification of caller-given rounds
# (cro_selftest_sm_legs_classify, cro_selftest_sram_classify)
SM_LEGS_COMPUTE, SM_LEGS_PRECISION = 0, 1


class SmCta(ctypes.Structure):
    """cro_sm_cta: what one CTA of a compute or precision leg publishes at the end of a round."""
    _fields_ = [("stamp", ctypes.c_uint64), ("t0", ctypes.c_uint64), ("t1", ctypes.c_uint64), ("cycles", ctypes.c_uint64),
                ("mismatches", ctypes.c_uint64), ("fold_mismatches", ctypes.c_uint64), ("fold", ctypes.c_uint64),
                ("smid", ctypes.c_uint32), ("nsmid", ctypes.c_uint32)]


class SramCta(ctypes.Structure):
    """cro_sram_cta: what one CTA of an SRAM leg publishes at the end of a round."""
    _fields_ = [("stamp", ctypes.c_uint64), ("t0", ctypes.c_uint64), ("t1", ctypes.c_uint64), ("cycles", ctypes.c_uint64),
                ("count", ctypes.c_uint64 * SRAM_ELEMENTS), ("last", ctypes.c_uint64), ("fold_x", ctypes.c_uint64),
                ("fold_s", ctypes.c_uint64), ("fold_w", ctypes.c_uint64), ("smid", ctypes.c_uint32), ("nsmid", ctypes.c_uint32),
                ("rank", ctypes.c_uint32), ("block", ctypes.c_uint32)]


class SramRecord(ctypes.Structure):
    """cro_sram_record: one word record of an SRAM leg as the device keeps it (peer_block resolved through `round`)."""
    _fields_ = [("element", ctypes.c_uint32), ("iteration", ctypes.c_uint32), ("smid", ctypes.c_uint32),
                ("peer_block", ctypes.c_uint32), ("round", ctypes.c_uint32), ("word", ctypes.c_uint32),
                ("expected", ctypes.c_uint64), ("actual", ctypes.c_uint64)]


# test hook: one sweep kernel between guard bands (cro_selftest_sweep)
(SELFTEST_SWEEP_FILL, SELFTEST_SWEEP_COPY_LDG, SELFTEST_SWEEP_COPY_TMA, SELFTEST_SWEEP_COPY_FUSED, SELFTEST_SWEEP_READ_LDG,
 SELFTEST_SWEEP_READ_TMA, SELFTEST_SWEEP_READ_LDG256, SELFTEST_SWEEP_LOCATE, SELFTEST_SWEEP_FORCE_WORDS,
 SELFTEST_SWEEP_LINK_READ, SELFTEST_SWEEP_LINK_WRITE) = range(1, 12)
SELFTEST_LAYOUT_SRC_DST, SELFTEST_LAYOUT_DST_SRC, SELFTEST_LAYOUT_APART = 1, 2, 3
SELFTEST_GUARD_BYTES, SELFTEST_F_INTERIORS = 2 << 20, 1


class SelftestSweepOpts(ctypes.Structure):
    _fields_ = [("kernel", ctypes.c_uint32), ("layout", ctypes.c_uint32), ("offset", ctypes.c_uint64),
                ("bytes", ctypes.c_uint64), ("seed", ctypes.c_uint64), ("canary", ctypes.c_uint64),
                ("invert", ctypes.c_uint64), ("word0", ctypes.c_uint64), ("force_first", ctypes.c_uint64 * 2),
                ("force_count", ctypes.c_uint64 * 2), ("force_and", ctypes.c_uint64 * 2), ("force_or", ctypes.c_uint64 * 2),
                ("flags", ctypes.c_uint32), ("reserved", ctypes.c_uint32)]


class SelftestSweepOut(ctypes.Structure):
    """cro_selftest_sweep_out: the kernel's slot, the buffer's size and interiors, each interior's fold after the
    kernel, and the word-checking kernels' counters and granules."""
    _fields_ = [("sweep", SweepResult), ("buf_bytes", ctypes.c_uint64), ("at", ctypes.c_uint64 * 2),
                ("after_xor", ctypes.c_uint64 * 2), ("after_sum", ctypes.c_uint64 * 2), ("after_wsum", ctypes.c_uint64 * 2),
                ("mismatches", ctypes.c_uint64), ("claims", ctypes.c_uint64), ("granules", ctypes.c_uint64),
                ("granule_min", ctypes.c_uint64), ("granule_max", ctypes.c_uint64)]

    def after(self, k: int) -> Tuple[int, int, int]:
        """Checksum (xor, sum, weighted sum) of interior k once the kernel was done."""
        return (self.after_xor[k], self.after_sum[k], self.after_wsum[k])


assert ctypes.sizeof(ProbeResult) == 512, ctypes.sizeof(ProbeResult)
assert ctypes.sizeof(ComputeResult) == 600 and ctypes.sizeof(ComputeSm) == 208, ctypes.sizeof(ComputeResult)
assert ctypes.sizeof(PrecisionResult) == 808 and ctypes.sizeof(PrecisionSm) == 288 and ctypes.sizeof(PrecisionFault) == 32 \
    and ctypes.sizeof(PrecisionOpts) == 48, ctypes.sizeof(PrecisionResult)
assert ctypes.sizeof(FaultReport) == 928 and ctypes.sizeof(LocatePass) == 120, ctypes.sizeof(FaultReport)
assert ctypes.sizeof(LinkResult) == 984 and ctypes.sizeof(PciPath) == 272, ctypes.sizeof(LinkResult)
assert ctypes.sizeof(ScanReport) == 12632 and ctypes.sizeof(ScanOpts) == 72, ctypes.sizeof(ScanReport)
assert ctypes.sizeof(SramResult) == 568 and ctypes.sizeof(SramSm) == 168 and ctypes.sizeof(SramFault) == 48, ctypes.sizeof(SramResult)
assert ctypes.sizeof(L2Result) == 616 and ctypes.sizeof(L2Sm) == 128 and ctypes.sizeof(L2Fault) == 56, ctypes.sizeof(L2Result)
assert ctypes.sizeof(SmCta) == 64 and ctypes.sizeof(SramCta) == 128 and ctypes.sizeof(SramRecord) == 40, ctypes.sizeof(SramCta)

# Every symbol include/croprobe.h declares; tests check the library exports all of them.
EXPORTS = [
    "cro_probe_init", "cro_probe_destroy", "cro_device_count", "cro_enumerate", "cro_emit_csv",
    "cro_parse_gpu_csv", "cro_parse_proc_csv", "cro_proc_information_to_line", "cro_check_gpu_visible",
    "cro_normalize", "cro_probe_device", "cro_probe_all", "cro_result_device_ptr", "cro_hbm_fill",
    "cro_hbm_read_checksum", "cro_hbm_copy", "cro_hbm_read_checksum_dst", "cro_hbm_expected_checksum",
    "cro_inject_fault", "cro_read_words", "cro_hbm_read_loop", "cro_hbm_copy_loop", "cro_hbm_fill_loop",
    "cro_device_seed", "cro_launch_count", "cro_emit_status_json", "cro_emit_scalar_status_json",
    "cro_emit_fm_scale_up", "cro_emit_fm_scale_down", "cro_emit_cm_scale_up", "cro_emit_cm_scale_down",
    "cro_emit_sunfish_request", "cro_emit_probe_annotations_json", "cro_fm_parse_scale_up_response",
    "cro_reconcile_attach", "cro_strerror", "cro_last_error", "cro_version", "cro_cm_check_adding_resources",
    "cro_sim_create", "cro_sim_destroy", "cro_sim_apply", "cro_sim_delete", "cro_sim_plant", "cro_sim_run",
    "cro_sim_reconcile_request", "cro_sim_dump", "cro_probe_begin", "cro_probe_end",
    "cro_check_no_gpu_loads", "cro_check_gpu_drain_status", "cro_check_device_file_scan",
    "cro_scan_device_file_holders", "cro_sim_reconcile_resource", "cro_sim_sync_upstream",
    "cro_fabric_check_resource", "cro_fabric_get_resources", "cro_fabric_list_devices",
    "cro_local_node_op", "cro_scan_cmdline_for", "cro_token_from_reply",
    "cro_selftest_exception_barrier", "cro_probe_sweep_times", "cro_p2p_detail_get", "cro_fullbox_times",
    "cro_chase_end", "cro_validate_env", "cro_node_inventory", "cro_probe_uuid", "cro_set_latency_hops", "cro_local_exec", "cro_metrics_text", "cro_describe_wire_type",
    "cro_selftest_probe_finalize", "cro_selftest_p2p_finalize", "cro_selftest_chase", "cro_selftest_sweep",
    "cro_locate_faults", "cro_emit_fault_annotations_json",
    "cro_probe_host_link", "cro_probe_host_link_uuid", "cro_pci_link_path", "cro_emit_link_annotations_json",
    "cro_probe_compute", "cro_probe_compute_uuid", "cro_compute_expected", "cro_emit_compute_annotations_json",
    "cro_probe_precision", "cro_probe_precision_uuid", "cro_precision_expected", "cro_emit_precision_annotations_json",
    "cro_scan_hbm", "cro_scan_hbm_uuid", "cro_read_hbm_health", "cro_emit_scan_annotations_json",
    "cro_probe_sram", "cro_probe_sram_uuid", "cro_read_sram_health", "cro_emit_sram_annotations_json",
    "cro_probe_l2", "cro_probe_l2_uuid", "cro_read_l2_health", "cro_emit_l2_annotations_json", "cro_selftest_l2_classify",
    "cro_selftest_sm_legs_classify", "cro_selftest_sram_classify",
]

# Slot map of a device's sweep-slot array (cro_sweep_slot, 64 bytes each); the cro_selftest_* hooks take such arrays.
SLOT_FILL, SLOT_SWEEP0, MAX_SWEEPS_EACH, SLOT_EXPECT, SLOT_PREFIX, SLOT_P2P0 = 0, 1, 30, 62, 63, 64
SLOT_SCRATCH = SLOT_P2P0 + 3 * MAX_DEVICES
SLOT_COUNT = SLOT_SCRATCH + 4
SLOT_BYTES = 64


def _load() -> ctypes.CDLL:
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "libcroprobe.so is not built (%s): run `python -c 'import __graft_entry__ as g; g.build()'` or "
            "`make -C composable-resource-operator_b200/csrc`.  There is no CPU fallback for the probe path."
            % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    c, sz, psz = ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t)
    vp, i32, u32, u64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint32, ctypes.c_uint64
    out = [c, sz, psz]
    sig = {
        "cro_probe_init": (i32, [ctypes.POINTER(Opts), ctypes.POINTER(vp)]),
        "cro_probe_destroy": (None, [vp]),
        "cro_device_count": (i32, [vp, ctypes.POINTER(i32)]),
        "cro_enumerate": (i32, [vp, ctypes.POINTER(DevInfo), i32, ctypes.POINTER(i32)]),
        "cro_emit_csv": (i32, [ctypes.POINTER(DevInfo), i32, c] + out),
        "cro_parse_gpu_csv": (i32, [c, c, c, c] + out),
        "cro_parse_proc_csv": (i32, [c, c, c, c] + out),
        "cro_proc_information_to_line": (i32, [c] + out),
        "cro_check_gpu_visible": (i32, [ctypes.POINTER(DevInfo), i32, c, ctypes.POINTER(i32)]),
        "cro_normalize": (i32, [i32, c] + out),
        "cro_probe_device": (i32, [vp, i32, ctypes.POINTER(ProbeResult)]),
        "cro_probe_all": (i32, [vp, ctypes.POINTER(ProbeResult), i32, ctypes.POINTER(i32)]),
        "cro_probe_begin": (i32, [vp, i32]),
        "cro_probe_end": (i32, [vp, i32, ctypes.POINTER(ProbeResult)]),
        "cro_result_device_ptr": (i32, [vp, i32, ctypes.POINTER(u64)]),
        "cro_hbm_fill": (i32, [vp, i32, ctypes.POINTER(SweepResult)]),
        "cro_hbm_fill_loop": (i32, [vp, i32, u32, ctypes.POINTER(SweepResult)]),
        "cro_hbm_read_checksum": (i32, [vp, i32, u32, ctypes.POINTER(SweepResult)]),
        "cro_hbm_read_checksum_dst": (i32, [vp, i32, u32, ctypes.POINTER(SweepResult)]),
        "cro_hbm_read_loop": (i32, [vp, i32, u32, u32, ctypes.POINTER(SweepResult)]),
        "cro_hbm_copy": (i32, [vp, i32, u32, ctypes.POINTER(SweepResult)]),
        "cro_hbm_copy_loop": (i32, [vp, i32, u32, u32, ctypes.POINTER(SweepResult)]),
        "cro_hbm_expected_checksum": (i32, [vp, i32, ctypes.POINTER(SweepResult)]),
        "cro_inject_fault": (i32, [vp, i32, u64, u64]),
        "cro_read_words": (i32, [vp, i32, u64, u64, ctypes.POINTER(u64)]),
        "cro_device_seed": (i32, [vp, i32, ctypes.POINTER(u64)]),
        "cro_probe_sweep_times": (i32, [vp, i32, ctypes.POINTER(SweepTime), i32, ctypes.POINTER(i32)]),
        "cro_p2p_detail_get": (i32, [vp, i32, i32, ctypes.POINTER(P2PDetail)]),
        "cro_fullbox_times": (i32, [vp, ctypes.POINTER(FullBoxTime)]),
        "cro_chase_end": (i32, [i32, i32, u32, ctypes.POINTER(u32)]),
        "cro_set_latency_hops": (i32, [vp, u32]),
        "cro_metrics_text": (i32, [vp] + out),
        "cro_validate_env": (i32, [c, c, c, sz]),
        "cro_node_inventory": (i32, [c, ctypes.POINTER(DevInfo), i32, ctypes.POINTER(DevInfo), i32, ctypes.POINTER(i32)]),
        "cro_probe_uuid": (i32, [vp, c, ctypes.POINTER(ProbeResult)]),
        "cro_launch_count": (u64, [vp]),
        "cro_emit_status_json": (i32, [c, c, c, c] + out),
        "cro_emit_scalar_status_json": (i32, [c, c, c, c, c] + out),
        "cro_emit_fm_scale_up": (i32, [c, c, c, c] + out),
        "cro_emit_fm_scale_down": (i32, [c, c, c, c] + out),
        "cro_emit_cm_scale_up": (i32, [c, i32] + out),
        "cro_emit_cm_scale_down": (i32, [c, i32, c] + out),
        "cro_emit_sunfish_request": (i32, [c, ctypes.c_longlong, c, c] + out),
        "cro_emit_probe_annotations_json": (i32, [ctypes.POINTER(ProbeResult)] + out),
        "cro_fm_parse_scale_up_response": (i32, [c, c, c, c, c, sz, c, sz, c, sz]),
        "cro_reconcile_attach": (i32, [vp, c] + out),
        "cro_cm_check_adding_resources": (i32, [c, c, c, c, c, sz, ctypes.POINTER(i32), c, sz, c, sz, c, sz]),
        "cro_sim_create": (i32, [vp, c, ctypes.POINTER(vp)]),
        "cro_sim_destroy": (None, [vp]),
        "cro_sim_apply": (i32, [vp, c, c, sz]),
        "cro_sim_plant": (i32, [vp, c, c, sz]),
        "cro_sim_delete": (i32, [vp, c]),
        "cro_sim_run": (i32, [vp, ctypes.c_longlong] + out),
        "cro_sim_reconcile_request": (i32, [vp, c, c, sz]),
        "cro_sim_dump": (i32, [vp] + out),
        "cro_fabric_check_resource": (i32, [c, c, c, c, c, c, sz]),
        "cro_fabric_get_resources": (i32, [c, c, c, c] + out),
        "cro_fabric_list_devices": (i32, [c] + out),
        "cro_token_from_reply": (i32, [c] + out),
        "cro_selftest_exception_barrier": (i32, [i32]),
        "cro_selftest_probe_finalize": (i32, [vp, i32, ctypes.POINTER(ProbeResult), vp, u64, u64, u64, u32, u32, u32, u32,
                                              ctypes.POINTER(ProbeResult)]),
        "cro_selftest_p2p_finalize": (i32, [vp, i32, ctypes.POINTER(ProbeResult), vp, ctypes.POINTER(vp), ctypes.POINTER(u64),
                                            ctypes.POINTER(u64), ctypes.POINTER(u32), u32, u32, u32, u32, u32, u64, u64]),
        "cro_selftest_chase": (i32, [vp, i32, ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int32), u32, u32,
                                     ctypes.POINTER(u64)]),
        "cro_selftest_sweep": (i32, [vp, i32, ctypes.POINTER(SelftestSweepOpts), ctypes.POINTER(SelftestSweepOut), vp, u64,
                                     ctypes.POINTER(FaultWord), i32, ctypes.POINTER(i32)]),
        "cro_locate_faults": (i32, [vp, i32, ctypes.POINTER(LocateOpts), ctypes.POINTER(FaultReport), ctypes.POINTER(FaultWord),
                                    i32, ctypes.POINTER(i32)]),
        "cro_emit_fault_annotations_json": (i32, [ctypes.POINTER(FaultReport), ctypes.POINTER(FaultWord), i32] + out),
        "cro_probe_host_link": (i32, [vp, i32, ctypes.POINTER(LinkOpts), ctypes.POINTER(LinkResult), ctypes.POINTER(LinkFault),
                                      i32, ctypes.POINTER(i32)]),
        "cro_probe_host_link_uuid": (i32, [vp, c, ctypes.POINTER(LinkOpts), i32, ctypes.POINTER(LinkResult),
                                           ctypes.POINTER(LinkFault), i32, ctypes.POINTER(i32), ctypes.POINTER(u64)]),
        "cro_pci_link_path": (i32, [c, c, ctypes.POINTER(PciPath)]),
        "cro_emit_link_annotations_json": (i32, [ctypes.POINTER(LinkResult)] + out),
        "cro_probe_compute": (i32, [vp, i32, ctypes.POINTER(ComputeOpts), ctypes.POINTER(ComputeResult),
                                    ctypes.POINTER(ComputeSm), i32, ctypes.POINTER(i32), ctypes.POINTER(ComputeFault), i32,
                                    ctypes.POINTER(i32)]),
        "cro_probe_compute_uuid": (i32, [vp, c, ctypes.POINTER(ComputeOpts), i32, ctypes.POINTER(ComputeResult),
                                         ctypes.POINTER(ComputeSm), i32, ctypes.POINTER(i32), ctypes.POINTER(ComputeFault), i32,
                                         ctypes.POINTER(i32), ctypes.POINTER(u64)]),
        "cro_compute_expected": (i32, [i32, u64, ctypes.POINTER(ctypes.c_int32)]),
        "cro_emit_compute_annotations_json": (i32, [ctypes.POINTER(ComputeResult)] + out),
        "cro_probe_precision": (i32, [vp, i32, ctypes.POINTER(PrecisionOpts), ctypes.POINTER(PrecisionResult),
                                      ctypes.POINTER(PrecisionSm), i32, ctypes.POINTER(i32), ctypes.POINTER(PrecisionFault), i32,
                                      ctypes.POINTER(i32)]),
        "cro_probe_precision_uuid": (i32, [vp, c, ctypes.POINTER(PrecisionOpts), i32, ctypes.POINTER(PrecisionResult),
                                           ctypes.POINTER(PrecisionSm), i32, ctypes.POINTER(i32), ctypes.POINTER(PrecisionFault),
                                           i32, ctypes.POINTER(i32), ctypes.POINTER(u64)]),
        "cro_precision_expected": (i32, [i32, u64, ctypes.POINTER(ctypes.c_int64)]),
        "cro_emit_precision_annotations_json": (i32, [ctypes.POINTER(PrecisionResult)] + out),
        "cro_scan_hbm": (i32, [vp, i32, ctypes.POINTER(ScanOpts), ctypes.POINTER(ScanReport), ctypes.POINTER(FaultWord), i32,
                               ctypes.POINTER(i32)]),
        "cro_scan_hbm_uuid": (i32, [vp, c, ctypes.POINTER(ScanOpts), ctypes.POINTER(ScanReport), ctypes.POINTER(FaultWord), i32,
                                    ctypes.POINTER(i32)]),
        "cro_read_hbm_health": (i32, [c, ctypes.POINTER(HbmHealth)]),
        "cro_emit_scan_annotations_json": (i32, [ctypes.POINTER(ScanReport)] + out),
        "cro_probe_sram": (i32, [vp, i32, ctypes.POINTER(SramOpts), ctypes.POINTER(SramResult), ctypes.POINTER(SramSm), i32,
                                 ctypes.POINTER(i32), ctypes.POINTER(SramFault), i32, ctypes.POINTER(i32)]),
        "cro_probe_sram_uuid": (i32, [vp, c, ctypes.POINTER(SramOpts), ctypes.POINTER(SramResult), ctypes.POINTER(SramSm), i32,
                                      ctypes.POINTER(i32), ctypes.POINTER(SramFault), i32, ctypes.POINTER(i32)]),
        "cro_read_sram_health": (i32, [c, ctypes.POINTER(SramHealth)]),
        "cro_emit_sram_annotations_json": (i32, [ctypes.POINTER(SramResult)] + out),
        "cro_probe_l2": (i32, [vp, i32, ctypes.POINTER(L2Opts), ctypes.POINTER(L2Result), ctypes.POINTER(L2Sm), i32,
                               ctypes.POINTER(i32), ctypes.POINTER(L2Fault), i32, ctypes.POINTER(i32)]),
        "cro_probe_l2_uuid": (i32, [vp, c, ctypes.POINTER(L2Opts), ctypes.POINTER(L2Result), ctypes.POINTER(L2Sm), i32,
                                    ctypes.POINTER(i32), ctypes.POINTER(L2Fault), i32, ctypes.POINTER(i32)]),
        "cro_read_l2_health": (i32, [c, ctypes.POINTER(L2Health)]),
        "cro_emit_l2_annotations_json": (i32, [ctypes.POINTER(L2Result)] + out),
        "cro_selftest_l2_classify": (i32, [ctypes.POINTER(L2Result), ctypes.POINTER(L2Sm), i32, ctypes.POINTER(L2Fault), i32]),
        "cro_selftest_sm_legs_classify": (i32, [i32, u32, ctypes.POINTER(u32), u32, u64, ctypes.POINTER(u32),
                                                ctypes.POINTER(SmCta), ctypes.POINTER(u64), ctypes.POINTER(u64), vp, vp, vp, i32,
                                                ctypes.POINTER(i32), vp, i32, ctypes.POINTER(i32)]),
        "cro_selftest_sram_classify": (i32, [u32, u32, u32, u64, u32, u32, u32, u64, ctypes.POINTER(u32),
                                             ctypes.POINTER(SramCta), ctypes.POINTER(u64), ctypes.POINTER(SramRecord),
                                             ctypes.POINTER(SramResult), ctypes.POINTER(SramSm), i32, ctypes.POINTER(i32),
                                             ctypes.POINTER(SramFault), i32, ctypes.POINTER(i32)]),
        "cro_local_node_op": (i32, [vp, c] + out),
        "cro_local_exec": (i32, [c] + out),
        "cro_describe_wire_type": (i32, [c] + out),
        "cro_scan_cmdline_for": (i32, [c, c, ctypes.POINTER(i32)]),
        "cro_sim_reconcile_resource": (i32, [vp, c, c, sz]),
        "cro_sim_sync_upstream": (i32, [vp, c, ctypes.c_longlong, c, sz]),
        "cro_check_no_gpu_loads": (i32, [c, c, c, c, c, c, i32, c, sz]),
        "cro_check_gpu_drain_status": (i32, [c, c, c, c, c, ctypes.POINTER(i32), c, sz]),
        "cro_check_device_file_scan": (i32, [c, c, c, i32, c, sz]),
        "cro_scan_device_file_holders": (i32, [c, c, i32] + out),
        "cro_strerror": (c, [i32]),
        "cro_last_error": (i32, [vp, c, sz]),
        "cro_version": (c, []),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)   # AttributeError == a declared symbol is not exported
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()


def strerror(code: int) -> str:
    return lib.cro_strerror(code).decode()


def version() -> str:
    return lib.cro_version().decode()


def _b(s) -> Optional[bytes]:
    if s is None:
        return None
    return s if isinstance(s, bytes) else s.encode("utf-8", "surrogateescape")


def _text_call(fn, *args, cap: int = 1 << 16) -> Tuple[int, bytes]:
    buf = ctypes.create_string_buffer(cap)
    n = ctypes.c_size_t(0)
    rc = fn(*args, buf, cap, ctypes.byref(n))
    if rc == ERR_BUFFER_SMALL and n.value + 1 > cap:
        return _text_call(fn, *args, cap=n.value + 1)
    return rc, buf.raw[: n.value]


def _text(fn, *args) -> str:
    rc, raw = _text_call(fn, *args)
    if rc != OK:
        raise ProbeError(rc, raw.decode("utf-8", "replace"))
    return raw.decode("utf-8", "surrogateescape")


# ---- host-side mirror of the reference text path (no GPU needed) -------------------
def getGPUInfoFromNvidiaSmiOutput(std_out: str, std_err: str, exec_err: Optional[str], queryArgs: str) -> Tuple[int, str]:
    """Parse rule of getGPUInfoFromNvidiaPod (internal/utils/gpus.go:896-916).
    Returns (code, text): Go JSON of the []map[string]string, or the error text."""
    rc, raw = _text_call(lib.cro_parse_gpu_csv, _b(std_out), _b(std_err), _b(exec_err), _b(queryArgs))
    return rc, raw.decode("utf-8", "surrogateescape")


def getGPUInfoFromProcOutput(std_out: str, std_err: str, exec_err: Optional[str], queryArgs: str) -> Tuple[int, str]:
    """Parse rule of getGPUInfoFromProcInCroNodeAgentPod (internal/utils/gpus.go:1045-1089)."""
    rc, raw = _text_call(lib.cro_parse_proc_csv, _b(std_out), _b(std_err), _b(exec_err), _b(queryArgs))
    return rc, raw.decode("utf-8", "surrogateescape")


def proc_information_to_line(text: str) -> str:
    return _text(lib.cro_proc_information_to_line, _b(text))


def normalize(kind: int, s: str) -> str:
    return _text(lib.cro_normalize, kind, _b(s))


def emit_csv(devs: List[DevInfo], query: str) -> str:
    arr = (DevInfo * max(1, len(devs)))(*devs)
    return _text(lib.cro_emit_csv, arr, len(devs), _b(query))


def CheckGPUVisible(devs: List[DevInfo], device_id: str) -> bool:
    """internal/utils/gpus.go:73-84 over an enumerated device list."""
    arr = (DevInfo * max(1, len(devs)))(*devs)
    v = ctypes.c_int(0)
    rc = lib.cro_check_gpu_visible(arr, len(devs), _b(device_id), ctypes.byref(v))
    if rc != OK:
        raise ProbeError(rc)
    return bool(v.value)


def emit_status_json(state: str, error: str = "", device_id: str = "", cdi_device_id: str = "") -> str:
    return _text(lib.cro_emit_status_json, _b(state), _b(error), _b(device_id), _b(cdi_device_id))


def emit_scalar_status_json(state: str, device_id: str = "", cdi_device_id: str = "", node_name: str = "",
                            error: str = "") -> str:
    return _text(lib.cro_emit_scalar_status_json, _b(state), _b(device_id), _b(cdi_device_id), _b(node_name), _b(error))


def emit_fm_scale_up(tenant: str, mach: str, res_type: str, model: str) -> str:
    return _text(lib.cro_emit_fm_scale_up, _b(tenant), _b(mach), _b(res_type), _b(model))


def emit_fm_scale_down(tenant: str, mach: str, res_type: str, res_uuid: str) -> str:
    return _text(lib.cro_emit_fm_scale_down, _b(tenant), _b(mach), _b(res_type), _b(res_uuid))


def emit_cm_scale_up(spec_uuid: str, device_count: int) -> str:
    return _text(lib.cro_emit_cm_scale_up, _b(spec_uuid), device_count)


def emit_cm_scale_down(spec_uuid: str, device_count: int, device_id: str) -> str:
    return _text(lib.cro_emit_cm_scale_down, _b(spec_uuid), device_count, _b(device_id))


def emit_sunfish_request(name: str, count: int, proc_type: str, model: str) -> str:
    return _text(lib.cro_emit_sunfish_request, _b(name), count, _b(proc_type), _b(model))


def emit_probe_annotations_json(r: ProbeResult) -> str:
    return _text(lib.cro_emit_probe_annotations_json, ctypes.byref(r))


def emit_fault_annotations_json(report: FaultReport, words: List[FaultWord]) -> str:
    """Additive cohdi.io/probe-fault-* annotations of a locate_faults report (Go-marshalled map[string]string)."""
    arr = (FaultWord * max(1, len(words)))(*words)
    return _text(lib.cro_emit_fault_annotations_json, ctypes.byref(report), arr, len(words))


def emit_link_annotations_json(r: LinkResult) -> str:
    """Additive cohdi.io/probe-link-* annotations of a probe_host_link result (Go-marshalled map[string]string)."""
    return _text(lib.cro_emit_link_annotations_json, ctypes.byref(r))


def emit_compute_annotations_json(r: ComputeResult) -> str:
    """Additive cohdi.io/probe-compute-* annotations of a probe_compute result (Go-marshalled map[string]string)."""
    return _text(lib.cro_emit_compute_annotations_json, ctypes.byref(r))


def emit_precision_annotations_json(r: PrecisionResult) -> str:
    """Additive cohdi.io/probe-precision-* annotations of a probe_precision result (Go-marshalled map[string]string)."""
    return _text(lib.cro_emit_precision_annotations_json, ctypes.byref(r))


def emit_scan_annotations_json(r: ScanReport) -> str:
    """Additive cohdi.io/hbm-scan-* annotations of a scan report (Go-marshalled map[string]string)."""
    return _text(lib.cro_emit_scan_annotations_json, ctypes.byref(r))


def read_hbm_health(uuid: str) -> HbmHealth:
    """cro_read_hbm_health: the GPU's DRAM ECC counts and row-remapping state from NVML (no context, no CUDA)."""
    h = HbmHealth()
    rc = lib.cro_read_hbm_health(_b(uuid), ctypes.byref(h))
    if rc != OK:
        raise ProbeError(rc, "cro_read_hbm_health")
    return h


def emit_sram_annotations_json(r: SramResult) -> str:
    """Additive cohdi.io/probe-sram-* annotations of an SRAM probe result (Go-marshalled map[string]string)."""
    return _text(lib.cro_emit_sram_annotations_json, ctypes.byref(r))


def read_sram_health(uuid: str) -> SramHealth:
    """cro_read_sram_health: the GPU's volatile SRAM ECC counts and threshold flag from NVML (no context, no CUDA)."""
    h = SramHealth()
    rc = lib.cro_read_sram_health(_b(uuid), ctypes.byref(h))
    if rc != OK:
        raise ProbeError(rc, "cro_read_sram_health")
    return h


def emit_l2_annotations_json(r: L2Result) -> str:
    """Additive cohdi.io/probe-l2-* annotations of an L2 probe result (Go-marshalled map[string]string)."""
    return _text(lib.cro_emit_l2_annotations_json, ctypes.byref(r))


def read_l2_health(uuid: str) -> L2Health:
    """cro_read_l2_health: the GPU's volatile SRAM and L2 ECC counts and SRAM error status from NVML (no context, no
    CUDA)."""
    h = L2Health()
    rc = lib.cro_read_l2_health(_b(uuid), ctypes.byref(h))
    if rc != OK:
        raise ProbeError(rc, "cro_read_l2_health")
    return h


def _l2_opts(bytes: int, iterations: int, a1_counters: int, a2_counters: int, deadline_ms: int,
             inject: Optional[Tuple[int, int, int, int, int, int]]) -> L2Opts:
    o = L2Opts()
    o.bytes, o.iterations, o.a1_counters, o.a2_counters, o.deadline_ms = bytes, iterations, a1_counters, a2_counters, deadline_ms
    if inject is not None:
        (o.test_inject_leg, o.test_inject_sm, o.test_inject_element, o.test_inject_iteration, o.test_inject_word,
         o.test_inject_mask) = inject
    return o


def probe_l2_uuid(ctx: Optional["ProbeContext"], uuid: str, bytes: int = 0, iterations: int = 0, a1_counters: int = 0,
                  a2_counters: int = 0, deadline_ms: int = 0, inject: Optional[Tuple[int, int, int, int, int, int]] = None,
                  cap: int = 256) -> Tuple[L2Result, List[L2Sm], List[L2Fault]]:
    """cro_probe_l2_uuid: the L2 probe of any GPU on the node, run by the helper process (ctx may be None).
    Returns the result (its status is OK, ERR_CHECKSUM or ERR_CUDA), one entry per SM seen and up to `cap` records."""
    o = _l2_opts(bytes, iterations, a1_counters, a2_counters, deadline_ms, inject)
    handle = ctx.handle if ctx is not None else None
    rc, out = _per_sm(lib.cro_probe_l2_uuid, (handle, _b(uuid), ctypes.byref(o)), L2Result, L2Sm, L2_MAX_SMS, L2Fault, cap)
    if rc not in (OK, ERR_CHECKSUM, ERR_CUDA):
        raise _helper_error(rc, handle)
    return out


def selftest_l2_classify(r: L2Result, sms: List[L2Sm], faults: List[L2Fault]) -> Tuple[L2Result, List[L2Sm], List[L2Fault]]:
    """cro_selftest_l2_classify: the L2 probe's classification of the given counts and records, on copies."""
    out = L2Result.from_buffer_copy(r)
    s = (L2Sm * max(1, len(sms)))(*sms)
    f = (L2Fault * max(1, len(faults)))(*faults)
    rc = lib.cro_selftest_l2_classify(ctypes.byref(out), s, len(sms), f, len(faults))
    if rc != OK:
        raise ProbeError(rc, "cro_selftest_l2_classify")
    return out, list(s[:len(sms)]), list(f[:len(faults)])


def _legs_rounds(n_legs: int, legs: int, rounds, claims, records, cta, words: int, fault):
    """The flat arrays of the selftest hooks: per leg of `legs`, rounds[l] as (CTA records, coverage words) pairs and
    records[l]; `words` 0 means the rounds carry no coverage words."""
    ran = [l for l in range(n_legs) if legs >> l & 1]
    ctas = [x for l in ran for got, _ in rounds[l] for x in got]
    bits = [b for l in ran for _, got in rounds[l] for b in got]
    recs = [x for l in ran for x in records[l]]
    assert all(len(got) == words for l in ran for _, got in rounds[l])
    return ((ctypes.c_uint32 * n_legs)(*[len(rounds[l]) if l in ran else 0 for l in range(n_legs)]),
            (cta * max(1, len(ctas)))(*ctas), (ctypes.c_uint64 * max(1, len(bits)))(*bits),
            (ctypes.c_uint64 * n_legs)(*claims), (fault * max(1, len(recs)))(*recs))


def selftest_sm_legs_classify(probe: int, iterations: List[int], grid: int, call: int, rounds, claims: List[int],
                              records, legs: int = 0):
    """cro_selftest_sm_legs_classify: the compute (SM_LEGS_COMPUTE) or precision probe's classification of call `call`
    on `grid` SMs.  Per leg l (every list is indexed by leg; legs 0: all): rounds[l] a list of (grid SmCta, the
    COMPUTE_MAX_SMS // 64 coverage words) per round, claims[l] and records[l] (ComputeFault / PrecisionFault, the first
    min(claims[l], RECORDS)).  Returns (result, SM entries, faults); the result's status may be OK, ERR_CHECKSUM or
    ERR_UNSUPPORTED."""
    compute = probe == SM_LEGS_COMPUTE
    n_legs = COMPUTE_LEGS if compute else PRECISION_LEGS
    result, sm, fault = (ComputeResult, ComputeSm, ComputeFault) if compute else (PrecisionResult, PrecisionSm, PrecisionFault)
    ran = legs or (1 << n_legs) - 1
    nr, ctas, bits, cl, recs = _legs_rounds(n_legs, ran, rounds, claims, records, SmCta, COMPUTE_MAX_SMS // 64, fault)
    it = (ctypes.c_uint32 * n_legs)(*iterations)
    cap = sum(len(records[l]) for l in range(n_legs) if ran >> l & 1)
    rc, out = _per_sm(lib.cro_selftest_sm_legs_classify, (probe, legs, it, grid, call, nr, ctas, bits, cl,
                                                          recs), result, sm, COMPUTE_MAX_SMS, fault, cap)
    if rc not in (OK, ERR_CHECKSUM, ERR_UNSUPPORTED):
        raise ProbeError(rc, "cro_selftest_sm_legs_classify")
    return out


def selftest_sram_classify(iterations: int, n_words: int, seed: int, cluster: int, sm_count: int, net_grid: int, call: int,
                           rounds, claims: List[int], records, legs: int = 0):
    """cro_selftest_sram_classify: the SRAM probe's classification of call `call`.  Per leg l (legs 0: both): rounds[l] a
    list of rounds, each a list of SramCta (sm_count of them for the local leg, net_grid for the network leg),
    claims[l] and records[l] (SramRecord, the first min(claims[l], SRAM_RECORDS)).  Returns (result, SM entries,
    faults); the result's status may be OK, ERR_CHECKSUM or ERR_UNSUPPORTED."""
    ran = legs or SRAM_ALL_LEGS
    nr, ctas, _, cl, recs = _legs_rounds(SRAM_LEGS, ran, [[(x, []) for x in r] for r in rounds], claims, records, SramCta, 0,
                                         SramRecord)
    cap = sum(len(records[l]) for l in range(SRAM_LEGS) if ran >> l & 1)
    rc, out = _per_sm(lib.cro_selftest_sram_classify, (legs, iterations, n_words, seed, cluster, sm_count, net_grid, call, nr,
                                                       ctas, cl, recs), SramResult, SramSm, SRAM_MAX_SMS, SramFault, cap)
    if rc not in (OK, ERR_CHECKSUM, ERR_UNSUPPORTED):
        raise ProbeError(rc, "cro_selftest_sram_classify")
    return out


def _sram_opts(legs: int, iterations: int, cluster: int, max_rounds: int, deadline_ms: int,
               inject: Optional[Tuple[int, int, int, int, int, int]]) -> SramOpts:
    o = SramOpts()
    o.legs, o.iterations, o.cluster, o.max_rounds, o.deadline_ms = legs, iterations, cluster, max_rounds, deadline_ms
    if inject is not None:
        (o.test_inject_leg, o.test_inject_sm, o.test_inject_element, o.test_inject_iteration, o.test_inject_word,
         o.test_inject_mask) = inject
    return o


def probe_sram_uuid(ctx: Optional["ProbeContext"], uuid: str, legs: int = SRAM_ALL_LEGS, iterations: int = 0, cluster: int = 0,
                    max_rounds: int = 0, deadline_ms: int = 0, inject: Optional[Tuple[int, int, int, int, int, int]] = None,
                    cap: int = 256) -> Tuple[SramResult, List[SramSm], List[SramFault]]:
    """cro_probe_sram_uuid: the SRAM probe of any GPU on the node, run by the helper process (ctx may be None).
    Returns the result (its status is OK, ERR_CHECKSUM or ERR_CUDA), one entry per SM seen and up to `cap` records."""
    o = _sram_opts(legs, iterations, cluster, max_rounds, deadline_ms, inject)
    handle = ctx.handle if ctx is not None else None
    rc, out = _per_sm(lib.cro_probe_sram_uuid, (handle, _b(uuid), ctypes.byref(o)), SramResult, SramSm, SRAM_MAX_SMS, SramFault,
                      cap)
    if rc not in (OK, ERR_CHECKSUM, ERR_CUDA):
        raise _helper_error(rc, handle)
    return out


def _helper_error(rc: int, handle) -> "ProbeError":
    buf = ctypes.create_string_buffer(1024)
    lib.cro_last_error(handle, buf, 1024)
    return ProbeError(rc, buf.value.decode("utf-8", "replace"))


def _per_sm(fn, head: tuple, result, sm, max_sms: int, fault, cap: int, tail: tuple = ()):
    """One call of a per-SM probe (compute, precision, SRAM, L2; in process or by UUID):
    fn(*head, result, sms, max_sms, n_sms, faults, cap, n, *tail) on fresh arrays.  Returns the return code and
    (result, the SM entries, the faults)."""
    r = result()
    sms = (sm * max_sms)()
    arr = (fault * max(1, cap))()
    n_sms, n = ctypes.c_int(), ctypes.c_int()
    rc = fn(*head, ctypes.byref(r), sms, max_sms, ctypes.byref(n_sms), arr, cap, ctypes.byref(n), *tail)
    return rc, (r, [sms[i] for i in range(n_sms.value)], [arr[i] for i in range(n.value)])


def _link_opts(bytes: int, hops: int, ctas: int, inject: Optional[Tuple[int, int, int]]) -> LinkOpts:
    o = LinkOpts()
    o.bytes, o.hops, o.ctas = bytes, hops, ctas
    if inject is not None:
        o.test_inject_check, o.test_inject_word, o.test_inject_mask = inject
    return o


def probe_host_link_uuid(ctx: Optional["ProbeContext"], uuid: str, bytes: int = 0, hops: int = 0, ctas: int = 0,
                         deadline_ms: int = 0, inject: Optional[Tuple[int, int, int]] = None,
                         cap: int = 256) -> Tuple[LinkResult, List[LinkFault], int]:
    """cro_probe_host_link_uuid: the host link probe of any GPU on the node, run by the helper process (ctx may be
    None).  bytes = 0: 256 MiB (the helper's sweep region is L).  Returns the result (its status is OK, ERR_CHECKSUM or
    ERR_CUDA), up to `cap` mismatching words and the helper's spawn-to-exit time in ns."""
    o = _link_opts(bytes, hops, ctas, inject)
    r = LinkResult()
    arr = (LinkFault * max(1, cap))()
    n, ns = ctypes.c_int(), ctypes.c_uint64()
    handle = ctx.handle if ctx is not None else None
    rc = lib.cro_probe_host_link_uuid(handle, _b(uuid), ctypes.byref(o), deadline_ms, ctypes.byref(r), arr, cap, ctypes.byref(n),
                                      ctypes.byref(ns))
    if rc not in (OK, ERR_CHECKSUM, ERR_CUDA):
        raise _helper_error(rc, handle)
    return r, [arr[i] for i in range(n.value)], ns.value


def _compute_opts(iterations: int, alu_iterations: int, legs: int, max_rounds: int,
                  inject: Optional[Tuple[int, int, int, int, int, int]]) -> ComputeOpts:
    o = ComputeOpts()
    o.iterations, o.alu_iterations, o.legs, o.max_rounds = iterations, alu_iterations, legs, max_rounds
    if inject is not None:
        (o.test_inject_leg, o.test_inject_sm, o.test_inject_iteration, o.test_inject_row, o.test_inject_col,
         o.test_inject_mask) = inject
    return o


def probe_compute_uuid(ctx: Optional["ProbeContext"], uuid: str, iterations: int = 0, alu_iterations: int = 0,
                       legs: int = COMPUTE_ALL_LEGS, max_rounds: int = 0, deadline_ms: int = 0,
                       inject: Optional[Tuple[int, int, int, int, int, int]] = None,
                       cap: int = 256) -> Tuple[ComputeResult, List[ComputeSm], List[ComputeFault], int]:
    """cro_probe_compute_uuid: the compute probe of any GPU on the node, run by the helper process (ctx may be None).
    Returns the result (its status is OK, ERR_CHECKSUM or ERR_CUDA), one entry per SM seen, up to `cap` element records
    and the helper's spawn-to-exit time in ns."""
    o = _compute_opts(iterations, alu_iterations, legs, max_rounds, inject)
    ns = ctypes.c_uint64()
    handle = ctx.handle if ctx is not None else None
    rc, out = _per_sm(lib.cro_probe_compute_uuid, (handle, _b(uuid), ctypes.byref(o), deadline_ms), ComputeResult, ComputeSm,
                      COMPUTE_MAX_SMS, ComputeFault, cap, (ctypes.byref(ns),))
    if rc not in (OK, ERR_CHECKSUM, ERR_CUDA):
        raise _helper_error(rc, handle)
    return out + (ns.value,)


def _precision_opts(iterations: int, alu_iterations: int, legs: int, max_rounds: int,
                    inject: Optional[Tuple[int, int, int, int, int, int]]) -> PrecisionOpts:
    o = PrecisionOpts()
    o.iterations, o.alu_iterations, o.legs, o.max_rounds = iterations, alu_iterations, legs, max_rounds
    if inject is not None:
        (o.test_inject_leg, o.test_inject_sm, o.test_inject_iteration, o.test_inject_row, o.test_inject_col,
         o.test_inject_mask) = inject
    return o


def probe_precision_uuid(ctx: Optional["ProbeContext"], uuid: str, iterations: int = 0, alu_iterations: int = 0,
                         legs: int = PRECISION_ALL_LEGS, max_rounds: int = 0, deadline_ms: int = 0,
                         inject: Optional[Tuple[int, int, int, int, int, int]] = None,
                         cap: int = 256) -> Tuple[PrecisionResult, List[PrecisionSm], List[PrecisionFault], int]:
    """cro_probe_precision_uuid: the precision probe of any GPU on the node, run by the helper process (ctx may be None).
    Returns the result (its status is OK, ERR_CHECKSUM or ERR_CUDA), one entry per SM seen, up to `cap` element records
    and the helper's spawn-to-exit time in ns."""
    o = _precision_opts(iterations, alu_iterations, legs, max_rounds, inject)
    ns = ctypes.c_uint64()
    handle = ctx.handle if ctx is not None else None
    rc, out = _per_sm(lib.cro_probe_precision_uuid, (handle, _b(uuid), ctypes.byref(o), deadline_ms), PrecisionResult,
                      PrecisionSm, PRECISION_MAX_SMS, PrecisionFault, cap, (ctypes.byref(ns),))
    if rc not in (OK, ERR_CHECKSUM, ERR_CUDA):
        raise _helper_error(rc, handle)
    return out + (ns.value,)


def _scan_opts(max_bytes: int, reserve_bytes: int, seed: int, deadline_ms: int, chunk_bytes: int,
               force: Optional[Tuple[int, int, int, int]]) -> ScanOpts:
    o = ScanOpts()
    o.max_bytes, o.reserve_bytes, o.seed, o.deadline_ms, o.test_chunk_bytes = max_bytes, reserve_bytes, seed, deadline_ms, chunk_bytes
    if force is not None:
        o.test_force_first, o.test_force_count, o.test_force_and, o.test_force_or = force
    return o


def scan_hbm_uuid(ctx: Optional["ProbeContext"], uuid: str, max_bytes: int = 0, reserve_bytes: int = 0, seed: int = 0,
                  deadline_ms: int = 0, cap: int = 256, chunk_bytes: int = 0,
                  force: Optional[Tuple[int, int, int, int]] = None) -> Tuple[ScanReport, List[FaultWord]]:
    """cro_scan_hbm_uuid: the whole-HBM scan of any GPU on the node, run by the helper process (ctx may be None).
    Returns the report (its status is OK, ERR_CHECKSUM or ERR_CUDA) and up to `cap` mismatching words."""
    o = _scan_opts(max_bytes, reserve_bytes, seed, deadline_ms, chunk_bytes, force)
    rep = ScanReport()
    arr = (FaultWord * max(1, cap))()
    n = ctypes.c_int()
    handle = ctx.handle if ctx is not None else None
    rc = lib.cro_scan_hbm_uuid(handle, _b(uuid), ctypes.byref(o), ctypes.byref(rep), arr, cap, ctypes.byref(n))
    if rc not in (OK, ERR_CHECKSUM, ERR_CUDA):
        raise _helper_error(rc, handle)
    return rep, [arr[i] for i in range(n.value)]


def precision_expected(answer: int, seed: int) -> List[int]:
    """cro_precision_expected: the PRECISION_ANSWER_* answer tile of the operands of `seed`, int64 values, row-major
    (PRECISION_M x PRECISION_F64_N for the wide answer, PRECISION_M x PRECISION_N otherwise; host arithmetic, no GPU)."""
    arr = (ctypes.c_int64 * (PRECISION_M * PRECISION_N))()
    rc = lib.cro_precision_expected(answer, seed, arr)
    if rc != OK:
        raise ProbeError(rc, "cro_precision_expected")
    return list(arr)[:PRECISION_M * (PRECISION_F64_N if answer == PRECISION_ANSWER_WIDE else PRECISION_N)]


def compute_expected(answer: int, seed: int) -> List[int]:
    """cro_compute_expected: the COMPUTE_ANSWER_S8 / _SMALL answer tile of the operands of `seed`, COMPUTE_M * COMPUTE_N
    int32 values, row-major (host arithmetic, no GPU)."""
    arr = (ctypes.c_int32 * (COMPUTE_M * COMPUTE_N))()
    rc = lib.cro_compute_expected(answer, seed, arr)
    if rc != OK:
        raise ProbeError(rc, "cro_compute_expected")
    return list(arr)


def pci_link_path(bus_id: str, sys_root: Optional[str] = None) -> PciPath:
    """cro_pci_link_path: the device's PCIe path as sysfs under sys_root (default /sys) describes it.  No GPU needed."""
    p = PciPath()
    rc = lib.cro_pci_link_path(_b(sys_root), _b(bus_id), ctypes.byref(p))
    if rc != OK:
        raise ProbeError(rc)
    return p


def fm_parse_scale_up_response(body: str, name: str, res_type: str, model: str) -> Tuple[str, str, str]:
    """(deviceID, CDIDeviceID, err) per internal/cdi/fti/fm/client.go:184-213."""
    dev, cdi, err = (ctypes.create_string_buffer(256) for _ in range(3))
    err = ctypes.create_string_buffer(1024)
    rc = lib.cro_fm_parse_scale_up_response(_b(body), _b(name), _b(res_type), _b(model), dev, 256, cdi, 256, err, 1024)
    if rc != OK:
        return "", "", err.value.decode()
    return dev.value.decode(), cdi.value.decode(), ""


def cm_check_adding_resources(machine_body: str, existing_device_ids: List[str], res_type: str, model: str):
    """(specUUID, deviceCount, deviceID, CDIDeviceID, err) per internal/cdi/fti/cm/client.go:432-459."""
    spec, dev, cdi = (ctypes.create_string_buffer(256) for _ in range(3))
    err = ctypes.create_string_buffer(1024)
    n = ctypes.c_int(0)
    lib.cro_cm_check_adding_resources(_b(machine_body), _b("\n".join(existing_device_ids)), _b(res_type), _b(model),
                                      spec, 256, ctypes.byref(n), dev, 256, cdi, 256, err, 1024)
    return spec.value.decode(), n.value, dev.value.decode(), cdi.value.decode(), err.value.decode()


def reconcile_attach(ctx: Optional["ProbeContext"], request: Dict) -> Dict:
    """One pass of handleAttachingState (composableresource_controller.go:200-287).
    ``ctx`` may be None when ``request['enumeration']`` supplies the exec output."""
    handle = ctx.handle if ctx is not None else None
    rc, raw = _text_call(lib.cro_reconcile_attach, handle, _b(json.dumps(request)))
    if rc != OK:
        raise ProbeError(rc, raw.decode("utf-8", "replace"))
    out = json.loads(raw.decode("utf-8"))
    out["_raw"] = raw.decode("utf-8")
    return out


# ---- the probe context (needs an H100) -----------------------------------------------
class ProbeContext:
    """Long-lived probe context: resident sweep buffers, streams, events.

    Takes the slot of utils.RunNvidiaSmi + utils.CheckGPUVisible
    (internal/utils/gpus.go:666-689, 54-86)."""

    def __init__(self, sweep_bytes: int = 0, devices: Optional[List[int]] = None, flags: int = 0,
                 read_sweeps: int = 0, copy_sweeps: int = 0, read_variant: int = READ_AUTO,
                 copy_variant: int = COPY_AUTO, p2p_bytes: int = 0, latency_hops: int = 0,
                 deadline_ms: int = 0, seed_base: int = 0, rank_base: int = 0, world: int = 0,
                 inject: Optional[Tuple[int, int, int]] = None) -> None:
        o = Opts()
        o.abi_version = ABI_VERSION
        o.flags = flags
        o.sweep_bytes = sweep_bytes
        o.p2p_bytes = p2p_bytes
        o.seed_base = seed_base
        o.read_sweeps, o.copy_sweeps = read_sweeps, copy_sweeps
        o.latency_hops = latency_hops
        o.read_variant, o.copy_variant = read_variant, copy_variant
        o.deadline_ms = deadline_ms
        o.rank_base, o.world_override = rank_base, world
        if inject is not None:            # (after sweep number, word index, xor mask): fault injection inside the probe
            o.flags |= F_TEST_INJECT
            o.test_inject_after, o.test_inject_word, o.test_inject_mask = inject
        if devices:
            o.n_devices = len(devices)
            for i, d in enumerate(devices):
                o.devices[i] = d
        h = ctypes.c_void_p()
        rc = lib.cro_probe_init(ctypes.byref(o), ctypes.byref(h))
        if rc != OK:
            why = ctypes.create_string_buffer(1024)
            lib.cro_last_error(None, why, 1024)       # the context died with the init: its text is per-thread
            detail = why.value.decode("utf-8", "replace")
            raise ProbeError(rc, "cro_probe_init" + (": " + detail if detail else ""))
        self.handle = h

    def close(self) -> None:
        if getattr(self, "handle", None):
            lib.cro_probe_destroy(self.handle)
            self.handle = None

    def __enter__(self) -> "ProbeContext":
        return self

    def __exit__(self, *a) -> None:
        self.close()

    def __del__(self) -> None:
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int, allow=()) -> int:
        if rc != OK and rc not in allow:
            buf = ctypes.create_string_buffer(1024)
            lib.cro_last_error(self.handle, buf, 1024)
            raise ProbeError(rc, buf.value.decode("utf-8", "replace"))
        return rc

    def last_error(self) -> str:
        """Text of this thread's most recent failing (or degrading) call on the context."""
        buf = ctypes.create_string_buffer(1024)
        lib.cro_last_error(self.handle, buf, 1024)
        return buf.value.decode("utf-8", "replace")

    def device_count(self) -> int:
        n = ctypes.c_int()
        self._check(lib.cro_device_count(self.handle, ctypes.byref(n)))
        return n.value

    def enumerate(self) -> List[DevInfo]:
        n = ctypes.c_int()
        arr = (DevInfo * MAX_DEVICES)()
        self._check(lib.cro_enumerate(self.handle, arr, MAX_DEVICES, ctypes.byref(n)))
        return [arr[i] for i in range(n.value)]

    def own_devices(self) -> List[DevInfo]:
        """The devices this context probes in process, by dev_index (enumerate() lists the whole NODE, fresh)."""
        mine = [d for d in self.enumerate() if d.flags & DEV_IN_PROCESS]
        return sorted(mine, key=lambda d: d.dev_index)

    def seed(self, dev: int = 0) -> int:
        s = ctypes.c_uint64()
        self._check(lib.cro_device_seed(self.handle, dev, ctypes.byref(s)))
        return s.value

    def probe_device(self, dev: int = 0, allow_checksum_error: bool = False) -> ProbeResult:
        r = ProbeResult()
        self._check(lib.cro_probe_device(self.handle, dev, ctypes.byref(r)),
                    allow=(ERR_CHECKSUM,) if allow_checksum_error else ())
        return r

    def probe_begin(self, dev: int = 0) -> None:
        self._check(lib.cro_probe_begin(self.handle, dev))

    def probe_end(self, dev: int = 0) -> ProbeResult:
        r = ProbeResult()
        self._check(lib.cro_probe_end(self.handle, dev, ctypes.byref(r)))
        return r

    def probe_all(self) -> List[ProbeResult]:
        arr = (ProbeResult * MAX_DEVICES)()
        n = ctypes.c_int()
        self._check(lib.cro_probe_all(self.handle, arr, MAX_DEVICES, ctypes.byref(n)))
        return [arr[i] for i in range(n.value)]

    def result_device_ptr(self, dev: int = 0) -> int:
        p = ctypes.c_uint64()
        self._check(lib.cro_result_device_ptr(self.handle, dev, ctypes.byref(p)))
        return p.value

    def _sweep(self, fn, *args) -> SweepResult:
        r = SweepResult()
        self._check(fn(self.handle, *args, ctypes.byref(r)))
        return r

    def hbm_fill(self, dev: int = 0, iters: int = 1) -> SweepResult:
        return self._sweep(lib.cro_hbm_fill_loop, dev, iters)

    def hbm_read_checksum(self, dev: int = 0, variant: int = READ_AUTO, iters: int = 1, dst: bool = False) -> SweepResult:
        if dst:
            return self._sweep(lib.cro_hbm_read_checksum_dst, dev, variant)
        return self._sweep(lib.cro_hbm_read_loop, dev, variant, iters)

    def hbm_copy(self, dev: int = 0, variant: int = COPY_AUTO, iters: int = 1) -> SweepResult:
        return self._sweep(lib.cro_hbm_copy_loop, dev, variant, iters)

    def hbm_expected_checksum(self, dev: int = 0) -> SweepResult:
        return self._sweep(lib.cro_hbm_expected_checksum, dev)

    def inject_fault(self, dev: int, word_index: int, mask: int) -> None:
        self._check(lib.cro_inject_fault(self.handle, dev, word_index, mask))

    def read_words(self, dev: int, first: int, n: int) -> List[int]:
        arr = (ctypes.c_uint64 * n)()
        self._check(lib.cro_read_words(self.handle, dev, first, n, arr))
        return list(arr)

    def locate_faults(self, dev: int = 0, retest: bool = True, cap: int = 256,
                      force: Optional[Tuple[int, int, int, int]] = None) -> Tuple[FaultReport, List[FaultWord]]:
        """cro_locate_faults: which words of the sweep region differ from their pattern, typically right after a probe
        returned ERR_CHECKSUM.  Pass 0 compares what the region holds now; retest adds the fresh-pattern and complement
        passes.  force = (first, count, and_mask, or_mask) is the test-only stand-in for stuck cells, applied after
        each retest fill.  Returns the report (its status is OK or ERR_CHECKSUM) and up to `cap` words by index."""
        o = LocateOpts()
        o.flags = LOCATE_RETEST if retest else 0
        if force is not None:
            o.test_force_first, o.test_force_count, o.test_force_and, o.test_force_or = force
        rep = FaultReport()
        arr = (FaultWord * max(1, cap))()
        n = ctypes.c_int()
        self._check(lib.cro_locate_faults(self.handle, dev, ctypes.byref(o), ctypes.byref(rep), arr, cap, ctypes.byref(n)),
                    allow=(ERR_CHECKSUM,))
        return rep, [arr[i] for i in range(n.value)]

    def probe_host_link(self, dev: int = 0, bytes: int = 0, hops: int = 0, inject: Optional[Tuple[int, int, int]] = None,
                        cap: int = 256, ctas: int = 0) -> Tuple[LinkResult, List[LinkFault]]:
        """cro_probe_host_link: moves fresh patterns over the device's PCIe link in both directions (copy engines and
        SMs, each direction alone and both at once), checks every byte, chases through host memory and reads the
        link's path from sysfs.  bytes = 0: min(256 MiB, S); hops = 0: 1024; ctas = 0: the default grid of the SM
        legs.  inject = (check, word, mask) is the test-only fault.  Returns the result (its status is OK or
        ERR_CHECKSUM) and up to `cap` mismatching words."""
        o = _link_opts(bytes, hops, ctas, inject)
        r = LinkResult()
        arr = (LinkFault * max(1, cap))()
        n = ctypes.c_int()
        self._check(lib.cro_probe_host_link(self.handle, dev, ctypes.byref(o), ctypes.byref(r), arr, cap, ctypes.byref(n)),
                    allow=(ERR_CHECKSUM,))
        return r, [arr[i] for i in range(n.value)]

    def probe_compute(self, dev: int = 0, iterations: int = 0, alu_iterations: int = 0, legs: int = COMPUTE_ALL_LEGS,
                      max_rounds: int = 0, inject: Optional[Tuple[int, int, int, int, int, int]] = None,
                      cap: int = 256) -> Tuple[ComputeResult, List[ComputeSm], List[ComputeFault]]:
        """cro_probe_compute: every SM computes the answer tile with its tensor cores (s8, bf16, e4m3) and CUDA cores
        (FFMA, IMAD) and checks it exactly.  iterations = 0 / alu_iterations = 0 / max_rounds = 0: the defaults.
        inject = (leg, sm, iteration, row, col, mask) is the test-only wrong answer (sm, row, col: -1 for every one).
        Returns the result (its status is OK or ERR_CHECKSUM), one entry per SM seen and up to `cap` element records."""
        o = _compute_opts(iterations, alu_iterations, legs, max_rounds, inject)
        rc, out = _per_sm(lib.cro_probe_compute, (self.handle, dev, ctypes.byref(o)), ComputeResult, ComputeSm, COMPUTE_MAX_SMS,
                          ComputeFault, cap)
        self._check(rc, allow=(ERR_CHECKSUM,))
        return out

    def probe_precision(self, dev: int = 0, iterations: int = 0, alu_iterations: int = 0, legs: int = PRECISION_ALL_LEGS,
                        max_rounds: int = 0, inject: Optional[Tuple[int, int, int, int, int, int]] = None,
                        cap: int = 256) -> Tuple[PrecisionResult, List[PrecisionSm], List[PrecisionFault]]:
        """cro_probe_precision: every SM computes its answer tiles in FP64 (DMMA, DFMA), TF32, FP16 (f32 and f16
        accumulation, HFMA2) and E5M2 and checks each value bit for bit.  iterations (F64, TF32, F16, F16ACC, E5M2) /
        alu_iterations (DFMA, HFMA2) / max_rounds = 0: the defaults.  inject = (leg, sm, iteration, row, col, mask) is the
        test-only wrong answer (sm, row, col: -1 for every one; mask up to the leg's element width).  Returns the result
        (its status is OK or ERR_CHECKSUM), one entry per SM seen and up to `cap` element records."""
        o = _precision_opts(iterations, alu_iterations, legs, max_rounds, inject)
        rc, out = _per_sm(lib.cro_probe_precision, (self.handle, dev, ctypes.byref(o)), PrecisionResult, PrecisionSm,
                          PRECISION_MAX_SMS, PrecisionFault, cap)
        self._check(rc, allow=(ERR_CHECKSUM,))
        return out

    def scan_hbm(self, dev: int = 0, max_bytes: int = 0, reserve_bytes: int = 0, seed: int = 0, cap: int = 256,
                 chunk_bytes: int = 0, force: Optional[Tuple[int, int, int, int]] = None) -> Tuple[ScanReport, List[FaultWord]]:
        """cro_scan_hbm: fills every chunk of the free memory this process can allocate (min(max_bytes, free -
        reserve_bytes); 0 = all / 1 GiB) with a pattern, compares, fills its complement, compares.  seed = 0: a fresh
        one, reported.  chunk_bytes and force = (first, count, and_mask, or_mask) are the test-only chunk size and stuck
        cells.  Returns the report (its status is OK, ERR_CHECKSUM or ERR_CUDA) and up to `cap` mismatching words;
        report.place(word) is its (chunk, offset)."""
        o = _scan_opts(max_bytes, reserve_bytes, seed, 0, chunk_bytes, force)
        rep = ScanReport()
        arr = (FaultWord * max(1, cap))()
        n = ctypes.c_int()
        self._check(lib.cro_scan_hbm(self.handle, dev, ctypes.byref(o), ctypes.byref(rep), arr, cap, ctypes.byref(n)),
                    allow=(ERR_CHECKSUM, ERR_CUDA))
        return rep, [arr[i] for i in range(n.value)]

    def probe_sram(self, dev: int = 0, legs: int = SRAM_ALL_LEGS, iterations: int = 0, cluster: int = 0, max_rounds: int = 0,
                   inject: Optional[Tuple[int, int, int, int, int, int]] = None,
                   cap: int = 256) -> Tuple[SramResult, List[SramSm], List[SramFault]]:
        """cro_probe_sram: March C- over every SM's shared memory (SRAM_LEG_SMEM) and the words of each cluster written
        and read across the SM-to-SM network (SRAM_LEG_DSMEM, `cluster` CTAs: 2, 4 or 8).  iterations = 0 / cluster = 0 /
        max_rounds = 0: the defaults.  inject = (leg, sm, element, iteration, word, mask) is the test-only stand-in for a
        bad cell (sm, word: -1 for every one).  Returns the result (its status is OK, ERR_CHECKSUM or ERR_CUDA), one entry
        per SM seen and up to `cap` word records."""
        o = _sram_opts(legs, iterations, cluster, max_rounds, 0, inject)
        rc, out = _per_sm(lib.cro_probe_sram, (self.handle, dev, ctypes.byref(o)), SramResult, SramSm, SRAM_MAX_SMS, SramFault, cap)
        self._check(rc, allow=(ERR_CHECKSUM, ERR_CUDA))
        return out

    def probe_l2(self, dev: int = 0, bytes: int = 0, iterations: int = 0, a1_counters: int = 0, a2_counters: int = 0,
                 inject: Optional[Tuple[int, int, int, int, int, int]] = None,
                 cap: int = 256) -> Tuple[L2Result, List[L2Sm], List[L2Fault]]:
        """cro_probe_l2: March C- over an L2-resident buffer of `bytes` whose blocks change SM from element to element,
        and the L2 atomic units' A1 (red.add / red.xor) and A2 (atom.add tickets) legs.  0: the defaults.
        inject = (leg, sm, element, iteration, word, mask) is the test-only stand-in for a fault (L2_MARCH: sm, element,
        word -1 for every one; L2_A1 / L2_A2: word is the counter).  Returns the result (its status is OK,
        ERR_CHECKSUM or ERR_CUDA), one entry per SM seen and up to `cap` word records."""
        o = _l2_opts(bytes, iterations, a1_counters, a2_counters, 0, inject)
        rc, out = _per_sm(lib.cro_probe_l2, (self.handle, dev, ctypes.byref(o)), L2Result, L2Sm, L2_MAX_SMS, L2Fault, cap)
        self._check(rc, allow=(ERR_CHECKSUM, ERR_CUDA))
        return out

    def launch_count(self) -> int:
        return int(lib.cro_launch_count(self.handle))

    def sweep_times(self, dev: int = 0) -> List[SweepTime]:
        """Per-sweep CUDA-event and %globaltimer times of the device's last probe (fill, copies, reads)."""
        arr = (SweepTime * 64)()
        n = ctypes.c_int()
        self._check(lib.cro_probe_sweep_times(self.handle, dev, arr, 64, ctypes.byref(n)))
        return [arr[i] for i in range(n.value)]

    def p2p_detail(self, dev: int, peer: int) -> P2PDetail:
        d = P2PDetail()
        self._check(lib.cro_p2p_detail_get(self.handle, dev, peer, ctypes.byref(d)))
        return d

    def metrics_text(self) -> str:
        """Prometheus text exposition of the context's counters and per-GPU gauges."""
        rc, raw = _text_call(lib.cro_metrics_text, self.handle)
        self._check(rc)
        return raw.decode()

    def set_latency_hops(self, hops: int) -> None:
        self._check(lib.cro_set_latency_hops(self.handle, hops))

    def fullbox_times(self) -> FullBoxTime:
        t = FullBoxTime()
        self._check(lib.cro_fullbox_times(self.handle, ctypes.byref(t)))
        return t

    # ---- test hooks: the verdict kernels on crafted inputs (never used by the probe path) ----
    def selftest_probe_finalize(self, dev: int, tmpl: bytes, slots: bytes, seed: int, nonce: int, sweep_bytes: int,
                                read_sweeps: int, copy_sweeps: int, read_variant: int, copy_variant: int) -> bytes:
        """probe_finalize_kernel over a 512-byte template and SLOT_COUNT packed slots; returns the 512 bytes it wrote."""
        assert len(tmpl) == 512 and len(slots) == SLOT_COUNT * SLOT_BYTES
        t, out = ProbeResult.from_buffer_copy(tmpl), ProbeResult()
        sl = ctypes.create_string_buffer(slots, len(slots))
        self._check(lib.cro_selftest_probe_finalize(self.handle, dev, ctypes.byref(t), sl, seed, nonce, sweep_bytes,
                                                    read_sweeps, copy_sweeps, read_variant, copy_variant, ctypes.byref(out)))
        return bytes(out)

    def selftest_p2p_finalize(self, dev: int, result: bytes, slots: bytes, peer_slots: List[Optional[bytes]],
                              peer_stamp: List[int], chase_out: List[int], chase_expect: List[int], n: int, self_index: int,
                              hops: int, have_push: int, push_folded: int, p2p_bytes: int, stamp: int) -> bytes:
        """p2p_finalize_kernel over a result struct, this device's slots and peer j's slots (None = no such peer);
        returns the result struct it left."""
        assert len(result) == 512 and len(slots) == SLOT_COUNT * SLOT_BYTES and len(peer_slots) <= MAX_DEVICES
        r = ProbeResult.from_buffer_copy(result)
        sl = ctypes.create_string_buffer(slots, len(slots))
        keep = [ctypes.create_string_buffer(p, len(p)) if p is not None else None for p in peer_slots]
        ps = (ctypes.c_void_p * MAX_DEVICES)(*[ctypes.cast(k, ctypes.c_void_p) if k is not None else None for k in keep])
        st = (ctypes.c_uint64 * MAX_DEVICES)(*peer_stamp)
        co = (ctypes.c_uint64 * (2 * MAX_DEVICES))(*chase_out)
        ce = (ctypes.c_uint32 * MAX_DEVICES)(*chase_expect)
        self._check(lib.cro_selftest_p2p_finalize(self.handle, dev, ctypes.byref(r), sl, ps, st, co, ce, n, self_index, hops,
                                                  have_push, push_folded, p2p_bytes, stamp))
        return bytes(r)

    def selftest_chase(self, dev: int, pairs: List[Optional[Tuple[int, int]]], hops: int) -> List[int]:
        """chase_kernel over tables built for (minor_src, minor_dst) pairs (None = a row without a table);
        returns the 2 * len(pairs) output words."""
        n = len(pairs)
        src = (ctypes.c_int32 * n)(*[p[0] if p is not None else -1 for p in pairs])
        dst = (ctypes.c_int32 * n)(*[p[1] if p is not None else -1 for p in pairs])
        out = (ctypes.c_uint64 * (2 * n))()
        self._check(lib.cro_selftest_chase(self.handle, dev, src, dst, n, hops, out))
        return list(out)

    def selftest_sweep(self, dev: int, kernel: int, bytes: int, offset: int = 0, layout: int = 0, seed: int = 0,
                       canary: int = 0, invert: int = 0, word0: int = 0, force: List[Tuple[int, int, int, int]] = (),
                       interiors: bool = False, alloc=bytearray, cap: int = 16):
        """One SELFTEST_SWEEP_* kernel on a buffer of the hook's own: guards holding canary words (word j of guard g:
        pattern_word(canary, g * 2^32 + j)) around the interior(s), a copy's in the SELFTEST_LAYOUT_* given.  force: up
        to two (first, count, and_mask, or_mask) interior ranges.  Returns (SelftestSweepOut, the buffer as alloc(buf_bytes) made it, with the guards and,
        if interiors, the interiors at their offsets, and up to `cap` of the kernel's records by word)."""
        o = SelftestSweepOpts()
        o.kernel, o.layout, o.offset, o.bytes, o.seed, o.canary = kernel, layout, offset, bytes, seed, canary
        o.invert, o.word0 = invert, word0
        for r, (first, count, and_mask, or_mask) in enumerate(force):
            o.force_first[r], o.force_count[r], o.force_and[r], o.force_or[r] = first, count, and_mask, or_mask
        o.flags = SELFTEST_F_INTERIORS if interiors else 0
        out = SelftestSweepOut()
        arr = (FaultWord * max(1, cap))()
        n = ctypes.c_int()
        self._check(lib.cro_selftest_sweep(self.handle, dev, ctypes.byref(o), ctypes.byref(out), None, 0, arr, cap,
                                           ctypes.byref(n)), allow=(ERR_BUFFER_SMALL,))
        buf = alloc(out.buf_bytes)
        raw = (ctypes.c_char * out.buf_bytes).from_buffer(buf)
        self._check(lib.cro_selftest_sweep(self.handle, dev, ctypes.byref(o), ctypes.byref(out), raw, out.buf_bytes, arr,
                                           cap, ctypes.byref(n)))
        del raw                                   # release the export: the caller may resize a bytearray
        return out, buf, [arr[i] for i in range(n.value)]


def node_inventory(proc_root: Optional[str], in_process: List[DevInfo]) -> List[DevInfo]:
    """What cro_enumerate answers for a context managing `in_process` on a node whose /proc is at proc_root:
    the driver's registry is re-read, devices attached later are flagged DEV_NEEDS_HELPER, removed ones are dropped."""
    arr = (DevInfo * max(1, len(in_process)))(*in_process)
    out = (DevInfo * 64)()
    n = ctypes.c_int()
    rc = lib.cro_node_inventory(_b(proc_root), arr, len(in_process), out, 64, ctypes.byref(n))
    if rc != OK:
        raise ProbeError(rc, "cro_node_inventory")
    return [out[i] for i in range(n.value)]


def probe_uuid(ctx: Optional["ProbeContext"], uuid: str) -> ProbeResult:
    """cro_probe_uuid: in-process probe, or the helper process for a GPU attached after init (ctx may be None)."""
    r = ProbeResult()
    rc = lib.cro_probe_uuid(ctx.handle if ctx is not None else None, _b(uuid), ctypes.byref(r))
    if rc not in (OK, ERR_CHECKSUM):
        buf = ctypes.create_string_buffer(1024)
        lib.cro_last_error(ctx.handle if ctx is not None else None, buf, 1024)
        raise ProbeError(rc, buf.value.decode("utf-8", "replace"))
    return r


def chase_end(minor_src: int, minor_dst: int, hops: int) -> int:
    """Slot reached after `hops` steps of the latency permutation of the directed pair (host arithmetic)."""
    e = ctypes.c_uint32()
    rc = lib.cro_chase_end(minor_src, minor_dst, hops, ctypes.byref(e))
    if rc != OK:
        raise ProbeError(rc, "cro_chase_end")
    return e.value


def validate_env(name: Optional[str] = None, value: Optional[str] = None) -> str:
    """"" when the CRO_* knob (or, with no name, the process environment) is legal, else the reference-style
    sentence "the env variable X has an invalid value: 'v'" (composableresource_adapter.go:44)."""
    err = ctypes.create_string_buffer(512)
    rc = lib.cro_validate_env(_b(name), _b(value), err, 512)
    return "" if rc == OK else err.value.decode("utf-8", "replace")


def fabric_check_resource(kind: str, machine_body: str, res_type: str, model: str, device_id: str) -> str:
    """CdiProvider.CheckResource decision (fm/client.go:314-359, cm/client.go:262-304); "" = healthy."""
    err = ctypes.create_string_buffer(2048)
    lib.cro_fabric_check_resource(_b(kind), _b(machine_body), _b(res_type), _b(model), _b(device_id), err, 2048)
    return err.value.decode("utf-8", "surrogateescape")


def fabric_get_resources(kind: str, machine_body: str, node_name: str, machine_uuid: str) -> List[Dict]:
    """CdiProvider.GetResources decode for one node (fm/client.go:385-410, cm/client.go:335-343)."""
    return json.loads(_text(lib.cro_fabric_get_resources, _b(kind), _b(machine_body), _b(node_name), _b(machine_uuid)))


def fabric_list_devices(request: Dict) -> Dict:
    """CdiProvider.GetResources of the FM / CM client over a scripted fabric (what the UpstreamSyncer
    tick reads: upstreamsyncer_controller.go:77-84).  request = {"env": {...}, "fabric": {...}}."""
    return json.loads(_text(lib.cro_fabric_list_devices, _b(json.dumps(request))))


def token_from_reply(reply: Dict) -> Dict:
    """What fti.CachedToken.Token makes of the id_manager's answer (fti/token.go:96-175):
    reply = {"secret_error","transport_error","status","body"} -> {"error", "expiry"}."""
    return json.loads(_text(lib.cro_token_from_reply, _b(json.dumps(reply))))


def local_node_op(ctx: Optional["ProbeContext"], request: Dict) -> Dict:
    """One node-side operation of internal/utils/gpus.go run locally (scans native, read-only commands spawned,
    mutating ones only with allow_mutation).  See cro_local_node_op in include/croprobe.h."""
    return json.loads(_text(lib.cro_local_node_op, ctx.handle if ctx is not None else None, _b(json.dumps(request))))


def describe_wire_type(name: str) -> Dict:
    """The reply struct a fabric decoder walks, as the library describes it (declaration order)."""
    return json.loads(_text(lib.cro_describe_wire_type, _b(name)))


def local_exec(argv: List[str], allow_mutation: bool = False, exec_deadline_ms: int = 0, native_nvml: bool = True,
               nvml_lib: str = "") -> Dict:
    """One command through the node-local executor (read-only allow-list while allow_mutation is false; deadline).
    The detach side's nvidia-smi invocations (compute apps, drain -q/-m/-r, -pm) are answered through NVML in this
    process when it is there ("how": "native"); nvml_lib names another libnvidia-ml (tests load a stand-in)."""
    req = {"argv": argv, "allow_mutation": allow_mutation, "native_nvml": native_nvml}
    if nvml_lib:
        req["nvml_lib"] = nvml_lib
    if exec_deadline_ms:
        req["exec_deadline_ms"] = exec_deadline_ms
    return json.loads(_text(lib.cro_local_exec, _b(json.dumps(req))))


def scan_cmdline_for(proc_root: str, needle: str) -> bool:
    found = ctypes.c_int(0)
    rc = lib.cro_scan_cmdline_for(_b(proc_root), _b(needle), ctypes.byref(found))
    if rc != OK:
        raise ProbeError(rc, "cro_scan_cmdline_for")
    return bool(found.value)


def CheckNoGPULoadsFromOutput(std_out: str, std_err: str, exec_err: Optional[str], pod_name: str, node_name: str,
                              target_uuid: Optional[str], driver_enabled: bool) -> str:
    """utils.CheckNoGPULoads parse + decision (internal/utils/gpus.go:145-186); returns the error text ("" = nil)."""
    err = ctypes.create_string_buffer(4096)
    lib.cro_check_no_gpu_loads(_b(std_out), _b(std_err), _b(exec_err), _b(pod_name), _b(node_name), _b(target_uuid),
                               int(driver_enabled), err, 4096)
    return err.value.decode("utf-8", "surrogateescape")


def checkGPUDrainStatusFromOutput(std_out: str, std_err: str, exec_err: Optional[str], node_name: str,
                                  bus_id: str) -> Tuple[bool, str]:
    """checkGPUDrainStatus (internal/utils/gpus.go:964-1012); returns (draining, error text)."""
    err = ctypes.create_string_buffer(4096)
    d = ctypes.c_int(0)
    lib.cro_check_gpu_drain_status(_b(std_out), _b(std_err), _b(exec_err), _b(node_name), _b(bus_id), ctypes.byref(d), err, 4096)
    return bool(d.value), err.value.decode("utf-8", "surrogateescape")


def CheckDeviceFileScanResult(std_out: str, std_err: str, exec_err: Optional[str], rke2: bool = False) -> str:
    err = ctypes.create_string_buffer(4096)
    lib.cro_check_device_file_scan(_b(std_out), _b(std_err), _b(exec_err), int(rke2), err, 4096)
    return err.value.decode("utf-8", "surrogateescape")


def scan_device_file_holders(target: str, proc_root: Optional[str] = None, rke2: bool = False) -> str:
    """Native fd scan (replaces the shell scripts at internal/utils/gpus.go:236-260, 441-457)."""
    return _text(lib.cro_scan_device_file_holders, _b(proc_root), _b(target), int(rke2))


class Cluster:
    """In-memory API server + both reconcilers (cro_sim_*): the caller of the hot path.

    Mirrors ComposabilityRequestReconciler / ComposableResourceReconciler
    (internal/controller/*.go); drives the storm / churn configs."""

    def __init__(self, config: Dict, ctx: Optional[ProbeContext] = None) -> None:
        h = ctypes.c_void_p()
        rc = lib.cro_sim_create(ctx.handle if ctx is not None else None, _b(json.dumps(config)), ctypes.byref(h))
        if rc != OK:
            raise ProbeError(rc, "cro_sim_create")
        self.handle = h
        self._ctx = ctx   # keep the probe context alive

    def close(self) -> None:
        if getattr(self, "handle", None):
            lib.cro_sim_destroy(self.handle)
            self.handle = None

    def __enter__(self) -> "Cluster":
        return self

    def __exit__(self, *a) -> None:
        self.close()

    def _err_call(self, fn, arg: str) -> str:
        err = ctypes.create_string_buffer(1024)
        fn(self.handle, _b(arg), err, 1024)
        return err.value.decode("utf-8", "replace")

    def apply(self, name: str, resource: Dict) -> str:
        """kubectl apply of a ComposabilityRequest; returns "" or the admission error."""
        return self._err_call(lib.cro_sim_apply, json.dumps({"name": name, "resource": resource}))

    def plant(self, obj: Dict) -> str:
        return self._err_call(lib.cro_sim_plant, json.dumps(obj))

    def delete(self, name: str) -> bool:
        return lib.cro_sim_delete(self.handle, _b(name)) == OK

    def reconcile_request(self, name: str) -> str:
        """One Reconcile of the request controller; returns the reconcile error ("" = nil)."""
        return self._err_call(lib.cro_sim_reconcile_request, name)

    def reconcile_resource(self, name: str) -> str:
        """One Reconcile of the ComposableResource controller; returns the reconcile error ("" = nil)."""
        return self._err_call(lib.cro_sim_reconcile_resource, name)

    def sync_upstream(self, devices: List[Dict], now_s: int) -> str:
        """One UpstreamSyncer tick (upstreamsyncer_controller.go:77-136) at time now_s."""
        err = ctypes.create_string_buffer(1024)
        lib.cro_sim_sync_upstream(self.handle, _b(json.dumps(devices)), now_s, err, 1024)
        return err.value.decode("utf-8", "replace")

    def run(self, max_reconciles: int = 0) -> Dict:
        rc, raw = _text_call(lib.cro_sim_run, self.handle, max_reconciles, cap=1 << 16)
        if rc != OK:
            raise ProbeError(rc)
        return json.loads(raw.decode())

    def dump(self) -> Dict:
        rc, raw = _text_call(lib.cro_sim_dump, self.handle, cap=1 << 22)
        if rc != OK:
            raise ProbeError(rc)
        return json.loads(raw.decode())
