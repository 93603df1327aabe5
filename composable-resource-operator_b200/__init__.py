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
        ("test_inject_after", ctypes.c_uint32), ("test_inject_count", ctypes.c_uint32),
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


# SM sparse probe (cro_probe_sparse, cro_sparse_expected); verdicts and marks are COMPUTE_*
SPARSE_LEG_S8, SPARSE_LEG_E4M3, SPARSE_LEG_E5M2, SPARSE_LEG_BF16, SPARSE_LEG_F16, SPARSE_LEG_TF32 = range(6)
SPARSE_LEGS, SPARSE_ALL_LEGS = 6, 0x3F
SPARSE_ANSWER_S8, SPARSE_ANSWER_SMALL, SPARSE_ANSWER_SMALL256, SPARSE_ANSWER_SMALL128 = range(4)
SPARSE_ANSWERS = 4
SPARSE_M, SPARSE_N, SPARSE_K, SPARSE_K16, SPARSE_TF32_K = 128, 256, 512, 256, 128
SPARSE_RECORDS, SPARSE_MAX_SMS, SPARSE_MAX_ITERATIONS, SPARSE_MAX_ROUNDS = 4096, 256, 65536, 64


class SparseOpts(ctypes.Structure):
    _fields_ = [("iterations", ctypes.c_uint32), ("legs", ctypes.c_uint32), ("max_rounds", ctypes.c_uint32),
                ("test_inject_leg", ctypes.c_int32), ("test_inject_sm", ctypes.c_int32),
                ("test_inject_iteration", ctypes.c_uint32), ("test_inject_row", ctypes.c_int32),
                ("test_inject_col", ctypes.c_int32), ("test_inject_mask", ctypes.c_uint64), ("test_meta", ctypes.c_uint32),
                ("test_meta_leg", ctypes.c_int32), ("test_meta_sm", ctypes.c_int32), ("test_meta_iteration", ctypes.c_uint32),
                ("test_meta_row", ctypes.c_uint32), ("test_meta_group", ctypes.c_uint32)]


class SparseResult(ctypes.Structure):
    """cro_sparse_result: status, verdict and per-leg counts, coverage and times of one sparse probe call."""
    _fields_ = [("status", ctypes.c_int32), ("verdict", ctypes.c_uint32), ("seed", ctypes.c_uint64),
                ("call", ctypes.c_uint64), ("sm_count", ctypes.c_uint32), ("legs", ctypes.c_uint32),
                ("host_ref_ns", ctypes.c_uint64), ("nsmid", ctypes.c_uint32), ("bad_sms", ctypes.c_uint32),
                ("bad_sm", ctypes.c_uint16 * 16), ("leg", ComputeLeg * SPARSE_LEGS)]


class SparseSm(ctypes.Structure):
    """One SM seen by a sparse probe call, with its counts, times and COMPUTE_PERSISTENT / _INTERMITTENT mark per leg."""
    _fields_ = [("smid", ctypes.c_uint32), ("reserved", ctypes.c_uint32), ("leg", ComputeSmLeg * SPARSE_LEGS)]


class SparseFault(ctypes.Structure):
    """One wrong element of a last iteration's answer: leg, SM, row, column, the exact answer and the raw 32 bits got."""
    _fields_ = [("leg", ctypes.c_uint32), ("smid", ctypes.c_uint32), ("row", ctypes.c_uint32), ("col", ctypes.c_uint32),
                ("expected", ctypes.c_int32), ("actual_bits", ctypes.c_uint32)]


# SM warp-MMA probe (cro_probe_warpmma, cro_warpmma_expected); verdicts and marks are COMPUTE_*
WARPMMA_LEG_S8, WARPMMA_LEG_F16, WARPMMA_LEG_BF16, WARPMMA_LEG_TF32, WARPMMA_LEG_F16ACC, WARPMMA_LEG_MOVE = range(6)
WARPMMA_LEGS, WARPMMA_ALL_LEGS = 6, 0x3F
WARPMMA_ANSWER_S8, WARPMMA_ANSWER_SMALL, WARPMMA_ANSWER_SMALL128, WARPMMA_ANSWER_NARROW, WARPMMA_ANSWER_MOVE = range(5)
WARPMMA_ANSWERS = 5
WARPMMA_M, WARPMMA_N, WARPMMA_K, WARPMMA_TF32_K = 128, 256, 256, 128
WARPMMA_RECORDS, WARPMMA_MAX_SMS, WARPMMA_MAX_ITERATIONS, WARPMMA_MAX_ROUNDS = 4096, 256, 65536, 64


class WarpMmaOpts(ctypes.Structure):
    _fields_ = [("iterations", ctypes.c_uint32), ("legs", ctypes.c_uint32), ("max_rounds", ctypes.c_uint32),
                ("test_inject_leg", ctypes.c_int32), ("test_inject_sm", ctypes.c_int32),
                ("test_inject_iteration", ctypes.c_uint32), ("test_inject_row", ctypes.c_int32),
                ("test_inject_col", ctypes.c_int32), ("test_inject_mask", ctypes.c_uint64), ("test_addr", ctypes.c_uint32),
                ("test_addr_leg", ctypes.c_int32), ("test_addr_sm", ctypes.c_int32), ("test_addr_iteration", ctypes.c_uint32),
                ("test_addr_row", ctypes.c_uint32), ("test_addr_kstep", ctypes.c_uint32)]


class WarpMmaResult(ctypes.Structure):
    """cro_warpmma_result: status, verdict and per-leg counts, coverage and times of one warp-MMA probe call."""
    _fields_ = [("status", ctypes.c_int32), ("verdict", ctypes.c_uint32), ("seed", ctypes.c_uint64),
                ("call", ctypes.c_uint64), ("sm_count", ctypes.c_uint32), ("legs", ctypes.c_uint32),
                ("host_ref_ns", ctypes.c_uint64), ("nsmid", ctypes.c_uint32), ("bad_sms", ctypes.c_uint32),
                ("bad_sm", ctypes.c_uint16 * 16), ("leg", ComputeLeg * WARPMMA_LEGS)]


class WarpMmaSm(ctypes.Structure):
    """One SM seen by a warp-MMA probe call, with its counts, times and COMPUTE_PERSISTENT / _INTERMITTENT mark per leg."""
    _fields_ = [("smid", ctypes.c_uint32), ("reserved", ctypes.c_uint32), ("leg", ComputeSmLeg * WARPMMA_LEGS)]


class WarpMmaFault(ctypes.Structure):
    """One wrong element of a last iteration's answer: leg, SM, row, column, the exact answer and the raw bits got."""
    _fields_ = [("leg", ctypes.c_uint32), ("smid", ctypes.c_uint32), ("row", ctypes.c_uint32), ("col", ctypes.c_uint32),
                ("expected", ctypes.c_int32), ("actual_bits", ctypes.c_uint32)]


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


# register-file probe (cro_probe_regfile, cro_probe_regfile_uuid, cro_selftest_regfile_classify)
REGFILE_SLOTS, REGFILE_THREADS, REGFILE_ELEMENTS, REGFILE_RECORDS, REGFILE_MAX_SMS = 224, 256, 2, 4096, 256
REGFILE_MAX_ITERATIONS, REGFILE_MAX_ROUNDS = 4096, 64
REGFILE_NONE, REGFILE_SM, REGFILE_ALL = 0, 1, 2
REGFILE_PERSISTENT, REGFILE_INTERMITTENT = 1, 2


class RegfileOpts(ctypes.Structure):
    _fields_ = [("iterations", ctypes.c_uint32), ("max_rounds", ctypes.c_uint32), ("deadline_ms", ctypes.c_int32),
                ("test_inject_sm", ctypes.c_int32), ("test_inject_warp", ctypes.c_int32), ("test_inject_lane", ctypes.c_int32),
                ("test_inject_slot", ctypes.c_int32), ("test_inject_element", ctypes.c_uint32),
                ("test_inject_iteration", ctypes.c_uint32), ("test_inject_mask", ctypes.c_uint32)]


class RegfileResult(ctypes.Structure):
    """cro_regfile_result: status, verdict, bad SMs, per-element counts, the fold and its closed form, coverage and
    times, the kernel's registers and NVML's SRAM health of one register-file probe call."""
    _fields_ = [("status", ctypes.c_int32), ("verdict", ctypes.c_uint32), ("seed", ctypes.c_uint64), ("call", ctypes.c_uint64),
                ("sm_count", ctypes.c_uint32), ("nsmid", ctypes.c_uint32), ("cuda_error", ctypes.c_int32),
                ("health", ctypes.c_uint32), ("iterations", ctypes.c_uint32), ("rounds", ctypes.c_uint32),
                ("slots", ctypes.c_uint32), ("threads", ctypes.c_uint32), ("num_regs", ctypes.c_uint32),
                ("regs_per_sm", ctypes.c_uint32), ("sms_covered", ctypes.c_uint32), ("complete", ctypes.c_uint32),
                ("ctas", ctypes.c_uint32), ("unpublished", ctypes.c_uint32), ("failed_sms", ctypes.c_uint32),
                ("bad_sms", ctypes.c_uint32), ("bad_sm", ctypes.c_uint16 * 16),
                ("mismatches", ctypes.c_uint64 * REGFILE_ELEMENTS), ("fold_mismatches", ctypes.c_uint64),
                ("recorded", ctypes.c_uint64), ("sms_listed", ctypes.c_uint32), ("reserved", ctypes.c_uint32),
                ("bits_checked", ctypes.c_uint64), ("ns", ctypes.c_uint64), ("timer_ns", ctypes.c_uint64),
                ("wall_ns", ctypes.c_uint64), ("helper_ns", ctypes.c_uint64), ("fold_xor", ctypes.c_uint64),
                ("fold_sum", ctypes.c_uint64), ("fold_wsum", ctypes.c_uint64), ("expect_xor", ctypes.c_uint64),
                ("expect_sum", ctypes.c_uint64), ("expect_wsum", ctypes.c_uint64), ("before", SramHealth),
                ("after", SramHealth)]

    @property
    def fold(self) -> Tuple[int, int, int]:
        return (self.fold_xor, self.fold_sum, self.fold_wsum)

    @property
    def expect(self) -> Tuple[int, int, int]:
        return (self.expect_xor, self.expect_sum, self.expect_wsum)


class RegfileSm(ctypes.Structure):
    """One SM seen by a register-file probe call: its per-element counts, fold mismatches, times and REGFILE_PERSISTENT /
    _INTERMITTENT mark."""
    _fields_ = [("smid", ctypes.c_uint32), ("mark", ctypes.c_uint32), ("mismatches", ctypes.c_uint64 * REGFILE_ELEMENTS),
                ("fold_mismatches", ctypes.c_uint64), ("ns", ctypes.c_uint64), ("cycles", ctypes.c_uint64),
                ("ctas", ctypes.c_uint32), ("reserved", ctypes.c_uint32)]


class RegfileFault(ctypes.Structure):
    """One failed compare: element, iteration, SM, warp, lane, slot, expected and actual word."""
    _fields_ = [("element", ctypes.c_uint32), ("iteration", ctypes.c_uint32), ("smid", ctypes.c_uint32),
                ("warp", ctypes.c_uint32), ("lane", ctypes.c_uint32), ("slot", ctypes.c_uint32),
                ("expected", ctypes.c_uint32), ("actual", ctypes.c_uint32)]


class RegfileCta(ctypes.Structure):
    """cro_regfile_cta: what one CTA of the register-file probe publishes at the end of a round."""
    _fields_ = [("stamp", ctypes.c_uint64), ("t0", ctypes.c_uint64), ("t1", ctypes.c_uint64), ("cycles", ctypes.c_uint64),
                ("count", ctypes.c_uint64 * REGFILE_ELEMENTS), ("last", ctypes.c_uint64), ("fold_x", ctypes.c_uint64),
                ("fold_s", ctypes.c_uint64), ("fold_w", ctypes.c_uint64), ("smid", ctypes.c_uint32), ("nsmid", ctypes.c_uint32),
                ("block", ctypes.c_uint32), ("reserved", ctypes.c_uint32)]


assert ctypes.sizeof(RegfileOpts) == 40 and ctypes.sizeof(RegfileResult) == 296 and ctypes.sizeof(RegfileSm) == 56 \
    and ctypes.sizeof(RegfileFault) == 32 and ctypes.sizeof(RegfileCta) == 96, ctypes.sizeof(RegfileResult)


# cross-lane probe (cro_probe_xlane, cro_probe_xlane_uuid, cro_xlane_expected, cro_selftest_xlane_classify)
XLANE_LEG_SHFL, XLANE_LEG_VOTE, XLANE_LEG_MATCH, XLANE_LEG_REDUX, XLANE_LEG_ATOMS = range(5)
XLANE_LEGS, XLANE_ALL_LEGS, XLANE_THREADS, XLANE_WARPS, XLANE_THREAD_RECORDS = 5, 0x1F, 256, 8, 4
XLANE_RECORDS, XLANE_MAX_SMS, XLANE_MAX_ITERATIONS, XLANE_MAX_ROUNDS = 4096, 256, 4096, 64
XLANE_SHFL_OPS, XLANE_VOTE_OPS, XLANE_MATCH_OPS, XLANE_REDUX_OPS, XLANE_ATOMS_OPS, XLANE_MAX_OPS = 177, 384, 64, 1296, 60, 1296
XLANE_OPS = [XLANE_SHFL_OPS, XLANE_VOTE_OPS, XLANE_MATCH_OPS, XLANE_REDUX_OPS, XLANE_ATOMS_OPS]
XLANE_NONE, XLANE_SM, XLANE_ALL = 0, 1, 2
XLANE_PERSISTENT, XLANE_INTERMITTENT = 1, 2


class XlaneOpts(ctypes.Structure):
    _fields_ = [("iterations", ctypes.c_uint32), ("legs", ctypes.c_uint32), ("max_rounds", ctypes.c_uint32),
                ("deadline_ms", ctypes.c_int32), ("test_inject_leg", ctypes.c_int32), ("test_inject_sm", ctypes.c_int32),
                ("test_inject_warp", ctypes.c_int32), ("test_inject_lane", ctypes.c_int32), ("test_inject_op", ctypes.c_uint32),
                ("test_inject_iteration", ctypes.c_uint32), ("test_inject_mask", ctypes.c_uint64)]


class XlaneResult(ctypes.Structure):
    """cro_xlane_result: status, verdict, bad SMs, per-leg counts, ops checked, folds and closed forms, coverage and
    times of one cross-lane probe call."""
    _fields_ = [("status", ctypes.c_int32), ("verdict", ctypes.c_uint32), ("seed", ctypes.c_uint64), ("call", ctypes.c_uint64),
                ("sm_count", ctypes.c_uint32), ("nsmid", ctypes.c_uint32), ("cuda_error", ctypes.c_int32), ("legs", ctypes.c_uint32),
                ("iterations", ctypes.c_uint32), ("rounds", ctypes.c_uint32), ("sms_covered", ctypes.c_uint32),
                ("complete", ctypes.c_uint32), ("ctas", ctypes.c_uint32), ("unpublished", ctypes.c_uint32),
                ("threads_unpublished", ctypes.c_uint32), ("failed_sms", ctypes.c_uint32), ("bad_sms", ctypes.c_uint32),
                ("failed_legs", ctypes.c_uint32), ("bad_sm", ctypes.c_uint16 * 16), ("recorded", ctypes.c_uint64),
                ("sms_listed", ctypes.c_uint32), ("reserved", ctypes.c_uint32), ("mismatches", ctypes.c_uint64 * XLANE_LEGS),
                ("ops_checked", ctypes.c_uint64 * XLANE_LEGS), ("fold_mismatches", ctypes.c_uint64 * XLANE_LEGS),
                ("leg_ns", ctypes.c_uint64 * XLANE_LEGS), ("fold", (ctypes.c_uint64 * 3) * XLANE_LEGS),
                ("expect", (ctypes.c_uint64 * 3) * XLANE_LEGS), ("ns", ctypes.c_uint64), ("timer_ns", ctypes.c_uint64),
                ("wall_ns", ctypes.c_uint64), ("helper_ns", ctypes.c_uint64)]


class XlaneSm(ctypes.Structure):
    """One SM seen by a cross-lane probe call: its failed legs, per-leg counts, fold mismatches, times and
    XLANE_PERSISTENT / _INTERMITTENT mark."""
    _fields_ = [("smid", ctypes.c_uint32), ("mark", ctypes.c_uint32), ("failed_legs", ctypes.c_uint32), ("ctas", ctypes.c_uint32),
                ("mismatches", ctypes.c_uint64 * XLANE_LEGS), ("fold_mismatches", ctypes.c_uint64), ("ns", ctypes.c_uint64),
                ("cycles", ctypes.c_uint64)]


class XlaneFault(ctypes.Structure):
    """One failed compare: leg, op, iteration, SM, warp, lane, the source lane of a shuffle's expected value (peer),
    expected and actual result."""
    _fields_ = [("leg", ctypes.c_uint32), ("op", ctypes.c_uint32), ("iteration", ctypes.c_uint32), ("smid", ctypes.c_uint32),
                ("warp", ctypes.c_uint32), ("lane", ctypes.c_uint32), ("peer", ctypes.c_uint32), ("reserved", ctypes.c_uint32),
                ("expected", ctypes.c_uint64), ("actual", ctypes.c_uint64)]


class XlaneThread(ctypes.Structure):
    """cro_xlane_thread: what one thread of the cross-lane probe publishes at the end of a launch."""
    _fields_ = [("stamp", ctypes.c_uint64), ("count", ctypes.c_uint64), ("last", ctypes.c_uint64), ("fold_x", ctypes.c_uint64),
                ("fold_s", ctypes.c_uint64), ("fold_w", ctypes.c_uint64)]


class XlaneCta(ctypes.Structure):
    """cro_xlane_cta: what thread 0 of a CTA of the cross-lane probe publishes at the end of a launch."""
    _fields_ = [("stamp", ctypes.c_uint64), ("t0", ctypes.c_uint64), ("t1", ctypes.c_uint64), ("cycles", ctypes.c_uint64),
                ("smid", ctypes.c_uint32), ("nsmid", ctypes.c_uint32), ("block", ctypes.c_uint32), ("reserved", ctypes.c_uint32)]


assert ctypes.sizeof(XlaneOpts) == 48 and ctypes.sizeof(XlaneResult) == 560 and ctypes.sizeof(XlaneSm) == 80 \
    and ctypes.sizeof(XlaneFault) == 48 and ctypes.sizeof(XlaneThread) == 48 and ctypes.sizeof(XlaneCta) == 48, \
    ctypes.sizeof(XlaneResult)


# ALU probe (cro_probe_alu, cro_probe_alu_uuid, cro_alu_expected, cro_selftest_alu_classify)
ALU_LEG_LOGIC, ALU_LEG_SHIFT, ALU_LEG_IADD, ALU_LEG_IMUL, ALU_LEG_FLOAT = range(5)
ALU_LEGS, ALU_ALL_LEGS, ALU_THREADS, ALU_WARPS, ALU_THREAD_RECORDS = 5, 0x1F, 256, 8, 4
ALU_RECORDS, ALU_MAX_SMS, ALU_MAX_ITERATIONS, ALU_MAX_ROUNDS = 4096, 256, 65536, 64
ALU_LOGIC_OPS, ALU_SHIFT_OPS, ALU_IADD_OPS, ALU_IMUL_OPS, ALU_FLOAT_OPS, ALU_MAX_OPS = 538, 76, 200, 100, 360, 538
ALU_OPS = [ALU_LOGIC_OPS, ALU_SHIFT_OPS, ALU_IADD_OPS, ALU_IMUL_OPS, ALU_FLOAT_OPS]
ALU_NONE, ALU_SM, ALU_ALL = 0, 1, 2
ALU_PERSISTENT, ALU_INTERMITTENT = 1, 2


class AluOpts(ctypes.Structure):
    _fields_ = [("iterations", ctypes.c_uint32), ("legs", ctypes.c_uint32), ("max_rounds", ctypes.c_uint32),
                ("deadline_ms", ctypes.c_int32), ("test_inject_leg", ctypes.c_int32), ("test_inject_sm", ctypes.c_int32),
                ("test_inject_warp", ctypes.c_int32), ("test_inject_lane", ctypes.c_int32), ("test_inject_op", ctypes.c_uint32),
                ("test_inject_iteration", ctypes.c_uint32), ("test_inject_operand", ctypes.c_uint32), ("reserved", ctypes.c_uint32),
                ("test_inject_mask", ctypes.c_uint64)]


class AluResult(ctypes.Structure):
    """cro_alu_result: the cross-lane result's fields (status, verdict, bad SMs, per-leg counts, folds, coverage and
    times) and the time the host took to build the call's table."""
    _fields_ = XlaneResult._fields_ + [("table_ns", ctypes.c_uint64)]


class AluSm(ctypes.Structure):
    """One SM seen by an ALU probe call: its failed legs, per-leg counts, fold mismatches, times and mark."""
    _fields_ = XlaneSm._fields_


class AluRecord(ctypes.Structure):
    """cro_alu_record: one table entry, the operands of one (leg, op, warp, lane) and the exact result."""
    _fields_ = [("in_", ctypes.c_uint64 * 4), ("out", ctypes.c_uint64 * 3), ("reserved", ctypes.c_uint64)]


class AluFault(ctypes.Structure):
    """One failed compare: leg, op, iteration, SM, warp, lane, the table's operands, expected and actual result."""
    _fields_ = [("leg", ctypes.c_uint32), ("op", ctypes.c_uint32), ("iteration", ctypes.c_uint32), ("smid", ctypes.c_uint32),
                ("warp", ctypes.c_uint32), ("lane", ctypes.c_uint32), ("reserved", ctypes.c_uint32 * 2), ("in_", ctypes.c_uint64 * 4),
                ("expected", ctypes.c_uint64 * 3), ("actual", ctypes.c_uint64 * 3)]


class AluThread(ctypes.Structure):
    """cro_alu_thread: what one thread of the ALU probe publishes at the end of a launch."""
    _fields_ = XlaneThread._fields_


class AluCta(ctypes.Structure):
    """cro_alu_cta: what thread 0 of a CTA of the ALU probe publishes at the end of a launch."""
    _fields_ = XlaneCta._fields_


assert ctypes.sizeof(AluOpts) == 56 and ctypes.sizeof(AluResult) == 568 and ctypes.sizeof(AluSm) == 80 \
    and ctypes.sizeof(AluRecord) == 64 and ctypes.sizeof(AluFault) == 112 and ctypes.sizeof(AluThread) == 48 \
    and ctypes.sizeof(AluCta) == 48, ctypes.sizeof(AluResult)


# Barrier probe (cro_probe_barrier, cro_probe_barrier_uuid, cro_barrier_expected, cro_selftest_barrier_classify)
BARRIER_LEG_BAR, BARRIER_LEG_MBAR, BARRIER_LEG_CLUSTER = range(3)
BARRIER_LEGS, BARRIER_ALL_LEGS, BARRIER_THREADS, BARRIER_WARPS, BARRIER_THREAD_RECORDS = 3, 0x7, 256, 8, 4
BARRIER_RECORDS, BARRIER_MAX_SMS, BARRIER_MAX_ITERATIONS, BARRIER_MAX_ROUNDS, BARRIER_MAX_PAIRS = 4096, 256, 65536, 64, 16
BARRIER_BAR_OPS, BARRIER_MBAR_OPS, BARRIER_CLUSTER_OPS, BARRIER_MAX_OPS = 64, 8, 17, 64
BARRIER_OPS = [BARRIER_BAR_OPS, BARRIER_MBAR_OPS, BARRIER_CLUSTER_OPS]
BARRIER_WAIT_NS = 20000000
(BARRIER_FORM_POPC, BARRIER_FORM_AND, BARRIER_FORM_OR, BARRIER_FORM_ARRIVE, BARRIER_FORM_TICKET, BARRIER_FORM_COUNT,
 BARRIER_FORM_DROP, BARRIER_FORM_TX, BARRIER_FORM_CBAR, BARRIER_FORM_ST_B32, BARRIER_FORM_ST_B64, BARRIER_FORM_ST_V2,
 BARRIER_FORM_ST_V4, BARRIER_FORM_RED_ADD, BARRIER_FORM_RED_ADD64, BARRIER_FORM_RED_MIN, BARRIER_FORM_RED_MAX,
 BARRIER_FORM_RED_MINS, BARRIER_FORM_RED_MAXS, BARRIER_FORM_RED_AND, BARRIER_FORM_RED_OR, BARRIER_FORM_RED_XOR,
 BARRIER_FORM_RED_INC, BARRIER_FORM_RED_DEC) = range(24)
BARRIER_KIND_VALUE, BARRIER_KIND_EARLY, BARRIER_KIND_TICKET, BARRIER_KIND_TIMEOUT = range(4)
BARRIER_NONE, BARRIER_SM, BARRIER_ALL, BARRIER_LINK = 0, 1, 2, 3
BARRIER_PERSISTENT, BARRIER_INTERMITTENT = 1, 2


class BarrierOpts(ctypes.Structure):
    _fields_ = [("iterations", ctypes.c_uint32), ("legs", ctypes.c_uint32), ("max_rounds", ctypes.c_uint32),
                ("deadline_ms", ctypes.c_int32), ("cluster", ctypes.c_uint32), ("test_inject_leg", ctypes.c_int32),
                ("test_inject_sm", ctypes.c_int32), ("test_inject_warp", ctypes.c_int32), ("test_inject_lane", ctypes.c_int32),
                ("test_inject_op", ctypes.c_uint32), ("test_inject_iteration", ctypes.c_uint32), ("reserved", ctypes.c_uint32),
                ("test_inject_mask", ctypes.c_uint64)]


class BarrierPair(ctypes.Structure):
    _fields_ = [("smid", ctypes.c_uint16), ("peer_smid", ctypes.c_uint16)]


class BarrierResult(ctypes.Structure):
    """cro_barrier_result: the cross-lane result's counts for three legs, the cluster size, the kept timeout records,
    the CLUSTER leg's coverage and failed (SM, peer SM) pairs, times and the host's table build time."""
    _fields_ = XlaneResult._fields_[:21] + [("cluster", ctypes.c_uint32)] + [
        ("mismatches", ctypes.c_uint64 * 3), ("ops_checked", ctypes.c_uint64 * 3), ("fold_mismatches", ctypes.c_uint64 * 3),
        ("leg_ns", ctypes.c_uint64 * 3), ("fold", (ctypes.c_uint64 * 3) * 3), ("expect", (ctypes.c_uint64 * 3) * 3),
        ("timeouts", ctypes.c_uint64), ("cluster_sms", ctypes.c_uint32), ("bad_pairs", ctypes.c_uint32),
        ("bad_pair", BarrierPair * 16), ("ns", ctypes.c_uint64), ("timer_ns", ctypes.c_uint64), ("wall_ns", ctypes.c_uint64),
        ("helper_ns", ctypes.c_uint64), ("table_ns", ctypes.c_uint64)]


class BarrierSm(ctypes.Structure):
    """One SM seen by a barrier probe call: its failed legs, per-leg counts, fold mismatches, times and mark."""
    _fields_ = [("smid", ctypes.c_uint32), ("mark", ctypes.c_uint32), ("failed_legs", ctypes.c_uint32), ("ctas", ctypes.c_uint32),
                ("mismatches", ctypes.c_uint64 * 3), ("fold_mismatches", ctypes.c_uint64), ("ns", ctypes.c_uint64),
                ("cycles", ctypes.c_uint64)]


class BarrierRow(ctypes.Structure):
    """cro_barrier_row: one row of the table."""
    _fields_ = [("form", ctypes.c_uint32), ("bar", ctypes.c_uint32), ("count", ctypes.c_uint32), ("warps", ctypes.c_uint32),
                ("producers", ctypes.c_uint32), ("phases", ctypes.c_uint32), ("held", ctypes.c_uint32), ("arriver", ctypes.c_uint32),
                ("expect", ctypes.c_uint64), ("pred", ctypes.c_uint32 * 8), ("next_rank", ctypes.c_uint8 * 8),
                ("slot_init", ctypes.c_uint64 * 8), ("slot_expect", ctypes.c_uint64 * 8)]


class BarrierFault(ctypes.Structure):
    """One failed check: leg, row, iteration, SM, warp, lane, kind, barrier id (or form), phase, slot, peer SM,
    expected and actual."""
    _fields_ = [("leg", ctypes.c_uint32), ("op", ctypes.c_uint32), ("iteration", ctypes.c_uint32), ("smid", ctypes.c_uint32),
                ("warp", ctypes.c_uint32), ("lane", ctypes.c_uint32), ("kind", ctypes.c_uint32), ("bar", ctypes.c_uint32),
                ("phase", ctypes.c_uint32), ("slot", ctypes.c_uint32), ("peer_smid", ctypes.c_uint32), ("reserved", ctypes.c_uint32),
                ("expected", ctypes.c_uint64), ("actual", ctypes.c_uint64)]


class BarrierThread(ctypes.Structure):
    """cro_barrier_thread: what one thread of the barrier probe publishes at the end of a launch."""
    _fields_ = XlaneThread._fields_


class BarrierCta(ctypes.Structure):
    """cro_barrier_cta: what thread 0 of a CTA of the barrier probe publishes at the end of a launch."""
    _fields_ = XlaneCta._fields_


assert ctypes.sizeof(BarrierOpts) == 56 and ctypes.sizeof(BarrierResult) == 488 and ctypes.sizeof(BarrierSm) == 64 \
    and ctypes.sizeof(BarrierRow) == 208 and ctypes.sizeof(BarrierFault) == 64 and ctypes.sizeof(BarrierThread) == 48 \
    and ctypes.sizeof(BarrierCta) == 48, ctypes.sizeof(BarrierResult)


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
SM_LEGS_COMPUTE, SM_LEGS_PRECISION, SM_LEGS_SPARSE, SM_LEGS_WARPMMA = 0, 1, 3, 4


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
SELFTEST_GUARD_BYTES, SELFTEST_F_INTERIORS, SELFTEST_F_XOR = 2 << 20, 1, 2


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
assert ctypes.sizeof(SparseResult) == 704 and ctypes.sizeof(SparseSm) == 248 and ctypes.sizeof(SparseFault) == 24 \
    and ctypes.sizeof(SparseOpts) == 64, ctypes.sizeof(SparseResult)
assert ctypes.sizeof(WarpMmaResult) == 704 and ctypes.sizeof(WarpMmaSm) == 248 and ctypes.sizeof(WarpMmaFault) == 24 \
    and ctypes.sizeof(WarpMmaOpts) == 64, ctypes.sizeof(WarpMmaResult)
assert ctypes.sizeof(FaultReport) == 928 and ctypes.sizeof(LocatePass) == 120, ctypes.sizeof(FaultReport)
assert ctypes.sizeof(LinkResult) == 984 and ctypes.sizeof(PciPath) == 272, ctypes.sizeof(LinkResult)
assert ctypes.sizeof(ScanReport) == 12632 and ctypes.sizeof(ScanOpts) == 72, ctypes.sizeof(ScanReport)
assert ctypes.sizeof(SramResult) == 568 and ctypes.sizeof(SramSm) == 168 and ctypes.sizeof(SramFault) == 48, ctypes.sizeof(SramResult)
assert ctypes.sizeof(L2Result) == 616 and ctypes.sizeof(L2Sm) == 128 and ctypes.sizeof(L2Fault) == 56, ctypes.sizeof(L2Result)
# health check (cro_check_health, cro_check_health_uuid): the six checks in one call
HEALTH_COMPUTE, HEALTH_PRECISION, HEALTH_SRAM, HEALTH_L2, HEALTH_LINK, HEALTH_SCAN = 0x01, 0x02, 0x04, 0x08, 0x10, 0x20
HEALTH_ALL = 0x3F
HEALTH_CHECKS = 6
HEALTH_NAMES = ("compute", "precision", "sram", "l2", "link", "scan")      # bit c, in run order


class HealthOpts(ctypes.Structure):
    """cro_health_opts: the checks to run (0: all) and each check's own options (zeroed: its defaults)."""
    _fields_ = [("checks", ctypes.c_uint32), ("reserved0", ctypes.c_uint32), ("compute", ComputeOpts),
                ("precision", PrecisionOpts), ("sram", SramOpts), ("l2", L2Opts), ("link", LinkOpts), ("scan", ScanOpts)]


class HealthResult(ctypes.Structure):
    """cro_health_result: the call's summary and each check's own result."""
    _fields_ = [("status", ctypes.c_int32), ("checks", ctypes.c_uint32), ("ran", ctypes.c_uint32), ("failed", ctypes.c_uint32),
                ("errored", ctypes.c_uint32), ("not_run", ctypes.c_uint32), ("incomplete", ctypes.c_uint32),
                ("reserved0", ctypes.c_uint32), ("check_status", ctypes.c_int32 * HEALTH_CHECKS),
                ("check_ns", ctypes.c_uint64 * HEALTH_CHECKS), ("seed_base", ctypes.c_uint64), ("helper_ns", ctypes.c_uint64),
                ("compute", ComputeResult), ("precision", PrecisionResult), ("sram", SramResult), ("l2", L2Result),
                ("link", LinkResult), ("scan", ScanReport)]


# (name, element type) of each list of cro_health_records, in order
HEALTH_LISTS = [("compute_sms", ComputeSm), ("compute_faults", ComputeFault), ("precision_sms", PrecisionSm),
                ("precision_faults", PrecisionFault), ("sram_sms", SramSm), ("sram_faults", SramFault), ("l2_sms", L2Sm),
                ("l2_faults", L2Fault), ("link_faults", LinkFault), ("scan_words", FaultWord)]


class HealthRecords(ctypes.Structure):
    """cro_health_records: the caller's {array, cap, n} per list of records."""
    _fields_ = [f for name, t in HEALTH_LISTS
                for f in ((name, ctypes.POINTER(t)), (name + "_cap", ctypes.c_int32), (name + "_n", ctypes.c_int32))]


assert ctypes.sizeof(HealthOpts) == 312 and ctypes.sizeof(HealthResult) == 16328 and ctypes.sizeof(HealthRecords) == 160
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
    "cro_selftest_p2p_plan",
    "cro_locate_faults", "cro_emit_fault_annotations_json",
    "cro_probe_host_link", "cro_probe_host_link_uuid", "cro_pci_link_path", "cro_emit_link_annotations_json",
    "cro_probe_compute", "cro_probe_compute_uuid", "cro_compute_expected", "cro_emit_compute_annotations_json",
    "cro_probe_precision", "cro_probe_precision_uuid", "cro_precision_expected", "cro_emit_precision_annotations_json",
    "cro_probe_sparse", "cro_probe_sparse_uuid", "cro_sparse_expected", "cro_emit_sparse_annotations_json",
    "cro_probe_warpmma", "cro_probe_warpmma_uuid", "cro_warpmma_expected", "cro_emit_warpmma_annotations_json",
    "cro_scan_hbm", "cro_scan_hbm_uuid", "cro_read_hbm_health", "cro_emit_scan_annotations_json",
    "cro_probe_sram", "cro_probe_sram_uuid", "cro_read_sram_health", "cro_emit_sram_annotations_json",
    "cro_probe_regfile", "cro_probe_regfile_uuid", "cro_emit_regfile_annotations_json", "cro_selftest_regfile_classify",
    "cro_probe_xlane", "cro_probe_xlane_uuid", "cro_xlane_expected", "cro_emit_xlane_annotations_json",
    "cro_selftest_xlane_classify",
    "cro_probe_alu", "cro_probe_alu_uuid", "cro_alu_expected", "cro_emit_alu_annotations_json", "cro_selftest_alu_classify",
    "cro_probe_barrier", "cro_probe_barrier_uuid", "cro_barrier_expected", "cro_emit_barrier_annotations_json",
    "cro_selftest_barrier_classify",
    "cro_probe_l2", "cro_probe_l2_uuid", "cro_read_l2_health", "cro_emit_l2_annotations_json", "cro_selftest_l2_classify",
    "cro_selftest_sm_legs_classify", "cro_selftest_sram_classify",
    "cro_selftest_locate_collect", "cro_selftest_scan_collect", "cro_selftest_link_classify",
    "cro_check_health", "cro_check_health_uuid", "cro_selftest_health_classify", "cro_emit_health_annotations_json",
]

# test hooks: the word checks' reports from caller-given device output
# (cro_selftest_locate_collect, cro_selftest_scan_collect, cro_selftest_link_classify)
class LocateCounters(ctypes.Structure):
    """cro_locate_counters: a word-checking kernel's exact counts of one pass or check."""
    _fields_ = [("mismatches", ctypes.c_uint64), ("claims", ctypes.c_uint64), ("bits", ctypes.c_uint64 * 64)]


class LocateRecord(ctypes.Structure):
    """cro_locate_record: one word a word-checking kernel recorded."""
    _fields_ = [("word", ctypes.c_uint64), ("expected", ctypes.c_uint64), ("actual", ctypes.c_uint64)]


class SweepSlot(ctypes.Structure):
    """cro_sweep_slot: one sweep's result slot as the kernels write it.  Its last word is the header's union of
    `mismatches` and `pad`: kept as `pad` here, read as `mismatches`."""
    _fields_ = [("x", ctypes.c_uint64), ("s", ctypes.c_uint64), ("w", ctypes.c_uint64), ("t0", ctypes.c_uint64),
                ("t1", ctypes.c_uint64), ("stamp", ctypes.c_uint64), ("n_words", ctypes.c_uint64), ("pad", ctypes.c_uint64)]

    @property
    def mismatches(self) -> int:
        """A comparing read's count of words that differ from the pattern (0 from a read that only folds)."""
        return self.pad


LINK_SLOTS = LINK_WORD_CHECKS + 5             # [k] check k's fold, two write roles, the closed forms of P1, P2, P3
SCAN_SLOTS = SCAN_PASSES * SCAN_MAX_CHUNKS + SCAN_MAX_CHUNKS
LOCATE_SLOTS = 3 * LOCATE_PASSES
assert ctypes.sizeof(LocateCounters) == 528 and ctypes.sizeof(LocateRecord) == 24 and ctypes.sizeof(SweepSlot) == 64

# Slot map of a device's sweep-slot array (cro_sweep_slot, 64 bytes each); the cro_selftest_* hooks take such arrays.
SLOT_FILL, SLOT_SWEEP0, MAX_SWEEPS_EACH, SLOT_EXPECT, SLOT_PREFIX, SLOT_P2P0 = 0, 1, 30, 62, 63, 64
SLOT_SCRATCH = SLOT_P2P0 + 3 * MAX_DEVICES
SLOT_COUNT = SLOT_SCRATCH + 4
SLOT_BYTES = 64

# test hook: the full-box probe's schedule (cro_selftest_p2p_plan)
P2P_PLAN_OPS, P2P_PLAN_ROUNDS = 4096, 16
P2P_OP_HBM, P2P_OP_PREFIX, P2P_OP_RECORD, P2P_OP_WAIT, P2P_OP_READ, P2P_OP_PUSH, P2P_OP_REREAD, P2P_OP_CHASE, \
    P2P_OP_FINALIZE = range(1, 10)
P2P_EV_HBM, P2P_EV_PUSH, P2P_EV_REREAD, P2P_EV_CHASE = range(1, 5)


class P2POp(ctypes.Structure):
    """cro_p2p_op: one stream operation of the full-box plan."""
    _fields_ = [("kind", ctypes.c_uint8), ("dev", ctypes.c_uint8), ("peer", ctypes.c_uint8), ("event", ctypes.c_uint8),
                ("round", ctypes.c_uint16), ("slot", ctypes.c_uint16), ("bytes", ctypes.c_uint64)]


class P2PFinalizePlan(ctypes.Structure):
    """cro_p2p_finalize_plan: one device's p2p_finalize arguments other than pointers, and the peers it checks and chases."""
    _fields_ = [("n", ctypes.c_uint32), ("self", ctypes.c_uint32), ("have_push", ctypes.c_uint32),
                ("push_folded", ctypes.c_uint32), ("p2p_bytes", ctypes.c_uint64), ("peer_mask", ctypes.c_uint32),
                ("chase_mask", ctypes.c_uint32)]


class P2PPlan(ctypes.Structure):
    """cro_p2p_plan: what cro_probe_all enqueues, in order."""
    _fields_ = [("p2p_bytes", ctypes.c_uint64), ("n_rounds", ctypes.c_uint32), ("n_ops", ctypes.c_uint32),
                ("n_pairs", ctypes.c_uint8 * P2P_PLAN_ROUNDS), ("pair", (ctypes.c_uint8 * MAX_DEVICES) * P2P_PLAN_ROUNDS),
                ("fin", P2PFinalizePlan * MAX_DEVICES), ("op", P2POp * P2P_PLAN_OPS)]


assert ctypes.sizeof(P2POp) == 16 and ctypes.sizeof(P2PFinalizePlan) == 32 and ctypes.sizeof(P2PPlan) == 66336


def selftest_p2p_plan(sweep_bytes: List[int], p2p_bytes: int, access: List[List[int]], flags: int = 0, unidir: bool = False,
                      write_variant: int = 3) -> P2PPlan:
    """cro_selftest_p2p_plan: the plan cro_probe_all walks on len(sweep_bytes) devices of those sizes, access[i] being
    device i's 8 p2p_access bytes, with cro_opts.flags `flags`, the CRO_P2P_UNIDIR knob and CRO_P2P_WRITE_VARIANT."""
    n = len(sweep_bytes)
    assert len(access) == n and all(len(row) == 8 for row in access)
    out = P2PPlan()
    rc = lib.cro_selftest_p2p_plan(n, (ctypes.c_uint64 * max(1, n))(*sweep_bytes), p2p_bytes,
                                   (ctypes.c_uint8 * max(8, 8 * n))(*[v for row in access for v in row]), flags, int(unidir),
                                   write_variant, ctypes.byref(out))
    if rc != OK:
        raise ProbeError(rc, "cro_selftest_p2p_plan")
    return out


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
        "cro_selftest_p2p_plan": (i32, [u32, ctypes.POINTER(u64), u64, ctypes.POINTER(ctypes.c_uint8), u32, u32, u32,
                                        ctypes.POINTER(P2PPlan)]),
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
        "cro_probe_sparse": (i32, [vp, i32, ctypes.POINTER(SparseOpts), ctypes.POINTER(SparseResult), ctypes.POINTER(SparseSm),
                                   i32, ctypes.POINTER(i32), ctypes.POINTER(SparseFault), i32, ctypes.POINTER(i32)]),
        "cro_probe_sparse_uuid": (i32, [vp, c, ctypes.POINTER(SparseOpts), i32, ctypes.POINTER(SparseResult),
                                        ctypes.POINTER(SparseSm), i32, ctypes.POINTER(i32), ctypes.POINTER(SparseFault), i32,
                                        ctypes.POINTER(i32), ctypes.POINTER(u64)]),
        "cro_sparse_expected": (i32, [i32, u64, ctypes.POINTER(ctypes.c_int32)]),
        "cro_emit_sparse_annotations_json": (i32, [ctypes.POINTER(SparseResult)] + out),
        "cro_probe_warpmma": (i32, [vp, i32, ctypes.POINTER(WarpMmaOpts), ctypes.POINTER(WarpMmaResult),
                                    ctypes.POINTER(WarpMmaSm), i32, ctypes.POINTER(i32), ctypes.POINTER(WarpMmaFault), i32,
                                    ctypes.POINTER(i32)]),
        "cro_probe_warpmma_uuid": (i32, [vp, c, ctypes.POINTER(WarpMmaOpts), i32, ctypes.POINTER(WarpMmaResult),
                                         ctypes.POINTER(WarpMmaSm), i32, ctypes.POINTER(i32), ctypes.POINTER(WarpMmaFault), i32,
                                         ctypes.POINTER(i32), ctypes.POINTER(u64)]),
        "cro_warpmma_expected": (i32, [i32, u64, ctypes.POINTER(ctypes.c_int32)]),
        "cro_emit_warpmma_annotations_json": (i32, [ctypes.POINTER(WarpMmaResult)] + out),
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
        "cro_probe_regfile": (i32, [vp, i32, ctypes.POINTER(RegfileOpts), ctypes.POINTER(RegfileResult), ctypes.POINTER(RegfileSm),
                                    i32, ctypes.POINTER(i32), ctypes.POINTER(RegfileFault), i32, ctypes.POINTER(i32)]),
        "cro_probe_regfile_uuid": (i32, [vp, c, ctypes.POINTER(RegfileOpts), ctypes.POINTER(RegfileResult),
                                         ctypes.POINTER(RegfileSm), i32, ctypes.POINTER(i32), ctypes.POINTER(RegfileFault), i32,
                                         ctypes.POINTER(i32)]),
        "cro_emit_regfile_annotations_json": (i32, [ctypes.POINTER(RegfileResult)] + out),
        "cro_selftest_regfile_classify": (i32, [u32, u64, u32, u64, u32, ctypes.POINTER(RegfileCta), u64,
                                                ctypes.POINTER(RegfileFault), ctypes.POINTER(RegfileResult),
                                                ctypes.POINTER(RegfileSm), i32, ctypes.POINTER(i32), ctypes.POINTER(RegfileFault),
                                                i32, ctypes.POINTER(i32)]),
        "cro_emit_sram_annotations_json": (i32, [ctypes.POINTER(SramResult)] + out),
        "cro_probe_xlane": (i32, [vp, i32, ctypes.POINTER(XlaneOpts), ctypes.POINTER(XlaneResult), ctypes.POINTER(XlaneSm),
                                  i32, ctypes.POINTER(i32), ctypes.POINTER(XlaneFault), i32, ctypes.POINTER(i32)]),
        "cro_probe_xlane_uuid": (i32, [vp, c, ctypes.POINTER(XlaneOpts), ctypes.POINTER(XlaneResult), ctypes.POINTER(XlaneSm),
                                       i32, ctypes.POINTER(i32), ctypes.POINTER(XlaneFault), i32, ctypes.POINTER(i32)]),
        "cro_xlane_expected": (i32, [i32, u64, u32, i32, ctypes.POINTER(u64)]),
        "cro_emit_xlane_annotations_json": (i32, [ctypes.POINTER(XlaneResult)] + out),
        "cro_selftest_xlane_classify": (i32, [u32, u32, u64, u32, u64, u32, ctypes.POINTER(XlaneCta), ctypes.POINTER(XlaneThread),
                                              ctypes.POINTER(XlaneFault), ctypes.POINTER(XlaneResult), ctypes.POINTER(XlaneSm), i32,
                                              ctypes.POINTER(i32), ctypes.POINTER(XlaneFault), i32, ctypes.POINTER(i32)]),
        "cro_probe_alu": (i32, [vp, i32, ctypes.POINTER(AluOpts), ctypes.POINTER(AluResult), ctypes.POINTER(AluSm),
                                i32, ctypes.POINTER(i32), ctypes.POINTER(AluFault), i32, ctypes.POINTER(i32)]),
        "cro_probe_alu_uuid": (i32, [vp, c, ctypes.POINTER(AluOpts), ctypes.POINTER(AluResult), ctypes.POINTER(AluSm),
                                     i32, ctypes.POINTER(i32), ctypes.POINTER(AluFault), i32, ctypes.POINTER(i32)]),
        "cro_alu_expected": (i32, [i32, u64, i32, ctypes.POINTER(AluRecord)]),
        "cro_emit_alu_annotations_json": (i32, [ctypes.POINTER(AluResult)] + out),
        "cro_selftest_alu_classify": (i32, [u32, u32, u64, u32, u64, u32, ctypes.POINTER(AluCta), ctypes.POINTER(AluThread),
                                            ctypes.POINTER(AluFault), ctypes.POINTER(AluResult), ctypes.POINTER(AluSm), i32,
                                            ctypes.POINTER(i32), ctypes.POINTER(AluFault), i32, ctypes.POINTER(i32)]),
        "cro_probe_barrier": (i32, [vp, i32, ctypes.POINTER(BarrierOpts), ctypes.POINTER(BarrierResult), ctypes.POINTER(BarrierSm),
                                    i32, ctypes.POINTER(i32), ctypes.POINTER(BarrierFault), i32, ctypes.POINTER(i32)]),
        "cro_probe_barrier_uuid": (i32, [vp, c, ctypes.POINTER(BarrierOpts), ctypes.POINTER(BarrierResult), ctypes.POINTER(BarrierSm),
                                         i32, ctypes.POINTER(i32), ctypes.POINTER(BarrierFault), i32, ctypes.POINTER(i32)]),
        "cro_barrier_expected": (i32, [i32, u64, u32, ctypes.POINTER(BarrierRow), ctypes.POINTER(u64)]),
        "cro_emit_barrier_annotations_json": (i32, [ctypes.POINTER(BarrierResult)] + out),
        "cro_selftest_barrier_classify": (i32, [u32, u32, u64, u32, u32, u64, u32, ctypes.POINTER(BarrierCta),
                                                ctypes.POINTER(BarrierThread), ctypes.POINTER(BarrierFault),
                                                ctypes.POINTER(BarrierResult), ctypes.POINTER(BarrierSm), i32, ctypes.POINTER(i32),
                                                ctypes.POINTER(BarrierFault), i32, ctypes.POINTER(i32)]),
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
        "cro_selftest_locate_collect": (i32, [u64, ctypes.POINTER(LocatePass), u32, ctypes.POINTER(LocateCounters),
                                              ctypes.POINTER(LocateRecord), ctypes.POINTER(u64), u64, ctypes.POINTER(SweepSlot),
                                              ctypes.POINTER(FaultReport), ctypes.POINTER(FaultWord), i32, ctypes.POINTER(i32)]),
        "cro_selftest_scan_collect": (i32, [i32, ctypes.POINTER(LocateCounters), ctypes.POINTER(LocateRecord),
                                            ctypes.POINTER(u64), u64, ctypes.POINTER(SweepSlot), ctypes.POINTER(ScanReport),
                                            ctypes.POINTER(FaultWord), i32, ctypes.POINTER(i32)]),
        "cro_selftest_link_classify": (i32, [u64, ctypes.POINTER(u64), u32, u32, ctypes.POINTER(LocateCounters),
                                             ctypes.POINTER(LocateRecord), ctypes.POINTER(u64), ctypes.POINTER(SweepSlot),
                                             ctypes.POINTER(u64), ctypes.POINTER(LinkResult), ctypes.POINTER(LinkFault), i32,
                                             ctypes.POINTER(i32)]),
        "cro_check_health": (i32, [vp, i32, ctypes.POINTER(HealthOpts), ctypes.POINTER(HealthResult), ctypes.POINTER(HealthRecords)]),
        "cro_check_health_uuid": (i32, [vp, c, ctypes.POINTER(HealthOpts), i32, ctypes.POINTER(HealthResult),
                                        ctypes.POINTER(HealthRecords), ctypes.POINTER(u64)]),
        "cro_selftest_health_classify": (i32, [u32, ctypes.POINTER(ctypes.c_int32), i32, ctypes.POINTER(HealthResult),
                                               ctypes.POINTER(u32)]),
        "cro_emit_health_annotations_json": (i32, [ctypes.POINTER(HealthResult)] + out),
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


def emit_sparse_annotations_json(r: SparseResult) -> str:
    """Additive cohdi.io/probe-sparse-* annotations of a probe_sparse result (Go-marshalled map[string]string)."""
    return _text(lib.cro_emit_sparse_annotations_json, ctypes.byref(r))


def emit_warpmma_annotations_json(r: WarpMmaResult) -> str:
    """Additive cohdi.io/probe-warpmma-* annotations of a probe_warpmma result (Go-marshalled map[string]string)."""
    return _text(lib.cro_emit_warpmma_annotations_json, ctypes.byref(r))


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


def emit_regfile_annotations_json(r: RegfileResult) -> str:
    """Additive cohdi.io/probe-regfile-* annotations of a register-file probe result (Go-marshalled map[string]string)."""
    return _text(lib.cro_emit_regfile_annotations_json, ctypes.byref(r))


def emit_xlane_annotations_json(r: XlaneResult) -> str:
    """Additive cohdi.io/probe-xlane-* annotations of a cross-lane probe result (Go-marshalled map[string]string)."""
    return _text(lib.cro_emit_xlane_annotations_json, ctypes.byref(r))


def xlane_expected(leg: int, seed: int, iteration: int, warp: int) -> List[int]:
    """cro_xlane_expected: every lane's expected result of every op of leg `leg` in iteration `iteration` of a call of
    seed `seed`, for warp `warp`: a list indexed op * 32 + lane (host arithmetic, no GPU)."""
    arr = (ctypes.c_uint64 * (XLANE_MAX_OPS * 32))()
    rc = lib.cro_xlane_expected(leg, seed, iteration, warp, arr)
    if rc != OK:
        raise ProbeError(rc, "cro_xlane_expected")
    return list(arr[:XLANE_OPS[leg] * 32])


def selftest_xlane_classify(legs: int, iterations: int, seed: int, sm_count: int, call: int, rounds, cap: Optional[int] = None):
    """cro_selftest_xlane_classify: the cross-lane probe's classification of call `call`.  rounds[leg index][round] =
    (sm_count XlaneCta, sm_count * XLANE_THREADS XlaneThread, sm_count * XLANE_THREADS * XLANE_THREAD_RECORDS
    XlaneFault), for each leg of `legs` in order, every leg the same number of rounds.  Returns (result, SM entries,
    faults); the result's status may be OK, ERR_CHECKSUM or ERR_UNSUPPORTED.  cap defaults to XLANE_RECORDS."""
    return _lane_classify("cro_selftest_xlane_classify", (legs, iterations, seed, sm_count, call), sm_count, rounds,
                          XLANE_RECORDS if cap is None else cap, XlaneCta, XlaneThread, XlaneFault, XLANE_THREADS,
                          XLANE_THREAD_RECORDS, XlaneResult, XlaneSm, XLANE_MAX_SMS)


def emit_alu_annotations_json(r: AluResult) -> str:
    """Additive cohdi.io/probe-alu-* annotations of an ALU probe result (Go-marshalled map[string]string)."""
    return _text(lib.cro_emit_alu_annotations_json, ctypes.byref(r))


def alu_expected(leg: int, seed: int, warp: int) -> List[AluRecord]:
    """cro_alu_expected: the table of a call of seed `seed` for leg `leg` and warp `warp`: a list of AluRecord indexed
    op * 32 + lane, each the operands and the exact result (host arithmetic, no GPU)."""
    arr = (AluRecord * (ALU_OPS[leg] * 32))()
    rc = lib.cro_alu_expected(leg, seed, warp, arr)
    if rc != OK:
        raise ProbeError(rc, "cro_alu_expected")
    return list(arr)


def selftest_alu_classify(legs: int, iterations: int, seed: int, sm_count: int, call: int, rounds, cap: Optional[int] = None):
    """cro_selftest_alu_classify: the ALU probe's classification of call `call`, as selftest_xlane_classify with
    AluCta, AluThread and AluFault.  Returns (result, SM entries, faults)."""
    return _lane_classify("cro_selftest_alu_classify", (legs, iterations, seed, sm_count, call), sm_count, rounds,
                          ALU_RECORDS if cap is None else cap, AluCta, AluThread, AluFault, ALU_THREADS, ALU_THREAD_RECORDS,
                          AluResult, AluSm, ALU_MAX_SMS)


def emit_barrier_annotations_json(r: BarrierResult) -> str:
    """Additive cohdi.io/probe-barrier-* annotations of a barrier probe result (Go-marshalled map[string]string)."""
    return _text(lib.cro_emit_barrier_annotations_json, ctypes.byref(r))


def barrier_expected(leg: int, seed: int, cluster: int = 2) -> Tuple[List[BarrierRow], List[int]]:
    """cro_barrier_expected: the table of a call of seed `seed` for leg `leg` (cluster: the CLUSTER leg's cluster
    size): its rows and its words, indexed (row * 256 + thread) * 2 + j (host arithmetic, no GPU)."""
    rows = (BarrierRow * BARRIER_OPS[leg])()
    words = (ctypes.c_uint64 * (BARRIER_OPS[leg] * BARRIER_THREADS * 2))()
    rc = lib.cro_barrier_expected(leg, seed, cluster, rows, words)
    if rc != OK:
        raise ProbeError(rc, "cro_barrier_expected")
    return list(rows), list(words)


def selftest_barrier_classify(legs: int, iterations: int, seed: int, cluster: int, sm_count: int, call: int, rounds,
                              cap: Optional[int] = None):
    """cro_selftest_barrier_classify: the barrier probe's classification of call `call`, as selftest_xlane_classify
    with BarrierCta, BarrierThread and BarrierFault.  Returns (result, SM entries, faults)."""
    return _lane_classify("cro_selftest_barrier_classify", (legs, iterations, seed, cluster, sm_count, call), sm_count, rounds,
                          BARRIER_RECORDS if cap is None else cap, BarrierCta, BarrierThread, BarrierFault, BARRIER_THREADS,
                          BARRIER_THREAD_RECORDS, BarrierResult, BarrierSm, BARRIER_MAX_SMS)


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
    """cro_selftest_sm_legs_classify: the compute (SM_LEGS_COMPUTE), precision (SM_LEGS_PRECISION), sparse
    (SM_LEGS_SPARSE) or warp-MMA (SM_LEGS_WARPMMA) probe's classification of call `call` on `grid` SMs.  Per leg l (every
    list is indexed by leg; legs 0: all): rounds[l] a list of (grid SmCta, the COMPUTE_MAX_SMS // 64 coverage words) per
    round, claims[l] and records[l] (ComputeFault / PrecisionFault / SparseFault / WarpMmaFault, the first min(claims[l],
    RECORDS)).  Returns (result, SM entries, faults); the result's status may be OK, ERR_CHECKSUM or ERR_UNSUPPORTED."""
    n_legs, result, sm, fault = {SM_LEGS_COMPUTE: (COMPUTE_LEGS, ComputeResult, ComputeSm, ComputeFault),
                                 SM_LEGS_SPARSE: (SPARSE_LEGS, SparseResult, SparseSm, SparseFault),
                                 SM_LEGS_WARPMMA: (WARPMMA_LEGS, WarpMmaResult, WarpMmaSm, WarpMmaFault)}.get(
        probe, (PRECISION_LEGS, PrecisionResult, PrecisionSm, PrecisionFault))
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


def selftest_regfile_classify(iterations: int, seed: int, sm_count: int, call: int, rounds: List[List[RegfileCta]],
                              claims: int, records: List[RegfileFault], cap: Optional[int] = None):
    """cro_selftest_regfile_classify: the register-file probe's classification of call `call`: rounds, each a list of
    sm_count RegfileCta, `claims` record claims and the first min(claims, REGFILE_RECORDS) records.  Returns (result, SM
    entries, faults); the result's status may be OK, ERR_CHECKSUM or ERR_UNSUPPORTED.  cap defaults to every record."""
    assert all(len(r) == sm_count for r in rounds) and len(records) == min(claims, REGFILE_RECORDS)
    flat = [x for r in rounds for x in r]
    ctas = (RegfileCta * max(1, len(flat)))(*flat)
    recs = (RegfileFault * max(1, len(records)))(*records)
    cap = len(records) if cap is None else cap
    rc, out = _per_sm(lib.cro_selftest_regfile_classify, (iterations, seed, sm_count, call, len(rounds), ctas, claims, recs),
                      RegfileResult, RegfileSm, REGFILE_MAX_SMS, RegfileFault, cap)
    if rc not in (OK, ERR_CHECKSUM, ERR_UNSUPPORTED):
        raise ProbeError(rc, "cro_selftest_regfile_classify")
    return out


def _word_checks(counters: List[LocateCounters], records, granules=None):
    """The flat arrays of the word-check hooks: counters, records[k] (the first min(claims, LOCATE_RECORDS) of each) in
    order, and granules[k] (each the same number of words) in order."""
    recs = [x for r in records for x in r]
    assert [len(r) for r in records] == [min(c.claims, LOCATE_RECORDS) for c in counters]
    gw = len(granules[0]) if granules else 0
    bits = [b for g in granules or [] for b in g]
    assert len(bits) == gw * len(counters)
    return ((LocateCounters * len(counters))(*counters), (LocateRecord * max(1, len(recs)))(*recs),
            (ctypes.c_uint64 * max(1, len(bits)))(*bits), gw)


def selftest_locate_collect(sweep_bytes: int, passes: List[LocatePass], counters: List[LocateCounters], records,
                            granules, slots: List[SweepSlot], cap: Optional[int] = None):
    """cro_selftest_locate_collect: the fault locator's report of len(passes) passes over a region of sweep_bytes, from
    pass p's counters[p], records[p] and granule words granules[p], and the LOCATE_SLOTS slots.  Returns (report,
    words); cap defaults to every located word."""
    ctr, recs, gran, gw = _word_checks(counters, records, granules)
    cap = sum(len(r) for r in records) if cap is None else cap
    out, words, n = FaultReport(), (FaultWord * max(1, cap))(), ctypes.c_int()
    rc = lib.cro_selftest_locate_collect(sweep_bytes, (LocatePass * len(passes))(*passes), len(passes), ctr, recs, gran, gw,
                                         (SweepSlot * LOCATE_SLOTS)(*slots), ctypes.byref(out), words, cap, ctypes.byref(n))
    if rc not in (OK, ERR_CHECKSUM):
        raise ProbeError(rc, "cro_selftest_locate_collect")
    return out, list(words[:n.value])


def selftest_scan_collect(chunks: List[Tuple[int, int]], elements_done: int, cuda_error: int, counters: List[LocateCounters],
                          records, granules, slots: List[SweepSlot], cap: Optional[int] = None):
    """cro_selftest_scan_collect: the scan's report over chunks [(word0, bytes)] after elements_done elements (and the
    CUDA error that stopped them, 0: none), from pass p's counters[p], records[p] and granule words granules[p], and
    the SCAN_SLOTS slots.  Returns (report, words); cap defaults to every recorded word."""
    ctr, recs, gran, gw = _word_checks(counters, records, granules)
    cap = sum(len(r) for r in records) if cap is None else cap
    out, words, n = ScanReport(), (FaultWord * max(1, cap))(), ctypes.c_int()
    out.n_chunks, out.elements_done = len(chunks), elements_done
    for k, (word0, nbytes) in enumerate(chunks):
        out.chunk[k].word0, out.chunk[k].bytes = word0, nbytes
    rc = lib.cro_selftest_scan_collect(cuda_error, ctr, recs, gran, gw, (SweepSlot * SCAN_SLOTS)(*slots), ctypes.byref(out),
                                       words, cap, ctypes.byref(n))
    if rc not in (OK, ERR_CHECKSUM, ERR_CUDA):
        raise ProbeError(rc, "cro_selftest_scan_collect")
    return out, list(words[:n.value])


def selftest_link_classify(bytes: int, seeds: List[int], minor: int, hops: int, counters: List[LocateCounters], records,
                           host: List[List[int]], slots: List[SweepSlot], chase_out: List[int], cap: Optional[int] = None):
    """cro_selftest_link_classify: the host link probe's word checks and chase of a call of L = bytes, from check k's
    counters[k], records[k] and host buffer host[k] (L / 8 words as the CPU read them), the LINK_SLOTS slots and the
    chase output (end slot, ns).  Returns (result, faults); cap defaults to every recorded fault."""
    ctr, recs, _, _ = _word_checks(counters, records)
    assert all(len(h) == bytes // 8 for h in host) and len(host) == LINK_WORD_CHECKS
    cap = sum(len(r) for r in records) if cap is None else cap
    out, faults, n = LinkResult(), (LinkFault * max(1, cap))(), ctypes.c_int()
    hw = (ctypes.c_uint64 * (LINK_WORD_CHECKS * (bytes // 8)))(*[w for h in host for w in h])
    rc = lib.cro_selftest_link_classify(bytes, (ctypes.c_uint64 * 3)(*seeds), minor, hops, ctr, recs, hw,
                                        (SweepSlot * LINK_SLOTS)(*slots), (ctypes.c_uint64 * 2)(*chase_out), ctypes.byref(out),
                                        faults, cap, ctypes.byref(n))
    if rc not in (OK, ERR_CHECKSUM):
        raise ProbeError(rc, "cro_selftest_link_classify")
    return out, list(faults[:n.value])


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


def _regfile_opts(iterations: int, max_rounds: int, deadline_ms: int,
                  inject: Optional[Tuple[int, int, int, int, int, int, int]]) -> RegfileOpts:
    o = RegfileOpts()
    o.iterations, o.max_rounds, o.deadline_ms = iterations, max_rounds, deadline_ms
    if inject is not None:
        (o.test_inject_sm, o.test_inject_warp, o.test_inject_lane, o.test_inject_slot, o.test_inject_element,
         o.test_inject_iteration, o.test_inject_mask) = inject
    return o


def probe_regfile_uuid(ctx: Optional["ProbeContext"], uuid: str, iterations: int = 0, max_rounds: int = 0, deadline_ms: int = 0,
                       inject: Optional[Tuple[int, int, int, int, int, int, int]] = None,
                       cap: int = 256) -> Tuple[RegfileResult, List[RegfileSm], List[RegfileFault]]:
    """cro_probe_regfile_uuid: the register-file probe of any GPU on the node, run by the helper process (ctx may be
    None).  Returns the result (its status is OK, ERR_CHECKSUM or ERR_CUDA), one entry per SM seen and up to `cap`
    records."""
    o = _regfile_opts(iterations, max_rounds, deadline_ms, inject)
    handle = ctx.handle if ctx is not None else None
    rc, out = _per_sm(lib.cro_probe_regfile_uuid, (handle, _b(uuid), ctypes.byref(o)), RegfileResult, RegfileSm, REGFILE_MAX_SMS,
                      RegfileFault, cap)
    if rc not in (OK, ERR_CHECKSUM, ERR_CUDA):
        raise _helper_error(rc, handle)
    return out


def _xlane_opts(iterations: int, legs: int, max_rounds: int, deadline_ms: int,
                inject: Optional[Tuple[int, int, int, int, int, int, int]]) -> XlaneOpts:
    o = XlaneOpts()
    o.iterations, o.legs, o.max_rounds, o.deadline_ms = iterations, legs, max_rounds, deadline_ms
    if inject is not None:
        (o.test_inject_leg, o.test_inject_sm, o.test_inject_warp, o.test_inject_lane, o.test_inject_op, o.test_inject_iteration,
         o.test_inject_mask) = inject
    return o


def probe_xlane_uuid(ctx: Optional["ProbeContext"], uuid: str, iterations: int = 0, legs: int = 0, max_rounds: int = 0,
                     deadline_ms: int = 0, inject: Optional[Tuple[int, int, int, int, int, int, int]] = None,
                     cap: int = 256) -> Tuple[XlaneResult, List[XlaneSm], List[XlaneFault]]:
    """cro_probe_xlane_uuid: the cross-lane probe of any GPU on the node, run by the helper process (ctx may be None).
    Returns the result (its status is OK, ERR_CHECKSUM or ERR_CUDA), one entry per SM seen and up to `cap` records."""
    o = _xlane_opts(iterations, legs, max_rounds, deadline_ms, inject)
    handle = ctx.handle if ctx is not None else None
    rc, out = _per_sm(lib.cro_probe_xlane_uuid, (handle, _b(uuid), ctypes.byref(o)), XlaneResult, XlaneSm, XLANE_MAX_SMS,
                      XlaneFault, cap)
    if rc not in (OK, ERR_CHECKSUM, ERR_CUDA):
        raise _helper_error(rc, handle)
    return out


def _alu_opts(iterations: int, legs: int, max_rounds: int, deadline_ms: int,
              inject: Optional[Tuple[int, int, int, int, int, int, int, int]]) -> AluOpts:
    o = AluOpts()
    o.iterations, o.legs, o.max_rounds, o.deadline_ms = iterations, legs, max_rounds, deadline_ms
    if inject is not None:
        (o.test_inject_leg, o.test_inject_sm, o.test_inject_warp, o.test_inject_lane, o.test_inject_op, o.test_inject_iteration,
         o.test_inject_operand, o.test_inject_mask) = inject
    return o


def probe_alu_uuid(ctx: Optional["ProbeContext"], uuid: str, iterations: int = 0, legs: int = 0, max_rounds: int = 0,
                   deadline_ms: int = 0, inject: Optional[Tuple[int, int, int, int, int, int, int, int]] = None,
                   cap: int = 256) -> Tuple[AluResult, List[AluSm], List[AluFault]]:
    """cro_probe_alu_uuid: the ALU probe of any GPU on the node, run by the helper process (ctx may be None).  Returns
    the result (its status is OK, ERR_CHECKSUM or ERR_CUDA), one entry per SM seen and up to `cap` records."""
    o = _alu_opts(iterations, legs, max_rounds, deadline_ms, inject)
    handle = ctx.handle if ctx is not None else None
    rc, out = _per_sm(lib.cro_probe_alu_uuid, (handle, _b(uuid), ctypes.byref(o)), AluResult, AluSm, ALU_MAX_SMS, AluFault, cap)
    if rc not in (OK, ERR_CHECKSUM, ERR_CUDA):
        raise _helper_error(rc, handle)
    return out


def _barrier_opts(iterations: int, legs: int, max_rounds: int, cluster: int, deadline_ms: int,
                  inject: Optional[Tuple[int, int, int, int, int, int, int]]) -> BarrierOpts:
    o = BarrierOpts()
    o.iterations, o.legs, o.max_rounds, o.cluster, o.deadline_ms = iterations, legs, max_rounds, cluster, deadline_ms
    if inject is not None:
        (o.test_inject_leg, o.test_inject_sm, o.test_inject_warp, o.test_inject_lane, o.test_inject_op, o.test_inject_iteration,
         o.test_inject_mask) = inject
    return o


def probe_barrier_uuid(ctx: Optional["ProbeContext"], uuid: str, iterations: int = 0, legs: int = 0, max_rounds: int = 0,
                       cluster: int = 0, deadline_ms: int = 0, inject: Optional[Tuple[int, int, int, int, int, int, int]] = None,
                       cap: int = 256) -> Tuple[BarrierResult, List[BarrierSm], List[BarrierFault]]:
    """cro_probe_barrier_uuid: the barrier probe of any GPU on the node, run by the helper process (ctx may be None).
    Returns the result (its status is OK, ERR_CHECKSUM or ERR_CUDA), one entry per SM seen and up to `cap` records."""
    o = _barrier_opts(iterations, legs, max_rounds, cluster, deadline_ms, inject)
    handle = ctx.handle if ctx is not None else None
    rc, out = _per_sm(lib.cro_probe_barrier_uuid, (handle, _b(uuid), ctypes.byref(o)), BarrierResult, BarrierSm, BARRIER_MAX_SMS,
                      BarrierFault, cap)
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


def _lane_classify(name: str, head: tuple, sm_count: int, rounds, cap: int, cta, thread, fault, threads: int,
                   thread_records: int, result, sm, max_sms: int):
    """One cro_selftest_<probe>_classify call of a lane probe (cross-lane, ALU, barrier): lib.<name>(*head, the round
    count, the CTA entries, thread entries and records of `rounds`, ...).  rounds[leg index][round] = (sm_count CTA
    entries, sm_count * threads thread entries, sm_count * threads * thread_records records), every leg the same number
    of rounds.  Returns (result, SM entries, faults); the result's status may be OK, ERR_CHECKSUM or ERR_UNSUPPORTED."""
    n_rounds = len(rounds[0]) if rounds else 0
    assert all(len(r) == n_rounds for r in rounds)
    flat = [rnd for leg in rounds for rnd in leg]
    ctas = (cta * max(1, sm_count * len(flat)))(*[x for rnd in flat for x in rnd[0]])
    thr = (thread * max(1, sm_count * threads * len(flat)))(*[x for rnd in flat for x in rnd[1]])
    recs = (fault * max(1, sm_count * threads * thread_records * len(flat)))(*[x for rnd in flat for x in rnd[2]])
    rc, out = _per_sm(getattr(lib, name), head + (n_rounds, ctas, thr, recs), result, sm, max_sms, fault, cap)
    if rc not in (OK, ERR_CHECKSUM, ERR_UNSUPPORTED):
        raise ProbeError(rc, name)
    return out


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


def _sparse_opts(iterations: int, legs: int, max_rounds: int, inject: Optional[Tuple[int, int, int, int, int, int]],
                 meta: Optional[Tuple[int, int, int, int, int]]) -> SparseOpts:
    o = SparseOpts()
    o.iterations, o.legs, o.max_rounds = iterations, legs, max_rounds
    if inject is not None:
        (o.test_inject_leg, o.test_inject_sm, o.test_inject_iteration, o.test_inject_row, o.test_inject_col,
         o.test_inject_mask) = inject
    if meta is not None:
        o.test_meta = 1
        o.test_meta_leg, o.test_meta_sm, o.test_meta_iteration, o.test_meta_row, o.test_meta_group = meta
    return o


def probe_sparse_uuid(ctx: Optional["ProbeContext"], uuid: str, iterations: int = 0, legs: int = SPARSE_ALL_LEGS,
                      max_rounds: int = 0, deadline_ms: int = 0, inject: Optional[Tuple[int, int, int, int, int, int]] = None,
                      meta: Optional[Tuple[int, int, int, int, int]] = None,
                      cap: int = 256) -> Tuple[SparseResult, List[SparseSm], List[SparseFault], int]:
    """cro_probe_sparse_uuid: the sparse probe of any GPU on the node, run by the helper process (ctx may be None).
    Returns the result (its status is OK, ERR_CHECKSUM or ERR_CUDA), one entry per SM seen, up to `cap` element records
    and the helper's spawn-to-exit time in ns."""
    o = _sparse_opts(iterations, legs, max_rounds, inject, meta)
    ns = ctypes.c_uint64()
    handle = ctx.handle if ctx is not None else None
    rc, out = _per_sm(lib.cro_probe_sparse_uuid, (handle, _b(uuid), ctypes.byref(o), deadline_ms), SparseResult, SparseSm,
                      SPARSE_MAX_SMS, SparseFault, cap, (ctypes.byref(ns),))
    if rc not in (OK, ERR_CHECKSUM, ERR_CUDA):
        raise _helper_error(rc, handle)
    return out + (ns.value,)


def _warpmma_opts(iterations: int, legs: int, max_rounds: int, inject: Optional[Tuple[int, int, int, int, int, int]],
                  addr: Optional[Tuple[int, int, int, int, int]]) -> WarpMmaOpts:
    o = WarpMmaOpts()
    o.iterations, o.legs, o.max_rounds = iterations, legs, max_rounds
    if inject is not None:
        (o.test_inject_leg, o.test_inject_sm, o.test_inject_iteration, o.test_inject_row, o.test_inject_col,
         o.test_inject_mask) = inject
    if addr is not None:
        o.test_addr = 1
        o.test_addr_leg, o.test_addr_sm, o.test_addr_iteration, o.test_addr_row, o.test_addr_kstep = addr
    return o


def probe_warpmma_uuid(ctx: Optional["ProbeContext"], uuid: str, iterations: int = 0, legs: int = WARPMMA_ALL_LEGS,
                       max_rounds: int = 0, deadline_ms: int = 0, inject: Optional[Tuple[int, int, int, int, int, int]] = None,
                       addr: Optional[Tuple[int, int, int, int, int]] = None,
                       cap: int = 256) -> Tuple[WarpMmaResult, List[WarpMmaSm], List[WarpMmaFault], int]:
    """cro_probe_warpmma_uuid: the warp-MMA probe of any GPU on the node, run by the helper process (ctx may be None).
    Returns the result (its status is OK, ERR_CHECKSUM or ERR_CUDA), one entry per SM seen, up to `cap` element records
    and the helper's spawn-to-exit time in ns."""
    o = _warpmma_opts(iterations, legs, max_rounds, inject, addr)
    ns = ctypes.c_uint64()
    handle = ctx.handle if ctx is not None else None
    rc, out = _per_sm(lib.cro_probe_warpmma_uuid, (handle, _b(uuid), ctypes.byref(o), deadline_ms), WarpMmaResult, WarpMmaSm,
                      WARPMMA_MAX_SMS, WarpMmaFault, cap, (ctypes.byref(ns),))
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


def emit_health_annotations_json(r: HealthResult) -> str:
    """Every ran check's own annotations and the cohdi.io/probe-health-* keys of a health result (one Go-marshalled
    map[string]string)."""
    return _text(lib.cro_emit_health_annotations_json, ctypes.byref(r))


def selftest_health_classify(checks: int, statuses: List[int]) -> Tuple[HealthResult, int]:
    """cro_selftest_health_classify: the stop and status rules for the selection `checks` (0: all) after the first
    len(statuses) checks to run returned `statuses`.  Returns the summary (status, checks, ran, failed, errored, not_run,
    check_status) and the HEALTH_* bit of the check to run next (0: none is left)."""
    out, nxt = HealthResult(), ctypes.c_uint32()
    rc = lib.cro_selftest_health_classify(checks, (ctypes.c_int32 * max(1, len(statuses)))(*statuses), len(statuses),
                                          ctypes.byref(out), ctypes.byref(nxt))
    if rc != OK:
        raise ProbeError(rc, "cro_selftest_health_classify")
    return out, nxt.value


def _health_opts(checks: int, compute=None, precision=None, sram=None, l2=None, link=None, scan=None) -> HealthOpts:
    """HealthOpts from the checks and each check's options, given as its struct or as a dict of the keyword arguments
    its own helper form takes (None: defaults)."""
    o = HealthOpts()
    o.checks = checks
    makers = {"compute": lambda a: _compute_opts(a.get("iterations", 0), a.get("alu_iterations", 0), a.get("legs", 0),
                                                 a.get("max_rounds", 0), a.get("inject")),
              "precision": lambda a: _precision_opts(a.get("iterations", 0), a.get("alu_iterations", 0), a.get("legs", 0),
                                                     a.get("max_rounds", 0), a.get("inject")),
              "sram": lambda a: _sram_opts(a.get("legs", 0), a.get("iterations", 0), a.get("cluster", 0), a.get("max_rounds", 0),
                                           a.get("deadline_ms", 0), a.get("inject")),
              "l2": lambda a: _l2_opts(a.get("bytes", 0), a.get("iterations", 0), a.get("a1_counters", 0), a.get("a2_counters", 0),
                                       a.get("deadline_ms", 0), a.get("inject")),
              "link": lambda a: _link_opts(a.get("bytes", 0), a.get("hops", 0), a.get("ctas", 0), a.get("inject")),
              "scan": lambda a: _scan_opts(a.get("max_bytes", 0), a.get("reserve_bytes", 0), a.get("seed", 0), a.get("deadline_ms", 0),
                                           a.get("chunk_bytes", 0), a.get("force"))}
    for name, given in (("compute", compute), ("precision", precision), ("sram", sram), ("l2", l2), ("link", link), ("scan", scan)):
        if given is not None:
            setattr(o, name, makers[name](given) if isinstance(given, dict) else given)
    return o


def _health_call(fn, head: tuple, tail: tuple, caps: Dict[str, int]):
    """fn(*head, result, records, *tail) with fresh arrays: caps[name] entries per list (per-SM lists default to
    every SM, the others to 256).  Returns the return code, the result and {list name: its records}."""
    r, rec, keep = HealthResult(), HealthRecords(), []
    for name, t in HEALTH_LISTS:
        cap = caps.get(name, 256 if not name.endswith("_sms") else COMPUTE_MAX_SMS)
        arr = (t * max(1, cap))()
        keep.append(arr)
        setattr(rec, name, ctypes.cast(arr, ctypes.POINTER(t)))
        setattr(rec, name + "_cap", cap)
    rc = fn(*head, ctypes.byref(r), ctypes.byref(rec), *tail)
    records = {name: [getattr(rec, name)[i] for i in range(getattr(rec, name + "_n"))] for name, _ in HEALTH_LISTS}
    return rc, r, records


def check_health_uuid(ctx: Optional["ProbeContext"], uuid: str, checks: int = 0, compute=None, precision=None, sram=None, l2=None,
                      link=None, scan=None, deadline_ms: int = 0, caps: Optional[Dict[str, int]] = None
                      ) -> Tuple[HealthResult, Dict[str, list], int]:
    """cro_check_health_uuid: the selected checks (0: all six) of any GPU on the node in one helper process (ctx may be
    None).  Each check's options: its struct, or a dict of the keyword arguments its own helper form takes (None:
    defaults).  caps: records asked for per list (HEALTH_LISTS names).  Returns the result (its status is OK,
    ERR_CHECKSUM, or the first other status a check returned), {list name: records} and the helper's spawn-to-exit ns.
    Raises ProbeError when no check ran: options refused, or no result from the helper."""
    o = _health_opts(checks, compute, precision, sram, l2, link, scan)
    ns = ctypes.c_uint64()
    handle = ctx.handle if ctx is not None else None
    rc, r, records = _health_call(lib.cro_check_health_uuid, (handle, _b(uuid), ctypes.byref(o), deadline_ms), (ctypes.byref(ns),),
                                  caps or {})
    if rc != OK and r.ran == 0:         # refused, or the helper gave no result: no check ran
        raise _helper_error(rc, handle)
    return r, records, ns.value


def sparse_expected(answer: int, seed: int) -> List[int]:
    """cro_sparse_expected: the SPARSE_ANSWER_* answer tile of the operands of `seed`, SPARSE_M x SPARSE_N int32
    values, row-major (host arithmetic, no GPU)."""
    arr = (ctypes.c_int32 * (SPARSE_M * SPARSE_N))()
    rc = lib.cro_sparse_expected(answer, seed, arr)
    if rc != OK:
        raise ProbeError(rc, "cro_sparse_expected")
    return list(arr)


def warpmma_expected(answer: int, seed: int) -> List[int]:
    """cro_warpmma_expected: the WARPMMA_ANSWER_* answer tile of the operands of `seed`, WARPMMA_M x WARPMMA_N int32
    values, row-major (host arithmetic, no GPU)."""
    arr = (ctypes.c_int32 * (WARPMMA_M * WARPMMA_N))()
    rc = lib.cro_warpmma_expected(answer, seed, arr)
    if rc != OK:
        raise ProbeError(rc, "cro_warpmma_expected")
    return list(arr)


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
                 inject: Optional[Tuple[int, ...]] = None) -> None:
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
        if inject is not None:            # (after sweep number, word index, xor mask[, words]): fault injection inside the probe
            o.flags |= F_TEST_INJECT
            o.test_inject_after, o.test_inject_word, o.test_inject_mask = inject[:3]
            o.test_inject_count = inject[3] if len(inject) > 3 else 0
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

    def probe_sparse(self, dev: int = 0, iterations: int = 0, legs: int = SPARSE_ALL_LEGS, max_rounds: int = 0,
                     inject: Optional[Tuple[int, int, int, int, int, int]] = None,
                     meta: Optional[Tuple[int, int, int, int, int]] = None,
                     cap: int = 256) -> Tuple[SparseResult, List[SparseSm], List[SparseFault]]:
        """cro_probe_sparse: every SM computes its answer tiles with 2:4 structured-sparsity wgmma in s8, E4M3, E5M2,
        BF16, F16 and TF32 (1:2) and checks each value exactly.  iterations / max_rounds = 0: the defaults.  inject =
        (leg, sm, iteration, row, col, mask) is the test-only accumulator XOR (sm, row, col: -1 for every one; mask at
        most 32 bits); meta = (leg, sm, iteration, row, group) the test-only metadata substitution (sm -1: every SM).
        Returns the result (its status is OK or ERR_CHECKSUM), one entry per SM seen and up to `cap` element records."""
        o = _sparse_opts(iterations, legs, max_rounds, inject, meta)
        rc, out = _per_sm(lib.cro_probe_sparse, (self.handle, dev, ctypes.byref(o)), SparseResult, SparseSm, SPARSE_MAX_SMS,
                          SparseFault, cap)
        self._check(rc, allow=(ERR_CHECKSUM,))
        return out

    def probe_warpmma(self, dev: int = 0, iterations: int = 0, legs: int = WARPMMA_ALL_LEGS, max_rounds: int = 0,
                      inject: Optional[Tuple[int, int, int, int, int, int]] = None,
                      addr: Optional[Tuple[int, int, int, int, int]] = None,
                      cap: int = 256) -> Tuple[WarpMmaResult, List[WarpMmaSm], List[WarpMmaFault]]:
        """cro_probe_warpmma: every SM computes its answer tiles with warp-synchronous mma.sync in s8, F16, BF16, TF32
        and F16 accumulation from ldmatrix fragments, and moves a tile through ldmatrix, movmatrix and stmatrix, and
        checks each value exactly.  iterations / max_rounds = 0: the defaults.  inject = (leg, sm, iteration, row, col,
        mask) is the test-only accumulator XOR (sm, row, col: -1 for every one; mask at most the leg's value width);
        addr = (leg, sm, iteration, row, kstep) the test-only fragment-address substitution (sm -1: every SM).  Returns
        the result (its status is OK or ERR_CHECKSUM), one entry per SM seen and up to `cap` element records."""
        o = _warpmma_opts(iterations, legs, max_rounds, inject, addr)
        rc, out = _per_sm(lib.cro_probe_warpmma, (self.handle, dev, ctypes.byref(o)), WarpMmaResult, WarpMmaSm,
                          WARPMMA_MAX_SMS, WarpMmaFault, cap)
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

    def probe_regfile(self, dev: int = 0, iterations: int = 0, max_rounds: int = 0,
                      inject: Optional[Tuple[int, int, int, int, int, int, int]] = None,
                      cap: int = 256) -> Tuple[RegfileResult, List[RegfileSm], List[RegfileFault]]:
        """cro_probe_regfile: every SM's registers hold REGFILE_SLOTS pattern words per thread, as 0 and as 1, across two
        barriers, and every word is compared.  iterations = 0 / max_rounds = 0: the defaults.  inject = (sm, warp, lane,
        slot, element, iteration, mask) is the test-only stand-in for a bad cell (sm, warp, lane, slot: -1 for every
        one).  Returns the result (its status is OK, ERR_CHECKSUM or ERR_CUDA), one entry per SM seen and up to `cap`
        slot records."""
        o = _regfile_opts(iterations, max_rounds, 0, inject)
        rc, out = _per_sm(lib.cro_probe_regfile, (self.handle, dev, ctypes.byref(o)), RegfileResult, RegfileSm, REGFILE_MAX_SMS,
                          RegfileFault, cap)
        self._check(rc, allow=(ERR_CHECKSUM, ERR_CUDA))
        return out

    def probe_xlane(self, dev: int = 0, iterations: int = 0, legs: int = 0, max_rounds: int = 0,
                    inject: Optional[Tuple[int, int, int, int, int, int, int]] = None,
                    cap: int = 256) -> Tuple[XlaneResult, List[XlaneSm], List[XlaneFault]]:
        """cro_probe_xlane: every lane of every warp of one CTA per SM checks each shuffle, vote, match, warp-reduce and
        shared-atomic form of the legs run (legs = 0: all) against an exact answer.  iterations / max_rounds = 0: the
        defaults.  inject = (leg, sm, warp, lane, op, iteration, mask) is the test-only operand XOR (sm, warp, lane: -1
        for every one).  Returns the result (its status is OK, ERR_CHECKSUM or ERR_CUDA), one entry per SM seen and up
        to `cap` records."""
        o = _xlane_opts(iterations, legs, max_rounds, 0, inject)
        rc, out = _per_sm(lib.cro_probe_xlane, (self.handle, dev, ctypes.byref(o)), XlaneResult, XlaneSm, XLANE_MAX_SMS,
                          XlaneFault, cap)
        self._check(rc, allow=(ERR_CHECKSUM, ERR_CUDA))
        return out

    def probe_alu(self, dev: int = 0, iterations: int = 0, legs: int = 0, max_rounds: int = 0,
                  inject: Optional[Tuple[int, int, int, int, int, int, int, int]] = None,
                  cap: int = 256) -> Tuple[AluResult, List[AluSm], List[AluFault]]:
        """cro_probe_alu: every lane of every warp of one CTA per SM runs each integer, bit-manipulation, DPX and
        directed-rounding floating-point form of the legs run (legs = 0: all) on the host table's operands and checks
        the result.  iterations / max_rounds = 0: the defaults.  inject = (leg, sm, warp, lane, op, iteration, operand,
        mask) is the test-only operand XOR (sm, warp, lane: -1 for every one).  Returns the result (its status is OK,
        ERR_CHECKSUM or ERR_CUDA), one entry per SM seen and up to `cap` records."""
        o = _alu_opts(iterations, legs, max_rounds, 0, inject)
        rc, out = _per_sm(lib.cro_probe_alu, (self.handle, dev, ctypes.byref(o)), AluResult, AluSm, ALU_MAX_SMS, AluFault, cap)
        self._check(rc, allow=(ERR_CHECKSUM, ERR_CUDA))
        return out

    def probe_barrier(self, dev: int = 0, iterations: int = 0, legs: int = 0, max_rounds: int = 0, cluster: int = 0,
                      inject: Optional[Tuple[int, int, int, int, int, int, int]] = None,
                      cap: int = 256) -> Tuple[BarrierResult, List[BarrierSm], List[BarrierFault]]:
        """cro_probe_barrier: one CTA of 8 warps per SM runs every row of the legs run (legs = 0: all) on the host's
        table: named barriers, mbarrier phases and transaction counts, and (clusters of `cluster`, 0: 2) cluster
        barriers with async remote stores.  iterations / max_rounds = 0: the defaults.  inject = (leg, sm, warp, lane,
        row, iteration, mask) is the test-only XOR into every value that row compares (sm, warp, lane: -1 for every one).
        Returns the result (its status is OK, ERR_CHECKSUM or ERR_CUDA), one entry per SM seen and up to `cap` records."""
        o = _barrier_opts(iterations, legs, max_rounds, cluster, 0, inject)
        rc, out = _per_sm(lib.cro_probe_barrier, (self.handle, dev, ctypes.byref(o)), BarrierResult, BarrierSm, BARRIER_MAX_SMS,
                          BarrierFault, cap)
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

    def check_health(self, dev: int = 0, checks: int = 0, compute=None, precision=None, sram=None, l2=None, link=None, scan=None,
                     caps: Optional[Dict[str, int]] = None) -> Tuple[HealthResult, Dict[str, list]]:
        """cro_check_health: the selected checks (0: all six) on in-process device `dev`, each through its own in-process
        call, with the options check_health_uuid takes.  Returns the result and {list name: records}."""
        o = _health_opts(checks, compute, precision, sram, l2, link, scan)
        rc, r, records = _health_call(lib.cro_check_health, (self.handle, dev, ctypes.byref(o)), (), caps or {})
        if r.ran == 0:
            self._check(rc)
        return r, records

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
                       interiors: bool = False, alloc=bytearray, cap: int = 16, xor: bool = False):
        """One SELFTEST_SWEEP_* kernel on a buffer of the hook's own: guards holding canary words (word j of guard g:
        pattern_word(canary, g * 2^32 + j)) around the interior(s), a copy's in the SELFTEST_LAYOUT_* given.  force: up
        to two (first, count, and_mask, or_mask) interior ranges; with xor, each word of a range is XORed with or_mask
        (and_mask all ones).  Returns (SelftestSweepOut, the buffer as alloc(buf_bytes) made it, with the guards and,
        if interiors, the interiors at their offsets, and up to `cap` of the kernel's records by word)."""
        o = SelftestSweepOpts()
        o.kernel, o.layout, o.offset, o.bytes, o.seed, o.canary = kernel, layout, offset, bytes, seed, canary
        o.invert, o.word0 = invert, word0
        for r, (first, count, and_mask, or_mask) in enumerate(force):
            o.force_first[r], o.force_count[r], o.force_and[r], o.force_or[r] = first, count, and_mask, or_mask
        o.flags = (SELFTEST_F_INTERIORS if interiors else 0) | (SELFTEST_F_XOR if xor else 0)
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
