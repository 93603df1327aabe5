"""The helper wire format without a GPU (csrc/helper_wire.h): every -raw command's option table against its cro_*_opts
struct as gcc lays it out, the decimal formatter and parser against each other and against the field's own type, and
the argument counts croprobe-cli takes."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "composable-resource-operator_b200", "csrc")
CLI = os.path.join(ROOT, "composable-resource-operator_b200", "croprobe-cli")
U = "GPU-5ca90000-0000-0000-0000-000000000002"

# each table, its options struct, and the fields deliberately left off argv
TABLES = [
    ("scan", "cro_scan_opts", ["deadline_ms", "reserved0"]),
    ("sram", "cro_sram_opts", ["deadline_ms"]),
    ("link", "cro_link_opts", ["reserved0"]),
    ("compute", "cro_compute_opts", []),
    ("precision", "cro_precision_opts", ["reserved"]),
    ("sparse", "cro_sparse_opts", []),
    ("l2", "cro_l2_opts", ["deadline_ms"]),
]
# what croprobe-cli has always taken: argv[0] and the command included
ARGC = {"scan-raw": 12, "sram-raw": 14, "l2-raw": 15, "link-raw": 11, "compute-raw": 15, "precision-raw": 15,
        "sparse-raw": 20, "health-raw": 65}

PROGRAM = r"""
#include <assert.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "helper_wire.h"

static int bad = 0;
#define CHECK(c, ...) do { if (!(c)) { printf("FAIL " __VA_ARGS__); printf("\n"); bad = 1; } } while (0)

static uint64_t rng = 0x9E3779B97F4A7C15ull;
static uint64_t next(void) {
    rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17;
    return rng;
}

/* Every byte of the struct covered exactly once by the table's fields and the skipped ones. */
static void coverage(const char *name, const cro_wire *w, size_t size, const size_t *skip_at, const size_t *skip_size, int n_skip) {
    unsigned char seen[512] = {0};
    for (uint32_t i = 0; i < w->n_fields; ++i)
        for (size_t b = 0; b < w->fields[i].size; ++b) seen[w->fields[i].at + b]++;
    for (int s = 0; s < n_skip; ++s)
        for (size_t b = 0; b < skip_size[s]; ++b) seen[skip_at[s] + b]++;
    for (size_t b = 0; b < size; ++b) CHECK(seen[b] == 1, "%s: byte %zu covered %d times", name, b, seen[b]);
    for (size_t b = size; b < sizeof seen; ++b) CHECK(seen[b] == 0, "%s: byte %zu past the struct", name, b);
}

/* The decimal the field's own type prints. */
static void natural(const cro_wire_field *f, const unsigned char *p, char *s) {
    if (f->size == 4 && f->is_signed) { int32_t v; memcpy(&v, p, 4); sprintf(s, "%d", v); }
    else if (f->size == 4) { uint32_t v; memcpy(&v, p, 4); sprintf(s, "%u", v); }
    else if (f->is_signed) { int64_t v; memcpy(&v, p, 8); sprintf(s, "%lld", (long long)v); }
    else { uint64_t v; memcpy(&v, p, 8); sprintf(s, "%llu", (unsigned long long)v); }
}

/* Field i set to v in a struct of random bytes: the formatter writes what the type prints, and parsing it into a copy
 * whose field is scrambled gives back the struct byte for byte. */
static void round_trip(const char *name, const cro_wire *w, size_t size, uint32_t i, uint64_t v) {
    unsigned char a[512], b[512];
    char s[24], want[24];
    for (size_t k = 0; k < size; ++k) a[k] = (unsigned char)next();
    const cro_wire_field *f = &w->fields[i];
    memcpy(a + f->at, &v, f->size);
    cro_wire_format(w, i, a, s, sizeof s);
    natural(f, a + f->at, want);
    CHECK(strcmp(s, want) == 0, "%s field %u: formatted %s, the type prints %s", name, i, s, want);
    memcpy(b, a, size);
    for (size_t k = 0; k < f->size; ++k) b[f->at + k] ^= 0xA5;
    cro_wire_parse(w, i, s, b);
    CHECK(memcmp(a, b, size) == 0, "%s field %u: %s does not parse back", name, i, s);
}

/* Every field of a random struct through argv and back into a zeroed one: the table's bytes come back. */
static void whole(const char *name, const cro_wire *w, size_t size) {
    unsigned char a[512] = {0}, b[512] = {0};
    char s[24];
    for (uint32_t i = 0; i < w->n_fields; ++i)
        for (size_t k = 0; k < w->fields[i].size; ++k) a[w->fields[i].at + k] = (unsigned char)next();
    for (uint32_t i = 0; i < w->n_fields; ++i) {
        cro_wire_format(w, i, a, s, sizeof s);
        cro_wire_parse(w, i, s, b);
    }
    CHECK(memcmp(a, b, size) == 0, "%s: a whole struct does not come back", name);
}

static void check(const char *name, const cro_wire *w, size_t size, const size_t *skip_at, const size_t *skip_size, int n_skip) {
    coverage(name, w, size, skip_at, skip_size, n_skip);
    for (uint32_t i = 0; i < w->n_fields; ++i) {
        const unsigned bits = 8u * w->fields[i].size;
        const uint64_t ones = bits == 64 ? ~0ull : (1ull << bits) - 1;
        const uint64_t min = w->fields[i].is_signed ? 1ull << (bits - 1) : 0, max = w->fields[i].is_signed ? ones >> 1 : ones;
        const uint64_t values[] = {0, 1, ones, min, max, min + 1, max - 1};
        for (size_t v = 0; v < sizeof values / sizeof *values; ++v) round_trip(name, w, size, i, values[v]);
        for (int r = 0; r < 2000; ++r) round_trip(name, w, size, i, next() >> (next() % 64));
    }
    for (int r = 0; r < 200; ++r) whole(name, w, size);
    printf("argc %s %d\n", w->cmd, cro_wire_argc(w));
}

int main(void) {
@BODY@
    printf("argc health-raw %d\n", cro_wire_health_at(CRO_HEALTH_CHECKS));
    /* health-raw's options: checks, reserved0 and each check's struct where the health table says */
    {
        unsigned char seen[sizeof(cro_health_opts)] = {0};
        for (size_t b = 0; b < 4; ++b) seen[offsetof(cro_health_opts, checks) + b]++, seen[offsetof(cro_health_opts, reserved0) + b]++;
        const size_t sizes[CRO_HEALTH_CHECKS] = {sizeof(cro_compute_opts), sizeof(cro_precision_opts), sizeof(cro_sram_opts),
                                                 sizeof(cro_l2_opts), sizeof(cro_link_opts), sizeof(cro_scan_opts)};
        for (int k = 0; k < CRO_HEALTH_CHECKS; ++k)
            for (size_t b = 0; b < sizes[k]; ++b) seen[cro_wire_health[k].opts_at + b]++;
        for (size_t b = 0; b < sizeof seen; ++b) CHECK(seen[b] == 1, "health opts: byte %zu covered %d times", b, seen[b]);
    }
    CHECK(cro_wire_health[0].wire == &cro_wire_compute && cro_wire_health[1].wire == &cro_wire_precision &&
          cro_wire_health[2].wire == &cro_wire_sram && cro_wire_health[3].wire == &cro_wire_l2 &&
          cro_wire_health[4].wire == &cro_wire_link && cro_wire_health[5].wire == &cro_wire_scan, "health run order");
    CHECK(cro_wire_health[2].result_at == offsetof(cro_health_result, sram) &&
          cro_wire_health[5].result_at == offsetof(cro_health_result, scan), "health result offsets");
    printf(bad ? "BAD\n" : "OK\n");
    return bad;
}
"""


def run_program(tmp_path):
    body = []
    for name, struct, skip in TABLES:
        at = ", ".join("offsetof(%s, %s)" % (struct, f) for f in skip) or "0"
        size = ", ".join("sizeof(((%s *)0)->%s)" % (struct, f) for f in skip) or "0"
        body.append("    { const size_t at[] = {%s}, size[] = {%s}; check(\"%s\", &cro_wire_%s, sizeof(%s), at, size, %d); }"
                    % (at, size, name, name, struct, len(skip)))
    src = tmp_path / "wire.c"
    src.write_text(PROGRAM.replace("@BODY@", "\n".join(body)))
    exe = tmp_path / "wire"
    subprocess.check_call(["gcc", "-std=c11", "-O1", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"),
                           "-I" + CSRC, str(src), "-o", str(exe)])
    return subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)


def test_tables_cover_their_structs_and_round_trip(tmp_path):
    out = run_program(tmp_path)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout[-4000:] + out.stderr
    argc = dict((ln.split()[1], int(ln.split()[2])) for ln in out.stdout.splitlines() if ln.startswith("argc "))
    assert argc == ARGC


@pytest.mark.parametrize("cmd", sorted(ARGC))
def test_cli_takes_exactly_its_argument_count(cmd):
    """One short and one long are refused (64); the exact count gets past the check to the device lookup."""
    n = ARGC[cmd]
    run = lambda k: subprocess.run([CLI, cmd, U] + ["0"] * (k - 3), capture_output=True, timeout=60).returncode
    assert run(n - 1) == 64 and run(n + 1) == 64
    assert run(n) != 64
