"""Re-verifies tests/golden/reference_kats.json against the reference tree.

Needs a checkout of the reference, given as the first argument; the test
suite does not run this.  For each vector, every
expected error / id string must occur verbatim in the cited file.
"""
import json
import os
import re
import sys

REF = sys.argv[1]
HERE = os.path.dirname(os.path.abspath(__file__))
kats = json.load(open(os.path.join(HERE, "reference_kats.json")))
cache = {}


def text_of(cite):
    path = re.match(r"([\w./-]+\.go)", cite).group(1)
    if path not in cache:
        cache[path] = open(os.path.join(REF, path)).read()
    return cache[path]


def go_quote(s):
    return s.replace("\\", "\\\\").replace('"', '\\"')


bad = 0
n = 0
for sec in ("parse", "attach", "env_errors"):
    for v in kats[sec]:
        t = text_of(v["cite"])
        strings = []
        exp = v.get("expected", v)
        if exp.get("error"):
            strings.append(exp["error"])
        for k in ("state", "error", "device_id", "cdi_device_id"):
            if isinstance(exp.get("status"), dict) and exp["status"].get(k):
                strings.append(exp["status"][k])
        if v.get("stdout"):
            strings.append(v["stdout"])
        en = v.get("enumeration") or {}
        for k in ("stdout", "stderr"):
            if en.get(k):
                strings.append(en[k])
        for s in strings:
            n += 1
            if go_quote(s) not in t:
                bad += 1
                print("MISSING in %s: %r" % (v["cite"], s))
print("%d strings checked, %d missing" % (n, bad))
sys.exit(1 if bad else 0)
