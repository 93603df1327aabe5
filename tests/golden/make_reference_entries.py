"""Extract the EXPECTATIONS of the reference's ComposableResource table tests into a fixture.
(reads the reference checkout named by $CRO_REFERENCE; the output tests/golden/reference_entries.json travels)

For every Entry(...) of internal/controller/composableresource_controller_test.go this records
  line, title, the Describe block it sits in, tenant/cluster uuid (they select the fake fabric's
  routes), the secret's username (selects the token scenario), the initial Status fields the entry
  sets, and what the entry expects: expectedReconcileError, the expected Status fields, or
  expectedRequestDeleted.
No Go code is copied: only string literals and field assignments the tests assert on.  The scenario
INPUTS (which objects exist, what nvidia-smi prints) are written by hand in
tests/test_reference_entries.py from the same entries."""
import json
import os
import re
import sys

SRC = os.path.join(os.environ["CRO_REFERENCE"], "internal", "controller", "composableresource_controller_test.go")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_entries.json")

STR = r'"((?:[^"\\]|\\.)*)"'


def unquote(s):
    return json.loads('"' + s + '"')


def block_assignments(block, opener):
    """Field assignments inside `<opener>: func() ... }(),`."""
    i = block.find(opener + ": func()")
    if i < 0:
        return None
    j = block.find("}(),", i)
    body = block[i:j]
    out = {}
    for m in re.finditer(r"composableResourceStatus\.(\w+) = " + STR, body):
        out[m.group(1)] = unquote(m.group(2))
    return out


def main():
    lines = open(SRC, errors="replace").read().split("\n")
    describes = []       # (line, title)
    entries = []
    for n, l in enumerate(lines, 1):
        m = re.search(r'\bDescribe\("((?:[^"\\]|\\.)*)"', l)
        if m:
            describes.append((n, l[:len(l) - len(l.lstrip())], unquote(m.group(1))))
        m = re.search(r'\bEntry\(' + STR, l)
        if m:
            entries.append((n, unquote(m.group(1))))
    out = []
    for k, (n, title) in enumerate(entries):
        end = entries[k + 1][0] - 1 if k + 1 < len(entries) else len(lines)
        block = "\n".join(lines[n - 1:end])
        # the enclosing Describe chain = the last Describe at each smaller indentation
        chain, indent = [], None
        for dn, dind, dtitle in reversed([d for d in describes if d[0] < n]):
            if indent is None or len(dind) < indent:
                chain.append(dtitle)
                indent = len(dind)
        e = {"line": n, "title": title, "context": list(reversed(chain))[1:]}
        for key in ("tenant_uuid", "cluster_uuid", "resourceName"):
            m = re.search(key + r":\s*" + STR, block)
            if m:
                e[key] = unquote(m.group(1))
        m = re.search(r'"username":\s*\[\]byte\(' + STR + r"\)", block)
        if m:
            e["username"] = unquote(m.group(1))
        m = re.search(r"expectedReconcileError:\s*(?:fmt\.Errorf\()?" + STR, block)
        if m:
            e["expected_error"] = unquote(m.group(1))
        if re.search(r"expectedRequestDeleted:\s*true", block):
            e["expected_deleted"] = True
        init = block_assignments(block, "resourceStatus")
        if init:
            e["initial_status"] = init
        exp = block_assignments(block, "expectedRequestStatus")
        if exp is not None:
            e["expected_status"] = exp
        if re.search(r"ignoreGet:\s*true", block):
            e["ignore_get"] = True
        if "DeletionTimestamp" in block or "k8sClient.Delete(ctx, composableResource" in block:
            e["deleted_by_user"] = True
        m = re.search(r"setErrorMode:\s*(\w+)", block)
        if m:
            e["set_error_mode"] = m.group(1)
        # which metal3 objects the entry's extraHandling creates, and with which annotations
        # (the target Node exists in every entry except the garbage-collection ones, which delete all Nodes last)
        objs = {"node": not e.get("expected_deleted", False),
                "node_annotation": '"machine.openshift.io/machine":' in block,
                "machine": "Metal3Machine{" in block, "machine_annotation": '"metal3.io/BareMetalHost":' in block,
                "bmh": "BareMetalHost{" in block, "secret": "corev1.Secret{" in block,
                # gpu-operator ClusterPolicy with spec.driver.enabled = true (absent: the RKE2 branches run)
                "cluster_policy": "gpuv1.ClusterPolicy{" in block}
        m = re.search(r'"cluster-manager\.cdi\.io/machine":\s*' + STR, block)
        if m:
            objs["bmh_machine_uuid"] = unquote(m.group(1))
        e["objects"] = objs
        # the entry's mock pod-exec (gomonkey patch of remotecommand.NewSPDYExecutor): an ordered chain of
        # `strings.Contains(url.RawQuery, needle)` -> newMockExecutor(stdout, stderr); a chain without `if` is one rule
        patches = [m.start() for m in re.finditer(r"remotecommand\.NewSPDYExecutor,", block)]
        if patches:
            seg = block[patches[-1]:]
            seg = seg[:seg.find("\n\t\t\t\t\t\t)") if "\n\t\t\t\t\t\t)" in seg else len(seg)]
            rules = []
            pos = 0
            for m in re.finditer(r"newMockExecutor\(" + STR + r",\s*" + STR + r"\)", seg):
                cond = seg[pos:m.start()]
                c = re.findall(r"strings\.Contains\(url\.RawQuery,\s*(?:neturl\.QueryEscape\(" + STR + r"\)|" + STR + r")\)", cond)
                needle = None
                if c:
                    esc, lit = c[-1]
                    needle = {"escape": unquote(esc)} if esc else {"literal": unquote(lit)}
                rules.append({"needle": needle, "stdout": unquote(m.group(1)), "stderr": unquote(m.group(2))})
                pos = m.end()
            e["exec_rules"] = rules
        # pods the entry creates (name, namespace, labels are literal in the block)
        pods = []
        for m in re.finditer(r"&corev1\.Pod\{\s*ObjectMeta: metav1\.ObjectMeta\{(.*?)\n\t+\},\s*Spec: corev1\.PodSpec\{(.*?)\n\t+\},", block, re.S):
            meta, spec = m.group(1), m.group(2)
            name = re.search(r"Name:\s*" + STR, meta)
            ns = re.search(r"Namespace:\s*" + STR, meta)
            labels = dict((unquote(a), unquote(b)) for a, b in re.findall(STR + r":\s*" + STR, meta[meta.find("Labels"):] if "Labels" in meta else ""))
            node = re.search(r"NodeName:\s*(?:" + STR + r"|(\w+))", spec)
            cont = re.findall(r"\{Name:\s*" + STR, spec)
            pods.append({"name": unquote(name.group(1)) if name else "", "namespace": unquote(ns.group(1)) if ns else "",
                         "labels": labels, "node": (unquote(node.group(1)) if node and node.group(1) else "worker-0") if node else "",
                         "containers": [unquote(x) for x in cont]})
        if pods:
            e["pods"] = pods
        out.append(e)
    # the fake fabric's route table (httptest handler, :663-930): path -> status + body
    routes = {}
    text = "\n".join(lines)
    for m in re.finditer(r'case ' + STR + r':\n(.*?)(?=\n\t\t\tcase |\n\t\t\tdefault:)', text, re.S):
        path, body = unquote(m.group(1)), m.group(2)
        if not path.startswith("/") or path.startswith("/id_manager"):   # the token endpoint is auth: not restated
            continue
        st = re.search(r"WriteHeader\(http\.Status(\w+)\)", body)
        r = {"status": {"OK": 200, "NotFound": 404, "Unauthorized": 401, "BadRequest": 400}[st.group(1)] if st else 200}
        lit = re.search(r"w\.Write\(\[\]byte\(`([^`]*)`\)\)", body) or re.search(r"w\.Write\(\[\]byte\(" + STR + r"\)\)", body)
        gen = re.search(r"w\.Write\((generate\w+)\(([^)]*)\)\)", body)
        if lit:
            r["body"] = lit.group(1) if "`" in lit.group(0) else unquote(lit.group(1))
        elif gen:
            args = [a.strip() for a in gen.group(2).split(",")]
            val = re.search(r'val := ' + STR, body)
            args = [(val.group(1) if (a == "&val" and val) else a) for a in args]
            r["generator"] = gen.group(1)
            r["args"] = [json.loads(a) if a in ("true", "false") else (None if a == "nil" else a.strip('"')) for a in args]
        else:
            r["body"] = ""
        routes[path] = r
    # the fake id_manager (:665-716): username of the Secret -> what the token endpoint answers.  An Encode()d map is kept
    # as its fields; the access token's middle part is symbolic ("payload": claims made at run time | raw text to encode)
    id_manager = {}
    idm = re.search(r'case "/id_manager[^"]*":\n(.*?)\n\t\t\tcase "/', text, re.S).group(1)
    for m in re.finditer(r'\n\t\t\t\tcase ' + STR + r':\n(.*?)(?=\n\t\t\t\tcase |\n\t\t\t\tdefault:)', idm, re.S):
        user, body = unquote(m.group(1)), m.group(2)
        st = re.search(r"WriteHeader\(http\.Status(\w+)\)", body)
        r = {"status": {"OK": 200, "Unauthorized": 401, "BadRequest": 400}[st.group(1)]}
        lit = re.search(r"w\.Write\(\[\]byte\(`([^`]*)`\)\)", body) or re.search(r"w\.Write\(\[\]byte\(" + STR + r"\)\)", body)
        if lit:
            r["body"] = lit.group(1) if "`" in lit.group(0) else unquote(lit.group(1))
        else:
            fields = {}
            enc = re.search(r"Encode\(map\[string\]interface\{\}\{(.*?)\n\t\t\t\t\t\}\)", body, re.S).group(1) + "\n"
            for k, v in re.findall(r"\n\s*" + STR + r":\s*(.*?),(?=\n)", enc):
                v = v.strip()
                if v.startswith('"') and "+" not in v:
                    fields[unquote(k)] = unquote(v[1:-1])
                elif "+" in v:
                    parts = [x.strip() for x in v.split("+")]
                    var = parts[1]
                    raw = re.search(var + r" := base64\.RawURLEncoding\.EncodeToString\(\[\]byte\(" + STR + r"\)\)", body)
                    hours = re.search(r"time\.Now\(\)\.Add\((\d+) \* time\.Hour\)", body)
                    fields[unquote(k)] = {"prefix": unquote(parts[0][1:-1]), "suffix": unquote(parts[2][1:-1]),
                                          "payload": {"raw": unquote(raw.group(1))} if raw else {"claims_exp_in_hours": int(hours.group(1))}}
                else:
                    fields[unquote(k)] = int(v)
            r["encode"] = fields
        id_manager[user] = r
    with open(OUT, "w") as f:
        json.dump({"_about": "expectations of the reference's ComposableResource table tests; made by make_reference_entries.py",
                   "source": "internal/controller/composableresource_controller_test.go", "routes": routes,
                   "id_manager": id_manager, "entries": out}, f, indent=1)
        f.write("\n")
    print(len(out), "entries ->", OUT)


if __name__ == "__main__":
    sys.exit(main())
