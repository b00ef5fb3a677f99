#!/usr/bin/env python
"""Kernel-by-kernel SASS comparison of two builds of libpwpp_b200.so (opcode + operands, addresses ignored).
usage: tools/sass_compare.py OLD.so NEW.so
Used to show that adding switched-off kernel variants leaves the device code of the default path bit-identical to a
build whose GPU parity run is on record (r01: the build of commit 7090554, profiles/r01_pytest_gpu.log)."""
import subprocess, re, sys, hashlib, collections
def funcs(lib):
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
    cur, d = None, collections.OrderedDict()
    for l in out.splitlines():
        m = re.search(r"Function : (\S+)", l)
        if m: cur = m.group(1); d[cur] = []; continue
        m = re.match(r"\s+/\*[0-9a-f]{4,5}\*/\s+(.*?)\s*/\*", l)
        if cur and m: d[cur].append(m.group(1))
    return d
a, b = funcs(sys.argv[1]), funcs(sys.argv[2])
names = subprocess.run(["c++filt"] + list(b), capture_output=True, text=True).stdout.split("\n")
for n, dn in zip(b, names):
    short = re.sub(r"\(.*", "", dn).replace("void pwpp::", "")
    if n not in a: print("NEW      ", len(b[n]), short); continue
    same = a[n] == b[n]
    print("IDENTICAL" if same else "DIFFERENT", len(a[n]), len(b[n]), short)
print("---- template kernels matched by dropping the new trailing 'false' parameter (or the whole parameter list of a kernel that became a template)")
da = {re.sub(r"\(.*", "", x).replace("void pwpp::", "").replace("pwpp::", ""): a[n] for n, x in zip(a, subprocess.run(["c++filt"] + list(a), capture_output=True, text=True).stdout.split("\n"))}
db = {re.sub(r"\(.*", "", x).replace("void pwpp::", "").replace("pwpp::", ""): b[n] for n, x in zip(b, names)}
for k, v in db.items():
    if k in da: continue
    k2 = k
    while k2 not in da and re.search(r", (false|\d+)>$", k2):   # template parameters appended since the old build (defaults)
        k2 = re.sub(r", (false|\d+)>$", ">", k2)
    if k2 == "k_bin_scan<4096>" or k2 not in da:
        k2 = re.sub(r"<[^<>]*>$", "", k2) if re.sub(r"<[^<>]*>$", "", k2) in da else k2   # a kernel that became a template
    if k2 in da: print("IDENTICAL" if da[k2] == v else "DIFFERENT", len(da[k2]), len(v), k)
