"""Compares the SASS of two builds function by function, so that a source change can be shown not to change the code.

Each side is an object file, or a directory whose .o files are matched by file name.  cuobjdump -sass of every object
is split per function and reduced to its instruction text (addresses and encodings dropped), with the
anonymous-namespace tag (_GLOBAL__N__<hash>_<len>_<file>_<hash>, which changes from build to build) normalised.
Functions are matched by demangled name without the parameter list; OLD=NEW pairs match a renamed function, such as a
kernel that became a template instantiation.  One line per function; exit code 1 on any difference or unmatched
function.  Needs the CUDA toolkit (cuobjdump, cu++filt), no GPU.

    python scripts/compare_sass.py before/csrc after/csrc 'arma_css_kernel=arma_css_kernel_t<false>' ...
"""
import difflib
import os
import re
import shutil
import subprocess
import sys

ANON = re.compile(r"_GLOBAL__N__[0-9a-f]+_\d+_\w*?_cu_[0-9a-f]{8}")
INSN = re.compile(r"/\*[0-9a-f]{4,}\*/\s*(.*?)\s*;")


def tool(name):
    path = shutil.which(name) or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)
    if not os.path.exists(path):
        sys.exit(f"compare_sass: {name} not found")
    return path


def short_name(demangled):
    """the function's name without namespaces, return type or parameters: 'arma_css_kernel_t<false>'"""
    s = demangled.replace("(anonymous namespace)", "").replace("<unnamed>", "")
    s = s.replace("(bool)0", "false").replace("(bool)1", "true")
    depth, start = 0, 0
    for i, ch in enumerate(s):
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif depth == 0 and ch == "(":
            return s[start:i]
        elif depth == 0 and (ch == " " or s.startswith("::", i)):
            start = i + (2 if ch == ":" else 1)
    return s[start:]


def functions(obj):
    """{short name: [instruction text]} of one object file ({} for an object without device code)"""
    out = subprocess.run([tool("cuobjdump"), "-sass", obj], capture_output=True, text=True)
    if out.returncode != 0:
        if "does not contain device code" in out.stderr + out.stdout:
            return {}
        sys.exit(f"compare_sass: cuobjdump -sass {obj} failed:\n{out.stderr}")
    names, bodies = [], []
    for line in out.stdout.splitlines():
        if "Function :" in line:
            names.append(line.split("Function :", 1)[1].strip())
            bodies.append([])
        elif bodies:
            m = INSN.search(line)
            if m:
                bodies[-1].append(ANON.sub("_GLOBAL__N_", m.group(1)))
    demangled = subprocess.run([tool("cu++filt")], input="\n".join(names) + "\n", capture_output=True,
                               text=True, check=True).stdout.splitlines()
    funcs = {}
    for name, body in zip(demangled, bodies):
        key = short_name(name)
        if key in funcs:
            sys.exit(f"compare_sass: {obj}: two functions named {key}")
        funcs[key] = body
    return funcs


def compare(label, old, new, renames):
    """prints one line per function of the object pair; True when all match"""
    a, b = functions(old), functions(new)
    if not a and not b:
        print(f"{label}: no device code")
        return True
    ok = True
    unmatched = dict(b)
    for name, body in a.items():
        other = renames.get(name, name)
        shown = name if other == name else f"{name} -> {other}"
        if other not in unmatched:
            print(f"{label}: {shown}: only in the old build")
            ok = False
            continue
        body_b = unmatched.pop(other)
        diff = [l for l in difflib.unified_diff(body, body_b, lineterm="", n=0)
                if l[:1] in "+-" and not l.startswith(("+++", "---"))]
        if diff:
            print(f"{label}: {shown}: {len(body)} / {len(body_b)} instructions, {len(diff)} lines differ")
            ok = False
        else:
            print(f"{label}: {shown}: {len(body)} instructions, identical")
    for name in unmatched:
        print(f"{label}: {name}: only in the new build")
        ok = False
    return ok


def main(argv):
    if len(argv) < 2 or any("=" not in r for r in argv[2:]):
        sys.exit(__doc__)
    old, new = argv[0], argv[1]
    renames = dict(r.split("=", 1) for r in argv[2:])
    if os.path.isdir(old) != os.path.isdir(new):
        sys.exit("compare_sass: compare two object files or two directories")
    if not os.path.isdir(old):
        return 0 if compare(os.path.basename(new), old, new, renames) else 1
    objs_a = {f for f in os.listdir(old) if f.endswith(".o")}
    objs_b = {f for f in os.listdir(new) if f.endswith(".o")}
    ok = True
    for f in sorted(objs_a | objs_b):
        if f in objs_a and f in objs_b:
            ok = compare(f, os.path.join(old, f), os.path.join(new, f), renames) and ok
        else:
            print(f"{f}: only in the {'old' if f in objs_a else 'new'} build")
            ok = False
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
