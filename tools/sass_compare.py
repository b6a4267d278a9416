"""Kernel-by-kernel comparison of two builds' SASS: python tools/sass_compare.py OLD.so|OLD.sass NEW.so|NEW.sass

Every kernel of OLD must have a kernel in NEW whose `cuobjdump -sass` instructions, encodings included, are byte-identical.
Kernels are matched by demangled name. A template parameter added since OLD with its old behaviour as the default (the
element type bf16, F16 = false, HALF = false) is dropped before matching, so `conv_wgmma_kernel<64, false, true, false>`
matches `conv_wgmma_kernel<64, false, true>`. This is how the bf16 kernels are checked to be untouched by the fp16 plans
(DESIGN.md §4e). Needs cuobjdump and c++filt, no GPU. Prints one line per differing or missing kernel and a summary; exits
1 if any."""
import re
import subprocess
import sys


def sass(path):
    if path.endswith(".sass"):
        return open(path).read()
    return subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout


def kernels(text):
    parts = re.split(r"\n\s*Function : (\S+)\n", text)
    return {parts[i]: re.sub(r"\s+", " ", parts[i + 1].split("\n\t\t..........")[0]) for i in range(1, len(parts), 2)}


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.split("\n")
    return dict(zip(names, out))


def norm(n):
    n = n[5:] if n.startswith("void ") else n
    for new, old in ((", false, false, false>", ", false, false>"), (", true, false, false>", ", true, false>"),
                     (", false, true, false>", ", false, true>"), ("<__nv_bfloat16>", ""),
                     ("<float, __nv_bfloat16>", "<float>"), ("<unsigned char, __nv_bfloat16>", "<unsigned char>"),
                     ("<false>(", "(")):
        n = n.replace(new, old)
    return n


def main():
    old, new = kernels(sass(sys.argv[1])), kernels(sass(sys.argv[2]))
    dold, dnew = demangle(list(old)), demangle(list(new))
    by_name = {}
    for k, body in new.items():
        by_name.setdefault(norm(dnew[k]), []).append(body)
    bad = 0
    for k, body in old.items():
        cand = by_name.get(norm(dold[k]))
        if not cand or body not in cand:
            bad += 1
            print(("DIFFERS " if cand else "MISSING ") + dold[k][:200])
    print(f"{len(old)} kernels in the old build, {len(old) - bad} byte-identical in the new one ({len(new)} kernels)")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
