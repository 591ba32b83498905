"""Compare the SASS of two builds of libpob_b200.so kernel by kernel, with no GPU: `cuobjdump -sass` of each, names demangled by
`cu++filt`, parameter lists dropped.  Every kernel of the OLD build must appear in the NEW one with identical instructions.  The G1
instantiations of the curve-generic MSM kernels (k_msm_sum<MsmBases<MsmCurve<Fq>>>, ...) are matched to the names they had before
msm.cuh became a template (k_msm_sum<MsmBases>, ...).  Kernels only in NEW are listed.  Exit code 1 on any difference.

    python tools/sass_diff.py OLD.so NEW.so
"""
import os
import re
import subprocess
import sys

CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")


def kernels(so):
    sass = subprocess.run([os.path.join(CUDA, "bin", "cuobjdump"), "-sass", so], check=True, capture_output=True, text=True).stdout
    sass = subprocess.run([os.path.join(CUDA, "bin", "cu++filt")], input=sass, check=True, capture_output=True, text=True).stdout
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (.*)", line)
        if m:
            cur = out.setdefault(name(m.group(1).strip()), [])
        elif cur is not None and re.search(r"/\*[0-9a-f]{4,}\*/", line):
            cur.append(re.sub(r"\s+", " ", line.strip()))
    return out


def name(n):
    n = re.sub(r"\((?:[^()]|\([^()]*\))*\)$", "", n).replace("void ", "")
    g1 = "<unnamed>::MsmCurve<pob::Fq>"
    for k in ("MsmBases", "MsmPartials"):
        n = n.replace("<<unnamed>::%s<%s>>" % (k, g1), "<<unnamed>::%s>" % k)
    for k in ("k_msm_final", "k_msm_reduce"):
        n = n.replace("%s<%s>" % (k, g1), k)
    return n


def main():
    old, new = kernels(sys.argv[1]), kernels(sys.argv[2])
    bad = 0
    for k, v in old.items():
        w = new.get(k)
        state = "missing" if w is None else "identical" if w == v else "DIFFERS (%d instructions new)" % len(w)
        bad += state != "identical"
        print("%-75s %6d  %s" % (k[:75], len(v), state))
    for k in sorted(set(new) - set(old)):
        print("%-75s %6d  new" % (k[:75], len(new[k])))
    print("kernels of the old build that differ or are missing: %d" % bad)
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
