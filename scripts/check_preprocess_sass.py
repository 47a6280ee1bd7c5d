"""Compare the SASS of the packed-only pre-process kernels of two builds of preprocess.cu (object files or their
`cuobjdump -sass` listings): a change that adds input formats must leave the kernels packed-frame calls launch
instruction for instruction as they were.

    python scripts/check_preprocess_sass.py OLD.o NEW.o

Kernels are matched on (kernel, element type, tap capacity); in NEW only the instantiations whose YUV template argument
is false take part.  Exit status 0 when every matched body is identical."""
import re
import subprocess
import sys

CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"


def listing(path):
    if path.endswith(".o"):
        return subprocess.run([CUOBJDUMP, "-sass", path], check=True, capture_output=True, text=True).stdout
    return open(path).read()


def kernels(text):
    """{(kernel, dtype, taps): [instruction lines]} of the packed-only pre-process kernels in a SASS listing"""
    out = {}
    for part in re.split(r"\n\s*Function : ", text)[1:]:
        name, body = part.split("\n", 1)
        m = re.match(r"_ZN3vpb\d+(preprocess_pil_kernel|preprocess_direct_kernel)INS_\d+(F16|BF16)E(?:Li(\d+)E)?(Lb([01])E)?E",
                     name.strip())
        if not m or m.group(5) == "1":
            continue
        ins = [re.sub(r"/\*[0-9a-f]{4,}\*/", "", l).strip() for l in body.splitlines() if re.search(r"/\*[0-9a-f]{4}\*/", l)]
        out[(m.group(1), m.group(2), m.group(3))] = ins
    return out


def main(old, new):
    a, b = kernels(listing(old)), kernels(listing(new))
    if not a or sorted(a) != sorted(b):
        print(f"kernel sets differ: {sorted(a)} vs {sorted(b)}")
        return 1
    bad = 0
    for key in sorted(a):
        same = a[key] == b[key]
        bad += not same
        print(f"{'identical' if same else 'DIFFERENT'}  {key[0]}<{key[1]}{', ' + key[2] if key[2] else ''}>  "
              f"{len(a[key])} / {len(b[key])} instructions")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main(*sys.argv[1:3]))
