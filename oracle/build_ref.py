"""TEST/BENCH INFRASTRUCTURE ONLY — makes the UNMODIFIED reference importable from inside the repository tree.

The reference (neonbjb/tortoise-tts) is pure Python: "building" it is copying its package where the shims
(oracle/ref_shims.py) can import it. Where a checkout of the reference exists (TORTOISE_REFERENCE_ROOT), this recipe copies
`tortoise/` (sources + the small data assets + three voice clips used by BASELINE configs[1]) to `oracle/_ref/tortoise`,
which is git-ignored (the sources never enter this repository's history) but travels with a copy of the built tree,
like a built .so. `__graft_entry__.build()` runs it whenever the checkout is present.

  python -m oracle.build_ref
"""
import os
import shutil

SRC = os.environ.get("TORTOISE_REFERENCE_ROOT", "/root/reference")
DST = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")
KEEP_VOICES = ("angie", "cond_latent_example")


def build(force=False):
    src = os.path.join(SRC, "tortoise")
    if not os.path.isdir(src):
        return None                                  # no checkout here: use the copy made earlier, if any
    dst = os.path.join(DST, "tortoise")
    stamp = os.path.join(DST, ".stamp")
    want = str(sorted((os.path.relpath(os.path.join(d, f), src), os.path.getsize(os.path.join(d, f)))
                      for d, _, fs in os.walk(src) for f in fs if f.endswith(".py")))
    if not force and os.path.exists(stamp) and open(stamp).read() == want:
        return dst
    if os.path.isdir(dst):
        shutil.rmtree(dst)

    def ignore(d, names):
        if os.path.basename(d) == "voices":
            return [n for n in names if n not in KEEP_VOICES]
        return [n for n in names if n == "__pycache__"]
    shutil.copytree(src, dst, ignore=ignore)
    with open(stamp, "w") as f:
        f.write(want)
    return dst


if __name__ == "__main__":
    print(build(force=True))
