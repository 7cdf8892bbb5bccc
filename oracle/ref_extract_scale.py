"""Generate the reference's own source for the deformable-robot pin build (`make -C oracle ref`), under oracle/_ref/scaled/ (git-ignored).

TEST INFRASTRUCTURE.  Runs oracle/ref_extract.py unchanged into oracle/_ref/scaled/_ref/gen/ and then edits only the copy:
  * sw_methods.inc loses the verbatim getScale / getDotScale (sw_manager.hpp:495-518, the hook a user edits for a deforming
    robot) and includes oracle/ref_scale_hook.inc instead (ours: this project's schedule as getScale);
  * sw_macros.inc gets `#undef useScale` / `#define useScale true` after the verbatim macros (the reference's switch, :17).
It also copies oracle/ref_path_shim.cpp next to that gen/ directory, so that the copy's `#include "_ref/gen/..."` lines resolve to
the edited fragments; oracle/ref_path_scaled_shim.cpp includes the copy and adds the schedule's C entry points.

    python oracle/ref_extract_scale.py [--ref /root/reference]
"""
from __future__ import annotations

import argparse
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_extract  # noqa: E402

OUT = os.path.join(HERE, "_ref", "scaled")


def main(ref: str) -> None:
    gen = os.path.join(OUT, "_ref", "gen")
    ref_extract.extract(ref, gen)
    swm = ref_extract.Source(os.path.join(ref, "src", "swept_volume/include/swept_volume/sw_manager.hpp"))
    hook = [swm.block(r"^\s*inline Eigen::Matrix3d getScale\(", expect_lines=(485, 510)),
            swm.block(r"^\s*inline Eigen::Matrix3d getDotScale\(", expect_lines=(500, 525))]
    p = os.path.join(gen, "sw_methods.inc")
    with open(p, encoding="utf-8", errors="surrogateescape") as fh:
        text = fh.read()
    for b in hook:
        assert text.count(b) == 1, "getScale / getDotScale not found verbatim in sw_methods.inc"
        text = text.replace(b, "")
    text += "// ---- ours: getScale = this project's schedule (oracle/ref_scale_hook.inc)\n#include \"ref_scale_hook.inc\"\n"
    with open(p, "w", encoding="utf-8", errors="surrogateescape") as fh:
        fh.write(text)
    with open(os.path.join(gen, "sw_macros.inc"), "a", encoding="utf-8") as fh:
        fh.write("// ---- ours: the deformable-robot build\n#undef useScale\n#define useScale true\n")
    for f in ("ref_path_shim.cpp", "ref_shape_scaffold.inc"):  # the scaffold's `_ref/gen/` includes must resolve to the copy too
        shutil.copyfile(os.path.join(HERE, f), os.path.join(OUT, f))
    print("ref_extract_scale: wrote", OUT)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default="/root/reference")
    a = ap.parse_args()
    if not os.path.isdir(a.ref):
        print("ref_extract_scale: no reference tree at", a.ref, file=sys.stderr)
        sys.exit(2)
    main(a.ref)
