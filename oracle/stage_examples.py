#!/usr/bin/env python
"""Copy the reference's example-only model code, where it lies under $COGDL_REFERENCE (default /root/reference), into
oracle/_ref/examples/ (git-ignored; it travels with the tree to a machine that has no reference checkout).

TEST INFRASTRUCTURE ONLY, like oracle/build_ref.py: the files are copied unmodified into the ignored directory and
nothing from them enters the repository.  The reference package that build_ref.py installs leaves examples/ out, so
layers defined only in an example are staged here:

  simple_hgn/conv.py   the Simple-HGN layer myGATConv, run under cogdl_b200.install_simple_hgn by
                       tests/test_gpu_simple_hgn.py (child tests/simple_hgn_refpkg_check.py)

Without a reference checkout, whatever oracle/_ref/examples/ already holds is kept.
"""
import os
import shutil

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("COGDL_REFERENCE", "/root/reference")
OUT = os.path.join(HERE, "_ref", "examples")
FILES = ["simple_hgn/conv.py"]


def main():
    src_root = os.path.join(REF, "examples")
    if not os.path.isdir(src_root):
        print(f"[stage_examples] {src_root} not present: keeping whatever is staged in {OUT}")
        return
    for rel in FILES:
        src, dst = os.path.join(src_root, rel), os.path.join(OUT, rel)
        if os.path.exists(dst) and os.path.getmtime(dst) >= os.path.getmtime(src):
            continue
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        shutil.copyfile(src, dst)
    print("[stage_examples]", OUT)


if __name__ == "__main__":
    main()
