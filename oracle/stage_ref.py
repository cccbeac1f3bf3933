"""ORACLE TEST INFRASTRUCTURE: stage the UNMODIFIED reference modules of the decode hot path into oracle/_ref/.

The reference is pure Python, so "building" it is a byte-for-byte copy of the handful of files the path lives in
(SURVEY.md 8a) from /root/reference into oracle/_ref/accessory/...  oracle/_ref/ is git-ignored (reference sources never
enter the history); a copy of the working tree made after build() carries it to a machine without the reference tree,
where tests and bench.py's CPU leg / --impl reference can then run the reference itself instead of the port.
Called by __graft_entry__.build(); idempotent; a no-op where the reference tree is absent.
"""
import filecmp
import os
import shutil

HERE = os.path.dirname(os.path.abspath(__file__))
SRC_ROOT = os.environ.get("B200_REFERENCE_SRC", "/root/reference")
DST_ROOT = os.path.join(HERE, "_ref")

# every file the hot path (and the unmodified MetaModel.generate loop around it) is imported from
FILES = [
    "accessory/model/LLM/llama.py",      # Transformer, Attention, FeedForward, RoPE, forward_inference
    "accessory/model/LLM/mixtral.py",    # MoE / ExpertFeedForward
    "accessory/model/components.py",     # RMSNorm
    "accessory/model/meta.py",           # MetaModel.generate / stream_generate / sample_top_p
    "accessory/util/tensor_type.py",     # default_tensor_type (imported by llama.py / mixtral.py)
    "LICENSE",
]


def staged() -> bool:
    return all(os.path.isfile(os.path.join(DST_ROOT, f)) for f in FILES if f != "LICENSE")


def stage(verbose=False) -> bool:
    """Copy FILES from the reference tree; returns True when oracle/_ref is complete afterwards."""
    if not os.path.isfile(os.path.join(SRC_ROOT, FILES[0])):
        return staged()
    for f in FILES:
        src, dst = os.path.join(SRC_ROOT, f), os.path.join(DST_ROOT, f)
        if not os.path.isfile(src):
            continue
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        if not (os.path.isfile(dst) and filecmp.cmp(src, dst, shallow=False)):
            shutil.copyfile(src, dst)
            if verbose:
                print("staged", f)
    return staged()


if __name__ == "__main__":
    print("oracle/_ref complete:", stage(verbose=True))
