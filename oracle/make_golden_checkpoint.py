"""ORACLE TEST INFRASTRUCTURE: what the UNMODIFIED accessory/util/tensor_parallel.py makes of the tensor-parallel
checkpoint folders this repo writes (llama2_accessory_b200.checkpoint.save_tensor_parallel_shards), for
tests/test_checkpoint_cpu.py::test_merge_and_inference_agree_with_the_reference_loader.

Needs the reference tree (oracle/ref_import.py).  The folders hold the seeded tiny LLaMA of that test at TP = 2 in both
formats; recorded per format: the inferred (format, mp size), the shard file names, the merged TP = 1 state dict (key,
dtype, shape, sha256 of the bytes) and the keys the reference Transformer reports missing after loading it; and which
malformed folders the reference refuses.

  python -m oracle.make_golden_checkpoint   ->  tests/golden/checkpoint_loader.json
"""
import contextlib
import hashlib
import importlib
import io
import json
import os
import tempfile

import torch

from llama2_accessory_b200 import checkpoint as ck

from . import cases, ref_import

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "checkpoint_loader.json")


def tensor_digest(t):
    t = t.detach().contiguous().cpu()
    return [str(t.dtype), list(t.shape), hashlib.sha256(t.view(torch.uint8).numpy().tobytes()).hexdigest()]


def main():
    ref_import.load("llama")
    tp = importlib.import_module("accessory.util.tensor_parallel")
    args = cases.TINY_LLAMA
    sd = cases.master_state_dict("llama", args, seed=3)
    model = ref_import.build_reference_model("llama", dict(args), sd, torch.float16)
    holder = torch.nn.Module()
    holder.llma = model
    out = {"model": "TINY_LLAMA fp16 (oracle.cases, seed 3), TP = 2 folders", "formats": {}, "refused": []}
    with tempfile.TemporaryDirectory() as tmp:
        for fmt in ("consolidated", "meta_ori"):
            d = os.path.join(tmp, fmt)
            ck.save_tensor_parallel_shards(sd, d, 2, fmt)
            with contextlib.redirect_stdout(io.StringIO()):
                ref_sd = tp.load_tensor_parallel_model_state_dict(holder, d, fmt)
            res = holder.load_state_dict(ref_sd, strict=False)
            out["formats"][fmt] = {
                "inferred": list(tp.infer_checkpoint_format_and_mp_size(d)),
                "shard_file_names": list(tp.get_tensor_parallel_shards_file_name(fmt, 2)),
                "merged": {k: tensor_digest(v) for k, v in sorted(ref_sd.items())},
                "missing_after_load": sorted(res.missing_keys),
                "unexpected_after_load": sorted(res.unexpected_keys),
            }
        for bad in ("empty", "mixed"):
            d = os.path.join(tmp, bad)
            os.makedirs(d)
            if bad == "mixed":
                ck.save_tensor_parallel_shards(sd, d, 1, "consolidated")
                ck.save_tensor_parallel_shards(sd, d, 1, "meta_ori")
            else:
                with open(os.path.join(d, "x.txt"), "w") as f:
                    f.write("x")
            try:
                tp.infer_checkpoint_format_and_mp_size(d)
            except NotImplementedError:
                out["refused"].append(bad)
    with open(OUT, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
