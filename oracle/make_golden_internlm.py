"""ORACLE TEST INFRASTRUCTURE: generate tests/golden/internlm_*.npz FROM THE UNMODIFIED REFERENCE
(accessory/model/LLM/internlm.py), in the format of oracle/make_golden.py.

    python -m oracle.make_golden_internlm
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import cases, internlm  # noqa: E402
from oracle.make_golden import OUT, sd_digest  # noqa: E402


def main():
    assert internlm.reference_available(), "needs the reference tree (accessory/model/LLM/internlm.py)"
    torch.manual_seed(0)
    for name, (args, bits, gs, bsz, plen, ndec) in internlm.CASES.items():
        args, sd, sd_ref, recs, toks = internlm.build_case(name)
        res = {}
        for dt, tag in ((torch.float16, "fp16"), (torch.float32, "fp32")):
            model = internlm.reference_model(args, sd_ref, dt)
            res[tag] = cases.run_schedule(model, toks, plen, ndec).numpy()
        np.savez_compressed(
            os.path.join(OUT, f"{name}.npz"),
            logits_fp16=res["fp16"], logits_fp32=res["fp32"], tokens=toks.numpy(),
            weights_sha256=np.array(sd_digest(sd_ref)), prefill_len=np.array(plen), n_decode=np.array(ndec),
            torch_version=np.array(torch.__version__),
        )
        d = np.abs(res["fp16"] - res["fp32"]).max()
        print(f"{name}: logits {res['fp16'].shape}, |ref16-ref32|max={d:.3e}, absmax={np.abs(res['fp32']).max():.3f}")


if __name__ == "__main__":
    main()
