"""ORACLE TEST INFRASTRUCTURE: a plain-torch stand-in for the parts of megablocks (stanford-futuredata/megablocks) that
accessory/model/LLM/mixtral_sparse.py calls, so that the unmodified module runs on the CPU.  See megablocks/ops.py."""
