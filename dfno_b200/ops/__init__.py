"""Python wrappers (autograd, planning) around the sm_90a kernels in ``dfno_b200/csrc``."""
