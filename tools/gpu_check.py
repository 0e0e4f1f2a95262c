#!/usr/bin/env python
"""Run the GPU test groups in separate processes (a device trap in one group must not poison the
rest) and write logs + a summary under tool_out/.  Usage: python tools/gpu_check.py [group ...]"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tool_out")
os.makedirs(OUT, exist_ok=True)

GROUPS = {
    "loaded": ["tests/test_gpu_kernels.py::test_native_cuda_runtime_is_loaded"],
    "conv_fwd": ["tests/test_gpu_kernels.py::test_conv5x5_forward_and_stats"],
    "conv_exact": ["tests/test_gpu_kernels.py::test_conv_tma_im2col_exact"],
    "conv_bwd": ["tests/test_gpu_kernels.py::test_conv5x5_backward"],
    "bn_pool": ["tests/test_gpu_kernels.py::test_bn_relu_pool_forward_backward", "tests/test_gpu_kernels.py::test_generic_bn_kernels_match_torch"],
    "head_sgd": ["tests/test_gpu_kernels.py::test_linear_and_cross_entropy", "tests/test_gpu_kernels.py::test_fused_sgd_matches_torch"],
    "convnet": ["tests/test_gpu_kernels.py::test_convnet_fused_matches_unfused"],
    "ddp1": ["tests/test_gpu_kernels.py::test_single_gpu_ddp_and_graphed_step"],
    "adam": ["tests/test_adam.py"],
    "amsgrad": ["tests/test_adam_amsgrad.py"],
    "rmsprop_adagrad": ["tests/test_rmsprop_adagrad.py"],
    "nadam_radam": ["tests/test_nadam_radam.py"],
    "adamax_adadelta_asgd_rprop": ["tests/test_adamax_adadelta_asgd_rprop.py"],
    "clip": ["tests/test_clip_grad.py"],
    "average": ["tests/test_averaged_model.py"],
    "accum": ["tests/test_grad_accumulation.py"],
    "ce_options": ["tests/test_cross_entropy_options.py"],
    "syncbn": ["tests/test_syncbn_native.py", "tests/test_syncbn_large_mean.py"],
    "maxpool_ties": ["tests/test_maxpool_ties.py"],
    "input_grads": ["tests/test_convnet_input_grads.py"],
    "symm_emu": ["tests/test_symm_kernels_emulated.py"],
}


def main():
    want = sys.argv[1:] or list(GROUPS)
    summary = {}
    for name in want:
        t0 = time.time()
        log = os.path.join(OUT, f"check_{name}.log")
        cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "--timeout", "150", "-p", "no:cacheprovider"] + GROUPS[name]
        with open(log, "w") as f:
            try:
                rc = subprocess.run(cmd, cwd=ROOT, stdout=f, stderr=subprocess.STDOUT, timeout=400).returncode
            except subprocess.TimeoutExpired:
                rc = "timeout"
        tail = open(log).read().strip().splitlines()[-1:] or [""]
        summary[name] = {"rc": rc, "seconds": round(time.time() - t0, 1), "tail": tail[0][-200:]}
        print(name, summary[name], flush=True)
    with open(os.path.join(OUT, "check_summary.json"), "w") as f:
        json.dump(summary, f, indent=1)
    bad = [k for k, v in summary.items() if v["rc"] != 0]
    print("FAILED GROUPS:", bad if bad else "none")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
