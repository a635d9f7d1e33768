"""Local memory of the kernels in the built libppg_b200.so, read with `cuobjdump -res-usage` (no GPU needed).

The CBOX bounce kernels run 1024 threads per SM at 64 registers; a stack frame there is per-thread local memory that the path loop
reloads through L1, next to the D-tree nodes it reads through L1 on purpose (DESIGN.md 4.1).  What is left of their frame is register
spills (at most 96 bytes): every struct kernel parameter is __grid_constant__ (no per-thread copy of RenderParams, ~900 bytes), the staged
kernels have no BVH walk (its 512-byte stack) and no object whose address reaches a call that is not inlined.  Every other kernel keeps
at most the frame listed here."""
import os
import re
import shutil
import subprocess

import pytest

from ppg_b200 import capi

# stack frame (bytes) per kernel, at most
CEILING = {
    "trace_kernel<0,0>": 512, "trace_kernel<1,0>": 512, "trace_kernel<0,1>": 560, "trace_kernel<1,1>": 560,   # the BVH stack (2 x 64 entries)
    "commit_kernel<1>": 768, "commit_kernel<2>": 2816,
    "dtree_reset_kernel<0>": 768, "dtree_reset_kernel<1>": 768,                                               # the DFS stack (64 entries)
    "stree_refine_kernel": 0, "dtree_build_kernel": 0, "leaf_after_reset_kernel": 0, "adam_seq_kernel": 0, "adam_pack_kernel": 0,
    "adam_merge_kernel": 0, "tree_stats_kernel": 0, "adam_progress_kernel": 0,
    "op_record_kernel": 768, "op_emitter_sample_kernel": 608, "op_env_pdf_kernel": 0,
}
# bounce_kernel<FIRST, RECORD, NEE, SMEM, FULL>: at most this frame per (NEE, SMEM, FULL) family
BOUNCE_CEILING = {(0, 0, 0): 704, (0, 0, 1): 1168, (0, 1, 0): 112, (0, 1, 1): 496, (1, 0, 0): 848, (1, 0, 1): 1296, (1, 1, 0): 224, (1, 1, 1): 688}
CBOX = {(first, record, 0, 1, 0) for first in (0, 1) for record in (0, 1)}
CBOX_CEILING = 96        # register spills only


def _cuobjdump():
    for d in (os.environ.get("CUDA_HOME"), "/usr/local/cuda"):
        if d and os.path.exists(os.path.join(d, "bin", "cuobjdump")):
            return os.path.join(d, "bin", "cuobjdump")
    return shutil.which("cuobjdump")


def _frames():
    """{kernel key: stack bytes}; key = name<template args> from the mangled name, e.g. bounce_kernel<0,1,0,1,0>"""
    if not os.path.exists(capi.LIB_PATH):
        pytest.skip("libppg_b200.so has not been built")
    tool = _cuobjdump()
    assert tool, "cuobjdump not found (CUDA toolkit)"
    out = subprocess.run([tool, "-res-usage", capi.LIB_PATH], capture_output=True, text=True, check=True).stdout
    frames = {}
    for name, stack in re.findall(r"Function (\S+):\s*REG:\d+ STACK:(\d+)", out):
        pos, ident = name.find("N") + 1, None        # walk the length-prefixed names of the nested name to the one that ends in _kernel
        while pos and (m := re.compile(r"(\d+)").match(name, pos)):
            n = int(m.group(1)); ident = name[m.end():m.end() + n]; pos = m.end() + n
            if ident.endswith("_kernel"):
                break
        if not ident or not ident.endswith("_kernel"):
            continue
        t = re.compile(r"I((?:L[bi]\d+E)+)E").match(name, pos)
        args = re.findall(r"L[bi](\d+)E", t.group(1)) if t else []
        key = ident + ("<" + ",".join(args) + ">" if args else "")
        assert key not in frames, key
        frames[key] = int(stack)
    assert frames, "no kernels found in " + capi.LIB_PATH
    return frames


def test_cbox_bounce_kernels_keep_only_spills_in_local_memory():
    frames = _frames()
    keys = {"bounce_kernel<%d,%d,%d,%d,%d>" % k for k in CBOX}
    assert keys <= frames.keys(), keys - frames.keys()
    over = {k: frames[k] for k in keys if frames[k] > CBOX_CEILING}
    assert not over, over


def test_other_kernels_keep_their_stack_frames():
    frames = _frames()
    over = {}
    for key, limit in CEILING.items():
        assert key in frames, key
        if frames[key] > limit:
            over[key] = (frames[key], limit)
    bounce = [k for k in frames if k.startswith("bounce_kernel<")]
    assert len(bounce) == 40, len(bounce)
    for key in bounce:
        first, record, nee, smem, full = map(int, key[len("bounce_kernel<"):-1].split(","))
        limit = CBOX_CEILING if (first, record, nee, smem, full) in CBOX else BOUNCE_CEILING[(nee, smem, full)]
        if frames[key] > limit:
            over[key] = (frames[key], limit)
    assert not over, over
