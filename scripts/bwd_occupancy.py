#!/usr/bin/env python
"""Occupancy of the composite backward kernel on cuda:0: CTAs per SM as the CUDA occupancy calculator reports it for the
shipped instantiation (with its launch attributes and dynamic shared memory), next to the card's name, power limit and
clocks.  Nsight Compute is not needed.  Prints one JSON line.

    python scripts/bwd_occupancy.py
"""
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "comfyui-3d-pack_b200"), ROOT]

import torch  # noqa: E402

from gs_b200 import _lib  # noqa: E402


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    ctas, smem = C.c_int32(0), C.c_int32(0)
    _lib.check(_lib.lib.gs_b200_composite_bwd_occupancy(C.byref(ctas), C.byref(smem)))
    prop = torch.cuda.get_device_properties(0)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                          "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    print(json.dumps({"device": prop.name, "sms": prop.multi_processor_count, "nvidia_smi": smi.stdout.strip(),
                      "composite_bwd": {"ctas_per_sm": ctas.value, "warps_per_sm": 4 * ctas.value,
                                        "dynamic_smem_bytes": smem.value}}))


if __name__ == "__main__":
    main()
