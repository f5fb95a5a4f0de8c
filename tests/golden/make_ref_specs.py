#!/usr/bin/env python
"""Mint the state-dict layouts of the UNMODIFIED reference policies (run where the reference tree is available).

For each policy class and configuration the `state_dict()` of a freshly constructed reference model is recorded as an ordered
list of [key, shape].  The contract tests compare the hand-written specs of oracle/state_dict_spec.py against these records, so
they run without the reference.  Output: tests/golden/ref_state_dict_specs.json.gz."""
import gzip
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)


def main():
    from oracle import ref_shim, synth

    ref = ref_shim.load_reference()
    policies = sys.modules["vima.policy"]
    out = {}

    def record(name, cls, cfg):
        out[name] = [[k, list(v.shape)] for k, v in cls(**cfg).state_dict().items()]

    for model in ("2M", "20M"):
        record(f"VIMAPolicy/{model}", ref.VIMAPolicy, synth.MODEL_CFGS[model])
    record("VIMAFlamingoPolicy/flamingo_tiny", policies.VIMAFlamingoPolicy, synth.FLAMINGO_CFGS["flamingo_tiny"])
    record("VIMAGatoPolicy/gato_tiny", ref.VIMAGatoPolicy, synth.GATO_CFGS["gato_tiny"])
    record("VIMAGPTPolicy/gato_tiny", policies.VIMAGPTPolicy, synth.GATO_CFGS["gato_tiny"])
    with gzip.open(os.path.join(HERE, "ref_state_dict_specs.json.gz"), "wt") as fh:
        json.dump(out, fh, separators=(",", ":"))


if __name__ == "__main__":
    main()
