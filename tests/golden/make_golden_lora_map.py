"""Record the weight-name pairs of the reference's Wan -> diffusers checkpoint converter
(chronoedit_diffsynth/wan_video_dit_chronoedit.py, the state-dict converter's rename table) as tests/golden/LORA_KEY_MAP.json:
{"<diffusers name>": "<Wan name>"} for block 0 and for the modules outside the blocks.  tests/test_lora_cpu.py holds the
mirror's own map against it.  Needs the reference checkout (oracle/ref_loader.py)."""
import json
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from oracle import ref_loader  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "LORA_KEY_MAP.json")


def main():
    assert ref_loader.reference_available(), "needs the reference checkout"
    src = open(ref_loader.load_reference_diffsynth_dit().__file__).read()
    pairs = {}
    for dif, wan in re.findall(r'"([\w.]+\.weight)":\s*"([\w.]+\.weight)"', src):
        if not dif.startswith("blocks.") or dif.startswith("blocks.0."):
            pairs[dif] = wan
    with open(OUT, "w") as f:
        json.dump({"generated_by": "tests/golden/make_golden_lora_map.py", "weight_names": pairs}, f, indent=1, sort_keys=True)
    print(len(pairs), "pairs")


if __name__ == "__main__":
    main()
