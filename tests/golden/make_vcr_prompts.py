"""Generates tests/golden/vcr_prompts.json: the reference tokenizer's encodings of VCR's two prompt texts
(downstream/vcr/dataloader_joint.py:28-31), which merlot_b200.vcr_input holds as constants.

    python tests/golden/make_vcr_prompts.py PATH/TO/MERLOT    # a checkout of the reference (its utils/encode/encoder.py)
"""
import json
import os
import sys

if len(sys.argv) != 2:
    raise SystemExit(__doc__)
sys.path.insert(0, sys.argv[1])
from utils.encode.encoder import END, START, get_encoder  # noqa: E402

enc = get_encoder()
facts = {"specials": {"START": START, "END": END},
         "encode": {t: enc.encode(t) for t in (" answer question:", " provide rationale:")}}
out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "vcr_prompts.json")
with open(out, "w") as f:
    json.dump(facts, f, indent=1, sort_keys=True)
print("wrote", out)
