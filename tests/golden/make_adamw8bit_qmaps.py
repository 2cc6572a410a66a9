"""Writes tests/golden/adamw8bit_qmaps.json: the signed and unsigned 256-entry quantisation maps of optim.AdamW8bit
(`optim.dynamic_map`), as exact fp32 values.  tests/test_adamw8bit.py compares the maps with this table, so a change to the
construction shows up as a diff of the committed file.

    python tests/golden/make_adamw8bit_qmaps.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from t2v_b200.optim import dynamic_map  # noqa: E402

if __name__ == "__main__":
    out = os.path.join(ROOT, "tests", "golden", "adamw8bit_qmaps.json")
    with open(out, "w") as f:
        json.dump({"signed": dynamic_map(True).tolist(), "unsigned": dynamic_map(False).tolist()}, f, indent=1)
        f.write("\n")
    print("wrote", out)
