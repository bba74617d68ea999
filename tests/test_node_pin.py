"""tests/golden/knn_golden.json stores every float as Python's float.hex() string; its readers (tests/common.py,
tests/test_oracle.py) and tests/golden/make_golden_node.mjs, which checks the stored vectors against the reference's
own code on a machine with Node (RBK_REFERENCE=<checkout>), parse it back.  Pin the format the stored vectors are in."""
import json
from pathlib import Path

HERE = Path(__file__).resolve().parent


def test_python_hex_format_assumed_by_the_node_script():
    """make_golden_node.mjs parses/prints Python's float.hex() by hand: pin the format it assumes."""
    assert (0.5).hex() == "0x1.0000000000000p-1" and (-3.0).hex() == "-0x1.8000000000000p+1"
    assert (0.0).hex() == "0x0.0p+0" and float("nan").hex() == "nan"
    g = json.loads((HERE / "golden" / "knn_golden.json").read_text())
    import re
    pat = re.compile(r"^-?0x[01]\.[0-9a-f]{1,13}p[+-]\d+$")
    for c in g["cases"]:
        assert all(pat.match(x) for x in c["query"] + c["scan_scores"] + c["fms_scores"])
