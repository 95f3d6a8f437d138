"""Copy the sequence dictionaries vg's SAM header tests compare against out of the reference's test data into
tests/golden/sam/ (test/t/50_vg_giraffe.t:226-233 diffs `vg giraffe -o SAM --ref-paths` headers, M5 stripped, with them):
  test/small/xy.dict   @HD VN:1.5 SO:unknown, then @SQ x, y (1001 bp each)
  test/small/yx.dict   the same paths in the other order
Development container only; tests read the copies.   usage: python scripts/extract_sam_fixtures.py"""
import shutil
from pathlib import Path

REF = Path("/root/reference/test")
OUT = Path(__file__).resolve().parents[1] / "tests" / "golden" / "sam"
OUT.mkdir(parents=True, exist_ok=True)
for rel in ("small/xy.dict", "small/yx.dict"):
    shutil.copyfile(REF / rel, OUT / Path(rel).name)
    print(rel, "->", OUT / Path(rel).name)
