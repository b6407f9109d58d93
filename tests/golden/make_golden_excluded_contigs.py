"""Writes tests/golden/excluded_contigs.txt, one name per line: the UNMODIFIED reference list of contigs a genome-wide
call_variant leaves out (EXCLUDED_HUMAN_CONTIGS, pepper_variant/modules/python/ExcludeContigs.py, used at
ImageGenerationUI.py:117).  pepper_b200.exclude states the rule as name shapes; the fixture pins it to the list.
    python tests/golden/make_golden_excluded_contigs.py"""
import importlib.util
import os

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("PEPPER_REFERENCE", "/root/reference")
spec = importlib.util.spec_from_file_location("ExcludeContigs", os.path.join(REF, "pepper_variant/modules/python/ExcludeContigs.py"))
m = importlib.util.module_from_spec(spec)
spec.loader.exec_module(m)
with open(os.path.join(HERE, "excluded_contigs.txt"), "w") as f:
    f.write("".join(c + "\n" for c in m.EXCLUDED_HUMAN_CONTIGS))
print("wrote excluded_contigs.txt: %d names" % len(m.EXCLUDED_HUMAN_CONTIGS))
