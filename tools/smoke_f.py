#!/usr/bin/env python
"""One small pass over the 8(f) kernels for compute-sanitizer: index built on the device, gzip inflate + input
decode on the device, then the alignment kernels on that batch."""
import gzip
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sortmerna_b200 import api, hostio  # noqa: E402

g = os.path.join(ROOT, "tests", "golden")
al = api.Aligner(0)
al.set_params(api.default_params())
for k, n in enumerate(("db_arc.fasta", "db_bac.fasta")):
    assert al.build_index_device(k, os.path.join(g, n), hostio.load_references(os.path.join(g, n)), 60) == 1
text = open(os.path.join(g, "reads_mix.fq"), "rb").read()
gz = gzip.compress(text[: len(text) // 3], 6)
got, info = al.debug_inflate(gz, 4096)
assert got == text[: len(text) // 3], "inflate"
n = al.upload_fastx_gz(gz)
al.run_resident()
out = al.download()
print(f"smoke_f ok: {n} reads, {int(out['res']['is_hit'].sum())} aligned, inflate spans {info['spans']}")
al.close()
