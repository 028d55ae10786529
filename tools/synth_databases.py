#!/usr/bin/env python
"""Seeded stand-ins for the 8 bundled rRNA databases (data/rRNA_databases of the reference), for the benchmark.

The databases themselves are 76 MB of FASTA and are not part of this repository, so bench.py writes a synthetic set of
the same shape into a temporary directory: per database the same number of sequences and the same median sequence length
as the file it stands in for, organised the way a clustered rRNA database is -- every sequence descends from one database
ancestor through a clade ancestor (15 % substitutions from the ancestor, then 5 % from the clade), so a read drawn from
one sequence seeds against many others, as on the real databases.  Lengths vary +-10 % by trimming both ends.

The same seed gives the same bytes on every machine (numpy's PCG64).  The Gumbel parameters bench.py turns into minimal
scores are those the reference computes for the database each stand-in is named after (sortmerna_b200/gumbel_defaults.json).

  python tools/synth_databases.py OUT_DIR      # writes OUT_DIR/<name>.fasta for the 8 databases
"""
import os
import sys

import numpy as np

# name of the database stood in for, sequences, median length (data/rRNA_databases of the reference)
SHAPES = [("silva-bac-16s-id90", 12798, 1412), ("silva-bac-23s-id98", 4488, 2871), ("silva-arc-16s-id95", 3193, 1036),
          ("silva-arc-23s-id98", 251, 2918), ("silva-euk-18s-id95", 7348, 1741), ("silva-euk-28s-id98", 4935, 3026),
          ("rfam-5s-database-id98", 59513, 119), ("rfam-5.8s-database-id98", 13034, 155)]
SEED = 20261015
CLADE_SIZE = 50
CLADE_DIV, MEMBER_DIV = 0.15, 0.05


def _mutate(rng, seqs, rate):
    """i.i.d. substitutions (to one of the three other bases) at `rate` in a (n, L) uint8 array of 0..3 codes"""
    hit = rng.random(seqs.shape, dtype=np.float32) < rate
    return np.where(hit, (seqs + rng.integers(1, 4, seqs.shape, dtype=np.uint8)) & 3, seqs).astype(np.uint8)


def database(k, scale=1.0):
    """(ids, list of ACGT byte strings) of stand-in k; `scale` shrinks the sequence count (tests)."""
    name, nseq, med = SHAPES[k]
    nseq = max(1, int(nseq * scale))
    rng = np.random.default_rng([SEED, k])
    L = int(med * 1.1) + 1
    root = rng.integers(0, 4, L, dtype=np.uint8)
    nclade = (nseq + CLADE_SIZE - 1) // CLADE_SIZE
    clades = _mutate(rng, np.broadcast_to(root, (nclade, L)), CLADE_DIV)
    members = _mutate(rng, clades[np.arange(nseq) // CLADE_SIZE], MEMBER_DIV)
    lens = np.clip(rng.normal(med, 0.05 * med, nseq).astype(np.int64), max(20, int(0.9 * med)), L)
    lead = rng.integers(0, L - lens + 1)
    acgt = np.frombuffer(b"ACGT", np.uint8)
    seqs = [acgt[members[i, lead[i]:lead[i] + lens[i]]].tobytes() for i in range(nseq)]
    ids = [f"synth_{name}_{i:06d}" for i in range(nseq)]
    return ids, seqs


def file_name(k):
    return SHAPES[k][0] + ".fasta"


def write(out_dir, scale=1.0):
    """Writes the 8 stand-ins (skipping files already there); returns their paths in --ref order."""
    os.makedirs(out_dir, exist_ok=True)
    paths = []
    for k in range(len(SHAPES)):
        p = os.path.join(out_dir, file_name(k))
        if not os.path.exists(p):
            ids, seqs = database(k, scale)
            tmp = p + ".part"
            with open(tmp, "wb") as f:
                f.write(b"".join(b">" + i.encode() + b"\n" + s + b"\n" for i, s in zip(ids, seqs)))
            os.replace(tmp, p)
        paths.append(p)
    return paths


if __name__ == "__main__":
    print("\n".join(write(sys.argv[1])))
