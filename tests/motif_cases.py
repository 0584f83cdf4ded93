"""Shared inputs of the motif tests: the fixture's genome, sequences and .pfm files rebuilt on disk."""
import json
import os

import numpy as np

from conftest import GOLDEN

Z = np.load(os.path.join(GOLDEN, "motifs_small.npz"))
SIG = json.load(open(os.path.join(GOLDEN, "motifs_signature.json")))
JASPAR = np.load(os.path.join(GOLDEN, "jaspar_pfm.npz"))


def sequences():
    text, out, a = str(Z["seq_text"]), [], 0
    for n in Z["seq_len"]:
        out.append(text[a:a + int(n)])
        a += int(n)
    return out


def counts_list(z, names="pfm_name", lengths="pfm_len", counts="pfm_counts"):
    off = np.concatenate([[0], np.cumsum(z[lengths])])
    return [z[counts][:, off[i]:off[i + 1]] for i in range(len(z[names]))]


def write_pfms(directory, z=Z, names="pfm_name", lengths="pfm_len", counts="pfm_counts"):
    files = []
    for name, c in zip(z[names], counts_list(z, names, lengths, counts)):
        path = os.path.join(str(directory), str(name))
        with open(path, "w") as fh:
            for row in c:
                fh.write(" ".join(f"{int(v)}" for v in row) + "\n")
        files.append(path)
    return files


def write_meta(directory, z=Z):
    path = os.path.join(str(directory), "motif_to_gene.txt")
    with open(path, "w") as fh:
        for i, g in zip(z["meta_id"], z["meta_gene"]):
            fh.write(f"{i}\t{g}\n")
    return path


def write_fasta(directory, name="genome.fa"):
    path = os.path.join(str(directory), name)
    with open(path, "wb") as fh:
        fh.write(Z["fasta"].tobytes())
    return path


def random_genome(n, seed, n_runs=200, lower_runs=300):
    """A random sequence of n bases with runs of N and lowercase stretches, as a str."""
    rng = np.random.default_rng(seed)
    b = rng.choice(np.frombuffer(b"ACGT", np.uint8), n)
    for a in rng.integers(0, max(n - 100, 1), n_runs):
        b[a:a + int(rng.integers(1, 80))] = ord("N")
    for a in rng.integers(0, max(n - 500, 1), lower_runs):
        s = slice(a, a + int(rng.integers(5, 400)))
        b[s] = np.where(b[s] != ord("N"), b[s] | 0x20, b[s])
    return b.tobytes().decode()
