"""Occupancy and posting bandwidth of the k-mer ranker on the benchmark's headline shape (diagnostic, not the bench).

Prints, as JSON lines:
  - CTAs per SM of rank_kernel's full and short-query instances (cudaOccupancyMaxActiveBlocksPerMultiprocessor);
  - the ranker's kernel time (vsg_profile.rank_ms; median, min, max of --repeats) for the 32 768 queries of 250 nt
    bench.py ranks alone (100 000 x 1 500-nt database, wordlength 8, minwordmatches 12, tophits 41);
  - the posting bytes those queries stream: for every query, every shard and every distinct k-mer of the query, the
    k-mer's even and odd sub-lists as the index stores them (padded to vectors of 8 two-byte postings, the differences
    of the shard's list offsets), recomputed here from the database on the device; over the kernel time, and set
    against the H100 SXM data sheet's 3.35 TB/s;
  - the card's name, power limit and SM clock (nvidia-smi, read-only queries, sampled during the timed repeats).

    python tools/perf_rank_occupancy.py [--repeats 5] [--queries 32768]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
from vsearch_b200 import lib as vlib, synth  # noqa: E402

N_DB, DB_LEN, Q_LEN, DIV, SEED, K = 100_000, 1500, 250, 0.05, 2024, 8   # bench.py's headline workload
MINWORDMATCHES, TOPHITS = 12, 41
SHARD_STATIC = 32766
HBM_TBS = 3.35


def smi(fields):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader,nounits", "-i", "0"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except OSError:
        return ""


class ClockSampler(threading.Thread):
    """the SM clock every 200 ms until stop()"""

    def __init__(self):
        super().__init__(daemon=True)
        self.mhz, self.done = [], threading.Event()

    def run(self):
        while not self.done.is_set():
            v = smi("clocks.sm")
            if v.isdigit():
                self.mhz.append(int(v))
            self.done.wait(0.2)

    def stop(self):
        self.done.set()
        self.join()
        return self.mhz


def kmer_codes(m, k):
    """(n, L) ASCII ACGT matrix on the device -> (n, L - k + 1) k-mer codes, first base in the high bits"""
    b = torch.zeros_like(m, dtype=torch.int32)
    for ch, v in ((b"C", 1), (b"G", 2), (b"T", 3)):
        b[m == ch[0]] = v
    w = m.shape[1] - k + 1
    code = torch.zeros((m.shape[0], w), dtype=torch.int32, device=m.device)
    for j in range(k):
        code = (code << 2) | b[:, j:j + w]
    return code


def distinct_rows(code):
    """row-wise sorted codes with every repeat replaced by -1"""
    s, _ = torch.sort(code, dim=1)
    dup = torch.zeros_like(s, dtype=torch.bool)
    dup[:, 1:] = s[:, 1:] == s[:, :-1]
    return torch.where(dup, torch.full_like(s, -1), s)


def list_bytes_per_kmer(dbm, k, dev="cuda"):
    """bytes of postings the static index stores per k-mer, summed over the shards"""
    hashsize = 1 << (2 * k)
    total = torch.zeros(hashsize, dtype=torch.int64, device=dev)
    for t0 in range(0, dbm.shape[0], SHARD_STATIC):
        m = torch.from_numpy(dbm[t0:t0 + SHARD_STATIC]).to(dev)
        d = distinct_rows(kmer_codes(m, k))
        parity = (torch.arange(d.shape[0], device=dev) & 1).unsqueeze(1).expand_as(d)
        keep = d >= 0
        n = torch.bincount((2 * d[keep] + parity[keep]).long(), minlength=2 * hashsize)   # targets per sub-list
        padded = (n + 7) & ~7
        total += 2 * (padded[0::2] + padded[1::2])
    return total


def posting_bytes(dbm, qss, nq, k, dev="cuda"):
    """bytes of the posting lists queries [0, nq) of qss stream from the index of dbm"""
    per_kmer = list_bytes_per_kmer(dbm, k, dev)
    byts = 0
    for i0 in range(0, nq, 4096):
        rows = [qss.cat[qss.offs[i]:qss.offs[i] + qss.lens[i]] for i in range(i0, min(nq, i0 + 4096))]
        width = max(r.shape[0] for r in rows)
        m = np.full((len(rows), width), ord("A"), dtype=np.uint8)
        valid = np.zeros((len(rows), width - k + 1), dtype=bool)
        for j, r in enumerate(rows):
            m[j, :r.shape[0]] = r
            valid[j, :r.shape[0] - k + 1] = True
        code = kmer_codes(torch.from_numpy(m).to(dev), k)
        code = torch.where(torch.from_numpy(valid).to(dev), code, torch.full_like(code, -1))
        d = distinct_rows(code)
        byts += int(per_kmer[d[d >= 0].long()].sum().item())
    return byts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--queries", type=int, default=32768)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_rank_occupancy.py: no CUDA device")
    ctx = vlib.Context(0)
    full, short = ctx.rank_occupancy()
    print(json.dumps({"ctas_per_sm": {"full": full, "short": short}}), flush=True)

    dbm = synth.config2_db(N_DB, DB_LEN, SEED)
    qss, _ = synth.config2_query_batch(dbm, 65536, Q_LEN, DIV, SEED, batch=3)   # bench.py's first timed batch
    nq = a.queries
    db = ctx.seqset(synth.SeqSet.from_matrix(dbm))
    ix = ctx.index(db, K, 0)
    qs = ctx.seqset(qss)
    ref = ctx.rank(ix, qs, 0, nq, MINWORDMATCHES, TOPHITS)   # warm-up
    times = []
    sampler = ClockSampler()
    sampler.start()
    for _ in range(a.repeats):
        ctx.profile_reset()
        got = ctx.rank(ix, qs, 0, nq, MINWORDMATCHES, TOPHITS)
        times.append(ctx.profile().rank_ms)
        if not all(np.array_equal(x, y) for x, y in zip(got, ref)):
            raise SystemExit("a repeat's output differs from the first run's")
    mhz = sampler.stop()
    qs.close(); ix.close(); db.close(); ctx.close()

    byts = posting_bytes(dbm, qss, nq, K)
    med = statistics.median(times)
    name, plimit, maxmhz = (x.strip() for x in (smi("name,power.limit,clocks.max.sm").split(",") + ["", "", ""])[:3])
    print(json.dumps({"queries": nq, "query_len": Q_LEN, "tophits": TOPHITS, "rank_ms_median": round(med, 3),
                      "rank_ms_min": round(min(times), 3), "rank_ms_max": round(max(times), 3), "repeats": a.repeats,
                      "posting_bytes": byts, "posting_tb_per_s": round(byts / (med * 1e-3) / 1e12, 3),
                      "of_hbm_data_sheet": round(byts / (med * 1e-3) / 1e12 / HBM_TBS, 3)}), flush=True)
    print(json.dumps({"card": name, "power_limit_w": plimit, "sm_clock_max_mhz": maxmhz,
                      "sm_clock_mhz_during_repeats": {"median": statistics.median(mhz) if mhz else None,
                                                      "min": min(mhz, default=None), "max": max(mhz, default=None)}}),
          flush=True)


if __name__ == "__main__":
    main()
