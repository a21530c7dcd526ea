#!/usr/bin/env python3
"""covstats sampling, host route against device route, on a paired synthetic BAM.

    python tools/bench_covstats.py [--records 6000000] [--n 1000000] [--repeats 5] [--out DIR]

Writes a coordinate-sorted BAM of paired 150 bp reads with its .bai into a temporary directory, then calls
gl_bam_covstats_host and gl_bam_covstats alternately on one context: one warm-up call of each, then `repeats` timed calls of
each.  Both entries return after a device synchronise, so the wall clock around a call is the call.  Prints one JSON line:
wall times (median, min, max), the device route's phase times from the struct, compressed and inflated bytes, batches, the
host pool's thread count, and the card's name and power limit as nvidia-smi reports them in this run.  Needs a GPU."""
import argparse
import ctypes as C
import json
import os
import struct
import subprocess
import sys
import tempfile
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BLOCK = 65280
EOF_MEMBER = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def _member(chunk: bytes) -> bytes:
    c = zlib.compressobj(1, zlib.DEFLATED, -15)
    comp = c.compress(chunk) + c.flush()
    return (b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00" + struct.pack("<H", 18 + len(comp) + 8 - 1) + comp +
            struct.pack("<II", zlib.crc32(chunk) & 0xffffffff, len(chunk)))


def write_paired_bam(path: str, n_records: int, seed: int = 0, spacing: int = 5, sample: str = "S1") -> int:
    """A coordinate-sorted single-reference BAM of n_records paired 150 bp reads (150M; 45 % left mates of proper pairs, 45 %
    right mates, the rest duplicates, QC failures, unpaired and unmapped-with-coordinates) and path + ".bai".  Every record
    has the same size, so the index follows from arithmetic.  Returns n_records."""
    rng = np.random.default_rng(seed)
    name_len, rl = 8, 150
    rec = np.dtype([("bs", "<i4"), ("tid", "<i4"), ("pos", "<i4"), ("l_name", "u1"), ("mapq", "u1"), ("bin", "<u2"), ("n_cig", "<u2"),
                    ("flag", "<u2"), ("l_seq", "<i4"), ("mtid", "<i4"), ("mpos", "<i4"), ("tlen", "<i4"), ("name", "S8"), ("cigar", "<u4"),
                    ("seq", "u1", (rl + 1) // 2), ("qual", "u1", rl)])
    ref_len = n_records * spacing + 100_000
    text = ("@HD\tVN:1.6\tSO:coordinate\n@SQ\tSN:chr1\tLN:%d\n@RG\tID:a\tSM:%s\n" % (ref_len, sample)).encode()
    head = b"BAM\x01" + struct.pack("<i", len(text)) + text + struct.pack("<i", 1) + struct.pack("<i", 5) + b"chr1\0" + struct.pack("<i", ref_len)
    members, at = [], 0
    step = 200_000
    carry = head
    pool = ThreadPoolExecutor(max(2, min(16, os.cpu_count() or 2)))
    with open(path, "wb") as f:
        for r0 in range(0, n_records, step):
            m = min(step, n_records - r0)
            a = np.zeros(m, rec)
            a["bs"] = rec.itemsize - 4
            a["pos"] = (np.arange(r0, r0 + m, dtype=np.int64) * spacing).astype(np.int32)
            a["l_name"], a["mapq"], a["n_cig"], a["l_seq"], a["name"] = name_len, 60, 1, rl, b"read123"
            a["cigar"] = (rl << 4) | 0
            kind = rng.random(m)
            flag = np.where(kind < 0.45, 99, np.where(kind < 0.90, 147, np.where(kind < 0.93, 0x400 | 99, np.where(kind < 0.95, 0x200 | 163,
                            np.where(kind < 0.98, 0, 0x4 | 0x1 | 0x40)))))
            ins = np.clip(rng.normal(200, 50, m), -100, None).astype(np.int32)
            ins[rng.random(m) < 0.005] = rng.integers(5000, 200000)
            left = (flag & 0x20) != 0
            a["flag"] = flag
            a["mpos"] = np.where(left, a["pos"] + rl + ins, np.maximum(a["pos"] - rl - ins, 0))
            a["tlen"] = np.where(left, 2 * rl + ins, -(2 * rl + ins))
            a["seq"] = rng.integers(0, 4, (m, (rl + 1) // 2), dtype=np.uint8) * 17 + 17
            a["qual"] = rng.choice(np.array([2, 11, 25, 37], np.uint8), (m, rl), p=[0.03, 0.07, 0.2, 0.7])
            data = carry + a.tobytes()
            whole = len(data) // BLOCK * BLOCK
            for comp in pool.map(_member, [data[i:i + BLOCK] for i in range(0, whole, BLOCK)]):
                members.append(at); at += len(comp); f.write(comp)
            carry = data[whole:]
        if carry:
            comp = _member(carry)
            members.append(at); at += len(comp); f.write(comp)
        members.append(at)
        f.write(EOF_MEMBER)
    pool.shutdown()
    members = np.array(members, np.int64)

    def voff(byte_off):
        byte_off = np.asarray(byte_off, np.int64)
        return (members[byte_off // BLOCK].astype(np.uint64) << np.uint64(16)) | (byte_off % BLOCK).astype(np.uint64)
    pos_all = np.arange(n_records, dtype=np.int64) * spacing
    n_tiles = int((pos_all[-1] + rl - 1) >> 14) + 1
    first = np.searchsorted(pos_all + rl, np.arange(n_tiles, dtype=np.int64) * 16384, "right")        # first record whose end passes the tile's start
    lin = voff(len(head) + first * rec.itemsize)
    v0, v1 = int(voff(len(head))), int(voff(len(head) + n_records * rec.itemsize - 1)) + 1
    bai = b"BAI\x01" + struct.pack("<i", 1) + struct.pack("<i", 2)
    bai += struct.pack("<Ii", 0, 1) + struct.pack("<QQ", v0, v1)
    bai += struct.pack("<Ii", 37450, 2) + struct.pack("<4Q", v0, v1, n_records, 0)
    bai += struct.pack("<i", n_tiles) + lin.astype("<u8").tobytes() + struct.pack("<Q", 0)
    open(path + ".bai", "wb").write(bai)
    return n_records


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=6_000_000)
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--skip", type=int, default=100_000)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for bench_covstats.json (besides stdout)")
    args = ap.parse_args()
    from goleft_b200 import capi
    if capi.device_count() < 1:
        raise SystemExit("bench_covstats needs a CUDA device")
    capi.lib.glhost_pool_size.restype = C.c_int
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "paired.bam")
        t0 = time.time()
        write_paired_bam(path, args.records)
        res = {"bam_bytes": os.path.getsize(path), "records": args.records, "n": args.n, "skip": args.skip, "write_s": round(time.time() - t0, 1),
               "gpu": gpu[0] if gpu else "unknown", "host_threads": int(capi.lib.glhost_pool_size()), "repeats": args.repeats}
        with capi.Ctx(0) as ctx:
            bam = capi.Bam(path)
            routes = {"host": capi.bam_covstats_host, "device": capi.bam_covstats}
            walls = {k: [] for k in routes}
            last = {}
            for it in range(args.repeats + 1):                                  # the first round warms both routes up
                for k, fn in routes.items():
                    t = time.perf_counter()
                    st, H = fn(ctx, bam, args.n, args.skip)
                    ctx.sync()
                    dt = time.perf_counter() - t
                    if it:
                        walls[k].append(dt)
                    last[k] = (st, H)
            bam.close()
        (sh, Hh), (sd, Hd) = last["host"], last["device"]
        same = all(np.float64(getattr(sh, k)).tobytes() == np.float64(getattr(sd, k)).tobytes() for k in capi.CovStats.STATS + capi.CovStats.COUNTERS)
        res["identical"] = bool(same and Hh.tobytes() == Hd.tobytes())
        for k, w in walls.items():
            res[k + "_wall_s"] = {"median": round(float(np.median(w)), 4), "min": round(min(w), 4), "max": round(max(w), 4)}
        res["device_phases_s"] = {k: round(getattr(sd, k), 4) for k in ("read_s", "inflate_s", "index_s", "fields_s", "cut_s", "tail_s", "wall_s")}
        res["device"] = {"batches": sd.n_batches, "bytes_in": sd.bytes_in, "bytes_out": sd.bytes_out, "records_read": sd.n_records_read,
                         "n_insert": sd.n_insert, "h_len": sd.h_len}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        open(os.path.join(args.out, "bench_covstats.json"), "w").write(line + "\n")


if __name__ == "__main__":
    main()
