"""BAMs for the covstats cohort tests that the other helpers do not make."""
import struct


def odd_member(good):
    """a copy of `good` whose third BGZF member carries a subfield before BC (legal gzip the device route rejects), with
    its index shifted to match"""
    raw = open(good, "rb").read()
    offs, q = [], 0
    while q < len(raw):
        offs.append(q)
        q += struct.unpack_from("<H", raw, q + 16)[0] + 1
    m0, m1 = offs[2], offs[3]
    mem = raw[m0:m1]
    new = mem[:10] + struct.pack("<H", 10) + b"XX\x00\x00" + mem[12:16] + struct.pack("<H", len(mem) + 4 - 1) + mem[18:]
    odd = good[:-4] + ".odd.bam"
    open(odd, "wb").write(raw[:m0] + new + raw[m1:])
    bai = bytearray(open(good + ".bai", "rb").read())

    def shift(v):
        return v + (4 << 16) if (v >> 16) >= m1 else v
    o = 4
    n_ref = struct.unpack_from("<i", bai, o)[0]; o += 4
    for _ in range(n_ref):
        nb = struct.unpack_from("<i", bai, o)[0]; o += 4
        for _ in range(nb):
            b, nc = struct.unpack_from("<Ii", bai, o); o += 8
            for k in range(nc * 2):
                if b != 37450 or k < 2:
                    struct.pack_into("<Q", bai, o + 8 * k, shift(struct.unpack_from("<Q", bai, o + 8 * k)[0]))
            o += 16 * nc
        nl = struct.unpack_from("<i", bai, o)[0]; o += 4
        for k in range(nl):
            struct.pack_into("<Q", bai, o + 8 * k, shift(struct.unpack_from("<Q", bai, o + 8 * k)[0]))
        o += 8 * nl
    open(odd + ".bai", "wb").write(bytes(bai))
    return odd
