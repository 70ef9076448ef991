"""Test-only CSI index writer (`samtools index -c` layout, BGZF-compressed): per contig one ordinary bin and the pseudo-bin
holding (mapped, unmapped), which is what the native decoder's index statistics read."""
import struct

import bam_writer


def bgzf(data, block=4000):
    out = b"".join(bam_writer._bgzf_block(data[o:o + block]) for o in range(0, len(data), block))
    return out + bam_writer._bgzf_block(b"")


def write_csi(path, stats, min_shift=14, depth=5, aux=b""):
    """stats: [(contig, mapped)] in header order."""
    pseudo = ((1 << 3 * (depth + 1)) - 1) // 7 + 1
    body = b"CSI\1" + struct.pack("<iii", min_shift, depth, len(aux)) + aux + struct.pack("<i", len(stats))
    for k, (_, mapped) in enumerate(stats):
        body += struct.pack("<i", 2)
        body += struct.pack("<IQi", 0, 1000 * k, 1) + struct.pack("<QQ", 1000 * k, 1000 * k + 500)
        body += struct.pack("<IQi", pseudo, 0, 2) + struct.pack("<QQQQ", 1000 * k, 1000 * k + 500, mapped, 7)
    body += struct.pack("<Q", 2)
    with open(path, "wb") as f:
        f.write(bgzf(body))
