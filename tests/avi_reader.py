"""A small RIFF/AVI reader written for the tests, independent of video.MjpegAviWriter: it walks every RIFF segment, lists
the stream headers and the movi chunks in file order, and resolves every idx1, indx and ix## entry to the chunk it names
(asserting that a chunk of the right id and size sits there)."""
import struct


def _chunks(buf, start, end):
    at = start
    while at + 8 <= end:
        cid, size = buf[at:at + 4], struct.unpack_from("<I", buf, at + 4)[0]
        yield cid, at, size
        at += 8 + size + (size & 1)


def read(path):
    buf = open(path, "rb").read()
    out = {"segments": [], "strh": [], "strf": [], "indx": [], "movi_chunks": [], "idx1": None, "avih": None}
    for cid, at, size in _chunks(buf, 0, len(buf)):
        assert cid == b"RIFF", cid
        form = buf[at + 8:at + 12]
        out["segments"].append((form, at, size + 8))
        for sub, sat, ssize in _chunks(buf, at + 12, at + 8 + size):
            if sub == b"LIST" and buf[sat + 8:sat + 12] == b"hdrl":
                for h, hat, hsize in _chunks(buf, sat + 12, sat + 8 + ssize):
                    if h == b"avih":
                        out["avih"] = struct.unpack_from("<IIIIIIIIII", buf, hat + 8)
                    elif h == b"LIST" and buf[hat + 8:hat + 12] == b"strl":
                        for s, s_at, s_size in _chunks(buf, hat + 12, hat + 8 + hsize):
                            if s == b"strh":
                                out["strh"].append(struct.unpack_from("<4s4sIHHIIIIIIiIhhhh", buf, s_at + 8))
                            elif s == b"strf":
                                out["strf"].append(buf[s_at + 8:s_at + 8 + s_size])
                            elif s == b"indx":
                                lpe, sub_t, typ, n, chunk_id = struct.unpack_from("<HBBI4s", buf, s_at + 8)
                                assert (lpe, typ) == (4, 0)
                                out["indx"].append((chunk_id, [struct.unpack_from("<QII", buf, s_at + 32 + 16 * i)
                                                               for i in range(n)]))
            elif sub == b"LIST" and buf[sat + 8:sat + 12] == b"movi":
                movi = sat
                for c, cat, csize in _chunks(buf, sat + 12, sat + 8 + ssize):
                    if c[:2] != b"ix":
                        out["movi_chunks"].append((c, cat, csize))
            elif sub == b"idx1":
                out["idx1"] = [struct.unpack_from("<4sIII", buf, sat + 8 + 16 * i) for i in range(ssize // 16)]
                for cid2, flags, off, csize in out["idx1"]:
                    pos = movi + 8 + off
                    assert buf[pos:pos + 4] == cid2 and struct.unpack_from("<I", buf, pos + 4)[0] == csize
    # the OpenDML indices: every super-index entry names an ix## chunk, every ix## entry a chunk's data
    out["odml"] = []
    for chunk_id, entries in out["indx"]:
        listed = []
        for off, size, dur in entries:
            assert buf[off:off + 2] == b"ix"
            lpe, sub_t, typ, n, cid2, base = struct.unpack_from("<HBBI4sQ", buf, off + 8)
            assert (lpe, typ, cid2) == (2, 1, chunk_id) and size == 32 + 8 * n
            for i in range(n):
                rel, csize = struct.unpack_from("<II", buf, off + 32 + 8 * i)
                pos = base + rel - 8
                assert buf[pos:pos + 4] == chunk_id and struct.unpack_from("<I", buf, pos + 4)[0] == csize & 0x7FFFFFFF
                listed.append(pos)
        out["odml"].append((chunk_id, listed))
    out["data"] = lambda cid: [buf[at + 8:at + 8 + size] for c, at, size in out["movi_chunks"] if c == cid]
    return out
