"""Tokenizer and batch sources (reference progen_transformer/data.py).

Tokens: `ord(c) + 1`, 0 is pad / BOS / EOS (data.py:76-88).  Training rows have the reference's output contract
(data.py:64-70): uint16 `(B, seq_len + 1)`, a 0 (BOS) in front, `bytes + 1` truncated to seq_len, zero padded.
`iterator_from_tfrecords_folder` reads the reference's GZIP TFRecord files without tensorflow (length-prefixed records
with masked CRC32C, one bytes feature `seq` per tf.train.Example; data.py:25-72) — only the GCS source is out of scope;
`synthetic_iterator` produces the uniform-random rows BASELINE.json measures on, `iterator_from_sequences` turns strings
into rows."""
import numpy as np


def encode_token(token):
    return ord(token) + 1


def decode_token(token):
    if token < 0:
        return ''
    return str(chr(token))


def encode_tokens(tokens):
    return list(map(encode_token, tokens))


def decode_tokens(tokens, offset=1):
    return ''.join(list(map(decode_token, np.asarray(tokens).astype(np.int16) - offset)))


def collate(seqs, seq_len):
    """list of byte strings -> uint16 (B, seq_len + 1) rows exactly like data.py:29-35,64-70"""
    rows = np.zeros((len(seqs), seq_len + 1), np.uint16)
    for i, s in enumerate(seqs):
        t = np.frombuffer(s if isinstance(s, bytes) else s.encode(), dtype=np.uint8).astype(np.uint16)[:seq_len] + 1
        rows[i, 1:1 + len(t)] = t
    return rows


def iterator_from_sequences(seqs, seq_len, batch_size, skip=0, loop=False):
    seqs = list(seqs)[skip:]
    while True:
        for i in range(0, len(seqs), batch_size):
            yield collate(seqs[i:i + batch_size], seq_len)
        if not loop:
            return


def group_by_length(batches):
    """Length-grouped micro-batches: the rows of `batches` (the micro-batches of one effective batch, (b_i, n+1) integer
    rows each) sorted by counted length (`engine.counted_length`; stable, shortest first) and split again into
    micro-batches of the original sizes.  Every optimizer update sees the same sequences; each micro-step then runs at
    a cut length close to its rows' own (DESIGN.md §3.10).  Pure host work."""
    from .engine import counted_length
    if not batches:
        return []
    rows = np.concatenate([np.asarray(b) for b in batches])
    order = np.argsort(counted_length(rows[:, 1:]), kind='stable')
    out, r0 = [], 0
    for b in batches:
        out.append(rows[order[r0:r0 + len(b)]])
        r0 += len(b)
    return out


def synthetic_iterator(seq_len, batch_size, seed=42, vocab=256):
    """uniform-random [0, vocab) rows of seq_len + 1 tokens (BASELINE.json north_star), endless"""
    rng = np.random.default_rng(seed)
    while True:
        yield rng.integers(0, vocab, (batch_size, seq_len + 1)).astype(np.uint16)


# ---------------------------------------------------------------------------------------------------------------------
# TFRecord (GZIP) files without tensorflow — the reference's on-disk format (data.py:9-21 writer, :25-72 reader):
# a gzip stream of records [uint64 length][uint32 masked crc32c(length)][payload][uint32 masked crc32c(payload)], each
# payload a tf.train.Example with one bytes feature 'seq'.  File names end in `.<num_seqs>.<train|valid>.tfrecord.gz`
# (data.py:44-47 takes the sequence count from the 4th-from-last dotted field).
import glob as _glob
import gzip as _gzip
import os as _os
import struct as _struct

_CRC_TABLE = None


def _crc32c(data):
    global _CRC_TABLE
    if _CRC_TABLE is None:
        tbl = []
        for i in range(256):
            c = i
            for _ in range(8):
                c = (c >> 1) ^ 0x82F63B78 if c & 1 else c >> 1
            tbl.append(c)
        _CRC_TABLE = tbl
    crc = 0xFFFFFFFF
    for b in data:
        crc = _CRC_TABLE[(crc ^ b) & 0xFF] ^ (crc >> 8)
    return crc ^ 0xFFFFFFFF


def _masked_crc(data):
    crc = _crc32c(data)
    return ((((crc >> 15) | (crc << 17)) & 0xFFFFFFFF) + 0xA282EAD8) & 0xFFFFFFFF


def _varint(n):
    out = bytearray()
    while True:
        b = n & 0x7F
        n >>= 7
        out.append(b | (0x80 if n else 0))
        if not n:
            return bytes(out)


def _read_varint(buf, i):
    shift = val = 0
    while True:
        b = buf[i]
        i += 1
        val |= (b & 0x7F) << shift
        if not b & 0x80:
            return val, i
        shift += 7


def _len_field(tag, payload):
    return bytes([(tag << 3) | 2]) + _varint(len(payload)) + payload


def encode_example(seq_bytes, key=b'seq'):
    """tf.train.Example{features{feature{'seq': bytes_list{value: [seq_bytes]}}}} (data.py:10-12)"""
    bytes_list = _len_field(1, seq_bytes)
    feature = _len_field(1, bytes_list)
    entry = _len_field(1, key) + _len_field(2, feature)
    features = _len_field(1, entry)
    return _len_field(1, features)


def _fields(buf):
    i = 0
    while i < len(buf):
        tag, i = _read_varint(buf, i)
        wt = tag & 7
        if wt == 2:
            ln, i = _read_varint(buf, i)
            yield tag >> 3, buf[i:i + ln]
            i += ln
        elif wt == 0:
            _, i = _read_varint(buf, i)
        elif wt == 1:
            i += 8
        elif wt == 5:
            i += 4
        else:
            raise ValueError('unsupported protobuf wire type')


def decode_example(buf, key=b'seq'):
    for f1, features in _fields(buf):
        if f1 != 1:
            continue
        for f2, entry in _fields(features):
            k = v = None
            for f3, val in _fields(entry):
                if f3 == 1:
                    k = bytes(val)
                elif f3 == 2:
                    v = val
            if k == key and v is not None:
                for f4, bl in _fields(v):
                    if f4 == 1:                          # bytes_list
                        for f5, item in _fields(bl):
                            if f5 == 1:
                                return bytes(item)
    raise ValueError("no bytes feature 'seq' in record")


def write_tfrecords(path, seqs):
    """GZIP TFRecord writer (data.py:17-21)"""
    with _gzip.open(path, 'wb') as f:
        for s in seqs:
            rec = encode_example(s if isinstance(s, bytes) else s.encode())
            ln = _struct.pack('<Q', len(rec))
            f.write(ln + _struct.pack('<I', _masked_crc(ln)) + rec + _struct.pack('<I', _masked_crc(rec)))


def read_tfrecords(path, check_crc=True):
    with _gzip.open(path, 'rb') as f:
        while True:
            head = f.read(12)
            if len(head) < 12:
                return
            ln, = _struct.unpack('<Q', head[:8])
            if check_crc and _struct.unpack('<I', head[8:])[0] != _masked_crc(head[:8]):
                raise ValueError(f'{path}: corrupt record length')
            rec = f.read(ln)
            crc, = _struct.unpack('<I', f.read(4))
            if check_crc and crc != _masked_crc(rec):
                raise ValueError(f'{path}: corrupt record payload')
            yield decode_example(rec)


def iterator_from_tfrecords_folder(folder, data_type='train'):
    """Same contract as the reference (data.py:37-72): returns (num_seqs, iter_fn(seq_len, batch_size, skip, loop)) whose
    batches are uint16 (B, seq_len + 1) with a BOS 0 in front and tokens = byte + 1."""
    if str(folder).startswith('gs://'):
        raise NotImplementedError('GCS is out of scope (no network)')
    filenames = sorted(_glob.glob(_os.path.join(str(folder), '**', f'*.{data_type}.tfrecord.gz'), recursive=True))
    num_seqs = sum(int(_os.path.basename(t).split('.')[-4]) for t in filenames)

    def iter_fn(seq_len, batch_size, skip=0, loop=False):
        while True:
            batch, seen = [], 0
            for fn in filenames:
                for s in read_tfrecords(fn):
                    seen += 1
                    if seen <= skip:
                        continue
                    batch.append(s)
                    if len(batch) == batch_size:
                        yield collate(batch, seq_len)
                        batch = []
            if batch:
                yield collate(batch, seq_len)
            if not loop:
                return
            skip = 0

    return num_seqs, iter_fn
