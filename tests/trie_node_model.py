"""A CPU statement of the trie nodes served by path (phant_gpu_resident_state_trie_nodes, snap's GetTrieNodes), written from
the definition in include/phant_gpu.h: a plain recursive build of a secure trie that records the node starting at each
nibble path.  served() keeps the root and every node of 32 bytes or more (the nodes a parent references by hash); every
other path has no node.  Written independently of helpers.py::py_mptize, which the CPU tests use only as a cross-check."""
def _rlp_bytes(b):
    b = bytes(b)
    if len(b) == 1 and b[0] < 0x80:
        return b
    return _header(len(b), 0x80) + b


def _rlp_list(encoded):
    body = b"".join(encoded)
    return _header(len(body), 0xc0) + body


def _header(n, base):
    if n <= 55:
        return bytes([base + n])
    ll = (n.bit_length() + 7) // 8
    return bytes([base + 55 + ll]) + n.to_bytes(ll, "big")


def nibbles(key):
    return tuple(x for byte in key for x in (byte >> 4, byte & 15))


def _hex_prefix(nib, leaf):
    flag = (2 if leaf else 0) + (len(nib) & 1)
    if len(nib) & 1:
        head, rest = bytes([flag << 4 | nib[0]]), nib[1:]
    else:
        head, rest = bytes([flag << 4]), nib
    return head + bytes(rest[i] << 4 | rest[i + 1] for i in range(0, len(rest), 2))


def trie_nodes(keccak, kv):
    """kv: {32-byte key: stored value bytes}.  Returns (root, {nibble path (tuple): node RLP}) for EVERY node of the trie,
    embedded ones included; the empty trie has no node and the root keccak(0x80)."""
    items = sorted((nibbles(k), bytes(v)) for k, v in kv.items())
    nodes = {}

    def ref(enc):
        return enc if len(enc) < 32 else _rlp_bytes(keccak(enc))

    def build(its, depth):
        path = its[0][0][:depth]
        if len(its) == 1:
            enc = _rlp_list([_rlp_bytes(_hex_prefix(its[0][0][depth:], True)), _rlp_bytes(its[0][1])])
        else:
            common = 0
            while all(n[depth + common] == its[0][0][depth + common] for n, _ in its):
                common += 1
            if common:
                child = build(its, depth + common)
                enc = _rlp_list([_rlp_bytes(_hex_prefix(its[0][0][depth:depth + common], False)), ref(child)])
            else:
                kids = [b"\x80"] * 16
                for c in range(16):
                    group = [x for x in its if x[0][depth] == c]
                    if group:
                        kids[c] = ref(build(group, depth + 1))
                enc = _rlp_list(kids + [b"\x80"])
        nodes[path] = enc
        return enc

    if not items:
        return keccak(b"\x80"), {}
    return keccak(build(items, 0)), nodes


def served(nodes):
    """the nodes a GetTrieNodes server returns: the root and every node of 32 bytes or more"""
    return {p: e for p, e in nodes.items() if p == () or len(e) >= 32}


def storage_value(v32):
    """a slot's stored value: rlp of the value without leading zero bytes"""
    return _rlp_bytes(bytes(v32).lstrip(b"\x00"))


def state_nodes(keccak, m):
    """{(trie, nibble path): node RLP} served from the state of model m (resident_state_model.StateModel): trie None is the
    account trie, an account key its storage trie"""
    _, acc = trie_nodes(keccak, {k: m.leaf(k) for k in m.acc})
    out = {(None, p): e for p, e in served(acc).items()}
    for k, a in m.acc.items():
        if a.storage:
            _, st = trie_nodes(keccak, {sk: storage_value(v) for sk, v in a.storage.items()})
            out.update(((k, p), e) for p, e in served(st).items())
    return out


def pack(path):
    """a nibble path -> (32 bytes, high nibble first, zero padded; its length)"""
    nib = list(path) + [0] * (64 - len(path))
    return bytes(nib[i] << 4 | nib[i + 1] for i in range(0, 64, 2)), len(path)


def probe_paths(keys, rng=None, diverge=True):
    """paths around a set of keys: every prefix of every key (lengths 0..64) and, per key, a path that follows it for d
    nibbles and then differs, for every d < 64"""
    out = set()
    for k in keys:
        n = nibbles(k)
        out.update(n[:d] for d in range(65))
        if diverge:
            out.update(n[:d] + ((n[d] + 1 + (0 if rng is None else int(rng.integers(0, 15)))) % 16,) for d in range(64))
    return sorted(out)

