"""What the code store beside the resident world state holds (phant_gpu_resident_state_put_codes / _codes / _prune_codes),
stated on the Python model: codes by keccak(code), the empty code never stored, and a prune that keeps exactly the codes
some account names at a root the journal reaches.  The reachable roots are the states themselves here (the model's history),
not the undo records the device walks, so that the two statements can be held against each other."""
EMPTY_CODE_HASH = bytes.fromhex("c5d2460186f7233c927e7db2dcc703c0e500b653ca82273b7bfad8045d85a470")  # keccak("")


class CodeStore:
    def __init__(self, keccak):
        self.keccak = keccak
        self.held = {}  # hash -> code

    def put(self, codes):
        """returns the hashes in order"""
        out = []
        for c in codes:
            h = self.keccak(bytes(c))
            if c:
                self.held.setdefault(h, bytes(c))
            out.append(h)
        return out

    def lookup(self, h):
        """(held, code): keccak("") is always held, with b"" """
        if h == EMPTY_CODE_HASH:
            return True, b""
        return (True, self.held[h]) if h in self.held else (False, b"")

    @staticmethod
    def named(states):
        """every codeHash an account has in any of the states (StateModel)"""
        return {a.code_hash for m in states for a in m.acc.values()}

    def prune(self, states):
        """keep the held codes some account names in one of `states`: the current state and every state the journal reaches"""
        keep = self.named(states)
        self.held = {h: c for h, c in self.held.items() if h in keep}
