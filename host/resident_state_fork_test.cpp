// resident_state_fork_test.cpp -- forks of the resident world state in C++ (phant_host.hpp: ResidentStateTrie::fork), used to
// serve eth_getProof and snap's GetTrieNodes at the root before the last block while the state itself stays at the head.
// Reads the cases of resident_state_witness_test.cpp (written by tests/test_gpu_host_cpp_resident_state_fork.py from the
// fixture states):
//   case <pre state root hex> <post state root hex>
//   pre <address hex> <nonce> <balance hex, 32 bytes> <code hex or -> | pslot <address hex> <slot hex, 32 bytes> <value hex>
//   acct <address hex> <nonce> <balance hex, 32 bytes> <code hex or -> | del <address hex>
//   slot <address hex> <slot number hex, 32 bytes> <new value hex, 32 bytes>
//   end
// Per case: the pre-state is loaded with a journal of one block and the block applied (the post root); fork(1) must have the
// pre root while the state keeps the post root.  From the fork:
//   - getProofs of every pre-state account and slot, and of every account the block creates: phant_gpu_verify_witness over
//     the proofs' nodes must prove each pre-state account (its nonce and balance as getProofs returned them) and slot present
//     under the pre root, and each created account absent;
//   - getTrieNodes, healing the pre-state from its root level by level with wire-format pathsets: every blob hashes to the
//     reference its parent holds, and phant_gpu_verify_witness over the healed set proves every pre-state account and slot.
// Prints "ALL OK".
#include "phant_host.hpp"

#include <cstdio>
#include <fstream>
#include <iostream>
#include <sstream>

using namespace phant;

static Bytes unhex(const std::string& s)
{
    Bytes b(s.size() / 2);
    for (size_t i = 0; i < b.size(); ++i) b[i] = (uint8_t)std::stoi(s.substr(2 * i, 2), nullptr, 16);
    return b;
}
template <size_t N> static std::array<uint8_t, N> fixed(const std::string& s)
{
    const Bytes b = unhex(s);
    if (b.size() != N) throw std::invalid_argument("bad length: " + s);
    std::array<uint8_t, N> a;
    std::copy(b.begin(), b.end(), a.begin());
    return a;
}
static Hash32 hash(Gpu& g, const Bytes& b) { return hasher::keccak256_batch(g, {b})[0]; }
static const Hash32 kEmpty = {0x56, 0xe8, 0x1f, 0x17, 0x1b, 0xcc, 0x55, 0xa6, 0xff, 0x83, 0x45, 0xe6, 0x92, 0xc0, 0xf8, 0x6e,
                              0x5b, 0x48, 0xe0, 0x1b, 0x99, 0x6c, 0xad, 0xc0, 0x01, 0x62, 0x2f, 0xb5, 0xe3, 0x63, 0xb4, 0x21};

struct Case {
    Hash32 pre_root{}, post{};
    std::map<Address, state::AccountState> pre, live;
    std::set<Address> gone;
    state::HashedDiff::SlotChanges slots;
    std::map<Address, const state::AccountState*> touched() const
    {
        std::map<Address, const state::AccountState*> t;
        for (const auto& [a, s] : live) t[a] = &s;
        for (const Address& a : gone) t[a] = nullptr;
        return t;
    }
};

// ---- the minimum of RLP a healer needs to find a node's children ----
struct Item {
    bool list;
    size_t pay, len, end; // payload offset and length, the item's end
};
static Item item(const Bytes& b, size_t pos)
{
    const uint8_t x = b.at(pos);
    if (x < 0x80) return {false, pos, 1, pos + 1};
    const bool list = x >= 0xc0;
    const size_t s = x - (list ? 0xc0 : 0x80);
    if (s <= 55) return {list, pos + 1, s, pos + 1 + s};
    size_t n = 0;
    for (size_t i = 0; i < s - 55; ++i) n = n << 8 | b.at(pos + 1 + i);
    return {list, pos + 1 + (s - 55), n, pos + 1 + (s - 55) + n};
}
static std::vector<Item> items(const Bytes& b, const Item& l)
{
    std::vector<Item> v;
    for (size_t p = l.pay; p < l.pay + l.len; p = v.back().end) v.push_back(item(b, p));
    return v;
}
struct Want { // a node to fetch: its trie (storage: the trie of account `owner`), nibble path and the reference its parent holds
    bool storage;
    Hash32 owner;
    std::vector<uint8_t> path;
    Hash32 ref;
};
static Bytes compact(const std::vector<uint8_t>& nib)
{
    const bool odd = nib.size() & 1;
    Bytes c{(uint8_t)(odd ? 0x10 | nib[0] : 0)};
    for (size_t i = odd ? 1 : 0; i < nib.size(); i += 2) c.push_back((uint8_t)(nib[i] << 4 | nib[i + 1]));
    return c;
}
static Hash32 key_of(const std::vector<uint8_t>& nib)
{
    Hash32 k{};
    for (size_t i = 0; i < 64; ++i) k[i / 2] |= (uint8_t)(i & 1 ? nib[i] : nib[i] << 4);
    return k;
}
// below node l of blob b at w's path: what a healer asks for next; an account leaf's storage root into sroots
static void children(const Bytes& b, const Item& l, const Want& w, std::vector<Want>& next, std::map<Hash32, Hash32>& sroots)
{
    const std::vector<Item> it = items(b, l);
    auto child = [&](const Item& c, std::vector<uint8_t> path) {
        Want x{w.storage, w.owner, std::move(path), {}};
        if (c.list) return children(b, c, x, next, sroots); // embedded: walked in place
        if (c.len != 32) return;
        std::copy(b.begin() + c.pay, b.begin() + c.pay + 32, x.ref.begin());
        next.push_back(x);
    };
    if (it.size() == 17) {
        for (uint8_t i = 0; i < 16; ++i) {
            std::vector<uint8_t> p = w.path;
            p.push_back(i);
            child(it[i], p);
        }
        return;
    }
    std::vector<uint8_t> p = w.path;
    const uint8_t flag = b[it[0].pay] >> 4;
    for (size_t q = (flag & 1) ? 1 : 2; q < 2 * it[0].len; ++q) p.push_back(q & 1 ? b[it[0].pay + q / 2] & 15 : b[it[0].pay + q / 2] >> 4);
    if (flag < 2) return child(it[1], p);
    if (w.storage) return;
    const Item acct = item(b, it[1].pay); // the account: rlp([nonce, balance, storageRoot, codeHash])
    const Item sr = items(b, acct)[2];
    Hash32 root;
    std::copy(b.begin() + sr.pay, b.begin() + sr.pay + 32, root.begin());
    const Hash32 key = key_of(p);
    sroots[key] = root;
    if (root != kEmpty) next.push_back({true, key, {}, root});
}

// W over a node set: the status of each key under its root
static std::vector<uint8_t> prove_with_w(Gpu& g, const std::set<Bytes>& set, const Bytes& keys, const Bytes& roots)
{
    const uint64_t nk = keys.size() / 32;
    std::vector<uint8_t> status(nk);
    if (!nk) return status;
    Bytes nodes;
    std::vector<uint64_t> off{0};
    for (const Bytes& x : set) { nodes.insert(nodes.end(), x.begin(), x.end()); off.push_back(nodes.size()); }
    nodes.resize(nodes.size() + 64);
    std::vector<uint64_t> bitmap((nk + 63) / 64);
    const phant_gpu_witness w{off.size() - 1, nodes.data(), off.data(), off.back(), nk, keys.data(), roots.data(), nk};
    g.check(phant_gpu_verify_witness(g.ctx(), &w, bitmap.data(), status.data(), nullptr, nullptr), "verify_witness");
    return status;
}

static int run(Gpu& g, Case& c, int n)
{
    state::ResidentStateTrie st(g);
    std::map<Address, const state::AccountState*> load;
    for (const auto& [a, s] : c.pre) load[a] = &s;
    if (!load.empty() && st.apply(load) != c.pre_root) { std::cout << "case " << n << ": pre root mismatch\n"; return 1; }
    st.setJournal(1);
    if (st.apply(c.touched(), c.slots) != c.post) { std::cout << "case " << n << ": post root mismatch\n"; return 1; }
    std::unique_ptr<state::ResidentStateTrie> f = st.fork(1);
    if (f->root() != c.pre_root || st.root() != c.post) { std::cout << "case " << n << ": fork(1) is not at the pre root\n"; return 1; }

    // ---- eth_getProof at the pre root, from the fork ----
    state::ResidentStateTrie::ProofRequests req;
    for (const auto& [a, s] : c.pre)
        for (const auto& kv : s.storage)
            if (kv.second != std::array<uint8_t, 32>{}) req[a].push_back(kv.first);
    for (const auto& [a, s] : c.pre) req[a];
    for (const auto& [a, s] : c.live) req[a]; // accounts the block creates are absent at the pre root
    const auto proofs = f->getProofs(req);
    std::set<Bytes> pset;
    Bytes keys, roots;
    std::vector<uint8_t> want;
    for (const auto& [a, p] : proofs) {
        const auto pre = c.pre.find(a);
        if (pre != c.pre.end() && (p.nonce != pre->second.nonce || p.balance != pre->second.balance)) {
            std::cout << "case " << n << ": getProofs' account fields are not the pre-state's\n";
            return 1;
        }
        pset.insert(p.accountProof.begin(), p.accountProof.end());
        const Hash32 ak = hash(g, Bytes(a.begin(), a.end()));
        keys.insert(keys.end(), ak.begin(), ak.end());
        roots.insert(roots.end(), c.pre_root.begin(), c.pre_root.end());
        want.push_back(pre != c.pre.end() ? 1 : 2);
        for (const auto& sp : p.storageProof) {
            if (pre == c.pre.end() || sp.value != pre->second.storage.at(sp.key)) {
                std::cout << "case " << n << ": getProofs' slot value is not the pre-state's\n";
                return 1;
            }
            pset.insert(sp.proof.begin(), sp.proof.end());
            const Hash32 sk = hash(g, Bytes(sp.key.begin(), sp.key.end()));
            keys.insert(keys.end(), sk.begin(), sk.end());
            roots.insert(roots.end(), p.storageHash.begin(), p.storageHash.end());
            want.push_back(1);
        }
    }
    if (c.pre.empty()) { // the empty trie: every account is absent with an empty proof
        if (!pset.empty()) { std::cout << "case " << n << ": a proof under the empty root holds a node\n"; return 1; }
    } else if (prove_with_w(g, pset, keys, roots) != want) { std::cout << "case " << n << ": W does not accept the fork's proofs\n"; return 1; }

    // ---- GetTrieNodes at the pre root, from the fork: a heal, then W over the healed set ----
    std::set<Bytes> healed;
    std::map<Hash32, Hash32> sroots;
    std::vector<Want> frontier;
    if (!c.pre.empty()) frontier.push_back({false, {}, {}, c.pre_root});
    while (!frontier.empty()) {
        std::vector<state::ResidentStateTrie::PathSet> sets;
        std::vector<Want> order;
        std::map<Hash32, std::vector<const Want*>> by;
        for (const Want& w : frontier) {
            if (w.storage) { by[w.owner].push_back(&w); continue; }
            sets.push_back({compact(w.path)});
            order.push_back(w);
        }
        for (const auto& [o, ws] : by) {
            sets.push_back({Bytes(o.begin(), o.end())});
            for (const Want* w : ws) { sets.back().push_back(compact(w->path)); order.push_back(*w); }
        }
        const std::vector<Bytes> blobs = f->getTrieNodes(sets, 1ull << 40);
        if (blobs.size() != order.size()) { std::cout << "case " << n << ": " << blobs.size() << " blobs for " << order.size() << " paths\n"; return 1; }
        std::vector<Want> next;
        for (size_t i = 0; i < blobs.size(); ++i) {
            if (blobs[i].empty() || hash(g, blobs[i]) != order[i].ref) { std::cout << "case " << n << ": a blob does not hash to its reference\n"; return 1; }
            healed.insert(blobs[i]);
            children(blobs[i], item(blobs[i], 0), order[i], next, sroots);
        }
        frontier = std::move(next);
    }
    keys.clear();
    roots.clear();
    for (const auto& [a, s] : c.pre) {
        const Hash32 ak = hash(g, Bytes(a.begin(), a.end()));
        keys.insert(keys.end(), ak.begin(), ak.end());
        roots.insert(roots.end(), c.pre_root.begin(), c.pre_root.end());
        for (const auto& kv : s.storage) {
            if (kv.second == std::array<uint8_t, 32>{}) continue;
            const Hash32 sk = hash(g, Bytes(kv.first.begin(), kv.first.end()));
            const Hash32 sr = sroots[ak];
            keys.insert(keys.end(), sk.begin(), sk.end());
            roots.insert(roots.end(), sr.begin(), sr.end());
        }
    }
    for (uint8_t s : prove_with_w(g, healed, keys, roots))
        if (s != 1) { std::cout << "case " << n << ": the healed set does not prove every account and slot\n"; return 1; }
    if (st.root() != c.post || f->root() != c.pre_root) { std::cout << "case " << n << ": serving changed a root\n"; return 1; }
    return 0;
}

int main(int argc, char** argv)
{
    if (argc != 2) { std::cerr << "usage: resident_state_fork_test CASES\n"; return 2; }
    std::ifstream f(argv[1]);
    Gpu g(0);
    std::string line;
    Case c;
    int n = 0, bad = 0;
    while (std::getline(f, line)) {
        std::istringstream ls(line);
        std::string kind, a, b, x, y;
        ls >> kind >> a >> b >> x >> y;
        if (kind == "case") { c = Case{}; c.pre_root = fixed<32>(a); c.post = fixed<32>(b); }
        else if (kind == "pre" || kind == "acct") {
            state::AccountState s;
            s.nonce = std::stoull(b);
            s.balance = fixed<32>(x);
            if (y != "-") s.code = unhex(y);
            (kind == "pre" ? c.pre : c.live)[fixed<20>(a)] = s;
        } else if (kind == "pslot") c.pre[fixed<20>(a)].storage[fixed<32>(b)] = fixed<32>(x);
        else if (kind == "del") c.gone.insert(fixed<20>(a));
        else if (kind == "slot") c.slots[fixed<20>(a)][fixed<32>(b)] = fixed<32>(x);
        else if (kind == "end") { bad += run(g, c, n); ++n; }
    }
    if (n == 0 || bad) { std::cout << bad << " of " << n << " cases failed\n"; return 1; }
    std::cout << n << " cases\nALL OK\n";
    return 0;
}
