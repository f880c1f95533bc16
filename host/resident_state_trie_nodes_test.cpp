// resident_state_trie_nodes_test.cpp -- snap's GetTrieNodes from the resident world state in C++ (phant_host.hpp:
// ResidentStateTrie::getTrieNodes), driven as a healing peer drives it.  Reads the cases of resident_state_witness_test.cpp
// (written by tests/test_gpu_host_cpp_resident_state_trie_nodes.py from the fixture states) and uses their pre-states only:
//   case <pre state root hex> <post state root hex>
//   pre <address hex> <nonce> <balance hex, 32 bytes> <code hex or -> | pslot <address hex> <slot hex, 32 bytes> <value hex>
//   end (other lines are ignored)
// Per case: the pre-state is loaded and healed from its root with wire-format pathsets (compact paths; the storage paths of
// one account in one set led by its hash), level by level: every blob must hash to the reference its parent holds, and
// every child referenced by hash, and every account's storage root, is asked for next.  phant_gpu_verify_witness over the
// healed node set must then prove every account under the root and every slot under its account's storage root, present.
// A maxBytes below the answer's size must cut it after the blob that crosses it.  Prints "ALL OK".
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

struct Case {
    Hash32 pre_root{};
    std::map<Address, state::AccountState> pre;
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

struct Want { // a node to fetch: its trie (empty owner: the account trie), nibble path and the reference its parent holds
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
// the node `n` (inside blob b, as item l) at w's path: push what a healer asks for below it; an account leaf's storage root
// into sroots
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
    static const Hash32 empty = {0x56, 0xe8, 0x1f, 0x17, 0x1b, 0xcc, 0x55, 0xa6, 0xff, 0x83, 0x45, 0xe6, 0x92, 0xc0, 0xf8, 0x6e,
                                 0x5b, 0x48, 0xe0, 0x1b, 0x99, 0x6c, 0xad, 0xc0, 0x01, 0x62, 0x2f, 0xb5, 0xe3, 0x63, 0xb4, 0x21};
    if (root != empty) next.push_back({true, key, {}, root});
}

static int run(Gpu& g, const Case& c, int n)
{
    state::ResidentStateTrie st(g);
    std::map<Address, const state::AccountState*> load;
    for (const auto& [a, s] : c.pre) load[a] = &s;
    if (!load.empty() && st.apply(load) != c.pre_root) { std::cout << "case " << n << ": pre root mismatch\n"; return 1; }
    const Hash32 root = st.root();
    std::set<Bytes> healed;
    std::map<Hash32, Hash32> sroots;
    std::vector<Bytes> account_paths;
    std::vector<Want> frontier;
    if (!c.pre.empty()) frontier.push_back({false, {}, {}, root});
    while (!frontier.empty()) {
        std::vector<state::ResidentStateTrie::PathSet> sets;
        std::vector<Want> order;
        std::map<Hash32, std::vector<const Want*>> by;
        for (const Want& w : frontier) {
            if (w.storage) { by[w.owner].push_back(&w); continue; }
            sets.push_back({compact(w.path)});
            account_paths.push_back(compact(w.path));
            order.push_back(w);
        }
        for (const auto& [o, ws] : by) {
            sets.push_back({Bytes(o.begin(), o.end())});
            for (const Want* w : ws) { sets.back().push_back(compact(w->path)); order.push_back(*w); }
        }
        const std::vector<Bytes> blobs = st.getTrieNodes(sets, 1ull << 40);
        if (blobs.size() != order.size()) { std::cout << "case " << n << ": " << blobs.size() << " blobs for " << order.size() << " paths\n"; return 1; }
        std::vector<Want> next;
        for (size_t i = 0; i < blobs.size(); ++i) {
            if (blobs[i].empty() || hash(g, blobs[i]) != order[i].ref) { std::cout << "case " << n << ": a blob does not hash to its reference\n"; return 1; }
            healed.insert(blobs[i]);
            children(blobs[i], item(blobs[i], 0), order[i], next, sroots);
        }
        frontier = std::move(next);
    }
    if (st.root() != root) { std::cout << "case " << n << ": getTrieNodes changed the state\n"; return 1; }
    // every account and slot proven present from the healed set
    Bytes nodes, keys, roots;
    std::vector<uint64_t> off{0};
    for (const Bytes& x : healed) { nodes.insert(nodes.end(), x.begin(), x.end()); off.push_back(nodes.size()); }
    nodes.resize(nodes.size() + 64);
    for (const auto& [a, s] : c.pre) {
        const Hash32 ak = hash(g, Bytes(a.begin(), a.end()));
        keys.insert(keys.end(), ak.begin(), ak.end());
        roots.insert(roots.end(), root.begin(), root.end());
        for (const auto& kv : s.storage) {
            if (kv.second == std::array<uint8_t, 32>{}) continue;
            const Hash32 sk = hash(g, Bytes(kv.first.begin(), kv.first.end()));
            const Hash32 sr = sroots[ak];
            keys.insert(keys.end(), sk.begin(), sk.end());
            roots.insert(roots.end(), sr.begin(), sr.end());
        }
    }
    const uint64_t nk = keys.size() / 32;
    if (nk) {
        std::vector<uint8_t> status(nk);
        std::vector<uint64_t> bitmap((nk + 63) / 64);
        const phant_gpu_witness w{off.size() - 1, nodes.data(), off.data(), off.back(), nk, keys.data(), roots.data(), nk};
        g.check(phant_gpu_verify_witness(g.ctx(), &w, bitmap.data(), status.data(), nullptr, nullptr), "verify_witness");
        for (uint8_t s : status)
            if (s != 1) { std::cout << "case " << n << ": the healed set does not prove every account and slot\n"; return 1; }
    }
    // a response cut by maxBytes: the blobs up to and including the one that crosses it
    if (account_paths.size() > 1) {
        std::vector<state::ResidentStateTrie::PathSet> sets;
        for (const Bytes& p : account_paths) sets.push_back({p});
        const std::vector<Bytes> full = st.getTrieNodes(sets, 1ull << 40);
        const uint64_t cut = full[0].size() + 1;
        const std::vector<Bytes> part = st.getTrieNodes(sets, cut);
        uint64_t total = 0;
        size_t k = 0;
        while (k < full.size() && total <= cut) total += full[k++].size();
        if (part.size() != k || !std::equal(part.begin(), part.end(), full.begin())) { std::cout << "case " << n << ": maxBytes does not cut\n"; return 1; }
    }
    return 0;
}

int main(int argc, char** argv)
{
    if (argc != 2) { std::cerr << "usage: resident_state_trie_nodes_test CASES\n"; return 2; }
    std::ifstream f(argv[1]);
    Gpu g(0);
    std::string line;
    Case c;
    int n = 0, bad = 0;
    while (std::getline(f, line)) {
        std::istringstream ls(line);
        std::string kind, a, b, x, y;
        ls >> kind >> a >> b >> x >> y;
        if (kind == "case") { c = Case{}; c.pre_root = fixed<32>(a); }
        else if (kind == "pre") {
            state::AccountState s;
            s.nonce = std::stoull(b);
            s.balance = fixed<32>(x);
            if (y != "-") s.code = unhex(y);
            c.pre[fixed<20>(a)] = s;
        } else if (kind == "pslot") c.pre[fixed<20>(a)].storage[fixed<32>(b)] = fixed<32>(x);
        else if (kind == "end") { bad += run(g, c, n); ++n; }
    }
    if (n == 0 || bad) { std::cout << bad << " of " << n << " cases failed\n"; return 1; }
    std::cout << n << " cases\nALL OK\n";
    return 0;
}
