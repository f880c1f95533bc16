// range_proof_test.cpp -- a snap client's range-proof checks in C++ (phant_host.hpp: snap::verifyAccountRange /
// verifyStorageRanges) on answers served by ResidentStateTrie::accountRangeProof / storageRangeProof.  Reads the cases of
// resident_state_witness_test.cpp (written by tests/test_gpu_host_cpp_range_proofs.py from the fixture states):
//   case <pre state root hex> <post state root hex>
//   pre | acct <address hex> <nonce> <balance hex, 32 bytes> <code hex or -> | pslot | slot <address hex> <slot hex> <value hex>
//   del <address hex> | end
// Per case the pre-state is loaded and the block applied.  Every account range is served in chunks of 2 from the first key
// and from just after it, and every account's storage in chunks of 2: each answer is accepted with the range's `more`, and
// rejected against the pre-state's root (or the account's storage root before the block) when that root differs.  The
// accounts' whole storage tries go in one GetStorageRanges-shaped call with one proven partial range last, and a changed value
// in an answer is rejected.  Prints "ALL OK".
#include "phant_host.hpp"

#include <cstdio>
#include <fstream>
#include <iostream>
#include <sstream>

using namespace phant;
using Trie = state::ResidentStateTrie;

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
static Hash32 after(Hash32 k)
{
    for (int i = 31; i >= 0 && ++k[i] == 0; --i) {}
    return k;
}

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

// every account range of the current state from `origin`, chunk by chunk: accepted with `more`, rejected against `old_root`
static bool accounts_check(Gpu& g, Trie& st, Hash32 origin, const Hash32& root, const Hash32& old_root, size_t& answers)
{
    Hash32 all;
    all.fill(0xff);
    for (;;) {
        const Trie::AccountRangeProof p = st.accountRangeProof(origin, all, 2);
        if (snap::verifyAccountRange(g, root, origin, p.range.accounts, p.proof) != std::make_pair(true, p.range.more)) return false;
        if (old_root != root && snap::verifyAccountRange(g, old_root, origin, p.range.accounts, p.proof).first) return false;
        if (p.range.accounts.size() >= 1) {
            auto bad = p.range.accounts;
            bad[0].nonce ^= 1;
            if (snap::verifyAccountRange(g, root, origin, bad, p.proof).first) return false;
        }
        ++answers;
        if (!p.range.more) return true;
        origin = after(p.range.accounts.back().key);
    }
}

static int run(Gpu& g, Case& c, int n, size_t& answers)
{
    Trie st(g);
    std::map<Address, const state::AccountState*> load;
    for (const auto& [a, s] : c.pre) load[a] = &s;
    if (!load.empty() && st.apply(load) != c.pre_root) { std::cout << "case " << n << ": pre root mismatch\n"; return 1; }
    Hash32 zero{}, all;
    all.fill(0xff);
    const auto before = st.accountRange(zero, all, (uint32_t)c.pre.size() + 1);
    if (st.apply(c.touched(), c.slots) != c.post) { std::cout << "case " << n << ": apply root mismatch\n"; return 1; }
    const auto now = st.accountRange(zero, all, (uint32_t)(c.pre.size() + c.live.size()) + 1);
    if (!accounts_check(g, st, zero, c.post, c.pre_root, answers) ||
        (!now.accounts.empty() && !accounts_check(g, st, after(now.accounts[0].key), c.post, c.pre_root, answers))) {
        std::cout << "case " << n << ": an account range answer was not judged right\n";
        return 1;
    }
    std::map<Hash32, Hash32> old_sroot;
    for (const auto& e : before.accounts) old_sroot[e.key] = e.storageHash;
    std::map<Hash32, Address> addr_of;
    for (const auto* m : {&c.pre, &c.live})
        for (const auto& [a, s] : *m) addr_of[hash(g, Bytes(a.begin(), a.end()))] = a;
    std::vector<snap::StorageRangeAnswer> whole;
    for (const auto& e : now.accounts) {
        const Address& a = addr_of.at(e.key);
        Hash32 origin{};
        std::vector<std::pair<Hash32, std::array<uint8_t, 32>>> got;
        for (;;) {
            const Trie::SlotRangeProof p = st.storageRangeProof(a, origin, all, 2);
            const snap::StorageRangeAnswer ans{e.storageHash, origin, p.range.slots};
            const bool partial = origin != zero || p.range.more;
            if (snap::verifyStorageRanges(g, {ans}, p.proof, partial) != std::vector<std::pair<bool, bool>>{{true, p.range.more}}) {
                std::cout << "case " << n << ": a storage range answer was rejected\n";
                return 1;
            }
            const auto it = old_sroot.find(e.key);
            const Hash32 old = it == old_sroot.end() ? Hash32{} : it->second;
            if (old != e.storageHash && snap::verifyStorageRanges(g, {{old, origin, p.range.slots}}, p.proof, partial)[0].first) {
                std::cout << "case " << n << ": a storage range answer was accepted against the old storage root\n";
                return 1;
            }
            ++answers;
            got.insert(got.end(), p.range.slots.begin(), p.range.slots.end());
            if (!p.range.more) break;
            origin = after(p.range.slots.back().first);
        }
        whole.push_back({e.storageHash, zero, got});
    }
    // GetStorageRanges: every storage trie whole, then the first slots of the account with the most, proven
    size_t big = 0;
    for (size_t i = 0; i < whole.size(); ++i)
        if (whole[i].slots.size() > whole[big].slots.size()) big = i;
    if (!whole.empty() && whole[big].slots.size() >= 2) {
        const Trie::SlotRangeProof p = st.storageRangeProof(addr_of.at(now.accounts[big].key), zero, all, 1);
        std::vector<snap::StorageRangeAnswer> req = whole;
        req.push_back({whole[big].storageRoot, zero, p.range.slots});
        const auto r = snap::verifyStorageRanges(g, req, p.proof, true);
        bool ok = r.back() == std::make_pair(true, true);
        for (size_t i = 0; i + 1 < r.size(); ++i) ok &= r[i] == std::make_pair(true, false);
        req[big].slots.back().second[31] ^= 1;
        ok &= !snap::verifyStorageRanges(g, req, p.proof, true)[big].first;
        if (!ok) { std::cout << "case " << n << ": a GetStorageRanges answer was not judged right\n"; return 1; }
        ++answers;
    }
    return 0;
}

int main(int argc, char** argv)
{
    if (argc != 2) { std::cerr << "usage: range_proof_test CASES\n"; return 2; }
    std::ifstream f(argv[1]);
    Gpu g(0);
    std::string line;
    Case c;
    int n = 0, bad = 0;
    size_t answers = 0;
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
        else if (kind == "end") { bad += run(g, c, n, answers); ++n; }
    }
    if (n == 0 || bad) { std::cout << bad << " of " << n << " cases failed\n"; return 1; }
    std::cout << n << " cases, " << answers << " answers\nALL OK\n";
    return 0;
}
