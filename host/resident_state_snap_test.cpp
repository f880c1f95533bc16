// resident_state_snap_test.cpp -- snap GetAccountRange / GetStorageRanges answers from the resident world state in C++
// (phant_host.hpp: ResidentStateTrie::snapAccountRange / snapStorageRanges), driven as a syncing peer drives them and checked
// as it checks them (snap::verifySnapAccountRange / verifySnapStorageRanges, G).  Reads the cases of
// resident_state_witness_test.cpp (written by tests/test_gpu_host_cpp_resident_state_snap.py from the fixture states) and
// uses their pre-states only:
//   case <pre state root hex> <post state root hex>
//   pre <address hex> <nonce> <balance hex, 32 bytes> <code hex or -> | pslot <address hex> <slot hex, 32 bytes> <value hex>
//   end (other lines are ignored)
// Per case: the pre-state is loaded, then walked with small budgets -- the accounts from 0 (next origin = last + 1), then the
// storage of every account with storage, four accounts per request, a cut account continued from its last slot + 1.  Every
// answer must be accepted by G, the accounts must be exactly the pre-state's with its nonces and balances, and the slots
// exactly its non-zero slots.  A root other than the current one gets an empty answer.  Prints "ALL OK".
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

static Hash32 next_key(Hash32 k)
{
    for (int i = 31; i >= 0; --i)
        if (++k[i] != 0) break;
    return k;
}

static int run(Gpu& g, const Case& c, int n)
{
    state::ResidentStateTrie st(g);
    std::map<Address, const state::AccountState*> load;
    for (const auto& [a, s] : c.pre) load[a] = &s;
    if (!load.empty() && st.apply(load) != c.pre_root) { std::cout << "case " << n << ": pre root mismatch\n"; return 1; }
    const Hash32 root = st.root();
    Hash32 ff;
    ff.fill(0xff);
    // the accounts
    std::map<Hash32, state::ResidentStateTrie::AccountEntry> got;
    Hash32 origin{};
    for (;;) {
        const auto a = st.snapAccountRange(root, origin, ff, 300);
        const auto [ok, more] = snap::verifySnapAccountRange(g, root, origin, a.accounts, a.proof);
        if (!ok || (a.accounts.empty() && !c.pre.empty())) { std::cout << "case " << n << ": an account answer is not accepted\n"; return 1; }
        for (const auto& [k, body] : a.accounts) {
            state::ResidentStateTrie::AccountEntry e;
            snap::decodeSlimAccount(body, e);
            e.key = k;
            got[k] = e;
        }
        if (!more) break;
        origin = next_key(a.accounts.back().first);
    }
    std::map<Hash32, const state::AccountState*> want;
    std::map<Hash32, std::map<Hash32, std::array<uint8_t, 32>>> want_slots;
    size_t n_slots = 0;
    for (const auto& [a, s] : c.pre) {
        const Hash32 ak = hash(g, Bytes(a.begin(), a.end()));
        want[ak] = &s;
        for (const auto& kv : s.storage)
            if (kv.second != std::array<uint8_t, 32>{}) { want_slots[ak][hash(g, Bytes(kv.first.begin(), kv.first.end()))] = kv.second; ++n_slots; }
    }
    if (got.size() != want.size()) { std::cout << "case " << n << ": " << got.size() << " accounts for " << want.size() << "\n"; return 1; }
    for (const auto& [k, e] : got)
        if (!want.count(k) || want[k]->nonce != e.nonce || want[k]->balance != e.balance) { std::cout << "case " << n << ": an account differs\n"; return 1; }
    // the storage
    std::vector<Hash32> pending;
    for (const auto& [k, e] : got)
        if (e.storageHash != state::ResidentStateTrie::kEmptyRoot) pending.push_back(k);
    size_t seen = 0;
    Hash32 o{};
    while (!pending.empty()) {
        const std::vector<Hash32> batch(pending.begin(), pending.begin() + std::min<size_t>(4, pending.size()));
        const auto a = st.snapStorageRanges(root, batch, o, ff, 200);
        std::vector<Hash32> roots;
        for (size_t i = 0; i < a.slots.size(); ++i) roots.push_back(got[batch[i]].storageHash);
        const auto res = snap::verifySnapStorageRanges(g, roots, o, a.slots, a.proof);
        if (a.slots.empty()) { std::cout << "case " << n << ": no storage served\n"; return 1; }
        for (const auto& [ok, more] : res)
            if (!ok) { std::cout << "case " << n << ": a storage answer is not accepted\n"; return 1; }
        for (size_t i = 0; i < a.slots.size(); ++i)
            for (const auto& [k, body] : a.slots[i]) {
                const auto& w = want_slots[batch[i]];
                const auto it = w.find(k);
                if (it == w.end() || rlp::encode_bytes(it->second.data(), 32, true) != body) { std::cout << "case " << n << ": a slot differs\n"; return 1; }
                ++seen;
            }
        size_t done = a.slots.size();
        if (!a.proof.empty() && res.back().second) {
            o = next_key(a.slots.back().back().first);
            --done;
        } else {
            o = Hash32{};
        }
        pending.erase(pending.begin(), pending.begin() + done);
    }
    if (seen != n_slots) { std::cout << "case " << n << ": " << seen << " slots for " << n_slots << "\n"; return 1; }
    // another root: nothing served
    Hash32 other = root;
    other[0] ^= 1;
    if (!st.snapAccountRange(other, Hash32{}, ff).accounts.empty()) { std::cout << "case " << n << ": a past root was served\n"; return 1; }
    if (st.root() != root) { std::cout << "case " << n << ": the answers changed the state\n"; return 1; }
    return 0;
}

int main(int argc, char** argv)
{
    if (argc != 2) { std::cerr << "usage: resident_state_snap_test CASES\n"; return 2; }
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
