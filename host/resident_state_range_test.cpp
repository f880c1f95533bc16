// resident_state_range_test.cpp -- account and storage ranges of the resident world state in C++ (phant_host.hpp:
// ResidentStateTrie::accountRange / storageRange / dump).  Reads the cases of resident_state_witness_test.cpp (written by
// tests/test_gpu_host_cpp_resident_state_range.py from the fixture states):
//   case <pre state root hex> <post state root hex>
//   pre | acct <address hex> <nonce> <balance hex, 32 bytes> <code hex or -> | pslot | slot <address hex> <slot hex> <value hex>
//   del <address hex> | end
// Per case, with a journal of one apply: the pre-state is loaded and the block applied; dump() now must equal the post-state
// and dump(1) the pre-state, hashed (keccak(address) -> nonce, balance, keccak(code), keccak(slot) -> value); each dump loaded
// into a fresh state with one apply must give that state's root and the storage roots the dump reports; a whole
// accountRange and every storageRange must agree with the dump.  Prints "ALL OK".
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

using Dump = std::map<Hash32, state::ResidentStateTrie::DumpAccount>;

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
    std::map<Address, state::AccountState> post_state() const
    {
        std::map<Address, state::AccountState> p = pre;
        for (const Address& a : gone) p.erase(a);
        for (const auto& [a, s] : live) {
            auto old = p.count(a) ? p[a].storage : decltype(s.storage){};
            p[a] = s;
            p[a].storage = old;
            if (slots.count(a))
                for (const auto& [k, v] : slots.at(a)) p[a].storage[k] = v;
        }
        return p;
    }
};

// the dump equals `want` (hashed); fields other than the storage root compared
static bool same(Gpu& g, const Dump& d, const std::map<Address, state::AccountState>& want)
{
    size_t n = 0;
    for (const auto& [a, s] : want) {
        const auto it = d.find(hash(g, Bytes(a.begin(), a.end())));
        if (it == d.end()) return false;
        const auto& f = it->second.fields;
        if (f.nonce != s.nonce || f.balance != s.balance || f.codeHash != hash(g, s.code)) return false;
        std::map<Hash32, std::array<uint8_t, 32>> st;
        for (const auto& [k, v] : s.storage)
            if (v != std::array<uint8_t, 32>{}) st[hash(g, Bytes(k.begin(), k.end()))] = v;
        if (st != it->second.storage) return false;
        ++n;
    }
    return n == d.size();
}

// the dump loaded into a fresh state with one apply: its root, and the storage roots the dump reports
static bool reloads(Gpu& g, const Dump& d, const Hash32& root)
{
    Bytes k32, bal, code, skeys, svals, flags;
    std::vector<uint64_t> nonce;
    std::vector<uint32_t> sacc;
    std::vector<Hash32> sroots;
    for (const auto& [k, a] : d) {
        for (const auto& [sk, v] : a.storage) {
            sacc.push_back((uint32_t)nonce.size());
            skeys.insert(skeys.end(), sk.begin(), sk.end());
            svals.insert(svals.end(), v.begin(), v.end());
        }
        k32.insert(k32.end(), k.begin(), k.end());
        bal.insert(bal.end(), a.fields.balance.begin(), a.fields.balance.end());
        code.insert(code.end(), a.fields.codeHash.begin(), a.fields.codeHash.end());
        nonce.push_back(a.fields.nonce);
        flags.push_back(0);
        sroots.push_back(a.fields.storageHash);
    }
    phant_gpu_resident_state* s = nullptr;
    g.check(phant_gpu_resident_state_open(g.ctx(), &s), "open");
    Hash32 got{};
    Bytes out_sroots(32 * d.size() + 32);
    phant_gpu_state_diff diff{};
    diff.n_accounts = d.size();
    diff.account_keys32 = k32.data();
    diff.account_flags = flags.data();
    diff.nonce = nonce.data();
    diff.balance32 = bal.data();
    diff.code_hash32 = code.data();
    diff.n_slots = sacc.size();
    diff.slot_account = sacc.data();
    diff.slot_keys32 = skeys.data();
    diff.slot_vals32 = svals.data();
    const int rc = d.empty() ? phant_gpu_resident_state_root(s, got.data()) : phant_gpu_resident_state_apply(s, &diff, got.data(), out_sroots.data());
    phant_gpu_resident_state_close(s);
    if (rc != 0 || got != root) return false;
    for (size_t i = 0; i < sroots.size(); ++i)
        if (!std::equal(sroots[i].begin(), sroots[i].end(), out_sroots.begin() + 32 * i)) return false;
    return true;
}

// a whole accountRange and every account's whole storageRange agree with the dump (storageRange takes the address)
static bool ranges_agree(state::ResidentStateTrie& st, Gpu& g, const Dump& d, const std::map<Address, state::AccountState>& by_addr, uint32_t back)
{
    Hash32 lo{}, hi;
    hi.fill(0xff);
    const auto r = st.accountRange(lo, hi, (uint32_t)d.size() + 1, back);
    if (r.more || r.accounts.size() != d.size()) return false;
    size_t i = 0;
    for (const auto& [k, a] : d) {
        const auto& e = r.accounts[i++];
        if (e.key != k || e.nonce != a.fields.nonce || e.storageHash != a.fields.storageHash) return false;
    }
    for (const auto& [addr, s] : by_addr) {
        const auto& a = d.at(hash(g, Bytes(addr.begin(), addr.end())));
        const auto sr = st.storageRange(addr, lo, hi, (uint32_t)a.storage.size() + 1, back);
        if (sr.more || sr.slots.size() != a.storage.size()) return false;
        if (!a.storage.empty()) {
            const auto one = st.storageRange(addr, lo, hi, 1, back);
            if (one.slots.size() != 1 || one.slots[0].first != a.storage.begin()->first || one.more != (a.storage.size() > 1)) return false;
        }
    }
    return true;
}

static int run(Gpu& g, Case& c, int n)
{
    state::ResidentStateTrie st(g);
    st.setJournal(1);
    std::map<Address, const state::AccountState*> load;
    for (const auto& [a, s] : c.pre) load[a] = &s;
    if (!load.empty() && st.apply(load) != c.pre_root) { std::cout << "case " << n << ": pre root mismatch\n"; return 1; }
    if (st.apply(c.touched(), c.slots) != c.post) { std::cout << "case " << n << ": apply root mismatch\n"; return 1; }
    const auto post = c.post_state();
    const Dump now = st.dump(0, 5), before = st.dump(1, 3);
    if (!same(g, now, post)) { std::cout << "case " << n << ": the dump differs from the post-state\n"; return 1; }
    if (!same(g, before, c.pre)) { std::cout << "case " << n << ": the dump one apply back differs from the pre-state\n"; return 1; }
    if (!reloads(g, now, c.post) || !reloads(g, before, c.pre_root)) { std::cout << "case " << n << ": a reloaded dump has another root\n"; return 1; }
    if (!ranges_agree(st, g, now, post, 0) || !ranges_agree(st, g, before, c.pre, 1)) { std::cout << "case " << n << ": ranges differ\n"; return 1; }
    if (st.root() != c.post) { std::cout << "case " << n << ": a range call changed the state\n"; return 1; }
    return 0;
}

int main(int argc, char** argv)
{
    if (argc != 2) { std::cerr << "usage: resident_state_range_test CASES\n"; return 2; }
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
