// resident_state_read_test.cpp -- account and slot reads from the resident world state in C++ (phant_host.hpp:
// ResidentStateTrie::read), now and one apply back.  Reads the cases of resident_state_witness_test.cpp (written by
// tests/test_gpu_host_cpp_resident_state_read.py from the fixture states) and uses their pre-states only:
//   case <pre state root hex> <post state root hex>
//   pre <address hex> <nonce> <balance hex, 32 bytes> <code hex or -> | pslot <address hex> <slot hex, 32 bytes> <value hex>
//   end (other lines are ignored)
// Per case, with a journal of one apply: the pre-state is loaded; every account with every slot it holds and one slot it does
// not, and one absent account with two slots, are read and must equal the pre-state (storageHash: the one getProofs returns);
// then every account is destroyed, and the same reads must give every key absent now and the pre-state one apply back, with
// the pre root.  Prints "ALL OK".
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

// the values read for `req` are the pre-state's (pre == true) or every key absent
static bool same(Gpu& g, const Case& c, const state::ResidentStateTrie::ProofRequests& req,
                 const std::map<Address, state::ResidentStateTrie::AccountValues>& got,
                 const std::map<Address, state::ResidentStateTrie::AccountProof>& proofs, bool pre)
{
    const Hash32 empty_root = hash(g, Bytes{0x80}), empty_code = hash(g, Bytes{});
    for (const auto& [a, ks] : req) {
        const auto it = pre ? c.pre.find(a) : c.pre.end();
        const auto& v = got.at(a);
        if (v.exists != (it != c.pre.end())) return false;
        if (it != c.pre.end()) {
            const state::AccountState& s = it->second;
            if (v.nonce != s.nonce || v.balance != s.balance || v.codeHash != hash(g, s.code) || v.storageHash != proofs.at(a).storageHash)
                return false;
        } else if (v.nonce || v.balance != std::array<uint8_t, 32>{} || v.storageHash != empty_root || v.codeHash != empty_code)
            return false;
        if (v.storage.size() != std::set<std::array<uint8_t, 32>>(ks.begin(), ks.end()).size()) return false;
        for (const auto& k : ks) {
            std::array<uint8_t, 32> want{};
            if (it != c.pre.end() && it->second.storage.count(k)) want = it->second.storage.at(k);
            if (v.storage.at(k) != want) return false;
        }
    }
    return true;
}

static int run(Gpu& g, const Case& c, int n)
{
    state::ResidentStateTrie st(g);
    st.setJournal(1);
    std::map<Address, const state::AccountState*> load;
    for (const auto& [a, s] : c.pre) load[a] = &s;
    if (!load.empty() && st.apply(load) != c.pre_root) { std::cout << "case " << n << ": pre root mismatch\n"; return 1; }
    state::ResidentStateTrie::ProofRequests req;
    std::array<uint8_t, 32> extra{};
    extra[31] = 0x77;
    extra[0] = 0x5a;
    for (const auto& [a, s] : c.pre) {
        auto& ks = req[a];
        for (const auto& kv : s.storage) ks.push_back(kv.first);
        if (!s.storage.count(extra)) ks.push_back(extra);
    }
    Address ghost{};
    ghost.fill(0xee);
    req[ghost] = {extra, std::array<uint8_t, 32>{}};
    const auto proofs = st.getProofs(req);
    if (!same(g, c, req, st.read(req), proofs, true)) { std::cout << "case " << n << ": values now differ from the pre-state\n"; return 1; }
    if (load.empty()) return 0;
    std::map<Address, const state::AccountState*> destroy;
    for (const auto& [a, s] : c.pre) destroy[a] = nullptr;
    st.apply(destroy);
    const Hash32 after = st.root();
    if (!same(g, c, req, st.read(req), proofs, false)) { std::cout << "case " << n << ": a destroyed account is still read\n"; return 1; }
    if (!same(g, c, req, st.read(req, 1), proofs, true)) { std::cout << "case " << n << ": values one apply back differ\n"; return 1; }
    if (st.root() != after) { std::cout << "case " << n << ": read changed the state\n"; return 1; }
    return 0;
}

int main(int argc, char** argv)
{
    if (argc != 2) { std::cerr << "usage: resident_state_read_test CASES\n"; return 2; }
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
