// resident_state_code_test.cpp -- contract code beside the resident world state in C++ (phant_host.hpp: ResidentStateTrie::
// putCodes / codes / getCode / pruneCodes / witnessCodes).  Reads the cases of resident_state_witness_test.cpp (written by
// tests/test_gpu_host_cpp_resident_state_code.py from the fixture states):
//   case <pre state root hex> <post state root hex>
//   pre <address hex> <nonce> <balance hex, 32 bytes> <code hex or -> | pslot ... | del <address hex> | acct ... | slot ... | end
// Per case, with a journal of one apply: the pre-state's codes are put and the pre-state loaded; getCode of every account and
// of an absent one must give the pre-state's code; witnessCodes of the block must be the distinct codes of its accounts present
// before it, ordered by hash; after the post codes are put and the block applied, getCode gives the post-state's code now and
// the pre-state's one apply back, before and after pruneCodes.  Prints "ALL OK".
#include "phant_host.hpp"

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

struct Case {
    Hash32 pre_root{}, post{};
    std::map<Address, state::AccountState> pre, live;
    std::set<Address> gone;
    state::HashedDiff::SlotChanges slots;
};

static bool codes_are(state::ResidentStateTrie& st, const std::vector<Address>& addrs, const std::map<Address, Bytes>& want, uint32_t back)
{
    const auto got = st.getCode(addrs, back);
    for (const Address& a : addrs) {
        const auto it = want.find(a);
        const Bytes w = it == want.end() ? Bytes{} : it->second;
        if (!got.at(a) || *got.at(a) != w) return false;
    }
    return true;
}

static int run(Gpu& g, const Case& c, int n)
{
    state::ResidentStateTrie st(g);
    st.setJournal(1);
    std::map<Address, Bytes> pre_code, post_code;
    std::vector<Bytes> pre_codes, post_codes;
    for (const auto& [a, s] : c.pre) { pre_code[a] = s.code; pre_codes.push_back(s.code); }
    post_code = pre_code;
    for (const Address& a : c.gone) post_code.erase(a);
    for (const auto& [a, s] : c.live) { post_code[a] = s.code; post_codes.push_back(s.code); }
    std::vector<Address> everyone;
    for (const auto& kv : pre_code) everyone.push_back(kv.first);
    for (const auto& kv : c.live) everyone.push_back(kv.first);
    Address ghost{};
    ghost.fill(0xee);
    everyone.push_back(ghost);
    st.putCodes(pre_codes);
    std::map<Address, const state::AccountState*> load;
    for (const auto& [a, s] : c.pre) load[a] = &s;
    if (!load.empty() && st.apply(load) != c.pre_root) { std::cout << "case " << n << ": pre root mismatch\n"; return 1; }
    if (!codes_are(st, everyone, pre_code, 0)) { std::cout << "case " << n << ": getCode differs from the pre-state\n"; return 1; }
    std::map<Address, const state::AccountState*> touched;
    for (const auto& [a, s] : c.live) touched[a] = &s;
    for (const Address& a : c.gone) touched[a] = nullptr;
    std::map<Hash32, Bytes> want_wit;
    for (const auto& kv : touched) {
        const auto it = c.pre.find(kv.first);
        if (it != c.pre.end() && !it->second.code.empty()) want_wit[hasher::keccak256_batch(g, {it->second.code})[0]] = it->second.code;
    }
    std::vector<Bytes> want_list;
    for (const auto& kv : want_wit) want_list.push_back(kv.second);
    if (st.witnessCodes(touched) != want_list) { std::cout << "case " << n << ": witnessCodes differ\n"; return 1; }
    st.putCodes(post_codes);
    if (!touched.empty() && st.apply(touched, c.slots) != c.post) { std::cout << "case " << n << ": post root mismatch\n"; return 1; }
    for (int pruned = 0; pruned < 2; ++pruned) {
        if (!codes_are(st, everyone, post_code, 0)) { std::cout << "case " << n << ": getCode differs from the post-state\n"; return 1; }
        if (!touched.empty() && !codes_are(st, everyone, pre_code, 1)) { std::cout << "case " << n << ": getCode one apply back differs\n"; return 1; }
        st.pruneCodes();
    }
    return 0;
}

int main(int argc, char** argv)
{
    if (argc != 2) { std::cerr << "usage: resident_state_code_test CASES\n"; return 2; }
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
