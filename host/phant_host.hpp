// phant_host.hpp -- C++ host mirror of the phant functions that sit on the hot path, over the C ABI of
// include/phant_gpu.h.  phant's own host code is Zig; this image has no Zig toolchain, so the mirror is
// C++ (the reference is compiled code) with the same names, argument meaning and error behaviour:
//
//   hasher::keccak256 / keccak256WithPrefix      src/crypto/hasher.zig:4-17
//   mpt::KeyVal{init,lessThan}, mpt::mptize       src/mpt/mpt.zig:13-45
//   blockchain::calculateMPTRoot                  src/blockchain/blockchain.zig:209-235
//   engine_api::payloadListRoot                   src/engine_api/execution_payload.zig:125-139 (32-byte BE index keys)
//   state::StateDB::root                          hook src/blockchain/blockchain.zig:83-85 (missing in the reference)
//   state::StateDB::subtreeRoots / rootFromSubtreeRoots   the same root sharded over GPUs by top nibble (SURVEY.md 8e)
//   engine_api::verifyWitness                     hook src/engine_api/execution_payload.zig:177-178 (TODO in the reference)
//   engine_api::readPreState / stateDBFromWitness the pre-state a stateless block executes against (execution_payload.zig:20-25)
//   signer::getSenders                            src/signer/signer.zig:78-79 (erecover + keccak) for a whole block
//
// No arithmetic happens here: every hash and every root comes from libphantgpu.so.  Errors from the library
// surface as phant::GpuError (the Zig binding maps them to error.GpuBackend, INTEGRATION.md).
#pragma once
#include "../include/phant_gpu.h"

#include <algorithm>
#include <array>
#include <cstdint>
#include <cstring>
#include <map>
#include <set>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

namespace phant {

using Hash32 = std::array<uint8_t, 32>;
using Address = std::array<uint8_t, 20>;
using Bytes = std::vector<uint8_t>;

struct GpuError : std::runtime_error {
    int code;
    GpuError(int c, const std::string& where) : std::runtime_error(where + ": " + phant_gpu_strerror(c)), code(c) {}
};

// One device, one stream.  Not re-entrant: one per host thread (src/main.zig:143-149 runs handlers on worker threads).
class Gpu {
public:
    explicit Gpu(int device = 0)
    {
        if (phant_gpu_abi_version() != PHANT_GPU_ABI_VERSION) throw GpuError(PHANT_GPU_E_INVALID, "abi version");
        phant_gpu_config cfg{};
        cfg.device = device;
        const int rc = phant_gpu_create(&ctx_, &cfg);
        if (rc != 0) throw GpuError(rc, "phant_gpu_create"); // no device: the caller keeps its CPU path; nothing is emulated here
    }
    ~Gpu() { phant_gpu_destroy(ctx_); }
    Gpu(const Gpu&) = delete;
    Gpu& operator=(const Gpu&) = delete;
    phant_gpu_ctx* ctx() { return ctx_; }
    void check(int rc, const char* where) const
    {
        if (rc != 0) throw GpuError(rc, std::string(where) + " [" + phant_gpu_last_error(ctx_) + "]");
    }

private:
    phant_gpu_ctx* ctx_ = nullptr;
};

namespace hasher {
// many inputs at once (the shape the GPU wants); msgs[i] are independent byte strings
inline std::vector<Hash32> keccak256_batch(Gpu& g, const std::vector<Bytes>& msgs)
{
    Bytes flat;
    std::vector<uint64_t> off(msgs.size() + 1, 0);
    for (size_t i = 0; i < msgs.size(); ++i) {
        flat.insert(flat.end(), msgs[i].begin(), msgs[i].end());
        off[i + 1] = flat.size();
    }
    std::vector<Hash32> out(msgs.size());
    if (!msgs.empty())
        g.check(phant_gpu_keccak256_batch(g.ctx(), flat.data(), off.data(), msgs.size(), out[0].data()), "keccak256_batch");
    return out;
}
inline Hash32 keccak256(Gpu& g, const Bytes& data) { return keccak256_batch(g, {data})[0]; }
inline Hash32 keccak256WithPrefix(Gpu& g, const Bytes& prefix, const Bytes& data)
{
    Bytes m(prefix);
    m.insert(m.end(), data.begin(), data.end());
    return keccak256(g, m);
}
} // namespace hasher

namespace mpt {
inline const Hash32 empty_mpt_root = {0x56, 0xe8, 0x1f, 0x17, 0x1b, 0xcc, 0x55, 0xa6, 0xff, 0x83, 0x45, 0xe6, 0x92, 0xc0, 0xf8, 0x6e,
                                      0x5b, 0x48, 0xe0, 0x1b, 0x99, 0x6c, 0xad, 0xc0, 0x01, 0x62, 0x2f, 0xb5, 0xe3, 0x63, 0xb4, 0x21};

// mpt.zig:13-34
struct KeyVal {
    Bytes nibbles;
    Bytes value;
    static KeyVal init(const Bytes& key, const Bytes& value)
    {
        KeyVal kv;
        kv.nibbles.reserve(2 * key.size());
        for (uint8_t b : key) { kv.nibbles.push_back(b >> 4); kv.nibbles.push_back(b & 0x0f); }
        kv.value = value;
        return kv;
    }
    static bool lessThan(const KeyVal& a, const KeyVal& b) { return a.nibbles < b.nibbles; } // std::mem.lessThan on the nibbles
};

// mpt.zig:38-45: `list` must be sorted by key (the reference asserts); unsorted input -> GpuError(E_INVALID)
inline Hash32 mptize(Gpu& g, const std::vector<KeyVal>& list)
{
    Bytes keys, vals;
    std::vector<uint32_t> koff(list.size() + 1, 0);
    std::vector<uint64_t> voff(list.size() + 1, 0);
    for (size_t i = 0; i < list.size(); ++i) {
        const Bytes& nb = list[i].nibbles;
        if (nb.size() % 2) throw GpuError(PHANT_GPU_E_INVALID, "mptize: odd nibble count"); // KeyVal.init always makes pairs
        for (size_t j = 0; j < nb.size(); j += 2) keys.push_back((uint8_t)((nb[j] << 4) | nb[j + 1]));
        koff[i + 1] = (uint32_t)keys.size();
        vals.insert(vals.end(), list[i].value.begin(), list[i].value.end());
        voff[i + 1] = vals.size();
    }
    Hash32 root;
    g.check(phant_gpu_mpt_root(g.ctx(), keys.data(), koff.data(), vals.data(), voff.data(), list.size(), root.data()), "mptize");
    return root;
}
} // namespace mpt

namespace rlp {
inline Bytes encode_uint(uint64_t v)
{
    if (v == 0) return {0x80};
    Bytes be;
    for (int s = 56; s >= 0; s -= 8)
        if (!be.empty() || (v >> s) & 0xff) be.push_back((uint8_t)(v >> s));
    if (be.size() == 1 && be[0] < 0x80) return be;
    Bytes out{(uint8_t)(0x80 + be.size())};
    out.insert(out.end(), be.begin(), be.end());
    return out;
}
// list header in front of an already concatenated payload
inline Bytes wrap_list(const Bytes& payload)
{
    Bytes out;
    if (payload.size() < 56) out.push_back((uint8_t)(0xc0 + payload.size()));
    else {
        Bytes be;
        for (int s = 56; s >= 0; s -= 8)
            if (!be.empty() || ((uint64_t)payload.size() >> s) & 0xff) be.push_back((uint8_t)((uint64_t)payload.size() >> s));
        out.push_back((uint8_t)(0xf7 + be.size()));
        out.insert(out.end(), be.begin(), be.end());
    }
    out.insert(out.end(), payload.begin(), payload.end());
    return out;
}
} // namespace rlp

namespace blockchain {
// blockchain.zig:209-235: index trie of already-encoded items, keys rlp(i) visited in sorted order
// (1..0x7f, then 0 as 0x80, then 0x80.. as 0x81 xx ..)
inline Hash32 calculateMPTRoot(Gpu& g, const std::vector<Bytes>& encoded_items)
{
    std::vector<mpt::KeyVal> keyvals;
    keyvals.reserve(encoded_items.size());
    size_t i = 0;
    for (; i + 1 < encoded_items.size() && i + 1 != 0x80; ++i)
        keyvals.push_back(mpt::KeyVal::init({(uint8_t)(i + 1)}, encoded_items[i + 1]));
    if (!encoded_items.empty()) {
        keyvals.push_back(mpt::KeyVal::init({0x80}, encoded_items[0]));
        ++i;
    }
    for (; i < encoded_items.size(); ++i) keyvals.push_back(mpt::KeyVal::init(rlp::encode_uint(i), encoded_items[i]));
    return mpt::mptize(g, keyvals);
}
} // namespace blockchain

namespace state {
struct AccountState { // src/state/types.zig:13-33
    uint64_t nonce = 0;
    std::array<uint8_t, 32> balance{}; // u256, big endian
    Bytes code;
    std::map<std::array<uint8_t, 32>, std::array<uint8_t, 32>> storage; // slot -> value (zero values are deleted, statedb.zig:112-119)
};

class StateDB { // src/state/statedb.zig:16-30, plus the missing root()
public:
    std::map<Address, AccountState> db;

    // the body of the check commented out at src/blockchain/blockchain.zig:83-85
    Hash32 root(Gpu& g) const
    {
        Flat f(db, [](const Address&) { return true; });
        Hash32 r;
        g.check(phant_gpu_state_root(g.ctx(), &f.t, r.data()), "StateDB.root");
        return r;
    }

    // ---- root() sharded over GPUs by the top nibble of keccak(address) (SURVEY.md 8e) ----
    struct SubtreeRoots {
        std::array<uint8_t, 16 * 32> refs{}; // hash of the subtree under root-branch slot v, zero where this rank owns nothing
        uint32_t mask = 0;                   // populated slots
    };
    static int nibbleOwner(int v, int world) { return v * std::min(world, 16) / 16; }

    // this rank's share: the subtrees of the root-branch slots it owns (one K call for the address hashes, one S call)
    SubtreeRoots subtreeRoots(Gpu& g, int rank, int world) const
    {
        std::vector<Bytes> addrs;
        for (const auto& [a, acc] : db) addrs.emplace_back(a.begin(), a.end());
        const std::vector<Hash32> h = hasher::keccak256_batch(g, addrs);
        size_t i = 0;
        std::map<Address, int> slot;
        for (const auto& [a, acc] : db) slot[a] = h[i++][0] >> 4;
        Flat f(db, [&](const Address& a) { return nibbleOwner(slot[a], world) == rank; });
        SubtreeRoots out;
        g.check(phant_gpu_state_subtree_roots(g.ctx(), &f.t, out.refs.data(), &out.mask), "StateDB.subtreeRoots");
        return out;
    }

    // the same, with the exchange behind the ABI (phant_gpu_state_root_sharded: subtree roots here, ONE all-gather over the
    // communicator of phant_gpu_comm_init / _init_local, root branch hashed on every rank); call it on every rank
    Hash32 rootSharded(Gpu& g, int rank, int world) const
    {
        std::vector<Bytes> addrs;
        for (const auto& [a, acc] : db) addrs.emplace_back(a.begin(), a.end());
        const std::vector<Hash32> h = hasher::keccak256_batch(g, addrs);
        size_t i = 0;
        std::map<Address, int> slot;
        for (const auto& [a, acc] : db) slot[a] = h[i++][0] >> 4;
        Flat f(db, [&](const Address& a) { return phant_gpu_nibble_owner(slot[a], world) == rank; });
        Hash32 r;
        g.check(phant_gpu_state_root_sharded(g.ctx(), &f.t, r.data()), "StateDB.rootSharded");
        return r;
    }

    // after the all-gather (slots are disjoint between ranks, so summing / or-ing the shares is the gather): the root
    // branch rlp([ref_0 .. ref_15, ""]) hashed with one K call.  Needs >= 2 populated slots -- otherwise the root is not
    // a branch and the one rank that owns the populated slot holds every account: it calls root() on its share.
    static Hash32 rootFromSubtreeRoots(Gpu& g, const SubtreeRoots& all)
    {
        if (__builtin_popcount(all.mask) < 2) throw std::invalid_argument("root is not a branch: use root() on the owning rank");
        Bytes body;
        for (int v = 0; v < 16; ++v) {
            if ((all.mask >> v) & 1) { body.push_back(0xa0); body.insert(body.end(), all.refs.begin() + 32 * v, all.refs.begin() + 32 * v + 32); }
            else body.push_back(0x80);
        }
        body.push_back(0x80);
        return hasher::keccak256(g, rlp::wrap_list(body));
    }

private:
    struct Flat { // the SoA / CSR tables of phant_gpu_accounts over the accounts `keep` selects
        Bytes addr, bal, code, skeys, svals;
        std::vector<uint64_t> nonce, coff{0}, soff{0};
        phant_gpu_accounts t{};
        template <class Keep> Flat(const std::map<Address, AccountState>& db, Keep keep)
        {
            for (const auto& [a, acc] : db) {
                if (!keep(a)) continue;
                addr.insert(addr.end(), a.begin(), a.end());
                nonce.push_back(acc.nonce);
                bal.insert(bal.end(), acc.balance.begin(), acc.balance.end());
                code.insert(code.end(), acc.code.begin(), acc.code.end());
                coff.push_back(code.size());
                for (const auto& [k, v] : acc.storage) {
                    skeys.insert(skeys.end(), k.begin(), k.end());
                    svals.insert(svals.end(), v.begin(), v.end());
                }
                soff.push_back(skeys.size() / 32);
            }
            t.n_accounts = nonce.size();
            t.addr20 = addr.data(); t.nonce = nonce.data(); t.balance32 = bal.data();
            t.code = code.data(); t.code_off = coff.data();
            t.slot_keys32 = skeys.data(); t.slot_vals32 = svals.data(); t.slot_off = soff.data();
        }
    };
};

// StateDB.root() block after block (hook src/blockchain/blockchain.zig:83-85) without rebuilding the state: the account trie
// and every storage trie live on the device (phant_gpu_resident_state_*, DESIGN.md §4.3c); after a block the host hands over
// ONLY the accounts the block touched and, in the incremental form, the slots it wrote.  Addresses, slot numbers and code
// are hashed with K; the account leaves and storage roots are computed on the device.
// A block's changes as the C ABI takes them (phant_gpu_state_diff), addresses, slot numbers and code hashed with K: what the
// resident world state applies and what the transition roots apply to a witness.  `touched`: address -> new account state, or
// nullptr for a destroyed account.  changed == nullptr: each touched account's whole storage replaces what was there
// (CLEAR_STORAGE); otherwise only the listed slots (zero = deleted), and `recreated` accounts are sent with CLEAR_STORAGE.
struct HashedDiff {
    std::vector<Bytes> addrs, codes, slot_keys;
    std::vector<uint32_t> slot_account;
    Bytes slot_vals, flags, bal, k32, c32, s32;
    std::vector<uint64_t> nonce;
    using SlotChanges = std::map<Address, std::map<std::array<uint8_t, 32>, std::array<uint8_t, 32>>>;

    HashedDiff(Gpu& g, const std::map<Address, const AccountState*>& touched, const SlotChanges* changed, const std::set<Address>* recreated)
    {
        std::map<Address, uint32_t> index;
        for (const auto& [a, acc] : touched) {
            index[a] = (uint32_t)addrs.size();
            addrs.emplace_back(a.begin(), a.end());
            codes.push_back(acc ? acc->code : Bytes{});
            flags.push_back(acc ? (changed && !recreated->count(a) ? 0 : PHANT_GPU_ACCOUNT_CLEAR_STORAGE) : PHANT_GPU_ACCOUNT_DELETE);
            nonce.push_back(acc ? acc->nonce : 0);
            bal.insert(bal.end(), 32, 0);
            if (acc) std::copy(acc->balance.begin(), acc->balance.end(), bal.end() - 32);
            if (acc && !changed)
                for (const auto& [sk, sv] : acc->storage) {
                    slot_account.push_back(index[a]);
                    slot_keys.emplace_back(sk.begin(), sk.end());
                    slot_vals.insert(slot_vals.end(), sv.begin(), sv.end());
                }
        }
        if (recreated)
            for (const Address& a : *recreated)
                if (!touched.count(a) || !touched.at(a)) throw std::invalid_argument("a re-created account must be touched and live");
        if (changed)
            for (const auto& [a, slots] : *changed) {
                const auto it = index.find(a);
                if (it == index.end() || !touched.at(a)) throw std::invalid_argument("slots of an account that is not touched and live");
                for (const auto& [sk, sv] : slots) {
                    slot_account.push_back(it->second);
                    slot_keys.emplace_back(sk.begin(), sk.end());
                    slot_vals.insert(slot_vals.end(), sv.begin(), sv.end());
                }
            }
        const std::vector<Hash32> keys = hasher::keccak256_batch(g, addrs), code_hashes = hasher::keccak256_batch(g, codes);
        const std::vector<Hash32> hk = slot_keys.empty() ? std::vector<Hash32>{} : hasher::keccak256_batch(g, slot_keys);
        for (const Hash32& h : keys) k32.insert(k32.end(), h.begin(), h.end());
        for (const Hash32& h : code_hashes) c32.insert(c32.end(), h.begin(), h.end());
        for (const Hash32& h : hk) s32.insert(s32.end(), h.begin(), h.end());
    }
    phant_gpu_state_diff view() const
    {
        phant_gpu_state_diff d{};
        d.n_accounts = addrs.size();
        d.account_keys32 = k32.data();
        d.account_flags = flags.data();
        d.nonce = nonce.data();
        d.balance32 = bal.data();
        d.code_hash32 = c32.data();
        d.n_slots = slot_account.size();
        d.slot_account = slot_account.data();
        d.slot_keys32 = s32.data();
        d.slot_vals32 = slot_vals.data();
        return d;
    }
};

class ResidentStateTrie {
public:
    using SlotChanges = HashedDiff::SlotChanges; // address -> slot -> new value

    explicit ResidentStateTrie(Gpu& g) : g_(g) { g_.check(phant_gpu_resident_state_open(g_.ctx(), &s_), "ResidentStateTrie open"); }
    ~ResidentStateTrie() { phant_gpu_resident_state_close(s_); }
    ResidentStateTrie(const ResidentStateTrie&) = delete;
    ResidentStateTrie& operator=(const ResidentStateTrie&) = delete;

    Hash32 root()
    {
        Hash32 r;
        g_.check(phant_gpu_resident_state_root(s_, r.data()), "ResidentStateTrie root");
        return r;
    }
    // `touched`: address -> new account state, or nullptr for a destroyed account; each touched account's whole storage is
    // sent and replaces what the device held.  Returns the new state root.
    Hash32 apply(const std::map<Address, const AccountState*>& touched) { return send(touched, nullptr, nullptr); }
    // The incremental form: only the slots the block wrote (zero = deleted) are sent, and only the buckets they fall in are
    // re-hashed; every address in `changed_slots` is in `touched` with a live account.  `recreated`: touched live accounts the
    // block destroyed and created again -- their old storage is dropped before their changed slots apply.  No storage root is
    // computed here.
    Hash32 apply(const std::map<Address, const AccountState*>& touched, const SlotChanges& changed_slots, const std::set<Address>& recreated = {})
    {
        return send(touched, &changed_slots, &recreated);
    }
    // Keep on the device what undoes each of the last `depth` applies (0: nothing, the default), so that revert can take back
    // a block whose root does not match its header, or the blocks a reorg leaves.  With a journal, an apply with nothing
    // touched is still one block.
    void setJournal(uint32_t depth)
    {
        g_.check(phant_gpu_resident_state_set_journal(s_, depth), "ResidentStateTrie setJournal");
        journal_ = depth;
    }
    // Undo the last n applies, newest first; returns the root before the oldest of them.
    Hash32 revert(uint32_t n = 1)
    {
        Hash32 r;
        g_.check(phant_gpu_resident_state_revert(s_, n, r.data()), "ResidentStateTrie revert");
        return r;
    }
    // The execution witness of the block apply() would take with these arguments, from the state as it is now (which is not
    // changed): the pre-state trie nodes the block reads or changes, each once, ordered by digest.  With the block's codes
    // they make the witness engine_api::transitionRoot reads.
    std::vector<Bytes> witness(const std::map<Address, const AccountState*>& touched, const SlotChanges& changed_slots,
                               const std::set<Address>& recreated = {})
    {
        if (touched.empty()) return {};
        const HashedDiff hd(g_, touched, &changed_slots, &recreated);
        const phant_gpu_state_diff d = hd.view();
        phant_gpu_witness_size size{};
        g_.check(phant_gpu_resident_state_witness(s_, &d, &size), "ResidentStateTrie witness");
        Bytes all(size.nodes_bytes + 1);
        std::vector<uint64_t> off(size.n_nodes + 1);
        g_.check(phant_gpu_resident_state_witness_copy(s_, all.data(), off.data()), "ResidentStateTrie witness_copy");
        std::vector<Bytes> out;
        out.reserve(size.n_nodes);
        for (uint64_t i = 0; i < size.n_nodes; ++i) out.emplace_back(all.begin() + off[i], all.begin() + off[i + 1]);
        return out;
    }

private:
    Hash32 send(const std::map<Address, const AccountState*>& touched, const SlotChanges* changed, const std::set<Address>* recreated)
    {
        if (touched.empty()) {
            if (!journal_) return root();
            phant_gpu_state_diff d{};
            Hash32 r;
            g_.check(phant_gpu_resident_state_apply(s_, &d, r.data(), nullptr), "ResidentStateTrie apply");
            return r;
        }
        const HashedDiff hd(g_, touched, changed, recreated);
        const phant_gpu_state_diff d = hd.view();
        Hash32 r;
        g_.check(phant_gpu_resident_state_apply(s_, &d, r.data(), nullptr), "ResidentStateTrie apply");
        return r;
    }
    Gpu& g_;
    phant_gpu_resident_state* s_ = nullptr;
    uint32_t journal_ = 0;
};
} // namespace state

namespace signer {
// The tail of TxSigner.get_sender (src/signer/signer.zig:78-79) for many transactions at once: sigs65[i] = r || s || recid over
// the signing hash hashes[i]; addresses[i] is the sender, recovered[i] false where libsecp256k1 would have returned an error.
// validateSignatureFields and the EIP-155 `v` decoding (signer.zig:41-76) stay with the caller, as in the reference.
struct Senders {
    std::vector<Address> addresses;
    std::vector<uint8_t> recovered;
};
inline Senders getSenders(Gpu& g, const std::vector<Hash32>& hashes, const std::vector<std::array<uint8_t, 65>>& sigs65)
{
    if (hashes.size() != sigs65.size()) throw GpuError(PHANT_GPU_E_INVALID, "getSenders: one signature per hash");
    Senders out;
    out.addresses.resize(hashes.size());
    out.recovered.resize(hashes.size());
    if (!hashes.empty())
        g.check(phant_gpu_ecrecover_batch(g.ctx(), hashes[0].data(), sigs65[0].data(), hashes.size(), nullptr, out.addresses[0].data(),
                                          out.recovered.data()), "getSenders");
    return out;
}
} // namespace signer

namespace engine_api {
// execution_payload.zig:125-139: index trie keyed by the 32-byte big-endian index (phant's non-standard keys)
inline Hash32 payloadListRoot(Gpu& g, const std::vector<Bytes>& encoded_items)
{
    std::vector<mpt::KeyVal> kv;
    for (size_t i = 0; i < encoded_items.size(); ++i) {
        Bytes key(32, 0);
        for (int b = 0; b < 8; ++b) key[31 - b] = (uint8_t)((uint64_t)i >> (8 * b));
        kv.push_back(mpt::KeyVal::init(key, encoded_items[i]));
    }
    return mpt::mptize(g, kv); // big-endian fixed-width indices are already in sorted order
}

struct Witness {                       // flattened execution witness: one chain of nodes per key, root first
    Bytes nodes;
    std::vector<uint64_t> node_off{0};
    std::vector<uint64_t> proof_first{0};
    Bytes keys32;                      // hashed keys, 32 bytes each
    void add_proof(const std::vector<Bytes>& chain, const Hash32& hashed_key)
    {
        for (const Bytes& n : chain) { nodes.insert(nodes.end(), n.begin(), n.end()); node_off.push_back(nodes.size()); }
        proof_first.push_back(node_off.size() - 1);
        keys32.insert(keys32.end(), hashed_key.begin(), hashed_key.end());
    }
};
enum class ProofStatus : uint8_t { reject = 0, present = 1, absent = 2 };

// the TODO at execution_payload.zig:177-178: every proof of the witness must verify against `state_root`;
// returns per-proof status, throws only on backend errors (accept/reject is data)
inline std::vector<ProofStatus> verifyWitness(Gpu& g, const Hash32& state_root, const Witness& w)
{
    const uint64_t n = w.proof_first.size() - 1;
    std::vector<uint8_t> status(n);
    std::vector<uint64_t> bitmap((n + 63) / 64);
    phant_gpu_proof_batch b{};
    b.n_proofs = n;
    b.nodes = w.nodes.data(); b.node_off = w.node_off.data(); b.proof_first = w.proof_first.data();
    b.keys32 = w.keys32.data(); b.roots32 = state_root.data(); b.n_roots = 1;
    if (n) g.check(phant_gpu_verify_proofs(g.ctx(), &b, bitmap.data(), status.data(), nullptr, nullptr), "verifyWitness");
    std::vector<ProofStatus> out(n);
    for (uint64_t i = 0; i < n; ++i) out[i] = (ProofStatus)status[i];
    return out;
}

// ---- pre-state reads (phant_gpu_read_state): the StateDB a stateless block executes against (StatelessPayloadStatusV1,
// execution_payload.zig:20-25, TODO at :177-178), filled from the witness's `state` node set and `codes` ----
struct SlotRead {
    Address address;
    std::array<uint8_t, 32> slot; // the slot number, 32 bytes big endian (hashed here, as the storage trie keys it)
};
struct PreState {
    state::StateDB statedb;                        // every account proven present, with its code and its requested non-zero slots
    std::map<Address, uint8_t> account_status;     // 0 reject / 1 present / 2 absent / 3 node missing
    std::vector<uint8_t> slot_status;              // per requested slot, the same four values
    std::vector<Address> missing_code;             // present accounts whose codeHash no witness code hashes to
    bool complete() const
    {
        for (const auto& [a, s] : account_status)
            if (s != 1 && s != 2) return false;
        for (uint8_t s : slot_status)
            if (s != 1 && s != 2) return false;
        return missing_code.empty();
    }
};
struct IncompleteWitness : std::runtime_error {
    PreState pre; // what the witness did prove, for the caller's diagnostics
    explicit IncompleteWitness(PreState p) : std::runtime_error("execution witness does not prove the requested pre-state"), pre(std::move(p)) {}
};

// One K call for the addresses, one for the slot numbers, one P call; statuses are data (see PreState::complete)
inline PreState readPreState(Gpu& g, const Hash32& state_root, const std::vector<Bytes>& nodes, const std::vector<Bytes>& codes,
                             const std::vector<Address>& addresses, const std::vector<SlotRead>& slots)
{
    std::vector<Address> addrs;
    std::map<Address, uint32_t> idx;
    auto add = [&](const Address& a) { if (idx.emplace(a, (uint32_t)addrs.size()).second) addrs.push_back(a); };
    for (const Address& a : addresses) add(a);
    for (const SlotRead& s : slots) add(s.address);
    PreState out;
    out.slot_status.assign(slots.size(), 0);
    if (addrs.empty()) return out;
    std::vector<Bytes> am, sm;
    for (const Address& a : addrs) am.emplace_back(a.begin(), a.end());
    for (const SlotRead& s : slots) sm.emplace_back(s.slot.begin(), s.slot.end());
    const std::vector<Hash32> akeys = hasher::keccak256_batch(g, am), skeys = hasher::keccak256_batch(g, sm);
    auto flatten = [](const std::vector<Bytes>& items, Bytes& data, std::vector<uint64_t>& off) {
        off.assign(1, 0);
        for (const Bytes& b : items) { data.insert(data.end(), b.begin(), b.end()); off.push_back(data.size()); }
    };
    Bytes ndata, cdata;
    std::vector<uint64_t> noff, coff;
    flatten(nodes, ndata, noff);
    flatten(codes, cdata, coff);
    std::vector<uint32_t> sacc;
    for (const SlotRead& s : slots) sacc.push_back(idx[s.address]);
    const size_t na = addrs.size(), ns = slots.size();
    std::vector<uint8_t> ast(na), bal(32 * na), svals(32 * ns + 32);
    std::vector<uint64_t> nonce(na);
    std::vector<uint32_t> cidx(na);
    phant_gpu_state_reads in{};
    in.n_nodes = nodes.size(); in.nodes = ndata.data(); in.node_off = noff.data();
    in.n_codes = codes.size(); in.codes = cdata.data(); in.code_off = coff.data();
    in.roots32 = state_root.data(); in.n_roots = 1;
    in.n_accounts = na; in.account_keys32 = akeys[0].data();
    in.n_slots = ns; in.slot_keys32 = ns ? skeys[0].data() : nullptr; in.slot_account = sacc.data();
    phant_gpu_state_values v{};
    v.account_status = ast.data(); v.nonce = nonce.data(); v.balance32 = bal.data(); v.code_index = cidx.data();
    v.slot_status = out.slot_status.data(); v.slot_vals32 = svals.data();
    g.check(phant_gpu_read_state(g.ctx(), &in, &v), "readPreState");
    for (size_t i = 0; i < na; ++i) {
        out.account_status[addrs[i]] = ast[i];
        if (ast[i] != 1) continue;
        state::AccountState acc;
        acc.nonce = nonce[i];
        std::copy(bal.begin() + 32 * i, bal.begin() + 32 * i + 32, acc.balance.begin());
        if (cidx[i] == PHANT_GPU_CODE_MISSING) out.missing_code.push_back(addrs[i]);
        else if (cidx[i] != PHANT_GPU_CODE_EMPTY) acc.code = codes.at(cidx[i]);
        out.statedb.db[addrs[i]] = std::move(acc);
    }
    for (size_t j = 0; j < ns; ++j) {
        auto it = out.statedb.db.find(slots[j].address);
        if (out.slot_status[j] != 1 || it == out.statedb.db.end()) continue;
        std::array<uint8_t, 32> val;
        std::copy(svals.begin() + 32 * j, svals.begin() + 32 * j + 32, val.begin());
        it->second.storage[slots[j].slot] = val; // status 1 values are never zero
    }
    return out;
}

// The StateDB factory: the pre-state proven by the witness, or IncompleteWitness when any read is rejected (0), lacks a node
// (3) or a present account's code is not in `codes` -- the payload must then be refused before execution
inline state::StateDB stateDBFromWitness(Gpu& g, const Hash32& state_root, const std::vector<Bytes>& nodes, const std::vector<Bytes>& codes,
                                         const std::vector<Address>& addresses, const std::vector<SlotRead>& slots)
{
    PreState pre = readPreState(g, state_root, nodes, codes, addresses, slots);
    if (!pre.complete()) throw IncompleteWitness(std::move(pre));
    return std::move(pre.statedb);
}

// ---- state transition roots (phant_gpu_transition_roots): the post-state root a stateless client compares with the block
// header (StatelessPayloadStatusV1.state_root, execution_payload.zig:20-25; the check at blockchain.zig:83-85), from the
// witness's `state` node set, the parent state root and the block's changes, taken as ResidentStateTrie::apply takes them ----
struct TransitionResult {
    uint8_t status; // 1 computed / 0 a node breaks the rules / 3 the witness lacks a node the computation needs
    Hash32 root;    // zero unless status is 1
};
inline TransitionResult transitionRoot(Gpu& g, const Hash32& parent_root, const std::vector<Bytes>& nodes,
                                       const std::map<Address, const state::AccountState*>& touched,
                                       const state::HashedDiff::SlotChanges& changed_slots, const std::set<Address>& recreated = {})
{
    const state::HashedDiff hd(g, touched, &changed_slots, &recreated);
    const phant_gpu_state_diff d = hd.view();
    Bytes ndata;
    std::vector<uint64_t> noff(1, 0);
    for (const Bytes& b : nodes) { ndata.insert(ndata.end(), b.begin(), b.end()); noff.push_back(ndata.size()); }
    phant_gpu_transition t{};
    t.n_nodes = nodes.size(); t.nodes = ndata.data(); t.node_off = noff.data(); t.nodes_bytes = ndata.size();
    t.n_blocks = 1; t.pre_roots32 = parent_root.data();
    TransitionResult r{};
    g.check(phant_gpu_transition_roots(g.ctx(), &t, &d, r.root.data(), &r.status, nullptr), "transitionRoot");
    return r;
}
} // namespace engine_api

} // namespace phant
