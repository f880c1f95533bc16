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
//   snap::verifyAccountRange / verifyStorageRanges a snap client's checks of GetAccountRange / GetStorageRanges answers
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
#include <memory>
#include <optional>
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
// a byte string (an integer or a slot value with its leading zero bytes dropped first, when `trim`)
inline Bytes encode_bytes(const uint8_t* b, size_t n, bool trim = false)
{
    while (trim && n && !*b) { ++b; --n; }
    if (n == 1 && b[0] < 0x80) return {b[0]};
    Bytes out;
    if (n < 56) out.push_back((uint8_t)(0x80 + n));
    else {
        Bytes be;
        for (int s = 56; s >= 0; s -= 8)
            if (!be.empty() || ((uint64_t)n >> s) & 0xff) be.push_back((uint8_t)((uint64_t)n >> s));
        out.push_back((uint8_t)(0xb7 + be.size()));
        out.insert(out.end(), be.begin(), be.end());
    }
    out.insert(out.end(), b, b + n);
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
    // keccak(0x80), the empty trie's root, and keccak(""), the empty code's hash
    static constexpr Hash32 kEmptyRoot = {0x56, 0xe8, 0x1f, 0x17, 0x1b, 0xcc, 0x55, 0xa6, 0xff, 0x83, 0x45, 0xe6, 0x92, 0xc0, 0xf8, 0x6e,
                                          0x5b, 0x48, 0xe0, 0x1b, 0x99, 0x6c, 0xad, 0xc0, 0x01, 0x62, 0x2f, 0xb5, 0xe3, 0x63, 0xb4, 0x21};
    static constexpr Hash32 kEmptyCode = {0xc5, 0xd2, 0x46, 0x01, 0x86, 0xf7, 0x23, 0x3c, 0x92, 0x7e, 0x7d, 0xb2, 0xdc, 0xc7, 0x03, 0xc0,
                                          0xe5, 0x00, 0xb6, 0x53, 0xca, 0x82, 0x27, 0x3b, 0x7b, 0xfa, 0xd8, 0x04, 0x5d, 0x85, 0xa4, 0x70};

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
    // A new, independent state holding exactly what revert(back) would return to (back = 0: a copy of the state as it is
    // now); this one is not changed.  Every call works on the fork at that root -- getProofs, getTrieNodes, the range proofs,
    // witness, and apply for a side branch -- so a snap pivot or a recent block is served while this state moves on.  The
    // fork starts with no journal and an empty code store and shares no device memory with this state: either may be
    // destroyed first.
    std::unique_ptr<ResidentStateTrie> fork(uint32_t back = 0)
    {
        phant_gpu_resident_state* f = nullptr;
        g_.check(phant_gpu_resident_state_fork(s_, back, &f), "ResidentStateTrie fork");
        return std::unique_ptr<ResidentStateTrie>(new ResidentStateTrie(g_, f));
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
    // eth_getProof (EIP-1186) under the state as it is now (which is not changed): per requested address, the account proof and
    // fields and a proof of each requested slot (32-byte big-endian slot numbers), each proof a list of nodes, root first.  An
    // absent account gets the fields of an empty account -- nonce 0, balance 0, the empty trie root and keccak("") -- with a
    // proof of its absence; its slots have value 0 and empty proofs (they hang from the empty root).
    struct StorageProof {
        std::array<uint8_t, 32> key, value;
        std::vector<Bytes> proof;
    };
    struct AccountProof {
        std::vector<Bytes> accountProof;
        uint64_t nonce = 0;
        std::array<uint8_t, 32> balance{};
        Hash32 storageHash{}, codeHash{};
        std::vector<StorageProof> storageProof;
    };
    using ProofRequests = std::map<Address, std::vector<std::array<uint8_t, 32>>>;
    std::map<Address, AccountProof> getProofs(const ProofRequests& requests)
    {
        std::map<Address, AccountProof> out;
        if (requests.empty()) return out;
        const HashedRequest hq(g_, requests);
        const phant_gpu_proof_request q = hq.view();
        const uint64_t na = q.n_accounts, ms = q.n_slots, np = na + ms;
        phant_gpu_proof_size size{};
        g_.check(phant_gpu_resident_state_prove(s_, &q, &size), "ResidentStateTrie getProofs");
        Bytes nodes(size.nodes_bytes + 1), status(np), roots(32 * np), bal(32 * na), sroot(32 * na), code(32 * na), vals(32 * ms + 1);
        std::vector<uint64_t> off(size.n_nodes + 1), index(size.n_refs + 1), first(np + 1), nonce(na);
        phant_gpu_proofs r{nodes.data(), off.data(), index.data(), first.data(), roots.data(), status.data(), nonce.data(), bal.data(),
                           sroot.data(), code.data(), vals.data()};
        g_.check(phant_gpu_resident_state_prove_copy(s_, &r), "ResidentStateTrie getProofs copy");
        auto chain = [&](uint64_t p) {
            std::vector<Bytes> c;
            for (uint64_t e = first[p]; e < first[p + 1]; ++e) c.emplace_back(nodes.begin() + off[index[e]], nodes.begin() + off[index[e] + 1]);
            return c;
        };
        uint64_t i = 0, j = 0;
        for (const auto& [a, ks] : requests) {
            AccountProof& p = out[a];
            p.accountProof = chain(i);
            p.nonce = nonce[i];
            std::copy(bal.begin() + 32 * i, bal.begin() + 32 * i + 32, p.balance.begin());
            p.storageHash = kEmptyRoot;
            p.codeHash = kEmptyCode;
            if (status[i] == 1) {
                std::copy(sroot.begin() + 32 * i, sroot.begin() + 32 * i + 32, p.storageHash.begin());
                std::copy(code.begin() + 32 * i, code.begin() + 32 * i + 32, p.codeHash.begin());
            }
            for (const auto& k : ks) {
                StorageProof sp{k, {}, chain(na + j)};
                std::copy(vals.begin() + 32 * j, vals.begin() + 32 * j + 32, sp.value.begin());
                p.storageProof.push_back(std::move(sp));
                ++j;
            }
            ++i;
        }
        return out;
    }
    // snap GetTrieNodes at the state as it is now (compare root() with the request's root first: past roots are not served),
    // for a healing peer.  Pathsets as the wire carries them: {path} for a node of the account trie, {account hash (32 bytes),
    // path, ...} for nodes of that account's storage trie, each path compact-encoded (hex-prefix, flag nibble 0 even / 1 odd).
    // Returns one blob per path in request order: the node's RLP (the root, or a node its parent references by hash), empty
    // when there is no such node or the path does not decode.  It stops after the blob that takes the running total past
    // maxBytes.
    using PathSet = std::vector<Bytes>;
    std::vector<Bytes> getTrieNodes(const std::vector<PathSet>& pathsets, uint64_t maxBytes = 2u << 20)
    {
        std::map<Hash32, uint32_t> owner; // account hash -> index into the request's storage accounts
        std::vector<Hash32> owners;
        std::vector<int64_t> slot; // per path: its index in the device request, or -1
        Bytes paths, lens;
        std::vector<uint32_t> tries;
        for (const PathSet& ps : pathsets) {
            if (ps.empty()) continue;
            int64_t trie = 0;
            if (ps.size() > 1) {
                trie = -1;
                if (ps[0].size() == 32) {
                    Hash32 h;
                    std::copy(ps[0].begin(), ps[0].end(), h.begin());
                    auto it = owner.emplace(h, (uint32_t)owners.size()).first;
                    if (it->second == owners.size()) owners.push_back(h);
                    trie = 1 + it->second;
                }
            }
            for (size_t e = ps.size() > 1 ? 1 : 0; e < ps.size(); ++e) {
                uint8_t packed[32], n = 0;
                if (trie < 0 || !compactPath(ps[e], packed, n)) { slot.push_back(-1); continue; }
                slot.push_back((int64_t)lens.size());
                paths.insert(paths.end(), packed, packed + 32);
                lens.push_back(n);
                tries.push_back((uint32_t)trie);
            }
        }
        Bytes status, nodes;
        std::vector<uint64_t> off;
        if (!lens.empty()) {
            Bytes accts;
            for (const Hash32& h : owners) accts.insert(accts.end(), h.begin(), h.end());
            const phant_gpu_trie_node_request q{lens.size(), paths.data(), lens.data(), tries.data(), owners.size(),
                                                owners.empty() ? nullptr : accts.data()};
            phant_gpu_witness_size size{};
            g_.check(phant_gpu_resident_state_trie_nodes(s_, &q, &size), "ResidentStateTrie getTrieNodes");
            status.resize(lens.size());
            off.resize(lens.size() + 1);
            nodes.resize(size.nodes_bytes + 1);
            phant_gpu_trie_nodes r{status.data(), off.data(), nodes.data()};
            g_.check(phant_gpu_resident_state_trie_nodes_copy(s_, &r), "ResidentStateTrie getTrieNodes copy");
        }
        std::vector<Bytes> out;
        uint64_t total = 0;
        for (int64_t j : slot) {
            out.emplace_back();
            if (j >= 0 && status[j] == 1) out.back().assign(nodes.begin() + off[j], nodes.begin() + off[j + 1]);
            total += out.back().size();
            if (total > maxBytes) break;
        }
        return out;
    }
    // snap GetAccountRange / GetStorageRanges answered as a snap server puts them on the wire (DESIGN.md §4.3m), at the state
    // as it is now: an empty answer when `root` is not the current root (serve a pivot through fork()).  Budgets are capped
    // at 2 MiB, as geth's softResponseLimit.  Entries are (hashed key, body): an account's slim body rlp([nonce, balance,
    // storageRoot or "", codeHash or ""]), a slot's rlp(trimmed value).  The proof is the origin's chain, root first, then the
    // last entry's nodes not already listed.
    using SnapEntries = std::vector<std::pair<Hash32, Bytes>>;
    struct SnapAccountAnswer {
        SnapEntries accounts;
        std::vector<Bytes> proof;
    };
    struct SnapStorageAnswer {
        std::vector<SnapEntries> slots; // one list per served account, in request order
        std::vector<Bytes> proof;       // when not empty: the last served account's, whose list is partial
    };
    static constexpr uint64_t kSnapSoftLimit = 2u << 20;
    SnapAccountAnswer snapAccountRange(const Hash32& root, const Hash32& origin, const Hash32& limit, uint64_t bytes = kSnapSoftLimit)
    {
        SnapAccountAnswer a;
        if (root != this->root()) return a;
        const uint64_t b = std::min(bytes, kSnapSoftLimit);
        const phant_gpu_snap_request q{1, origin.data(), limit.data(), &b, 0, nullptr, nullptr, nullptr, nullptr, nullptr};
        SnapCopy r = snapCall(q);
        a.accounts = r.entries(r.account_keys, r.account_bodies, r.account_off, r.account_first[0], r.account_first[1]);
        a.proof = r.proof(0);
        return a;
    }
    SnapStorageAnswer snapStorageRanges(const Hash32& root, const std::vector<Hash32>& accounts, const Hash32& origin, const Hash32& limit,
                                        uint64_t bytes = kSnapSoftLimit)
    {
        SnapStorageAnswer a;
        if (root != this->root()) return a;
        const uint64_t b = std::min(bytes, kSnapSoftLimit), first[2] = {0, accounts.size()};
        Bytes accts;
        for (const Hash32& h : accounts) accts.insert(accts.end(), h.begin(), h.end());
        const phant_gpu_snap_request q{0, nullptr, nullptr, nullptr, 1, first, accts.empty() ? nullptr : accts.data(), origin.data(), limit.data(), &b};
        SnapCopy r = snapCall(q);
        for (uint64_t s = r.served_first[0]; s < r.served_first[1]; ++s)
            a.slots.push_back(r.entries(r.slot_keys, r.slot_bodies, r.slot_off, r.slot_first[s], r.slot_first[s + 1]));
        a.proof = r.proof(0);
        return a;
    }
private:
    // one snap_ranges call copied to the host
    struct SnapCopy {
        std::vector<uint64_t> account_first, account_off, served_first, slot_first, slot_off, proof_first, node_index, node_off;
        Bytes account_keys, account_bodies, slot_keys, slot_bodies, nodes;
        SnapEntries entries(const Bytes& keys, const Bytes& bodies, const std::vector<uint64_t>& off, uint64_t a, uint64_t b) const
        {
            SnapEntries out;
            for (uint64_t e = a; e < b; ++e) {
                Hash32 k;
                std::copy(keys.begin() + 32 * e, keys.begin() + 32 * e + 32, k.begin());
                out.emplace_back(k, Bytes(bodies.begin() + off[e], bodies.begin() + off[e + 1]));
            }
            return out;
        }
        std::vector<Bytes> proof(uint64_t r) const
        {
            std::vector<Bytes> out;
            for (uint64_t e = proof_first[r]; e < proof_first[r + 1]; ++e)
                out.emplace_back(nodes.begin() + node_off[node_index[e]], nodes.begin() + node_off[node_index[e] + 1]);
            return out;
        }
    };
    SnapCopy snapCall(const phant_gpu_snap_request& q)
    {
        phant_gpu_snap_size size{};
        g_.check(phant_gpu_resident_state_snap_ranges(s_, &q, &size), "ResidentStateTrie snap_ranges");
        const uint64_t n = q.n_account_requests, m = q.n_storage_requests;
        SnapCopy r;
        r.account_first.resize(n + 1); r.account_keys.resize(32 * size.n_accounts + 1); r.account_off.resize(size.n_accounts + 1);
        r.account_bodies.resize(size.account_bytes + 1); r.served_first.resize(m + 1); r.slot_first.resize(size.n_served + 1);
        r.slot_keys.resize(32 * size.n_slots + 1); r.slot_off.resize(size.n_slots + 1); r.slot_bodies.resize(size.slot_bytes + 1);
        r.proof_first.resize(n + m + 1); r.node_index.resize(size.n_refs + 1); r.nodes.resize(size.nodes_bytes + 1);
        r.node_off.resize(size.n_nodes + 1);
        phant_gpu_snap_ranges o{r.account_first.data(), r.account_keys.data(), r.account_off.data(), r.account_bodies.data(), r.served_first.data(),
                                r.slot_first.data(), r.slot_keys.data(), r.slot_off.data(), r.slot_bodies.data(), r.proof_first.data(),
                                r.node_index.data(), r.nodes.data(), r.node_off.data()};
        g_.check(phant_gpu_resident_state_snap_ranges_copy(s_, &o), "ResidentStateTrie snap_ranges copy");
        return r;
    }

public:
    // eth_getBalance / eth_getTransactionCount / eth_getStorageAt (and the codeHash behind eth_getCode) for many addresses in
    // one call, with no proof: at the state as it is now (back = 0) or as it was `back` applies ago (1 <= back <= the
    // journal's applies), which is not changed.  An absent account gets the fields of an empty account and value 0 for its
    // slots, as in getProofs.
    struct AccountValues {
        bool exists = false;
        uint64_t nonce = 0;
        std::array<uint8_t, 32> balance{};
        Hash32 storageHash{}, codeHash{};
        std::map<std::array<uint8_t, 32>, std::array<uint8_t, 32>> storage; // slot number -> value, big endian
    };
    std::map<Address, AccountValues> read(const ProofRequests& requests, uint32_t back = 0)
    {
        std::map<Address, AccountValues> out;
        if (requests.empty()) return out;
        const HashedRequest hq(g_, requests);
        const phant_gpu_proof_request q = hq.view();
        const uint64_t na = q.n_accounts, ms = q.n_slots;
        Bytes status(na), bal(32 * na), sroot(32 * na), code(32 * na), vals(32 * ms + 1);
        std::vector<uint64_t> nonce(na);
        phant_gpu_state_read_values v{status.data(), nonce.data(), bal.data(), sroot.data(), code.data(), nullptr, vals.data()};
        Hash32 root;
        g_.check(phant_gpu_resident_state_read(s_, &q, back, &v, root.data()), "ResidentStateTrie read");
        uint64_t i = 0, j = 0;
        for (const auto& [a, ks] : requests) {
            AccountValues& r = out[a];
            r.exists = status[i] == 1;
            r.nonce = nonce[i];
            std::copy(bal.begin() + 32 * i, bal.begin() + 32 * i + 32, r.balance.begin());
            r.storageHash = kEmptyRoot;
            r.codeHash = kEmptyCode;
            if (r.exists) {
                std::copy(sroot.begin() + 32 * i, sroot.begin() + 32 * i + 32, r.storageHash.begin());
                std::copy(code.begin() + 32 * i, code.begin() + 32 * i + 32, r.codeHash.begin());
            }
            for (const auto& k : ks) {
                std::copy(vals.begin() + 32 * j, vals.begin() + 32 * j + 32, r.storage[k].begin());
                ++j;
            }
            ++i;
        }
        return out;
    }
    // Contract code kept on the device beside the state, by keccak(code) (DESIGN.md §4.3i), for getCode, witnessCodes and
    // snap's GetByteCodes: put a block's new code before its apply.  A code already held is stored once, the empty code never.
    // Returns the hashes, in order.  Codes stay until pruneCodes finds no root the journal reaches that names them.
    std::vector<Hash32> putCodes(const std::vector<Bytes>& codes)
    {
        std::vector<Hash32> out(codes.size());
        if (codes.empty()) return out;
        Bytes all;
        std::vector<uint64_t> off{0};
        for (const Bytes& c : codes) {
            all.insert(all.end(), c.begin(), c.end());
            off.push_back(all.size());
        }
        all.push_back(0);
        g_.check(phant_gpu_resident_state_put_codes(s_, all.data(), off.data(), codes.size(), out[0].data()), "ResidentStateTrie putCodes");
        return out;
    }
    // snap GetByteCodes: the code behind each hash; nullopt where the store does not hold it (keccak("") is held: empty).
    std::vector<std::optional<Bytes>> codes(const std::vector<Hash32>& hashes)
    {
        const uint64_t n = hashes.size();
        std::vector<std::optional<Bytes>> out(n);
        if (!n) return out;
        Bytes status(n);
        std::vector<uint64_t> off(n + 1);
        g_.check(phant_gpu_resident_state_codes(s_, hashes[0].data(), n, status.data(), off.data(), nullptr, 0), "ResidentStateTrie codes");
        Bytes all(off[n] + 1);
        if (off[n]) g_.check(phant_gpu_resident_state_codes(s_, hashes[0].data(), n, status.data(), off.data(), all.data(), off[n]), "ResidentStateTrie codes");
        for (uint64_t i = 0; i < n; ++i)
            if (status[i] == 1) out[i] = Bytes(all.begin() + off[i], all.begin() + off[i + 1]);
        return out;
    }
    // eth_getCode for many addresses at the state as it is now (back = 0) or `back` applies ago: read's codeHash, then codes.
    // An absent account or one without code gives an empty code; nullopt when the store does not hold the code named.
    std::map<Address, std::optional<Bytes>> getCode(const std::vector<Address>& addresses, uint32_t back = 0)
    {
        std::map<Address, std::optional<Bytes>> out;
        if (addresses.empty()) return out;
        ProofRequests req;
        for (const Address& a : addresses) req[a];
        std::vector<Address> order;
        std::vector<Hash32> hashes;
        for (const auto& [a, v] : read(req, back)) {
            order.push_back(a);
            hashes.push_back(v.codeHash);
        }
        const std::vector<std::optional<Bytes>> got = codes(hashes);
        for (size_t i = 0; i < order.size(); ++i) out[order[i]] = got[i];
        return out;
    }
    // Drop the held codes that no account names now or at any root revert can return to.
    void pruneCodes() { g_.check(phant_gpu_resident_state_prune_codes(s_), "ResidentStateTrie pruneCodes"); }
    // The `codes` of the execution witness of the block apply() would take with `touched`: the distinct codes of every touched
    // account present now with code, ordered by hash.  Throws GpuError(PHANT_GPU_E_INVALID) naming the addresses whose code the
    // store does not hold: a witness without it could not be executed.
    std::vector<Bytes> witnessCodes(const std::map<Address, const AccountState*>& touched)
    {
        std::vector<Address> addrs;
        for (const auto& kv : touched) addrs.push_back(kv.first);
        std::map<Hash32, std::vector<Address>> by_hash;
        ProofRequests req;
        for (const Address& a : addrs) req[a];
        if (!req.empty())
            for (const auto& [a, v] : read(req))
                if (v.exists && v.codeHash != kEmptyCode) by_hash[v.codeHash].push_back(a);
        std::vector<Hash32> hashes;
        for (const auto& kv : by_hash) hashes.push_back(kv.first);
        const std::vector<std::optional<Bytes>> got = codes(hashes);
        std::vector<Bytes> out;
        std::string missing;
        for (size_t i = 0; i < hashes.size(); ++i) {
            if (got[i]) { out.push_back(*got[i]); continue; }
            for (const Address& a : by_hash[hashes[i]]) {
                missing += missing.empty() ? " 0x" : ", 0x";
                for (uint8_t b : a) { static const char* hx = "0123456789abcdef"; missing += hx[b >> 4]; missing += hx[b & 15]; }
            }
        }
        if (!missing.empty()) throw GpuError(PHANT_GPU_E_INVALID, "ResidentStateTrie witnessCodes: the code store does not hold the code of" + missing);
        return out;
    }
    // debug_accountRange / debug_storageRangeAt / snap's GetAccountRange and GetStorageRanges without proofs: the first `max`
    // keys in [origin, limit] (hashed keys, inclusive, ascending) at the state as it is now (back = 0) or `back` applies ago,
    // which is not changed; `more` says whether the range holds further keys.  Keys stay hashed: the state holds no preimages.
    struct AccountEntry {
        Hash32 key{};
        uint64_t nonce = 0;
        std::array<uint8_t, 32> balance{};
        Hash32 storageHash{}, codeHash{};
    };
    struct AccountRange {
        std::vector<AccountEntry> accounts;
        bool more = false;
    };
    struct SlotRange {
        std::vector<std::pair<Hash32, std::array<uint8_t, 32>>> slots; // hashed slot, value (big endian, never zero)
        bool more = false;
    };
    AccountRange accountRange(const Hash32& origin, const Hash32& limit, uint32_t max, uint32_t back = 0)
    {
        return std::move(range({{origin, limit, max}}, {}, back).first[0]);
    }
    SlotRange storageRange(const Address& address, const Hash32& origin, const Hash32& limit, uint32_t max, uint32_t back = 0)
    {
        const Hash32 akey = hasher::keccak256_batch(g_, {Bytes(address.begin(), address.end())})[0];
        return std::move(range({}, {{akey, origin, limit, max}}, back).second[0]);
    }
    // The whole state now or `back` applies ago, in calls of at most `chunk` entries: the accounts range by range, then the
    // slots of every account whose storageRoot is not the empty root, many accounts per call.  hashed address -> account.
    struct DumpAccount {
        AccountEntry fields;
        std::map<Hash32, std::array<uint8_t, 32>> storage; // hashed slot -> value
    };
    std::map<Hash32, DumpAccount> dump(uint32_t back = 0, uint32_t chunk = 1u << 20)
    {
        std::map<Hash32, DumpAccount> out;
        std::vector<std::pair<Hash32, Hash32>> pending; // (account, next origin)
        Hash32 origin{}, all;
        all.fill(0xff);
        for (;;) {
            AccountRange r = std::move(range({{origin, all, chunk}}, {}, back).first[0]);
            for (const AccountEntry& e : r.accounts) {
                out[e.key].fields = e;
                if (e.storageHash != kEmptyRoot) pending.push_back({e.key, Hash32{}});
            }
            if (!r.more) break;
            origin = next(r.accounts.back().key);
        }
        while (!pending.empty()) {
            const size_t nb = std::min<size_t>(pending.size(), chunk);
            const uint32_t each = std::max<uint32_t>(chunk / (uint32_t)nb, 1);
            std::vector<SlotRequest> req;
            for (size_t i = 0; i < nb; ++i) req.push_back({pending[i].first, pending[i].second, all, each});
            std::vector<SlotRange> got = range({}, req, back).second;
            pending.erase(pending.begin(), pending.begin() + nb);
            for (size_t i = 0; i < nb; ++i) {
                auto& st = out[req[i].account].storage;
                for (const auto& [k, v] : got[i].slots) st[k] = v;
                if (got[i].more) pending.push_back({req[i].account, next(got[i].slots.back().first)});
            }
        }
        return out;
    }

    // snap's GetAccountRange / GetStorageRanges for one account at the current root: accountRange / storageRange plus the
    // boundary proofs, one prove call on the origin and the last key returned (once when they are the same key).  `proof` is
    // the proofs' node set (a storage range's also holds its account's proof); snap::verifyAccountRange /
    // verifyStorageRanges take it as it is.
    struct AccountRangeProof {
        AccountRange range;
        std::vector<Bytes> proof;
    };
    struct SlotRangeProof {
        SlotRange range;
        std::vector<Bytes> proof;
    };
    AccountRangeProof accountRangeProof(const Hash32& origin, const Hash32& limit, uint32_t max)
    {
        AccountRangeProof p{accountRange(origin, limit, max), {}};
        Bytes k32(origin.begin(), origin.end());
        if (!p.range.accounts.empty() && p.range.accounts.back().key != origin)
            k32.insert(k32.end(), p.range.accounts.back().key.begin(), p.range.accounts.back().key.end());
        p.proof = proveNodes(k32, {}, {});
        return p;
    }
    SlotRangeProof storageRangeProof(const Address& address, const Hash32& origin, const Hash32& limit, uint32_t max)
    {
        SlotRangeProof p{storageRange(address, origin, limit, max), {}};
        const Hash32 akey = hasher::keccak256_batch(g_, {Bytes(address.begin(), address.end())})[0];
        Bytes s32(origin.begin(), origin.end());
        if (!p.range.slots.empty() && p.range.slots.back().first != origin)
            s32.insert(s32.end(), p.range.slots.back().first.begin(), p.range.slots.back().first.end());
        p.proof = proveNodes(Bytes(akey.begin(), akey.end()), std::vector<uint32_t>(s32.size() / 32, 0), s32);
        return p;
    }

private:
    // one prove call on hashed keys: the node set of every chain
    std::vector<Bytes> proveNodes(const Bytes& k32, const std::vector<uint32_t>& slot_account, const Bytes& s32)
    {
        const phant_gpu_proof_request q{k32.size() / 32, k32.data(), slot_account.size(), slot_account.data(), s32.data()};
        const uint64_t na = q.n_accounts, ms = q.n_slots, np = na + ms;
        phant_gpu_proof_size size{};
        g_.check(phant_gpu_resident_state_prove(s_, &q, &size), "ResidentStateTrie prove");
        Bytes nodes(size.nodes_bytes + 1), status(np), roots(32 * np), bal(32 * na), sroot(32 * na), code(32 * na), vals(32 * ms + 1);
        std::vector<uint64_t> off(size.n_nodes + 1), index(size.n_refs + 1), first(np + 1), nonce(na);
        phant_gpu_proofs r{nodes.data(), off.data(), index.data(), first.data(), roots.data(), status.data(), nonce.data(), bal.data(),
                           sroot.data(), code.data(), vals.data()};
        g_.check(phant_gpu_resident_state_prove_copy(s_, &r), "ResidentStateTrie prove copy");
        std::vector<Bytes> out;
        for (uint64_t i = 0; i < size.n_nodes; ++i) out.emplace_back(nodes.begin() + off[i], nodes.begin() + off[i + 1]);
        return out;
    }
    struct AccountRequest { Hash32 origin, limit; uint32_t max; };
    struct SlotRequest { Hash32 account, origin, limit; uint32_t max; };
    static Hash32 next(Hash32 k) // the hashed key after k (never the last key when more follows it)
    {
        for (int i = 31; i >= 0 && ++k[i] == 0; --i) {}
        return k;
    }
    // one phant_gpu_resident_state_range call
    std::pair<std::vector<AccountRange>, std::vector<SlotRange>> range(const std::vector<AccountRequest>& ar, const std::vector<SlotRequest>& sr,
                                                                       uint32_t back)
    {
        const size_t n = ar.size(), m = sr.size();
        Bytes ao, al, sa, so, sl;
        std::vector<uint32_t> amax, smax;
        uint64_t ea = 0, es = 0;
        for (const AccountRequest& r : ar) {
            ao.insert(ao.end(), r.origin.begin(), r.origin.end());
            al.insert(al.end(), r.limit.begin(), r.limit.end());
            amax.push_back(r.max);
            ea += r.max;
        }
        for (const SlotRequest& r : sr) {
            sa.insert(sa.end(), r.account.begin(), r.account.end());
            so.insert(so.end(), r.origin.begin(), r.origin.end());
            sl.insert(sl.end(), r.limit.begin(), r.limit.end());
            smax.push_back(r.max);
            es += r.max;
        }
        const phant_gpu_range_request q{n, ao.data(), al.data(), amax.data(), m, sa.data(), so.data(), sl.data(), smax.data()};
        std::vector<uint64_t> afirst(n + 1), sfirst(m + 1), nonce(ea + 1);
        Bytes amore(n + 1), smore(m + 1), akeys(32 * ea + 1), bal(32 * ea + 1), sroot(32 * ea + 1), code(32 * ea + 1), skeys(32 * es + 1), svals(32 * es + 1);
        phant_gpu_range_values v{afirst.data(), amore.data(), akeys.data(), nonce.data(), bal.data(), sroot.data(), code.data(),
                                 sfirst.data(), smore.data(), skeys.data(), svals.data()};
        Hash32 root;
        g_.check(phant_gpu_resident_state_range(s_, &q, back, &v, root.data()), "ResidentStateTrie range");
        std::pair<std::vector<AccountRange>, std::vector<SlotRange>> out;
        out.first.resize(n);
        out.second.resize(m);
        auto at = [](const Bytes& b, uint64_t e) { Hash32 h; std::copy(b.begin() + 32 * e, b.begin() + 32 * e + 32, h.begin()); return h; };
        for (size_t r = 0; r < n; ++r) {
            out.first[r].more = amore[r];
            for (uint64_t e = afirst[r]; e < afirst[r + 1]; ++e)
                out.first[r].accounts.push_back({at(akeys, e), nonce[e], at(bal, e), at(sroot, e), at(code, e)});
        }
        for (size_t r = 0; r < m; ++r) {
            out.second[r].more = smore[r];
            for (uint64_t e = sfirst[r]; e < sfirst[r + 1]; ++e) out.second[r].slots.push_back({at(skeys, e), at(svals, e)});
        }
        return out;
    }
    // a request's addresses and slot numbers hashed on the device, laid out for prove and read
    struct HashedRequest {
        Bytes k32, s32;
        std::vector<uint32_t> slot_account;
        HashedRequest(Gpu& g, const ProofRequests& requests)
        {
            std::vector<Bytes> addrs, slots;
            for (const auto& [a, ks] : requests) {
                for (const auto& k : ks) { slot_account.push_back((uint32_t)addrs.size()); slots.emplace_back(k.begin(), k.end()); }
                addrs.emplace_back(a.begin(), a.end());
            }
            for (const Hash32& h : hasher::keccak256_batch(g, addrs)) k32.insert(k32.end(), h.begin(), h.end());
            if (!slots.empty())
                for (const Hash32& h : hasher::keccak256_batch(g, slots)) s32.insert(s32.end(), h.begin(), h.end());
        }
        phant_gpu_proof_request view() const { return {k32.size() / 32, k32.data(), slot_account.size(), slot_account.data(), s32.data()}; }
    };
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
    // a compact-encoded trie path (flag nibble 0 even / 1 odd) -> its nibbles packed high nibble first, zero padded, and their
    // count; false when it does not decode as one or holds more than 64 nibbles
    static bool compactPath(const Bytes& c, uint8_t packed[32], uint8_t& n)
    {
        if (c.empty() || (c[0] >> 4) > 1 || ((c[0] >> 4) == 0 && (c[0] & 15))) return false;
        const bool odd = (c[0] >> 4) == 1;
        const size_t count = 2 * (c.size() - 1) + (odd ? 1 : 0);
        if (count > 64) return false;
        std::fill(packed, packed + 32, 0);
        for (size_t i = 0; i < count; ++i) {
            const size_t q = i + (odd ? 1 : 2); // nibble index in the encoded bytes
            const uint8_t v = (q & 1) ? (c[q >> 1] & 15) : (c[q >> 1] >> 4);
            packed[i >> 1] |= (i & 1) ? v : (uint8_t)(v << 4);
        }
        n = (uint8_t)count;
        return true;
    }
    ResidentStateTrie(Gpu& g, phant_gpu_resident_state* s) : g_(g), s_(s) {} // owns s (a fork)
    Gpu& g_;
    phant_gpu_resident_state* s_ = nullptr;
    uint32_t journal_ = 0;
};
} // namespace state

// ---- range proofs (phant_gpu_verify_ranges): a snap client's check of GetAccountRange / GetStorageRanges answers from a peer,
// taking what ResidentStateTrie::accountRangeProof / storageRangeProof return ----
namespace snap {
struct RangeStatus {
    uint8_t status; // 1 the entries are exactly the trie's contents in [origin, last] / 0 they are not / 3 a node is missing
    bool more;      // an accepted range's trie holds a key after its last entry
};
struct LeafRange {
    Hash32 root{}, origin{};
    std::vector<std::pair<Hash32, Bytes>> entries; // hashed key, leaf value bytes; ascending
    bool whole = false;                            // no boundary proof: the entries are the whole trie
};
// many ranges in one call over one node set holding every proven range's boundary proofs
inline std::vector<RangeStatus> verifyRanges(Gpu& g, const std::vector<LeafRange>& ranges, const std::vector<Bytes>& nodes)
{
    std::vector<RangeStatus> out(ranges.size());
    if (ranges.empty()) return out;
    Bytes ndata, roots, origins, flags, keys, vals;
    std::vector<uint64_t> noff(1, 0), first(1, 0), voff(1, 0);
    for (const Bytes& b : nodes) { ndata.insert(ndata.end(), b.begin(), b.end()); noff.push_back(ndata.size()); }
    for (const LeafRange& r : ranges) {
        roots.insert(roots.end(), r.root.begin(), r.root.end());
        origins.insert(origins.end(), r.origin.begin(), r.origin.end());
        flags.push_back(r.whole ? PHANT_GPU_RANGE_WHOLE : 0);
        for (const auto& [k, v] : r.entries) {
            keys.insert(keys.end(), k.begin(), k.end());
            vals.insert(vals.end(), v.begin(), v.end());
            voff.push_back(vals.size());
        }
        first.push_back(voff.size() - 1);
    }
    phant_gpu_range_proofs in{};
    in.n_nodes = nodes.size(); in.nodes = ndata.data(); in.node_off = noff.data(); in.nodes_bytes = ndata.size();
    in.n_ranges = ranges.size(); in.roots32 = roots.data(); in.origin32 = origins.data(); in.range_flags = flags.data();
    in.entry_first = first.data(); in.keys32 = keys.data(); in.vals = vals.data(); in.val_off = voff.data();
    Bytes status(ranges.size()), more(ranges.size());
    g.check(phant_gpu_verify_ranges(g.ctx(), &in, status.data(), more.data()), "snap verifyRanges");
    for (size_t r = 0; r < ranges.size(); ++r) out[r] = {status[r], more[r] != 0};
    return out;
}
// an account's leaf value: rlp([nonce, balance, storageRoot, codeHash])
inline Bytes accountValue(const state::ResidentStateTrie::AccountEntry& a)
{
    Bytes p = rlp::encode_uint(a.nonce);
    for (const Bytes& x : {rlp::encode_bytes(a.balance.data(), 32, true), rlp::encode_bytes(a.storageHash.data(), 32),
                           rlp::encode_bytes(a.codeHash.data(), 32)})
        p.insert(p.end(), x.begin(), x.end());
    return rlp::wrap_list(p);
}
// A GetAccountRange answer against the state root: (ok, more) -- ok when the accounts are exactly the state's accounts from
// `origin` to the last of them, more when accounts follow it.
inline std::pair<bool, bool> verifyAccountRange(Gpu& g, const Hash32& root, const Hash32& origin,
                                                const std::vector<state::ResidentStateTrie::AccountEntry>& accounts, const std::vector<Bytes>& proof)
{
    LeafRange r{root, origin, {}, false};
    for (const auto& a : accounts) r.entries.push_back({a.key, accountValue(a)});
    const RangeStatus s = verifyRanges(g, {r}, proof)[0];
    return {s.status == 1, s.more};
}
// A GetStorageRanges answer: per range its account's storageRoot, its origin and its slots (hashed slot, value).  Every range
// but the last is a whole storage trie; the last is too unless last_is_partial, when `proof` proves it from its origin.
struct StorageRangeAnswer {
    Hash32 storageRoot{}, origin{};
    std::vector<std::pair<Hash32, std::array<uint8_t, 32>>> slots;
};
inline std::vector<std::pair<bool, bool>> verifyStorageRanges(Gpu& g, const std::vector<StorageRangeAnswer>& ranges, const std::vector<Bytes>& proof,
                                                              bool last_is_partial)
{
    std::vector<LeafRange> rs;
    for (size_t i = 0; i < ranges.size(); ++i) {
        LeafRange r{ranges[i].storageRoot, ranges[i].origin, {}, !(last_is_partial && i + 1 == ranges.size())};
        for (const auto& [k, v] : ranges[i].slots) r.entries.push_back({k, rlp::encode_bytes(v.data(), 32, true)});
        rs.push_back(std::move(r));
    }
    std::vector<std::pair<bool, bool>> out;
    for (const RangeStatus& s : verifyRanges(g, rs, last_is_partial ? proof : std::vector<Bytes>{})) out.push_back({s.status == 1, s.more});
    return out;
}
// A snap slim account body rlp([nonce, balance, storageRoot or "", codeHash or ""]) expanded: false when it does not decode as
// four strings of the right lengths.  The empty fields become the empty root and keccak("").
inline bool decodeSlimAccount(const Bytes& b, state::ResidentStateTrie::AccountEntry& a)
{
    auto item = [&](size_t pos, size_t end, size_t& pay, size_t& len) -> size_t { // the item's end, 0 when it is not a short item
        if (pos >= end) return 0;
        const uint8_t x = b[pos];
        if (x < 0x80) { pay = pos; len = 1; return pos + 1; }
        if (x <= 0xb7) { pay = pos + 1; len = x - 0x80; return pay + len <= end ? pay + len : 0; }
        if (x < 0xc0) return 0;
        if (x <= 0xf7) { pay = pos + 1; len = x - 0xc0; }
        else if (x == 0xf8 && pos + 1 < end) { pay = pos + 2; len = b[pos + 1]; }
        else return 0;
        return pay + len <= end ? pay + len : 0;
    };
    size_t pay, len;
    if (b.empty() || b[0] < 0xc0 || item(0, b.size(), pay, len) != b.size()) return false;
    size_t f[4][2], pos = pay;
    for (int i = 0; i < 4; ++i) {
        if (pos < b.size() && b[pos] >= 0xc0) return false;
        const size_t e = item(pos, pay + len, f[i][0], f[i][1]);
        if (!e) return false;
        pos = e;
    }
    if (pos != pay + len || f[0][1] > 8 || f[1][1] > 32 || (f[2][1] != 0 && f[2][1] != 32) || (f[3][1] != 0 && f[3][1] != 32)) return false;
    a.nonce = 0;
    for (size_t i = 0; i < f[0][1]; ++i) a.nonce = a.nonce << 8 | b[f[0][0] + i];
    a.balance.fill(0);
    std::copy(b.begin() + f[1][0], b.begin() + f[1][0] + f[1][1], a.balance.end() - f[1][1]);
    a.storageHash = state::ResidentStateTrie::kEmptyRoot;
    a.codeHash = state::ResidentStateTrie::kEmptyCode;
    if (f[2][1]) std::copy(b.begin() + f[2][0], b.begin() + f[2][0] + 32, a.storageHash.begin());
    if (f[3][1]) std::copy(b.begin() + f[3][0], b.begin() + f[3][0] + 32, a.codeHash.begin());
    return true;
}
// A GetAccountRange answer as ResidentStateTrie::snapAccountRange returns it (slim bodies), checked with G: (ok, more).  A body
// that does not decode is not ok.
inline std::pair<bool, bool> verifySnapAccountRange(Gpu& g, const Hash32& root, const Hash32& origin,
                                                    const state::ResidentStateTrie::SnapEntries& accounts, const std::vector<Bytes>& proof)
{
    LeafRange r{root, origin, {}, false};
    for (const auto& [k, body] : accounts) {
        state::ResidentStateTrie::AccountEntry a;
        if (!decodeSlimAccount(body, a)) return {false, false};
        a.key = k;
        r.entries.push_back({k, accountValue(a)});
    }
    const RangeStatus s = verifyRanges(g, {r}, proof)[0];
    return {s.status == 1, s.more};
}
// A GetStorageRanges answer as snapStorageRanges returns it, checked with G: storageRoots of the served accounts, in order.
// Every list is checked whole, except the last when the answer carries a proof: that one from its origin (the request's
// origin for the first account, else 0).  Returns (ok, more) per list.
inline std::vector<std::pair<bool, bool>> verifySnapStorageRanges(Gpu& g, const std::vector<Hash32>& storageRoots, const Hash32& origin,
                                                                  const std::vector<state::ResidentStateTrie::SnapEntries>& slots,
                                                                  const std::vector<Bytes>& proof)
{
    std::vector<LeafRange> rs;
    for (size_t i = 0; i < slots.size(); ++i) {
        const bool partial = !proof.empty() && i + 1 == slots.size();
        rs.push_back({storageRoots.at(i), i == 0 ? origin : Hash32{}, slots[i], !partial});
    }
    std::vector<std::pair<bool, bool>> out;
    for (const RangeStatus& s : verifyRanges(g, rs, proof)) out.push_back({s.status == 1, s.more});
    return out;
}
} // namespace snap

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
