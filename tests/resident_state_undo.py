"""What undoes one apply of the resident world state (phant_gpu_resident_state_set_journal / _revert): the inverse diff,
computed from the model BEFORE it applies `diff`.  This is the statement of the undo record the device captures.

  listed account before the apply        the inverse holds
  absent, upserted                       DELETE
  absent, DELETE (a no-op)               nothing
  present, neither DELETE nor CLEAR      its old nonce, balance and codeHash, and the old value of every listed slot (zero
                                         where the slot was absent)
  present, DELETE or CLEAR_STORAGE       its old nonce, balance and codeHash with CLEAR_STORAGE, and every slot it held

The inverse never lists a slot under DELETE nor the same (account, slot) twice: apply accepts it as it is."""
from resident_state_model import CLEAR, DELETE, ZERO32, Diff


def inverse(model, diff):
    listed = {}
    for ai, skey, _ in diff.slots:
        listed.setdefault(ai, []).append(skey)
    accounts, slots = [], []
    for i, (key, flags, _, _, _) in enumerate(diff.accounts):
        a = model.acc.get(key)
        if a is None:
            if not flags & DELETE:
                accounts.append((key, DELETE, 0, ZERO32, ZERO32))
            continue
        j = len(accounts)
        if flags & (DELETE | CLEAR):
            accounts.append((key, CLEAR, a.nonce, a.balance, a.code_hash))
            slots += [(j, skey, v) for skey, v in a.storage.items()]
        else:
            accounts.append((key, 0, a.nonce, a.balance, a.code_hash))
            slots += [(j, skey, a.storage.get(skey, ZERO32)) for skey in listed.get(i, [])]
    return Diff(accounts, slots)


def snapshot(model):
    """the model's accounts as plain values, for exact comparisons"""
    return {k: (a.nonce, a.balance, a.code_hash, dict(a.storage)) for k, a in model.acc.items()}
