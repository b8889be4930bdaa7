"""OracleBackedStore + the sequence gather (b2rl_replay_gather_sequences), in numpy,
so that the device EpisodicReplayBuffer's host logic (episode table, eviction,
part liveness, recurrent-state ring, packing) runs on a machine without a GPU.
TEST INFRASTRUCTURE ONLY -- the product has no host fallback.  The packed order
is derived here from pack_sequence itself, not from the kernel's formula."""
import numpy as np
import torch
from torch.nn.utils.rnn import pack_sequence

from fake_store import OracleBackedStore
from pfrl_b200 import _lib


class EpisodicOracleStore(OracleBackedStore):
    def gather_sequences(self, first, length, end, obs_mode=0, obs_scale=1.0,
                         action_dtype=torch.int64, states=None):
        first = np.asarray(first, dtype=np.int64)
        length = np.asarray(length, dtype=np.int32)
        end = np.asarray(end, dtype=np.int64)
        B = len(first)
        live = len(self.records)
        ok = 1 <= B <= _lib.SEQ_MAX_B and all(
            L >= 1 and f >= 0 and f + L <= e <= live for f, L, e in zip(first, length, end)) \
            and all(a >= b for a, b in zip(length, length[1:]))
        if not ok:
            raise _lib.B2rlError(-4, "gather_sequences: invalid sequences")  # B2RL_ERR_RANGE
        # packed position of (b, t): pack the (b, t) labels themselves
        labels = [torch.tensor([[b, t] for t in range(int(L))]) for b, L in enumerate(length)]
        order = pack_sequence(labels).data.numpy()
        recs = [self.records[int(first[b] + t)] for b, t in order]
        out = {}
        for key, slot_key in (("state", "sp"), ("next_state", "nx")):
            raw = np.stack([self.parts[r[slot_key]].reshape(-1) for r in recs])
            if obs_mode == _lib.OBS_U8_TO_F32:
                out[key] = torch.from_numpy(raw.astype(np.float32) * np.float32(obs_scale))
            else:
                out[key] = torch.from_numpy(raw)
        abytes = np.stack([r["action"] for r in recs])
        out["action"] = torch.from_numpy(abytes).view(action_dtype).view(len(recs), -1)
        out["reward"] = torch.tensor([r["rewards"][0] for r in recs],
                                     dtype=torch.float64).float()
        out["is_state_terminal"] = torch.tensor([float(r["terminal"]) for r in recs])
        if states is not None:
            ring, present, leaves = states
            napp = self.napp
            npop = napp - live
            out["state_leaves"], out["next_state_leaves"] = [], []
            for off, d0, inner in leaves:
                for side, key in ((0, "state_leaves"), (1, "next_state_leaves")):
                    o = torch.zeros((d0, B, inner))
                    for b in range(B):
                        row = int((npop + first[b]) % ring.shape[0])
                        if present[row, side]:
                            o[:, b, :] = ring[row, side, off:off + d0 * inner].view(d0, inner)
                    out[key].append(o)
        return out
