"""fiatshamir.Transcript (fiat-shamir/transcript.go:19-127): named challenges in a fixed order, each the hash of its name, the raw
value of the challenge before it (all but the first) and the values bound to it, in the order they were bound."""
from __future__ import annotations


class Transcript:
    """NewTranscript(h, challengesID...).  `hf` is a hashlib constructor (e.g. hashlib.sha256): every challenge hashes with a fresh
    object, as the reference resets its hash.Hash before each one."""

    def __init__(self, hf, *challenge_ids: str):
        self._hf = hf
        self._position = {name: i for i, name in enumerate(challenge_ids)}
        self._bindings = {name: [] for name in challenge_ids}
        self._values = {}
        self._previous = None           # (position, raw value) of the last computed challenge

    def Bind(self, challenge_id: str, value: bytes) -> None:
        if challenge_id not in self._position:
            raise ValueError("challenge not recorded in the transcript")
        if challenge_id in self._values:
            raise ValueError("challenge already computed, cannot be binded to other values")
        self._bindings[challenge_id].append(bytes(value))

    def ComputeChallenge(self, challenge_id: str) -> bytes:
        """H(name || previous challenge || bound values), the previous challenge omitted for the first one; the raw digest"""
        if challenge_id not in self._position:
            raise ValueError("challenge not recorded in the transcript")
        if challenge_id in self._values:
            return self._values[challenge_id]
        pos = self._position[challenge_id]
        h = self._hf()
        h.update(challenge_id.encode())
        if pos != 0:
            if self._previous is None or self._previous[0] != pos - 1:
                raise ValueError("the previous challenge is needed and has not been computed")
            h.update(self._previous[1])
        for b in self._bindings[challenge_id]:
            h.update(b)
        value = h.digest()
        self._values[challenge_id] = value
        self._previous = (pos, value)
        return value
