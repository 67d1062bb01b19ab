"""CPU restatement of the inflight-load producer (requestcontrol/dataproducer/inflightload/producer.go) and of the engine's
counters for it: the token estimate, PreRequest over a scheduling call's decisions and details, ResponseBody releases and
endpoint resets.  Negative counts are kept, as the reference's concurrencyTracker keeps them.  The parity tests feed
these counters to the C oracle as ordinary ext columns (token count = column 0, request count = column 1)."""
from __future__ import annotations

import math

import numpy as np

NO = 0xFFFFFFFF
TOKEN_LOAD, ACTIVE_REQUEST = 6, 7
TOKEN_COL, REQUEST_COL = 0, 1


def est(prompt_len: int) -> int:
    """SimpleTokenEstimator.Estimate with RequestSizeBytes = prompt_len (token_estimator.go:55-56, 70-71):
    inputTokens = max(bytes / 4, 1) (integer division), outputTokens = math.Round(inputTokens * 1.5)."""
    i = max(int(prompt_len) // 4, 1)
    x = float(i) * 1.5                                   # exact while i < 2^52
    out = math.floor(x)
    if x - out >= 0.5:                                   # math.Round: halves away from zero
        out += 1
    return i + int(out)


class Counters:
    """InFlightLoad{Requests, Tokens} per slot."""

    def __init__(self, E: int):
        self.req = np.zeros(E, dtype=np.int64)
        self.tok = np.zeros(E, dtype=np.int64)

    def targets(self, dec, det=None, r=0):
        """TargetEndpoints[0] of every profile result of request r: pick, prefill pick, encode pick (those that ran and
        found an endpoint).  A Schedule error (status != 0) has no result, so PreRequest never runs.  dec / det are the
        engine's records or the C oracle's (which writes -1 for "no endpoint")."""
        if int(dec["status"][r]) != 0:
            return []
        eps = [int(dec["pick"][r]), int(dec["prefill_pick"][r])]
        if det is not None:
            eps.append(int(det["encode_pick"][r]))
        return [e & NO for e in eps if e & NO != NO]

    def pre_request(self, dec, lengths, det=None):
        """PreRequest (producer.go:110-129) for every request of one scheduling call."""
        for r in range(len(dec)):
            t = est(int(lengths[r]))
            for e in self.targets(dec, det, r):
                self.req[e] += 1
                self.tok[e] += t

    def release(self, eps, lengths):
        """ResponseBody's release (producer.go:170-178) of each (slot, prompt length); EPP_NO_ENDPOINT is skipped."""
        for e, L in zip(eps, lengths):
            if int(e) == NO:
                continue
            self.req[int(e)] -= 1
            self.tok[int(e)] -= est(int(L))

    def reset(self, ids):
        """DeleteEndpoint (producer.go:189-192): the slot's entries are gone, i.e. read as 0."""
        for e in ids:
            self.req[int(e)] = 0
            self.tok[int(e)] = 0

    def ext(self):
        """[2][E] f64 ext columns: tokens, requests."""
        return np.stack([self.tok, self.req]).astype(np.float64)


class Producer:
    """The reference plugin over endpoint names: PreRequest over a SchedulingResult {profile: [targets]}, ResponseBody with
    StartOfStream / EndOfStream, DeleteEndpoint.  What tests/test_inflight_cpu.py re-encodes producer_test.go with."""

    def __init__(self):
        self.requests, self.tokens = {}, {}

    def get(self, name):
        return self.requests.get(name, 0), self.tokens.get(name, 0)

    def _add(self, name, dr, dt):
        self.requests[name] = self.requests.get(name, 0) + dr
        self.tokens[name] = self.tokens.get(name, 0) + dt

    def PreRequest(self, prompt_len, result):
        for targets in result.values():
            if targets:
                self._add(targets[0], 1, est(prompt_len))

    def ResponseBody(self, prompt_len, result, start_of_stream=False, end_of_stream=False):
        if start_of_stream and result.get("prefill"):
            self._add(result["prefill"][0], -1, -est(prompt_len))
        if end_of_stream:
            for name, targets in result.items():
                if targets and name != "prefill":
                    self._add(targets[0], -1, -est(prompt_len))

    def DeleteEndpoint(self, name):
        self.requests.pop(name, None)
        self.tokens.pop(name, None)
