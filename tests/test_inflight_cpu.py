"""The inflight-load producer's restatement (tools/inflight_model.py) against the reference's own test cases: the token
estimate (token_estimator_test.go), the producer's lifecycle tests (producer_test.go) and the slot counters the engine's
GPU tests compare against.  No GPU."""
import numpy as np

from tools import inflight_model as M


def test_estimate_reference_cases():
    # token_estimator_test.go:53-96, the cases that go through a prompt, with the prompt's bytes as the request size
    assert M.est(len(b"123")) == 3
    assert M.est(len(b"1234")) == 3
    assert M.est(len(b"Hello, world!")) == 8
    assert M.est(0) == 3
    # producer_test.go:76: 16 bytes -> 4 input + 6 output
    assert M.est(16) == 10


def test_estimate_rounding_edges():
    # L = 0..7: one input token (max(L/4, 1)), 2 output tokens (1.5 rounds away from zero)
    assert [M.est(L) for L in range(8)] == [3] * 8
    # i odd: 1.5 i ends in .5 and rounds up; i even: exact
    for i in range(1, 200):
        assert M.est(4 * i) == i + (3 * i + 1) // 2, i
        assert M.est(4 * i + 3) == M.est(4 * i), i       # floor, not round, of L / 4
    assert M.est(8) == 5 and M.est(12) == 8 and M.est(20) == 13
    for L in (2**31 - 1, 2**32, 2**40 + 7, 2**50 + 3):
        i = L // 4
        assert M.est(L) == i + (3 * i + 1) // 2


def test_lifecycle():
    """TestInFlightLoadProducer_Lifecycle (producer_test.go:63-89)."""
    p = M.Producer()
    res = {"default": ["lifecycle-endpoint"]}
    p.PreRequest(16, res)
    assert p.get("lifecycle-endpoint") == (1, 10)
    p.ResponseBody(16, res, end_of_stream=True)
    assert p.get("lifecycle-endpoint") == (0, 0)


def test_multi_pod_lifecycle():
    """TestInFlightLoadProducer_MultiPodLifecycle (producer_test.go:91-129): prefill released at the first chunk,
    decode at the end of the stream."""
    p = M.Producer()
    res = {"prefill": ["pod-a"], "decode": ["pod-b"]}
    p.PreRequest(16, res)
    assert p.get("pod-a") == (1, 10) and p.get("pod-b") == (1, 10)
    p.ResponseBody(16, res, start_of_stream=True)
    assert p.get("pod-a") == (0, 0) and p.get("pod-b") == (1, 10)
    p.ResponseBody(16, res, end_of_stream=True)
    assert p.get("pod-a") == (0, 0) and p.get("pod-b") == (0, 0)
    # a single chunk carrying both flags releases each target once
    p.PreRequest(16, res)
    p.ResponseBody(16, res, start_of_stream=True, end_of_stream=True)
    assert p.get("pod-a") == (0, 0) and p.get("pod-b") == (0, 0)


def test_notification_cleanup_and_release_after_reset():
    """TestInFlightLoadProducer_NotificationCleanup (producer_test.go:131-158), then a release of a request added before
    the delete: the counter goes negative, as concurrencyTracker.add (:221-242) stores it."""
    p = M.Producer()
    p._add("deleted-endpoint", 10, 1000)
    p.DeleteEndpoint("deleted-endpoint")
    assert p.get("deleted-endpoint") == (0, 0)
    p.ResponseBody(16, {"default": ["deleted-endpoint"]}, end_of_stream=True)
    assert p.get("deleted-endpoint") == (-1, -10)


def _dec(rows):
    import epp_b200 as epp
    dec = np.zeros(len(rows), dtype=epp.DECISION_DTYPE)
    det = np.zeros(len(rows), dtype=epp.DETAIL_DTYPE)
    for r, (st, pick, pf, enc) in enumerate(rows):
        dec["status"][r], dec["pick"][r], dec["prefill_pick"][r], det["encode_pick"][r] = st, pick, pf, enc
    return dec, det


def test_counters_pre_request_release_reset():
    NO = M.NO
    c = M.Counters(4)
    dec, det = _dec([(0, 1, NO, NO),      # decode only
                     (0, 2, 2, NO),       # decode and prefill on the same slot: counted twice
                     (-1, NO, NO, NO),    # Schedule error: nothing
                     (0, 0, 3, 1)])       # decode, prefill and encode
    c.pre_request(dec, [16, 4, 100, 40], det)
    np.testing.assert_array_equal(c.req, [1, 2, 2, 1])
    np.testing.assert_array_equal(c.tok, [M.est(40), M.est(16) + M.est(40), 2 * M.est(4), M.est(40)])
    c.release([2, NO, 3], [4, 99, 40])
    np.testing.assert_array_equal(c.req, [1, 2, 1, 0])
    c.reset([1])
    c.release([1], [16])
    np.testing.assert_array_equal(c.req, [1, -1, 1, 0])
    np.testing.assert_array_equal(c.tok, [M.est(40), -M.est(16), M.est(4), 0])
    ext = c.ext()
    assert ext.shape == (2, 4) and ext[M.TOKEN_COL, 1] == -10.0 and ext[M.REQUEST_COL, 1] == -1.0
    # without details there is no encode pick
    c2 = M.Counters(4)
    c2.pre_request(dec, [16, 4, 100, 40])
    np.testing.assert_array_equal(c2.req, [1, 1, 2, 1])
