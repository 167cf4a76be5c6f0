"""GPU prover service: the reference's own plug-in seam (SURVEY.md §8(b) boundary B3, §8(f) f3).

An unmodified relayer started with `--prover-service-url http://gpu-box:PORT --prover-service-password PW`
(config/src/cli.rs:55-62) sends every proof job as an HTTP POST instead of proving locally
(workers/proof-manager/src/implementations/external_proof_manager/prover_service_client.rs):

    POST <url>/prove-valid-balance-create                    {statement, witness}            -> {proof}
    POST <url>/prove-intent-and-balance-validity             {statement, witness}            -> {proof, link_hint}
    POST <url>/prove-output-balance-validity                 {statement, witness}            -> {proof, link_hint}
    POST <url>/prove-intent-and-balance-private-settlement   {statement, witness, validity_link_hint_0/1,
                                                              output_balance_link_hint_0/1}  -> {proof, validity_link_proof_0/1,
                                                                                                output_balance_link_proof_0/1}
    ... 20 paths in all (prover_service_client.rs:101-147), HTTP basic auth user `admin` (:93, :186-205),
    request / response shapes of api_types.rs:81-130, 141-330.

This module is that server over `libb200prover`: requests are decoded, the circuit is synthesised by the registered
`SingleProverCircuit` (circuit_types.py), proofs run through the prover pool (several in flight per GPU; each HTTP worker
thread blocks only on its own ticket) and link proofs through the same pool, the way
`NativeProofManager::compute_private_settlement_link_proofs` forks them (native_proof_manager.rs:726-782).

Paths whose circuits are not registered answer 501 with a JSON error naming the circuit — the relayer surfaces that as
`ProofManagerError::Http` (error.rs:53-57).

Wire format.  The reference serialises with serde over upstream types (ark-mpc `Scalar`, jellyfish `Proof`) whose
serde impls are not vendored; the codec below is the single place to align them: scalars travel as decimal strings
(32-byte big-endian arrays are accepted too), group elements as {"x", "y"} hex strings of the canonical coordinates,
field names follow the reference's structs (plonk_proof_def.rs:168-222, mocks.rs:28-30, api_types.rs).
"""
from __future__ import annotations

import base64
import dataclasses
import hmac
import json
import threading
import typing
from http.server import BaseHTTPRequestHandler, ThreadingHTTPServer
from typing import Any, Callable, Dict, Optional

import numpy as np

from . import _lib
from . import circuit_types as ct
from .backend import B200LinkProof, B200Proof, GroupLayout, LinkingHint
from .fields import BASE_FIELD_MODULUS, SCALAR_FIELD_MODULUS, limbs_to_scalars, scalars_to_limbs

HTTP_BASIC_AUTH_USER = "admin"  # prover_service_client.rs:93
MAX_BODY_BYTES = 64 << 20

# the 20 paths of prover_service_client.rs:101-147
ALL_PATHS = [
    "/prove-valid-balance-create", "/prove-valid-deposit", "/prove-valid-order-cancellation", "/prove-valid-withdrawal",
    "/prove-intent-and-balance-validity", "/prove-intent-and-balance-first-fill-validity", "/prove-intent-only-validity",
    "/prove-intent-only-first-fill-validity", "/prove-new-output-balance-validity", "/prove-output-balance-validity",
    "/prove-intent-and-balance-bounded-settlement", "/prove-intent-and-balance-private-settlement",
    "/prove-intent-and-balance-public-settlement", "/prove-intent-only-bounded-settlement",
    "/prove-intent-only-public-settlement", "/prove-valid-note-redemption", "/prove-valid-private-protocol-fee-payment",
    "/prove-valid-private-relayer-fee-payment", "/prove-valid-public-protocol-fee-payment",
    "/prove-valid-public-relayer-fee-payment",
]


# ---------------------------------------------------------------------------------------------------------------
# codec
# ---------------------------------------------------------------------------------------------------------------
def encode_scalar(v: int) -> str:
    return str(int(v) % SCALAR_FIELD_MODULUS)


def decode_scalar(v: Any) -> int:
    if isinstance(v, bool):
        return int(v)
    if isinstance(v, int):
        return v % SCALAR_FIELD_MODULUS
    if isinstance(v, str):
        return int(v, 16 if v.startswith("0x") else 10) % SCALAR_FIELD_MODULUS
    if isinstance(v, list) and len(v) == 32:  # big-endian bytes
        return int.from_bytes(bytes(v), "big") % SCALAR_FIELD_MODULUS
    raise ValueError(f"not a scalar: {v!r}")


def to_json(obj: Any) -> Any:
    """dataclass / list / int / bool -> JSON value (ints as decimal strings: they are field elements)."""
    if dataclasses.is_dataclass(obj):
        return {f.name.rstrip("_"): to_json(getattr(obj, f.name)) for f in dataclasses.fields(obj)}
    if isinstance(obj, bool):
        return obj
    if isinstance(obj, int):
        return encode_scalar(obj)
    if isinstance(obj, (list, tuple)):
        return [to_json(v) for v in obj]
    raise TypeError(f"cannot encode {type(obj)}")


def from_json(tp: Any, data: Any) -> Any:
    """Inverse of `to_json`, driven by the dataclass type hints."""
    origin = typing.get_origin(tp)
    if dataclasses.is_dataclass(tp):
        hints = typing.get_type_hints(tp)
        kw = {}
        for f in dataclasses.fields(tp):
            key = f.name.rstrip("_")
            if key not in data:
                raise ValueError(f"{tp.__name__}: missing field {key}")
            kw[f.name] = from_json(hints[f.name], data[key])
        return tp(**kw)
    if tp is bool:
        return bool(data)
    if tp is int:
        return decode_scalar(data)
    if origin in (list, typing.List):
        (inner,) = typing.get_args(tp)
        return [from_json(inner, v) for v in data]
    if tp is tuple or origin is tuple:
        return tuple(decode_scalar(v) for v in data)
    raise TypeError(f"cannot decode {tp}")


def _g1_to_json(xy: np.ndarray) -> Dict[str, str]:
    x, y = limbs_to_scalars(np.asarray(xy, dtype=np.uint64).reshape(2, 4), BASE_FIELD_MODULUS)
    return {"x": hex(x), "y": hex(y)}


def _g1_from_json(d: Dict[str, str]) -> np.ndarray:
    return scalars_to_limbs([int(d["x"], 16), int(d["y"], 16)], BASE_FIELD_MODULUS).reshape(8)


def encode_proof(p: B200Proof) -> Dict[str, Any]:
    """`PlonkProof`, field names of plonk_proof_def.rs:197-222."""
    fr = lambda a: [encode_scalar(v) for v in limbs_to_scalars(np.array(a, dtype=np.uint64).reshape(-1, 4))]
    return {
        "wires_poly_comms": [_g1_to_json(np.array(c, dtype=np.uint64)) for c in p.wires_poly_comms],
        "prod_perm_poly_comm": _g1_to_json(np.array(p.prod_perm_poly_comm, dtype=np.uint64)),
        "split_quot_poly_comms": [_g1_to_json(np.array(c, dtype=np.uint64)) for c in p.split_quot_poly_comms],
        "opening_proof": _g1_to_json(np.array(p.opening_proof, dtype=np.uint64)),
        "shifted_opening_proof": _g1_to_json(np.array(p.shifted_opening_proof, dtype=np.uint64)),
        "poly_evals": {"wires_evals": fr(p.wires_evals), "wire_sigma_evals": fr(p.wire_sigma_evals),
                       "perm_next_eval": fr(p.perm_next_eval)[0]},
        "plookup_proof": None,
    }


def decode_proof(d: Dict[str, Any]) -> B200Proof:
    p = B200Proof()
    for i in range(5):
        p.wires_poly_comms[i][:] = [int(v) for v in _g1_from_json(d["wires_poly_comms"][i])]
        p.split_quot_poly_comms[i][:] = [int(v) for v in _g1_from_json(d["split_quot_poly_comms"][i])]
    p.prod_perm_poly_comm[:] = [int(v) for v in _g1_from_json(d["prod_perm_poly_comm"])]
    p.opening_proof[:] = [int(v) for v in _g1_from_json(d["opening_proof"])]
    p.shifted_opening_proof[:] = [int(v) for v in _g1_from_json(d["shifted_opening_proof"])]
    ev = d["poly_evals"]
    for i in range(5):
        p.wires_evals[i][:] = [int(v) for v in scalars_to_limbs([decode_scalar(ev["wires_evals"][i])])[0]]
    for i in range(4):
        p.wire_sigma_evals[i][:] = [int(v) for v in scalars_to_limbs([decode_scalar(ev["wire_sigma_evals"][i])])[0]]
    p.perm_next_eval[:] = [int(v) for v in scalars_to_limbs([decode_scalar(ev["perm_next_eval"])])[0]]
    return p


def encode_link_hint(h: LinkingHint) -> Dict[str, Any]:
    """`ProofLinkingHint` (plonk_proof_def.rs:143-150).  The polynomial's (n + 2) x 32 bytes travel base64-packed
    (Montgomery limbs, little-endian — the layout both ends hold in memory)."""
    poly = np.ascontiguousarray(h.linking_wire_poly, dtype=np.uint64)
    return {"linking_wire_poly": base64.b64encode(poly.tobytes()).decode(), "linking_wire_comm": _g1_to_json(h.linking_wire_comm)}


def decode_link_hint(d: Dict[str, Any]) -> LinkingHint:
    poly = np.frombuffer(base64.b64decode(d["linking_wire_poly"]), dtype=np.uint64).reshape(-1, 4).copy()
    return LinkingHint(linking_wire_poly=poly, linking_wire_comm=_g1_from_json(d["linking_wire_comm"]))


def encode_link_proof(lp: B200LinkProof) -> Dict[str, Any]:
    """`PlonkLinkProof` (mocks.rs:28-30)."""
    return {"quotient_commitment": _g1_to_json(np.array(lp.quotient_commitment, dtype=np.uint64)),
            "opening_proof": _g1_to_json(np.array(lp.opening_proof, dtype=np.uint64))}


def decode_link_proof(d: Dict[str, Any]) -> B200LinkProof:
    lp = B200LinkProof()
    lp.quotient_commitment[:] = [int(v) for v in _g1_from_json(d["quotient_commitment"])]
    lp.opening_proof[:] = [int(v) for v in _g1_from_json(d["opening_proof"])]
    return lp


# ---------------------------------------------------------------------------------------------------------------
# routes
# ---------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Route:
    """One `/prove-*` path: the circuit, how to decode its witness / statement, and the response kind
    ("proof" = ProofResponse, "proof_and_hint" = ProofAndHintResponse, "settlement" = SettlementProofResponse — one link
    proof —, "private_settlement" = PrivateSettlementProofResponse — four; api_types.rs:81-130)."""
    circuit: type
    decode_witness: Callable[[Any], Any]
    decode_statement: Callable[[Any], Any]
    response: str = "proof"
    # private settlement: [(request field of the hint, response field of the link proof, link group id)]
    links: Optional[list] = None


class ProverService:
    def __init__(self, routes: Dict[str, Route], password: str, srs_bases=None, pool=None, expedite_settlements=False):
        """`expedite_settlements`: the settlement routes' jobs are expedited on `pool` right after submit — they sit on
        a trade's critical path, so they overtake queued validity proofs and run on the pool's express workers."""
        self.routes, self.password, self.pool, self.srs_bases = routes, password, pool, srs_bases
        self.expedite_settlements = expedite_settlements
        self.stats = {"requests": 0, "proofs": 0, "link_proofs": 0, "errors": 0}
        self._lock = threading.Lock()
        self._idle = threading.Condition(self._lock)  # notified when the last request in flight is answered
        self._in_flight = 0
        self._stopping = False

    def shutdown(self, server=None) -> None:
        """Stop now, the way the reference's proof manager stops on its cancel channel: no request is accepted any more
        (503), `server` (what `make_server` returned) stops serving, every job on the pool is cancelled
        (`ProverPool.cancel_all`), so the requests still in flight are answered with a 500 at once instead of after their
        proofs, and once they all are, the pool is closed.  Without a pool the requests in flight run to their end."""
        with self._lock:
            self._stopping = True
        if server is not None:
            server.shutdown()
        with self._idle:
            while self._in_flight:
                if self.pool is not None:  # also the jobs a request submitted just after an earlier cancel_all
                    self.pool.cancel_all()
                self._idle.wait(0.05)
        if self.pool is not None:
            self.pool.close()
        if server is not None:
            server.server_close()

    # -- proving ------------------------------------------------------------------------------------------------
    def handle(self, path: str, body: Dict[str, Any]) -> Dict[str, Any]:
        route = self.routes[path]
        witness = route.decode_witness(body["witness"])
        statement = route.decode_statement(body["statement"])
        if self.pool is not None and route.response in ("settlement", "private_settlement"):
            return self._settle(route, witness, statement, body)
        proof, hint = route.circuit.prove_with_link_hint(witness, statement)
        with self._lock:
            self.stats["proofs"] += 1
        if route.response == "proof":
            return {"proof": encode_proof(proof)}
        if route.response == "proof_and_hint":
            return {"proof": encode_proof(proof), "link_hint": encode_link_hint(hint)}
        if route.response in ("settlement", "private_settlement"):  # SettlementProofResponse / PrivateSettlementProofResponse
            layouts = route.circuit.get_circuit_layout()
            out = {"proof": encode_proof(proof)}
            jobs = []
            for req_field, resp_field, group in route.links:
                other = decode_link_hint(body[req_field])
                lay = GroupLayout(layouts[group].alignment, layouts[group].offset, layouts[group].size)
                # validity / output-balance hint first, settlement hint second (intent_and_balance.rs:57-72)
                try:
                    jobs.append((resp_field, self._submit_link(other, hint, lay)))
                except _lib.B200Error as e:
                    raise ct.ProverError("Plonk", e) from e
            failure = None
            for resp_field, job in jobs:  # every queued job is waited for, also after a failure (its buffers live until then)
                try:
                    out[resp_field] = encode_link_proof(job())
                except _lib.B200Error as e:  # the two proofs do not hold the same values on the group (PlonkError)
                    failure = failure or e
            if failure is not None:
                raise ct.ProverError("Plonk", failure) from failure
            with self._lock:
                self.stats["link_proofs"] += len(jobs)
            return out
        raise ValueError(f"unknown response kind {route.response}")

    def _settle(self, route: Route, witness, statement, body: Dict[str, Any]) -> Dict[str, Any]:
        """A settlement route on the pool: ONE settlement job proves the statement and links every hint of the request
        (`SingleProverCircuit.prove_settlement`), with no host round trip between the proof and its links."""
        hints = [(decode_link_hint(body[req_field]), group) for req_field, _, group in route.links]
        res = route.circuit.prove_settlement_statuses(witness, statement, hints, pool=self.pool, srs_bases=self.srs_bases,
                                                      urgent=self.expedite_settlements)
        with self._lock:  # counted as on the two-step path: the proof once made, the link proofs once all are made
            self.stats["proofs"] += res[2][0] == _lib.B200_OK
        proof, link_proofs = ct.settlement_result(hints, *res)
        with self._lock:
            self.stats["link_proofs"] += len(link_proofs)
        out = {"proof": encode_proof(proof)}
        for (_, resp_field, _), lp in zip(route.links, link_proofs):
            out[resp_field] = encode_link_proof(lp)
        return out

    def _submit_link(self, a: LinkingHint, b: LinkingHint, layout: GroupLayout):
        """Queue one link proof; returns a function that waits for it."""
        srs = ct.system_srs()
        if self.pool is not None:
            tk = self.pool.submit_link(self.srs_bases or srs.powers_of_g, a, b, layout)
            return lambda: self.pool.wait(tk)
        from .backend import link_proofs
        lp, _ = link_proofs(srs.ctx, self.srs_bases or srs.powers_of_g, a, b, layout)
        return lambda: lp

    # -- HTTP ---------------------------------------------------------------------------------------------------
    def make_server(self, host: str = "127.0.0.1", port: int = 0) -> ThreadingHTTPServer:
        service = self
        expect = "Basic " + base64.b64encode(f"{HTTP_BASIC_AUTH_USER}:{self.password}".encode()).decode()

        class Handler(BaseHTTPRequestHandler):
            protocol_version = "HTTP/1.1"

            def log_message(self, *a):  # quiet
                pass

            def _send(self, code: int, obj: Any):
                data = json.dumps(obj).encode()
                self.send_response(code)
                self.send_header("Content-Type", "application/json")
                self.send_header("Content-Length", str(len(data)))
                self.end_headers()
                self.wfile.write(data)

            def do_GET(self):
                if self.path == "/ping":
                    return self._send(200, {"ok": True, "stats": service.stats, "paths": sorted(service.routes)})
                self._send(404, {"error": "not found"})

            def do_POST(self):
                with service._lock:
                    service.stats["requests"] += 1
                    if service._stopping:
                        self.close_connection = True
                        return self._send(503, {"error": "the prover service is shutting down"})
                    service._in_flight += 1
                try:
                    self._post()
                finally:
                    with service._lock:
                        service._in_flight -= 1
                        service._idle.notify_all()

            def _post(self):
                try:
                    n = int(self.headers.get("Content-Length", "0"))
                except ValueError:
                    n = -1
                if n < 0 or n > MAX_BODY_BYTES:  # the largest request (a private settlement with four link hints) is ~3 MB
                    self.close_connection = True
                    return self._send(413, {"error": "request body too large or Content-Length missing"})
                raw = self.rfile.read(n)
                if not hmac.compare_digest((self.headers.get("Authorization") or "").encode(), expect.encode()):
                    return self._send(401, {"error": "unauthorized"})
                if self.path not in ALL_PATHS:
                    return self._send(404, {"error": f"unknown path {self.path}"})
                if self.path not in service.routes:
                    return self._send(501, {"error": f"circuit for {self.path} is not registered with this prover service"})
                try:
                    body = json.loads(raw)
                    resp = service.handle(self.path, body)
                except (KeyError, ValueError, TypeError) as e:
                    with service._lock:
                        service.stats["errors"] += 1
                    return self._send(400, {"error": f"bad request: {e!r}"})
                except ct.ProverError as e:
                    with service._lock:
                        service.stats["errors"] += 1
                    return self._send(500, {"error": f"ProverError::{e}"})
                except _lib.B200Error as e:  # a job cancelled at shutdown on a path that does not wrap library errors
                    with service._lock:
                        service.stats["errors"] += 1
                    return self._send(500, {"error": f"ProverError::Plonk({e})"})
                self._send(200, resp)

        return ThreadingHTTPServer((host, port), Handler)


class ProofServiceClient:
    """The relayer side (prover_service_client.rs:186-205): POST JSON with basic auth, JSON back.  For tests and the
    bench's service leg."""

    def __init__(self, url: str, password: str):
        self.url = url.rstrip("/")
        self.auth = "Basic " + base64.b64encode(f"{HTTP_BASIC_AUTH_USER}:{password}".encode()).decode()

    def send_request(self, path: str, req: Dict[str, Any]):
        import urllib.error
        import urllib.request
        r = urllib.request.Request(self.url + path, data=json.dumps(req).encode(),
                                   headers={"Content-Type": "application/json", "Authorization": self.auth}, method="POST")
        try:
            with urllib.request.urlopen(r, timeout=120) as resp:
                return resp.status, json.loads(resp.read())
        except urllib.error.HTTPError as e:
            return e.code, json.loads(e.read() or b"{}")
