"""`/prove-*` routes of the GPU prover service (renegade_b200/service.py) for the statements restated in this package:
the request decoders (`{statement, witness[, link hints]}`, api_types.rs:141-264) bound to the `SingleProverCircuit`s of
statements.py.  The other four paths of prover_service_client.rs:101-147 are not registered here (their circuits verify Schnorr
signatures / ElGamal ciphertexts on BabyJubJub in-circuit and are not restated); the service answers 501 for them.

    python -m host_circuits.service_routes --port 3000 --password PW --srs /path/to/ptau [--device 0 --workers 6 --express 0 --express-sms 0]

`--express N` adds N express workers to the pool and expedites every settlement route's job onto them (b200express.h).
`--express-sms R` (with `--express N`, N >= 1) runs those workers on R reserved SMs, a multiple of 8, and the normal workers
on the rest (b200reserved.h).
"""
from __future__ import annotations

from typing import List

from renegade_b200.service import Route, from_json

from . import fees
from . import intent_and_balance_validity as val
from . import intent_only as io
from . import output_balance_validity as obv
from . import private_settlement as ps
from . import public_settlement as pub
from . import state_updates as su
from . import statements as st
from . import valid_balance_create as vbc


def routes():
    return {
        "/prove-valid-balance-create": Route(
            st.ValidBalanceCreate, lambda d: from_json(vbc.ValidBalanceCreateWitness, d),
            lambda d: from_json(vbc.ValidBalanceCreateStatement, d), "proof"),
        "/prove-valid-deposit": Route(
            st.ValidDeposit, lambda d: from_json(su.BalanceUpdateWitness, d), lambda d: from_json(su.ValidDepositStatement, d),
            "proof"),
        "/prove-valid-withdrawal": Route(
            st.ValidWithdrawal, lambda d: from_json(su.BalanceUpdateWitness, d),
            lambda d: from_json(su.ValidWithdrawalStatement, d), "proof"),
        "/prove-valid-order-cancellation": Route(
            st.ValidOrderCancellationCircuit, lambda d: from_json(su.ValidOrderCancellationWitness, d),
            lambda d: from_json(su.ValidOrderCancellationStatement, d), "proof"),
        "/prove-valid-note-redemption": Route(
            st.ValidNoteRedemption, lambda d: from_json(fees.NoteRedemptionWitness, d),
            lambda d: from_json(fees.NoteRedemptionStatement, d), "proof"),
        "/prove-valid-public-protocol-fee-payment": Route(
            st.ValidPublicProtocolFeePayment, lambda d: from_json(su.BalanceUpdateWitness, d),
            lambda d: from_json(fees.PublicFeePaymentStatement, d), "proof"),
        "/prove-valid-public-relayer-fee-payment": Route(
            st.ValidPublicRelayerFeePayment, lambda d: from_json(su.BalanceUpdateWitness, d),
            lambda d: from_json(fees.PublicFeePaymentStatement, d), "proof"),
        "/prove-intent-only-validity": Route(
            st.IntentOnlyValidityCircuit, lambda d: from_json(io.ValidityWitness, d), lambda d: from_json(io.ValidityStatement, d),
            "proof_and_hint"),
        "/prove-intent-only-first-fill-validity": Route(
            st.IntentOnlyFirstFillValidityCircuit, lambda d: from_json(io.FirstFillWitness, d),
            lambda d: from_json(io.FirstFillStatement, d), "proof_and_hint"),
        # SettlementProofResponse {proof, link_proof}: the request carries the validity proof's hint (api_types.rs:279-299)
        "/prove-intent-only-public-settlement": Route(
            st.IntentOnlyPublicSettlementCircuit, lambda d: from_json(io.PublicSettlementWitness, d),
            lambda d: from_json(io.PublicSettlementStatement, d), "settlement",
            links=[("validity_link_hint", "link_proof", io.INTENT_ONLY_SETTLEMENT_LINK)]),
        "/prove-intent-only-bounded-settlement": Route(
            st.IntentOnlyBoundedSettlementCircuit, lambda d: from_json(io.PublicSettlementWitness, d),
            lambda d: from_json(io.BoundedSettlementStatement, d), "settlement",
            links=[("validity_link_hint", "link_proof", io.INTENT_ONLY_SETTLEMENT_LINK)]),
        "/prove-intent-and-balance-validity": Route(
            st.IntentAndBalanceValidityCircuit, lambda d: from_json(val.Witness, d), lambda d: from_json(val.Statement, d),
            "proof_and_hint"),
        "/prove-output-balance-validity": Route(
            st.OutputBalanceValidityCircuit, lambda d: from_json(obv.Witness, d), lambda d: from_json(obv.Statement, d),
            "proof_and_hint"),
        # PublicSettlementProofResponse {proof, validity_link_proof, output_balance_link_proof} (api_types.rs:126-137, 238-277)
        "/prove-intent-and-balance-public-settlement": Route(
            st.IntentAndBalancePublicSettlementCircuit, lambda d: from_json(pub.Witness, d),
            lambda d: from_json(pub.PublicStatement, d), "settlement",
            links=[("validity_link_hint", "validity_link_proof", pub.PARTY_LINK),
                   ("output_balance_link_hint", "output_balance_link_proof", pub.OUTPUT_LINK)]),
        "/prove-intent-and-balance-bounded-settlement": Route(
            st.IntentAndBalanceBoundedSettlementCircuit, lambda d: from_json(pub.Witness, d),
            lambda d: from_json(pub.BoundedStatement, d), "settlement",
            links=[("validity_link_hint", "validity_link_proof", pub.PARTY_LINK),
                   ("output_balance_link_hint", "output_balance_link_proof", pub.OUTPUT_LINK)]),
        "/prove-intent-and-balance-private-settlement": Route(
            st.IntentAndBalancePrivateSettlementCircuit, lambda d: from_json(List[ps.PartyWitness], d),
            lambda d: from_json(ps.Statement, d), "private_settlement",
            links=[("validity_link_hint_0", "validity_link_proof_0", ps.PARTY_LINKS[0]),
                   ("validity_link_hint_1", "validity_link_proof_1", ps.PARTY_LINKS[1]),
                   ("output_balance_link_hint_0", "output_balance_link_proof_0", ps.OUTPUT_LINKS[0]),
                   ("output_balance_link_hint_1", "output_balance_link_proof_1", ps.OUTPUT_LINKS[1])]),
    }


def main():
    import argparse
    import numpy as np
    import renegade_b200 as rb
    from renegade_b200 import circuit_types as ct
    from renegade_b200.backend import ProverPool
    from renegade_b200.service import ProverService
    ap = argparse.ArgumentParser()
    ap.add_argument("--host", default="127.0.0.1")
    ap.add_argument("--port", type=int, default=3000)
    ap.add_argument("--password", required=True)
    ap.add_argument("--srs", required=True, help="ptau file (the reference's srs/srs00 chunks concatenated, or any prefix holding 2^14 + 3 powers)")
    ap.add_argument("--g2", help="256-byte file: the two G2 records h || tau*h (only needed by verifiers)")
    ap.add_argument("--check-srs", action="store_true",
                    help="check the loaded powers against h, tau*h (from --g2, else from the ptau's section 3) on the "
                         "device, and refuse to start on an SRS that fails")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--workers", type=int, default=6)
    ap.add_argument("--express", type=int, default=0,
                    help="express workers; > 0 also expedites the settlement routes' jobs (DESIGN.md §6, express lane)")
    ap.add_argument("--express-sms", type=int, default=0,
                    help="SMs reserved for the express workers, a multiple of 8; needs --express (DESIGN.md §6, reserved SMs)")
    args = ap.parse_args()
    if args.express_sms and args.express < 1:
        ap.error("--express-sms reserves SMs for express workers: it requires --express N with N >= 1")
    pool = ProverPool(args.device, workers=args.workers, express=args.express, express_sms=args.express_sms)
    ctx = pool.context(0)
    data = open(args.srs, "rb").read()
    params = rb.parse_ptau_file(ctx, data, count=(1 << 14) + 3)
    if args.g2:
        g2 = np.frombuffer(open(args.g2, "rb").read(), dtype=np.uint64)
    elif args.check_srs:
        g2 = np.concatenate(rb.read_ptau_g2(data))
    else:
        g2 = np.zeros(32, dtype=np.uint64)
    if args.check_srs:
        report = rb.check_srs(ctx, params.powers_of_g, g2[:16], g2[16:32])
        if not report.valid:
            params.powers_of_g.free()
            pool.close()
            raise SystemExit(f"--check-srs: {args.srs} is not a consistent SRS for this G2 pair: {report}")
        print(f"SRS checked: {len(params.powers_of_g)} powers consistent with h, tau*h", flush=True)
    ct.set_system_srs(ctx, params.powers_of_g, g2[:16], g2[16:32], pool=pool)
    for c in st.REGISTERED:  # `NativeProofManager::preprocess_circuits` (native_proof_manager.rs:305-331)
        c.proving_key()
    server = ProverService(routes(), args.password, pool=pool, expedite_settlements=args.express > 0).make_server(args.host, args.port)
    print(f"prover service on {args.host}:{server.server_address[1]} ({len(routes())} circuits)", flush=True)
    server.serve_forever()


if __name__ == "__main__":
    main()
