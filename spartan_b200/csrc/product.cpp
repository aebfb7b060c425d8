// spartan_b200 — product circuits (product_tree.rs) on the device: the layers of a batch of circuits and the batched proof of their products
// (ProductCircuitEvalProofBatched), run by SNARK::prove for SPARK's memory check (snark.cpp) and by the caller's own circuits (sp_prod_*).
#include "prover.hpp"
#include <algorithm>
#include <optional>

namespace sp {

void build_circuits(Ctx& ctx, std::vector<ProdCircuit*> cs, size_t from) {
  ProdCircuit& c0 = *cs[0];
  for (size_t k = from; k + 1 < c0.num_layers; k++) {
    const size_t h = c0.local_len(k) / 2;
    std::vector<u256*> outs; std::vector<const u256*> as, bs;
    if (k + 1 == c0.Ks) {
      DevBuf<u256> tmp(cs.size() * h);
      for (size_t i = 0; i < cs.size(); i++) { outs.push_back(tmp.p + i * h); as.push_back(cs[i]->layer(k)); bs.push_back(cs[i]->layer(k) + h); }
      dev::hadamard_many(outs.data(), as.data(), bs.data(), (int)cs.size(), h, ctx.stream);
      std::vector<const u256*> src(outs.begin(), outs.end());
      u256* g = ctx.allgather_cyclic(src.data(), (int)cs.size(), h);
      const size_t glen = h * (size_t)c0.W;
      for (size_t i = 0; i < cs.size(); i++) dev::d2d(cs[i]->layer(k + 1), g + i * glen, glen * sizeof(u256), ctx.stream);
      ctx.sync();   // tmp is released here
      continue;
    }
    for (auto* c : cs) { outs.push_back(c->layer(k + 1)); as.push_back(c->layer(k)); bs.push_back(c->layer(k) + h); }
    dev::hadamard_many(outs.data(), as.data(), bs.data(), (int)cs.size(), h, ctx.stream);
  }
}

void batched_prove(Ctx& ctx, std::vector<ProdCircuit*>& prods, std::vector<DotpCircuit>& dotps, Transcript& T, ProductCircuitEvalProofBatched& out,
                   std::vector<Fq>& rand_out) {
  const size_t np = prods.size(), nd = dotps.size();
  const size_t num_layers = prods[0]->num_layers;
  // the limit of one launch, which the layout's capacities for the evaluations, the bound entries and the staged last-layer entries rest on
  if (np + nd > (size_t)dev::SC_MAX_INST) throw SpError(SP_ERR_INTERNAL, "batched product proof of more than " + std::to_string(dev::SC_MAX_INST) + " instances");
  std::vector<Fq> claims_to_verify(np);
  {  // all evaluate()s with one sync
    uint8_t* stage = ctx.pinned + layout::PIN_STAGE.off;
    for (size_t i = 0; i < np; i++) dev::d2h(stage + 64 * i, prods[i]->layer(num_layers - 1), 64, ctx.stream);
    ctx.sync();
    for (size_t i = 0; i < np; i++) { Fq v[2]; memcpy(v, stage + 64 * i, 64); claims_to_verify[i] = v[0] * v[1]; }
  }
  const int W = prods[0]->W, rk = ctx.rank();
  const size_t Ks = prods[0]->Ks;
  // the shared eq table and its two ping-pong halves: local sizes while a layer is sharded, full sizes for the replicated layers
  const size_t max_half = std::max(prods[0]->local_len(0) / 2, Ks < num_layers ? prods[0]->local_len(Ks) / 2 : 1);
  DevBuf<u256> cpar_a(std::max<size_t>(max_half / 2, 1)), cpar_b(std::max<size_t>(max_half / 2, 1)), d_rand(64), eq_small(dev::eq_evals_scratch(num_layers));
  DevBuf<u256> cpar0(std::max<size_t>(max_half, 1));
  std::vector<Fq> rand;
  const size_t G_MIN = 2 * Ctx::SHARD_MIN_LOCAL;   // 16384 entries per table: the fused G kernel then always streams >= 32768
  u256* d_out = ctx.small.p + layout::SMALL_BATCH.off;   // ninst * 3 scalars
  u256* const h_out = ctx.host_res + layout::RES_OUT.off;   // where they reach the host
  DevBuf<u256> d_heads(3 * dev::SC_MAX_INST);
  const int logW = (int)log2_ceil(W);
  // a layer's sumcheck runs on tables of half = len/2 entries (num_rounds variables), lhalf of them on this rank while the layer is sharded
  struct Shape { size_t half, num_rounds, lhalf; bool sh; int logW; };
  auto shape_of = [&](size_t layer_id) {
    Shape s;
    s.half = prods[0]->layer_len(layer_id) / 2;
    s.num_rounds = log2_ceil(s.half);
    s.sh = prods[0]->sharded(layer_id);
    s.lhalf = s.sh ? s.half / W : s.half;
    s.logW = s.sh ? logW : 0;
    return s;
  };
  // eq-factored streaming rounds (kernels_sc.cu: k_sc_eval_g): rounds 0 .. jG-1, i.e. those whose evaluation streams >= G_MIN entries per table,
  // when no tau_j of them is zero (q(1) is recovered by a division by tau_j); rand[0] = r_layer is checked when the layer starts
  auto plan_jG = [&](const Shape& s, const Fq* rand_tail /* rand[1..] */) {
    size_t jG = 0;
    if (s.num_rounds >= 2) {
      while (jG + 1 < s.num_rounds && (s.lhalf >> jG) >= G_MIN) jG++;
      for (size_t j = 1; j < jG; j++) if (rand_tail[j - 1].is_zero()) jG = 0;
    }
    return jG;
  };
  // poly_C_par = eq(rand) with rand = [r_layer | rand_tail] (product_tree.rs:279-280).  Everything but the top variable is known once the layer
  // above has drawn its last challenge, so this builds E = eq(rand_tail, .) (times c_rank, leaving out the last logW variables, when sharded)
  // into cpar0 + lhalf/2 then, and the suffix levels of an eq-factored layer below it, all while the host still runs the layer above's tail
  // transcript; once r_layer is drawn, a layer without eq-factoring needs one eq_extend_top launch and an eq-factored one none.
  auto build_eq = [&](const Shape& s, const std::vector<Fq>& rand_tail) {
    const size_t n0 = s.lhalf / 2;
    if (!rand_tail.empty()) dev::h2d(d_rand.p, rand_tail.data(), rand_tail.size() * sizeof(u256), ctx.stream);
    dev::eq_evals(cpar0.p + n0, d_rand.p, (int)rand_tail.size() - s.logW, eq_small.p, ctx.stream);
    if (s.sh) dev::scale(cpar0.p + n0, shard_eq_scale(rand_tail, W, rk).m, n0, ctx.stream);   // c_rank: fixed by rand's last logW entries
    const size_t jG = plan_jG(s, rand_tail.data());
    if (jG > 1) dev::eq_suffix(cpar0.p, cpar0.p + n0, n0, (int)jG - 1, ctx.stream);
  };
  for (size_t layer_id = num_layers; layer_id-- > 0;) {
    const Shape shp = shape_of(layer_id);
    const size_t num_rounds = shp.num_rounds, lhalf = shp.lhalf;
    std::optional<FineTimer> fhead(std::in_place, ctx, "batched layer head");   // r_layer drawn .. round 0's evaluations on the host
    std::optional<FineTimer> fswitch;                                             // switch of an eq-factored layer .. its evaluations on the host
    if (num_rounds > 0 && rand.size() != num_rounds) throw SpError(SP_ERR_INTERNAL, "product layer sizes are not powers of two");
    // the suffix tables E_j = eq(rand[j+1..], .) of an eq-factored layer (E_0 at cpar0 + lhalf/2, the levels 1 .. jG-1 from cpar0 on, built by
    // build_eq); from round jG on the standard kernels run on C = eq(rand[jG..], .) = E_{jG-1} (times c_rank) and the host multiplies the product
    // instances' evaluations by prefix = prod_{j<jG} eq(tau_j, r_j).  Not applicable: the standard method from round 0 on C = [(1 - r_layer) E_0 | r_layer E_0].
    size_t jG = num_rounds > 0 ? plan_jG(shp, rand.data() + 1) : 0;
    if (jG && rand[0].is_zero()) jG = 0;
    std::vector<u256*> Elev(jG);
    if (jG) {
      const size_t n0 = lhalf / 2;
      Elev[0] = cpar0.p + n0;
      size_t off = 0;
      for (size_t k = 1; k < jG; k++) { Elev[k] = cpar0.p + off; off += n0 >> k; }
    } else if (num_rounds > 0) dev::eq_extend_top(cpar0.p, lhalf / 2, rand[0].m, ctx.stream);
    u256* const C0 = jG ? Elev[jG - 1] : cpar0.p;   // the shared C of the first standard round (read, never written)
    ScRounds sc{ctx, dev::SC_CUBIC3, {}, lhalf, shp.sh, d_out};
    for (size_t i = 0; i < np; i++) {
      dev::ScInst in;
      in.t[0] = prods[i]->layer(layer_id); in.t[1] = prods[i]->layer(layer_id) + lhalf; in.t[2] = C0; in.t[3] = nullptr;
      in.c_out = cpar_a.p; in.write_c = i == 0;
      sc.insts.push_back(in);
    }
    const bool with_dotp = layer_id == 0 && nd > 0;
    if (with_dotp) {
      for (size_t i = 0; i < nd; i++) {
        if (dotps[i].sharded != shp.sh) throw SpError(SP_ERR_INTERNAL, "dot-product circuits and product circuits disagree on sharding");
        dev::ScInst in;
        in.t[0] = dotps[i].left; in.t[1] = dotps[i].right; in.t[2] = dotps[i].weight; in.t[3] = nullptr;
        in.c_out = dotps[i].weight; in.write_c = 1;
        sc.insts.push_back(in);
        claims_to_verify.push_back(dotps[i].claim);   // DotProductCircuit::evaluate, taken on the unsharded tables by the caller
      }
    }
    const size_t ninst = sc.insts.size();
    // eq-factored rounds: the np product instances through the G kernels (2 values each), the dot-product circuits (their third table is not an
    // eq table) through the standard kernels in a second launch whose results land behind the first's
    const size_t ndi = ninst - np;
    auto launch_g = [&](size_t j, const Fq* r) {   // round j; r: bind with r first
      sc.sig = ctx.next_sig();
      if (!r) dev::sc_eval_g(sc.insts.data(), (int)np, sc.len, Elev[j], d_out, ctx.red.p, ctx.stream, sc.sig, sc.xr());
      else dev::sc_fold_eval_g(sc.insts.data(), (int)np, sc.len, r->m, Elev[j], d_out, ctx.red.p, ctx.stream, sc.sig, sc.xr());
      if (ndi) {
        sc.sig = ctx.next_sig();
        sc.sig.host_out = h_out + 3 * np;
        if (!r) dev::sc_eval(dev::SC_CUBIC3, sc.insts.data() + np, (int)ndi, sc.len, d_out + 3 * np, ctx.red.p, ctx.stream, sc.sig, sc.xr());
        else dev::sc_fold_eval(dev::SC_CUBIC3, sc.insts.data() + np, (int)ndi, sc.len, r->m, d_out + 3 * np, ctx.red.p, ctx.stream, sc.sig, sc.xr());
      }
      if (r) sc.len >>= 1;
    };
    // round 0's evaluations do not depend on the batching coefficients: launch them first, draw the coefficients while they run
    if (jG) launch_g(0, nullptr);
    else if (num_rounds > 0) sc.eval();
    std::vector<Fq> coeff_vec = T.challenge_vector("rand_coeffs_next_layer", claims_to_verify.size());
    Fq claim = Fq::zero();
    for (size_t i = 0; i < claims_to_verify.size(); i++) claim += claims_to_verify[i] * coeff_vec[i];

    std::vector<Fq> coeff_std = coeff_vec;            // the standard rounds' weights: after an eq-factored switch, prefix * coeff for the product instances
    LayerProofBatched lp;
    std::vector<Fq> rand_prod;
    Fq e = claim;
    std::vector<Fq> tau_inv(jG);   // batch inversion of tau_0 .. tau_{jG-1}
    Fq cP = Fq::zero(), eD = Fq::zero(), prefix = Fq::one();
    if (jG) {
      std::vector<Fq> pre(jG);
      Fq acc = Fq::one();
      for (size_t j = 0; j < jG; j++) { pre[j] = acc; acc *= rand[j]; }
      Fq inv = acc.inv();
      for (size_t j = jG; j-- > 0;) { tau_inv[j] = inv * pre[j]; inv *= rand[j]; }
      for (size_t i = 0; i < np; i++) cP += claims_to_verify[i] * coeff_vec[i];
      for (size_t i = np; i < ninst; i++) eD += claims_to_verify[i] * coeff_vec[i];
    }
    const Fq one = Fq::one();
    // the fold to two-entry tables (the last round's launch) publishes them, and the host binds the last variable itself (lp claims below)
    bool bound_on_host = false;
    for (size_t j = 0; j < num_rounds; j++) {
      FineTimer fw(ctx, "batched wait evals");
      const std::vector<Fq> ev = sc.wait();
      fw.stop();
      fhead.reset(); fswitch.reset();
      FineTimer fh(ctx, "batched host round");
      const bool eqf = j < jG;
      std::vector<Fq> evals(4), sD;
      Fq Q0 = Fq::zero(), Qinf = Fq::zero(), qb = Fq::zero(), omt = Fq::zero(), slope = Fq::zero();
      auto q_at = [&](const Fq& t) { return (Qinf * t + qb) * t + Q0; };
      if (eqf) {
        Fq D0 = Fq::zero(), D2 = Fq::zero(), D3 = Fq::zero();
        for (size_t i = 0; i < np; i++) { Q0 += ev[3 * i] * coeff_vec[i]; Qinf += ev[3 * i + 1] * coeff_vec[i]; }
        for (size_t i = np; i < ninst; i++) { D0 += ev[3 * i] * coeff_vec[i]; D2 += ev[3 * i + 1] * coeff_vec[i]; D3 += ev[3 * i + 2] * coeff_vec[i]; }
        const Fq& tau = rand[j];
        omt = one - tau;
        const Fq Q1 = (cP - omt * Q0) * tau_inv[j];            // c_j = (1 - tau_j) q(0) + tau_j q(1)
        qb = Q1 - Q0 - Qinf;
        slope = tau - omt;                                       // eq(tau_j, t) = (1 - tau_j) + t (2 tau_j - 1)
        sD = {D0, eD - D0, D2, D3};
        Fq t = Fq::zero(), lin = omt;
        for (int k = 0; k < 4; k++) { evals[k] = prefix * lin * q_at(t) + (ndi ? sD[k] : Fq::zero()); t += one; lin += slope; }
      } else {
        Fq c0 = Fq::zero(), c2 = Fq::zero(), c3 = Fq::zero();
        for (size_t i = 0; i < ninst; i++) { c0 += ev[3 * i] * coeff_std[i]; c2 += ev[3 * i + 1] * coeff_std[i]; c3 += ev[3 * i + 2] * coeff_std[i]; }  // sumcheck.rs:359-361
        evals = {c0, e - c0, c2, c3};
      }
      UniPoly poly = UniPoly::from_evals(evals);               // eq-factored: the same cubic the reference interpolates from its evaluations at 0, 1, 2, 3
      poly.append_to_transcript("poly", T);
      Fq r_j = T.challenge_scalar("challenge_nextround");
      rand_prod.push_back(r_j);
      if (j + 1 < jG) {
        launch_g(j + 1, &r_j);
      } else if (j + 1 == jG) {
        // switch: bind with r_j and evaluate round jG the standard way on C = E_{jG-1} = eq(rand[jG..], .) (this rank's slice, times c_rank, when
        // sharded); the factor prefix, the same on every rank, is applied to the product instances' evaluations on the host
        fswitch.emplace(ctx, "batched switch");
        sc.fold(r_j);
        sc.eval();
      } else if (j + 1 < num_rounds) {
        bound_on_host = j + 2 == num_rounds;
        sc.fold_eval(r_j, bound_on_host ? h_out + 3 * ninst : nullptr);
        // the product instances now read the shared C where instance 0 folded it, so the next fold writes it into the other ping-pong half;
        // after the shard exit they read its gathered copy instead and both halves are free
        for (size_t i = 0; i < np; i++)
          if (sc.insts[i].t[2] == sc.insts[i].c_out) sc.insts[i].c_out = sc.insts[i].c_out == cpar_a.p ? cpar_b.p : cpar_a.p;
      } else if (!bound_on_host) {
        sc.fold(r_j);   // the shared C's final value is never used by the prover (claims_prod.2 is dropped, product_tree.rs:336)
      }
      e = poly.evaluate(r_j);
      lp.proof.compressed_polys.push_back(poly.compress());
      if (eqf) {
        cP = q_at(r_j);
        prefix *= omt + r_j * slope;
        if (ndi) eD = UniPoly::from_evals(sD).evaluate(r_j);
        if (j + 1 == jG) for (size_t i = 0; i < np; i++) coeff_std[i] = coeff_vec[i] * prefix;
      }
    }
    // final claims: first element of every A / B (and C for the dot-product circuits)
    fhead.reset();
    FineTimer fl(ctx, "batched layer tail (claims d2h + transcript)");
    std::vector<Fq> heads(3 * ninst);
    if (bound_on_host) {   // a0 + r (a1 - a0): what the fold computes (fq_fold_const), on the two entries the last launch published
      std::vector<Fq> bound(6 * ninst);
      memcpy(bound.data(), h_out + 3 * ninst, 6 * ninst * sizeof(u256));
      const Fq& r = rand_prod.back();
      for (size_t k = 0; k < 3 * ninst; k++) heads[k] = bound[2 * k] + r * (bound[2 * k + 1] - bound[2 * k]);
      if (layer_id > 0) build_eq(shape_of(layer_id - 1), rand_prod);
    } else {  // layers of fewer than two rounds: a gather kernel that also publishes the values to the host.  It takes A and B of a product
              // instance and A, B and C of a dot-product circuit, at most 3 * SC_MAX_INST heads, in launches of at most HEADS_PER_LAUNCH; the last
              // one publishes the flag, after the earlier launches' values (stream order)
      std::vector<const u256*> hp;
      for (size_t i = 0; i < ninst; i++) {
        const dev::ScInst& in = sc.insts[i];
        hp.insert(hp.end(), {in.t[0], in.t[1]});
        if (i >= np) hp.push_back(in.t[2]);
      }
      dev::HostSig hs = ctx.next_sig();
      for (size_t at = 0; at < hp.size(); at += dev::HEADS_PER_LAUNCH) {
        const size_t cnt = std::min<size_t>(dev::HEADS_PER_LAUNCH, hp.size() - at);
        dev::HostSig part = hs;
        part.host_out = hs.host_out + at;
        if (at + cnt < hp.size()) part.flag = nullptr;
        dev::heads(d_heads.p + at, hp.data() + at, (int)cnt, ctx.stream, part);
      }
      if (layer_id > 0) build_eq(shape_of(layer_id - 1), rand_prod);
      ctx.wait_sig(hs);
      std::vector<Fq> got(hp.size());
      memcpy(static_cast<void*>(got.data()), h_out, hp.size() * sizeof(u256));
      for (size_t i = 0, at = 0; i < ninst; i++)
        for (size_t t = 0; t < (i >= np ? 3u : 2u); t++) heads[3 * i + t] = got[at++];
    }
    lp.claims_prod_left.resize(np); lp.claims_prod_right.resize(np);
    for (size_t i = 0; i < np; i++) { lp.claims_prod_left[i] = heads[3 * i]; lp.claims_prod_right[i] = heads[3 * i + 1]; }
    for (size_t i = 0; i < np; i++) {
      T.append_scalar("claim_prod_left", lp.claims_prod_left[i]);
      T.append_scalar("claim_prod_right", lp.claims_prod_right[i]);
    }
    if (with_dotp) {
      out.dotp_left.resize(nd); out.dotp_right.resize(nd); out.dotp_weight.resize(nd);
      for (size_t i = 0; i < nd; i++) {
        out.dotp_left[i] = heads[3 * (np + i)];
        out.dotp_right[i] = heads[3 * (np + i) + 1];
        out.dotp_weight[i] = heads[3 * (np + i) + 2];
        T.append_scalar("claim_dotp_left", out.dotp_left[i]);
        T.append_scalar("claim_dotp_right", out.dotp_right[i]);
        T.append_scalar("claim_dotp_weight", out.dotp_weight[i]);
      }
    }
    Fq r_layer = T.challenge_scalar("challenge_r_layer");
    claims_to_verify.resize(np);
    for (size_t i = 0; i < np; i++) claims_to_verify[i] = lp.claims_prod_left[i] + r_layer * (lp.claims_prod_right[i] - lp.claims_prod_left[i]);
    std::vector<Fq> ext = {r_layer};
    ext.insert(ext.end(), rand_prod.begin(), rand_prod.end());
    rand = ext;
    out.proof.push_back(std::move(lp));
  }
  rand_out = rand;
}

// ================================================================================================ the caller's circuits (sp_prod_*)
std::vector<Fq> prod_build(Ctx& ctx, std::vector<dev::ProdLeaves> leaves, std::vector<dev::DotpOperands> dotps, size_t n,
                           std::vector<std::unique_ptr<ProdCircuit>>& out, ProdDotps& dout) {
  const size_t k = leaves.size(), kd = dotps.size();
  out.clear();
  dout = ProdDotps();
  if (kd) {   // DotProductCircuit::split of each dot product d into its halves [0, n/2) and [n/2, n): circuits 2d and 2d + 1, the reference's order
    dout.ops.alloc(3 * n * kd);
    for (size_t d = 0; d < kd; d++) {
      dotps[d].out = dout.ops.p + 3 * n * d;
      for (size_t h = 0; h < 2; h++) {
        u256* base = dotps[d].out + h * (n / 2);
        dout.d.push_back(DotpCircuit{base, base + n, base + 2 * n, n / 2, false, Fq::zero()});
      }
    }
    dev::dotp_operands(dotps.data(), (int)kd, n, ctx.small.p + layout::SMALL_BATCH.off, ctx.red.p, ctx.stream);
  }
  for (size_t i = 0; i < k; i++) {
    out.emplace_back(new ProdCircuit);
    out[i]->alloc(ctx, n);   // no ShardScope: one rank's GPU, W = 1
    leaves[i].layer0 = out[i]->layer(0);
    leaves[i].layer1 = out[i]->num_layers > 1 ? out[i]->layer(1) : nullptr;
  }
  dev::prod_leaves(leaves.data(), (int)k, n, ctx.stream);
  // layers 2 .. num_layers - 1 in groups of at most 16 (hadamard_many's limit), the circuits split as evenly as the groups allow
  const size_t ngroups = (k + 15) / 16;
  for (size_t g = 0, first = 0; g < ngroups; g++) {
    const size_t cnt = k / ngroups + (g < k % ngroups ? 1 : 0);
    std::vector<ProdCircuit*> grp;
    for (size_t i = first; i < first + cnt; i++) grp.push_back(out[i].get());
    build_circuits(ctx, grp, 1);
    first += cnt;
  }
  // ProductCircuit::evaluate: the two entries of every last layer, and DotProductCircuit::evaluate of every half, with one synchronise
  uint8_t* stage = ctx.pinned + layout::PIN_STAGE.off;
  for (size_t i = 0; i < k; i++) dev::d2h(stage + 64 * i, out[i]->layer(out[i]->num_layers - 1), 64, ctx.stream);
  if (kd) dev::d2h(stage + 64 * k, ctx.small.p + layout::SMALL_BATCH.off, 2 * kd * sizeof(u256), ctx.stream);
  ctx.sync();
  std::vector<Fq> products(k);
  for (size_t i = 0; i < k; i++) { Fq v[2]; memcpy(static_cast<void*>(v), stage + 64 * i, 64); products[i] = v[0] * v[1]; }
  for (size_t j = 0; j < 2 * kd; j++) memcpy(static_cast<void*>(&dout.d[j].claim), stage + 64 * k + sizeof(u256) * j, sizeof(u256));
  return products;
}

void prod_prove(Ctx& ctx, std::vector<ProdCircuit*>& cs, std::vector<DotpCircuit>& dotps, Transcript& T, ProductCircuitEvalProofBatched& out,
                std::vector<Fq>& rand, std::vector<Fq>& leaf_evals, std::vector<Fq>& dotp_evals) {
  batched_prove(ctx, cs, dotps, T, out, rand);
  // the claims layer 0's proof leaves (product_tree.rs:373-375): left + r_layer (right - left), r_layer = rand[0]; for a dot product, its two
  // halves' final claims combined the same way, as the verifier combines claims_dotp[2k] and [2k + 1] (:385-485)
  const LayerProofBatched& l0 = out.proof.back();
  auto at_rand = [&](const Fq& lo, const Fq& hi) { return lo + rand[0] * (hi - lo); };
  leaf_evals.resize(cs.size());
  for (size_t i = 0; i < cs.size(); i++) leaf_evals[i] = at_rand(l0.claims_prod_left[i], l0.claims_prod_right[i]);
  dotp_evals.clear();
  for (size_t d = 0; d + 1 < dotps.size(); d += 2) {
    dotp_evals.push_back(at_rand(out.dotp_left[d], out.dotp_left[d + 1]));
    dotp_evals.push_back(at_rand(out.dotp_right[d], out.dotp_right[d + 1]));
    dotp_evals.push_back(at_rand(out.dotp_weight[d], out.dotp_weight[d + 1]));
  }
}

}  // namespace sp
