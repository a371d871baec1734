// distributions.js -- the `ld` log-density surface of rasmusab/bayes.js (distributions.js:63-284) for the H100 sampler.
//
// Inside log_post the calls are recorded from source (amwg_rewrite.js / amwg_trace.js) and become device opcodes whose
// implementation (csrc/amwg_ld.cuh) follows the reference operation by operation; this module is what `ld.norm(183, 180, 5)`
// evaluates to OUTSIDE log_post: the same device function, run on the GPU through the addon (amwg_ld_eval). There is no CPU
// implementation in the product.
(function (root, factory) {
  if (typeof define === "function" && define.amd) { define(["./amwg_trace", "./amwg_native"], factory); }
  else if (typeof module === "object" && module.exports) { module.exports = factory(require("./amwg_trace"), require("./amwg_native")); }
  else { root.ld = factory(root.amwg_trace, root.amwg_native); }
}(this, function (tracer, native) {
  "use strict";
  var OP = tracer.OP;
  function dev(op, arity, name) {
    return function () {
      var args = [], i;
      if (arguments.length !== arity) { throw "ld." + name + " takes " + arity + " arguments"; }
      for (i = 0; i < arity; i++) { args.push(Number(arguments[i])); }
      return native.ld_eval(OP[op], [args])[0];
    };
  }
  function at(a, i) { return a[i]; }
  var ld = {
    lgamma: dev("LGAMMA", 1, "lgamma"), lfactorial: dev("LFACTORIAL", 1, "lfactorial"), lchoose: dev("LCHOOSE", 2, "lchoose"), lbeta: dev("LBETA", 2, "lbeta"),
    beta: dev("LD_BETA", 3, "beta"), cauchy: dev("LD_CAUCHY", 3, "cauchy"), norm: dev("LD_NORM", 3, "norm"), laplace: dev("LD_LAPLACE", 3, "laplace"),
    gamma: dev("LD_GAMMA", 3, "gamma"), invgamma: dev("LD_INVGAMMA", 3, "invgamma"), lnorm: dev("LD_LNORM", 3, "lnorm"), pareto: dev("LD_PARETO", 3, "pareto"),
    t: dev("LD_T", 4, "t"), weibull: dev("LD_WEIBULL", 3, "weibull"), logis: dev("LD_LOGIS", 3, "logis"), exp: dev("LD_EXP", 2, "exp"),
    unif: dev("LD_UNIF", 3, "unif"), bern: dev("LD_BERN", 2, "bern"), binom: dev("LD_BINOM", 3, "binom"), nbinom: dev("LD_NBINOM", 3, "nbinom"),
    hyper: dev("LD_HYPER", 4, "hyper"), pois: dev("LD_POIS", 2, "pois")
  };
  ld.dexp = ld.laplace;                                            // distributions.js:140
  // the array-valued ones, composed on the device one primitive at a time in the reference's operation order
  function e1(op, x) { return native.ld_eval(OP[op], [[x]])[0]; }
  function e2(op, x, y) { return native.ld_eval(OP[op], [[x, y]])[0]; }
  ld.bivarnorm = function (x, mean, sd, corr) {                    // distributions.js:125-133
    var x0 = at(x, 0), x1 = at(x, 1), m0 = at(mean, 0), m1 = at(mean, 1), s0 = at(sd, 0), s1 = at(sd, 1), r = corr;
    var z = e2("POW", x0 - m0, 2) / e2("POW", s0, 2) + e2("POW", x1 - m1, 2) / e2("POW", s1, 2) - (2 * r * (x0 - m0) * (x1 - m1)) / (s0 * s1);
    var nf = -(e1("LOG", 2) + e1("LOG", Math.PI) + e1("LOG", s0) + e1("LOG", s1) + 0.5 * e1("LOG", 1 - e2("POW", r, 2)));
    return nf - z / (2 * (1 - e2("POW", r, 2)));
  };
  ld.dirichlet = function (x, alpha) {                             // distributions.js:203-214
    var sum_alpha = 0, sum_lg = 0, s = 0, i;
    for (i = 0; i < alpha.length; i++) { sum_alpha = sum_alpha + alpha[i]; sum_lg = sum_lg + e1("LGAMMA", alpha[i]); s = s + (alpha[i] - 1) * e1("LOG", x[i]); }
    return e1("LGAMMA", sum_alpha) - sum_lg + s;
  };
  ld.cat = function (x, probs) {                                   // distributions.js:232-238
    if (x < 1 || x > probs.length) { return -Infinity; }
    return e1("LOG", probs[x - 1]);
  };
  return ld;
}));
