// mcmc.js -- the JavaScript host side of the H100-native AMWG sampler: a drop-in for rasmusab/bayes.js' `mcmc` module on the one
// path this package accelerates,
//
//     var sampler = new mcmc.AmwgSampler(params, log_post, data, options);      // reference: mcmc.js:1090-1092, 940-966
//     sampler.burn(1000); var samples = sampler.sample(5000);                    //            mcmc.js:1035-1039, 1005-1030
//
// Same names, argument meaning and thrown strings as the reference; the stepping happens in libamwg_b200.so (CUDA, sm_90a)
// for `options.chains` independent chains at once, reached through the N-API addon js/amwg_napi.cc (`require("./amwg_native")`,
// a thin wrapper over include/amwg.h). log_post is recorded from its source (amwg_rewrite.js) and lowered to the device program
// (amwg_trace.js). Nothing here computes a log density or draws a proposal: there is no CPU path.
//
// New, non-reference options: `chains` (default 1: output shaped exactly like the reference's), `seed`, `device`, `first_chain`,
// `faithful` (no factorised likelihood plates: bit-faithful sums, slower), `scope` ({name: value} for identifiers log_post uses
// from an enclosing scope that a recording from source cannot see), `init_radius` (over-dispersed starting points drawn on the
// device, DESIGN.md §2), `superchain_size` (chains per superchain that start at one point, DESIGN.md §4.6), `temperatures` (parallel
// tempering: ladders of K neighbouring chains at T_0 = 1 < ... < T_{K-1} that swap states after every sweep; sample() returns the
// T = 1 chains, DESIGN.md §2). New methods: `sampler.set_state(values)` places the chains anywhere; `sampler.checkpoint()` and
// `sampler.restore(images)` stop and resume a run bit for bit.
(function (root, factory) {
  if (typeof define === "function" && define.amd) { define(["./amwg_trace", "./amwg_native"], factory); }
  else if (typeof module === "object" && module.exports) { module.exports = factory(require("./amwg_trace"), require("./amwg_native")); }
  else { root.mcmc = factory(root.amwg_trace, root.amwg_native); }
}(this, function (tracer, native) {
  "use strict";

  var TYPE_CODE = {"real": 0, "int": 1, "binary": 2};
  var STEPPER_OPTIONS = [["prop_log_scale", 0], ["batch_size", 50], ["max_adaptation", 0.33], ["initial_adaptation", 1.0],
                         ["target_accept_rate", 0.44], ["is_adapting", true]];

  // ---------------------------------------------------------------------------------------------- helpers (mcmc.js:131-303)
  function is_array(a) { return Object.prototype.toString.call(a) === "[object Array]"; }
  function is_number(x) { return typeof x === "number"; }
  function own_keys(o) { var k, out = []; for (k in o) { if (o.hasOwnProperty(k)) { out.push(k); } } return out; }
  function create_array(dim, init) {
    var out = [], i;
    if (dim.length < 1) { throw "create_array can't create a dimensionless array"; }
    for (i = 0; i < dim[0]; i++) { out.push(dim.length === 1 ? (typeof init === "function" ? init() : init) : create_array(dim.slice(1), init)); }
    return out;
  }
  function array_dim(a) { return (a.length > 0 && is_array(a[0])) ? [a.length].concat(array_dim(a[0])) : [a.length]; }
  function array_equal(a, b) {
    var i;
    if (a.length !== b.length) { return false; }
    for (i = 0; i < a.length; i++) {
      if (is_array(a[i]) && is_array(b[i])) { if (!array_equal(a[i], b[i])) { return false; } }
      else if (a[i] !== b[i]) { return false; }
    }
    return true;
  }
  function flatten(a, out) {
    var i;
    out = out || [];
    if (is_array(a)) { for (i = 0; i < a.length; i++) { flatten(a[i], out); } } else { out.push(a); }
    return out;
  }
  function nest(flat, dim) {
    var out = [], i, step;
    if (dim.length === 1) { return flat.slice(0, dim[0]); }
    step = flat.length / dim[0];
    for (i = 0; i < dim[0]; i++) { out.push(nest(flat.slice(i * step, (i + 1) * step), dim.slice(1))); }
    return out;
  }
  function product(dim) { var n = 1, i; for (i = 0; i < dim.length; i++) { n *= dim[i]; } return n; }
  function deep_clone(v) {
    var out, k, i;
    if (is_array(v)) { out = []; for (i = 0; i < v.length; i++) { out.push(deep_clone(v[i])); } return out; }
    if (v !== null && typeof v === "object") { out = {}; for (k in v) { if (v.hasOwnProperty(k)) { out[k] = deep_clone(v[k]); } } return out; }
    return v;
  }
  function get_option(name, options, default_value) {       // mcmc.js:280-285: undefined and null fall back, 0 / false do not
    var v = options ? options[name] : undefined;
    return (v === undefined || v === null) ? default_value : v;
  }
  function get_multidim_option(name, options, dim, default_value) {     // mcmc.js:293-303
    var value = get_option(name, options, default_value);
    if (!is_array(value)) { value = create_array(dim, value); }
    if (!array_equal(array_dim(value), dim)) { throw "The option " + name + " is of dimension [" + array_dim(value) + "] but should be [" + dim + "]."; }
    return value;
  }

  // ---------------------------------------------------------------------------------------------- parameters (mcmc.js:313-403)
  function param_init_fixed(type, lower, upper) {
    if (lower > upper) { throw "Can not initialize parameter where lower bound > upper bound"; }
    if (type === "real") {
      if (lower === -Infinity && upper === Infinity) { return 0.5; }
      if (lower === -Infinity) { return upper - 0.5; }
      if (upper === Infinity) { return lower + 0.5; }
      return (lower + upper) / 2;
    }
    if (type === "int") {
      if (lower === -Infinity && upper === Infinity) { return 1; }
      if (lower === -Infinity) { return upper - 1; }
      if (upper === Infinity) { return lower + 1; }
      return Math.round((lower + upper) / 2);
    }
    if (type === "binary") { return 1; }
    throw "Could not initialize parameter of type " + type + "[" + lower + ", " + upper + "]";
  }
  function complete_params(params_to_complete, param_init) {
    var params = deep_clone(params_to_complete), names = own_keys(params), i, p, make;
    param_init = param_init || param_init_fixed;
    for (i = 0; i < names.length; i++) {
      p = params[names[i]];
      if (!p.hasOwnProperty("type")) { p.type = "real"; }
      if (!p.hasOwnProperty("dim")) { p.dim = [1]; }
      if (is_number(p.dim)) { p.dim = [p.dim]; }
      if (p.type === "binary") { p.upper = 1; p.lower = 0; }
      if (!p.hasOwnProperty("upper")) { p.upper = Infinity; }
      if (!p.hasOwnProperty("lower")) { p.lower = -Infinity; }
      if (p.hasOwnProperty("init")) {
        if (array_equal(p.dim, [1]) && typeof p.init === "function") { p.init = p.init(); }
        else if (!array_equal(p.dim, [1]) && !is_array(p.init)) { p.init = create_array(p.dim, p.init); }
      } else if (array_equal(p.dim, [1])) {
        p.init = param_init(p.type, p.lower, p.upper);
      } else {
        make = (function (q) { return function () { return param_init(q.type, q.lower, q.upper); }; }(p));
        p.init = create_array(p.dim, make);
      }
    }
    return params;
  }

  // ---------------------------------------------------------------------------------------------- exported RNG helpers (mcmc.js:31-54)
  // Math.random() of the helpers := the Philox stream of the sampler (DESIGN.md "RNG contract"), drawn on the device.
  var host_stream = {seed: 1835232611, chain: 4294967295, n: 0, block: [], block0: 0};
  function stream_random() {
    var k = host_stream.n - host_stream.block0, want, i, idx = [];
    if (!(k >= 0 && k < host_stream.block.length)) {
      want = 1024;
      for (i = 0; i < want; i++) { idx.push(host_stream.n + i); }
      host_stream.block = native.stream_uniforms(host_stream.seed, host_stream.chain, host_stream.n, want);
      host_stream.block0 = host_stream.n;
      k = 0;
    }
    host_stream.n++;
    return host_stream.block[k];
  }
  function set_random_stream(seed, chain, position) { host_stream.seed = seed; host_stream.chain = chain || 0; host_stream.n = position || 0; host_stream.block = []; host_stream.block0 = 0; }
  function runif(min, max) { return stream_random() * (max - min) + min; }
  function runif_discrete(min, max) { return Math.floor(stream_random() * (max - min + 1)) + min; }
  function rnorm(mean, sd) {                                   // Leva's ratio of uniforms; the log is the device's Math.log
    var u, v, x, y, q;
    do {
      u = stream_random();
      v = 1.7156 * (stream_random() - 0.5);
      x = u - 0.449871;
      y = Math.abs(v) + 0.386595;
      q = x * x + y * (0.19600 * y - 0.25472 * x);
    } while (q > 0.27597 && (q > 0.27846 || v * v > -4 * native.device_log(u) * u * u));
    return (v / u) * sd + mean;
  }

  // ---------------------------------------------------------------------------------------------- option resolution
  function truthy(v) { return !!v; }
  // AmwgStepper's per-parameter merge (mcmc.js:871-878) with its quirks: `a || b` lets falsy values fall through, and
  // options.params[name] is mutated in place
  function resolve_stepper_options(params, names, options, direct) {
    var out = {}, i, k, name, p, po, param_options, key, r;
    for (i = 0; i < names.length; i++) {
      name = names[i]; p = params[name];
      if (!TYPE_CODE.hasOwnProperty(p.type)) { throw "AmwgStepper can't handle parameter " + name + " with type " + p.type; }
      if (direct) { param_options = options || {}; }
      else {
        options = options || {};
        po = truthy(options.params) ? options.params[name] : undefined;
        param_options = truthy(po) ? po : {};
        for (k = 0; k < STEPPER_OPTIONS.length; k++) { key = STEPPER_OPTIONS[k][0]; param_options[key] = truthy(param_options[key]) ? param_options[key] : options[key]; }
      }
      r = {};
      if (p.type !== "binary") {
        for (k = 0; k < STEPPER_OPTIONS.length; k++) {
          key = STEPPER_OPTIONS[k][0];
          r[key] = array_equal(p.dim, [1]) ? [get_option(key, param_options, STEPPER_OPTIONS[k][1])] : flatten(get_multidim_option(key, param_options, p.dim, STEPPER_OPTIONS[k][1]));
        }
      }
      out[name] = r;
    }
    return out;
  }

  // ---------------------------------------------------------------------------------------------- the device model
  // options.temperatures -> [1 / T_r]; throws unless 2..256 finite, T_0 = 1, strictly increasing, and their number divides n_chains
  function ladder_betas(temps, n_chains) {
    var i, out = [];
    if (!is_array(temps)) { throw "options.temperatures must be a list of numbers"; }
    for (i = 0; i < temps.length; i++) { if (!is_number(temps[i])) { throw "options.temperatures must be a list of numbers"; } }
    if (temps.length < 2 || temps.length > 256) { throw "options.temperatures must have between 2 and 256 entries"; }
    for (i = 0; i < temps.length; i++) { if (!isFinite(temps[i])) { throw "options.temperatures must be finite"; } }
    if (temps[0] !== 1) { throw "options.temperatures must start at 1"; }
    for (i = 1; i < temps.length; i++) { if (!(temps[i - 1] < temps[i])) { throw "options.temperatures must be strictly increasing"; } }
    if (n_chains % temps.length !== 0) { throw "options.temperatures: their number must divide options.chains"; }
    for (i = 0; i < temps.length; i++) { out.push(1.0 / temps[i]); }
    return out;
  }

  function DeviceModel(params, names, log_post, data, options, resolved) {
    var i, j, c, name, p, ncomp, off, flat, r, o, n_comp = 0, prog, seed, radius, size, failed, temps;
    this.params = params; this.names = names; this.offsets = {};
    for (i = 0; i < names.length; i++) { this.offsets[names[i]] = n_comp; n_comp += product(params[names[i]].dim); }
    this.n_comp = n_comp;
    this.n_chains = Math.floor(get_option("chains", options, 1));
    if (!(this.n_chains >= 1)) { throw "options.chains must be >= 1"; }
    seed = get_option("seed", options, null);
    this.seed = seed === null ? Math.floor(Math.random() * 9007199254740992) : seed;
    this.device = get_option("device", options, 0);
    this.first_chain = get_option("first_chain", options, 0);
    radius = get_option("init_radius", options, null);            // over-dispersed starting points (DESIGN.md §2)
    if (radius !== null && !(typeof radius === "number" && isFinite(radius) && radius > 0)) { throw "options.init_radius must be a finite number > 0"; }
    size = get_option("superchain_size", options, null);           // chains per superchain (nested R-hat, DESIGN.md §4.6)
    if (size !== null) {
      if (!(typeof size === "number" && isFinite(size) && size >= 1 && size === Math.floor(size))) { throw "options.superchain_size must be an integer >= 1"; }
      if (this.n_chains % size !== 0) { throw "options.superchain_size must divide options.chains"; }
    }
    this.superchain_size = size;
    temps = get_option("temperatures", options, null);              // parallel tempering (DESIGN.md §2 "Tempered ladders")
    this.temperatures = temps;
    this.betas = temps === null ? null : ladder_betas(temps, this.n_chains);
    if (this.betas !== null && size !== null) { throw "options.superchain_size cannot be combined with options.temperatures: superchains of tempered chains are not defined"; }
    if (this.betas !== null && this.first_chain % this.betas.length !== 0) { throw "options.first_chain must be a multiple of the number of temperatures"; }
    this.n_cold = this.betas === null ? this.n_chains : this.n_chains / this.betas.length;     // the chains sample() returns
    prog =tracer.trace(log_post, names, params, this.offsets, n_comp, data, {faithful: !!get_option("faithful", options, false), scope: get_option("scope", options, null),
                                                                                base_state: get_option("base_state", options, null)});
    this.program = prog;
    this.derived_names = prog.derived_names;
    var desc = {params: [], init: [], comp_options: [], code: prog.code, logpost_prog: prog.logpost_prog, derived_prog: prog.derived_prog,
                n_derived: prog.derived_names.length, consts: prog.consts.length ? prog.consts : [0], columns: prog.columns, plates: prog.plates,
                fold_prog: prog.fold_prog, fold_dst: prog.fold_dst, n_terms: prog.n_terms, comp_prog: prog.comp_prog, touch_off: prog.touch_off,
                touch_terms: prog.touch_terms, block_params: prog.block_params, term_block_comp: prog.term_block_comp, stat_prog: prog.stat_prog,
                n_sum_terms: prog.stat_prog >= 0 ? prog.n_sum_terms : prog.n_terms, variant_comps: prog.variant_comps,
                variant_logpost: prog.variant_logpost, variant_derived: prog.variant_derived};
    for (i = 0; i < names.length; i++) {
      name = names[i]; p = params[name]; ncomp = product(p.dim); off = this.offsets[name];
      desc.params.push({type: TYPE_CODE[p.type], n_comp: ncomp, dim0: p.dim[0], comp_offset: off, lower: p.lower, upper: p.upper});
      flat = flatten(p.init);
      if (flat.length !== ncomp) { throw "The init of parameter " + name + " does not match its dim"; }
      for (j = 0; j < ncomp; j++) { desc.init.push(flat[j]); }
      r = resolved[name];
      for (c = 0; c < ncomp; c++) {
        if (p.type === "binary") { o = {prop_log_scale: 0, batch_size: 50, max_adaptation: 0.33, initial_adaptation: 1.0, target_accept_rate: 0.44, is_adapting: 0}; }
        else {
          o = {prop_log_scale: r.prop_log_scale[c], batch_size: r.batch_size[c], max_adaptation: r.max_adaptation[c], initial_adaptation: r.initial_adaptation[c],
               target_accept_rate: r.target_accept_rate[c], is_adapting: r.is_adapting[c] ? 1 : 0};
        }
        desc.comp_options.push(o);
      }
    }
    this.handle = native.create(desc, this.n_chains, this.first_chain, this.seed, this.device);
    if (this.betas !== null) { native.set_ladder(this.handle, this.betas); }
    if (radius !== null) {
      failed = size === null ? native.disperse_state(this.handle, radius) : native.disperse_state(this.handle, radius, size);
      if (failed > 0) {
        native.destroy(this.handle);
        this.handle = null;
        throw "options.init_radius: " + failed + " of " + this.n_chains + " chains found no starting point with a finite log_post in 100 attempts";
      }
    }
  }
  DeviceModel.prototype.state_keys = function () { return this.names.concat(this.derived_names); };
  DeviceModel.prototype.entries = function (name) {
    var out = [], i, n;
    if (this.offsets.hasOwnProperty(name)) { n = product(this.params[name].dim); for (i = 0; i < n; i++) { out.push(this.offsets[name] + i); } return out; }
    i = this.derived_names.indexOf(name);
    return i >= 0 ? [this.n_comp + i] : [];
  };
  // raw: flat [rows][n_entries][chains]; -> reference-shaped draws of `name` (entries s..s+ln): [rows] of numbers / nested arrays for one
  // chain, [rows][chains] of the same otherwise
  DeviceModel.prototype.shape_out = function (name, raw, rows, n_entries, s, ln, chains) {
    var dim = this.params.hasOwnProperty(name) ? this.params[name].dim : [1], C = chains === undefined ? this.n_chains : chains, out = [], r, c, e, one, row,
        scalar = array_equal(dim, [1]);
    for (r = 0; r < rows; r++) {
      row = [];
      for (c = 0; c < C; c++) {
        if (scalar) { row.push(raw[(r * n_entries + s) * C + c]); }
        else {
          one = [];
          for (e = 0; e < ln; e++) { one.push(raw[(r * n_entries + s + e) * C + c]); }
          row.push(nest(one, dim));
        }
      }
      out.push(C === 1 ? row[0] : row);
    }
    return out;
  };
  DeviceModel.prototype.state = function () {
    var keys = this.state_keys(), n_entries = this.n_comp + this.derived_names.length, raw = native.get_state(this.handle), out = {}, i, e;
    for (i = 0; i < keys.length; i++) { e = this.entries(keys[i]); out[keys[i]] = this.shape_out(keys[i], raw, 1, n_entries, e[0], e.length)[0]; }
    return out;
  };
  // values: {name: value shaped like state()[name], or like one chain's value (given to every chain)} -> amwg_set_state
  DeviceModel.prototype.set_state = function (values) {
    var C = this.n_chains, D = this.n_comp, raw = native.get_state(this.handle), block = [], keys, i, k, c, name, dim, n, off, v, got, one, per, flat, scalar;
    if (values === null || typeof values !== "object" || is_array(values)) { throw "set_state expects an object keyed by parameter name"; }
    for (i = 0; i < D * C; i++) { block.push(raw[i]); }
    keys = own_keys(values);
    for (i = 0; i < keys.length; i++) {
      name = keys[i];
      if (this.derived_names.indexOf(name) >= 0) { throw "set_state: " + name + " is a derived quantity, not a parameter"; }
      if (!this.offsets.hasOwnProperty(name)) { throw "set_state: " + name + " is not a parameter of this sampler"; }
      dim = this.params[name].dim; n = product(dim); off = this.offsets[name]; v = values[name];
      scalar = array_equal(dim, [1]);
      one = scalar ? [] : dim;
      per = [C].concat(one);
      got = is_array(v) ? array_dim(v) : [];
      flat = flatten(v);
      if ((array_equal(got, one) || array_equal(got, dim)) && flat.length === n) {
        for (k = 0; k < n; k++) { for (c = 0; c < C; c++) { block[(off + k) * C + c] = flat[k]; } }
      } else if (array_equal(got, per) && flat.length === C * n) {
        for (k = 0; k < n; k++) { for (c = 0; c < C; c++) { block[(off + k) * C + c] = flat[c * n + k]; } }
      } else {
        throw "set_state: " + name + " is of dimension [" + got + "] but should be [" + dim + "] or [" + per + "]";
      }
    }
    native.set_state(this.handle, block);
  };
  DeviceModel.prototype.sample = function (n, thin, monitored) {
    var entries = [], spans = {}, i, e, rows, raw, out = {}, j, col;
    monitored = monitored === null ? this.state_keys() : monitored;
    for (i = 0; i < monitored.length; i++) { e = this.entries(monitored[i]); spans[monitored[i]] = [entries.length, e.length]; entries = entries.concat(e); }
    n = Math.floor(n);
    thin = Math.abs(Math.floor(thin));
    if (thin === 0 || !(thin === thin)) {              // i % 0 is NaN: nothing is ever recorded, the chains still step (mcmc.js:1021)
      native.burn(this.handle, Math.max(n, 0));
      for (i = 0; i < monitored.length; i++) { out[monitored[i]] = []; }
      return out;
    }
    rows = n <= 0 ? 0 : Math.ceil(n / thin);
    raw = native.sample(this.handle, n, thin, entries);
    for (i = 0; i < monitored.length; i++) {
      e = spans[monitored[i]];
      if (e[1] === 0) { col = []; for (j = 0; j < rows; j++) { col.push(undefined); } out[monitored[i]] = col; }      // JS: state[name] is undefined
      else { out[monitored[i]] = this.shape_out(monitored[i], raw, rows, entries.length, e[0], e[1], this.n_cold); }
    }
    return out;
  };
  DeviceModel.prototype.info = function () {
    var inf = native.info(this.handle), C = this.n_chains, per = {}, i, name, p, e, self = this;
    function per_chain(arr, ent, dim) {
      var c, k, vals, out = [];
      for (c = 0; c < C; c++) { vals = []; for (k = 0; k < ent.length; k++) { vals.push(arr[ent[k] * C + c]); } out.push(array_equal(dim, [1]) ? vals[0] : nest(vals, dim)); }
      return C === 1 ? out[0] : out;
    }
    function invariant(idx, ent, dim, as_bool) {
      var k, vals = [];
      for (k = 0; k < ent.length; k++) { vals.push(as_bool ? inf.scalars[ent[k] * 3 + idx] !== 0 : inf.scalars[ent[k] * 3 + idx]); }
      return array_equal(dim, [1]) ? vals[0] : nest(vals, dim);
    }
    for (i = 0; i < this.names.length; i++) {
      name = this.names[i]; p = this.params[name];
      if (p.type === "binary") { per[name] = {}; continue; }        // BinaryStepper inherits Stepper.info -> {} (mcmc.js:465-468)
      e = self.entries(name);
      per[name] = {prop_log_scale: per_chain(inf.prop_log_scale, e, p.dim), is_adapting: invariant(0, e, p.dim, true),
                   acceptance_count: per_chain(inf.acceptance_count, e, p.dim), iterations_since_adaption: invariant(1, e, p.dim, false),
                   batch_count: invariant(2, e, p.dim, false)};
    }
    return per;
  };

  // ---------------------------------------------------------------------------------------------- Sampler / AmwgSampler (mcmc.js:940-1099)
  function Sampler(params, log_post, data, options) {
    this.data = data;
    this.param_names = own_keys(params);
    this.param_init_fun = get_option("param_init_fun", options, param_init_fixed);
    this.thin(get_option("thin", options, 1));
    this.monitor(get_option("monitor", options, null));
    this.options = options;
    this.params = complete_params(params, this.param_init_fun);
    this.steppers = this.create_stepper_ensamble(this.params, null, log_post, this.options);
  }
  Sampler.prototype.create_stepper_ensamble = function () { throw "Every Sampler needs to implement create_stepper_ensamble()"; };
  Sampler.prototype.thin = function (k) { this.thinning_interval = k; };
  Sampler.prototype.monitor = function (names) { this.monitored_params = names; };

  function AmwgSampler(params, log_post, data, options) { Sampler.call(this, params, log_post, data, options); }
  AmwgSampler.prototype = Object.create(Sampler.prototype);
  AmwgSampler.prototype.constructor = AmwgSampler;
  AmwgSampler.prototype.create_stepper_ensamble = function (params, state, log_post, options) {
    options = options || {};
    this.model = new DeviceModel(params, this.param_names, log_post, this.data, options, resolve_stepper_options(params, this.param_names, options, false));
    this.n_chains = this.model.n_chains;
    return ["AmwgStepper"];
  };
  AmwgSampler.prototype.burn = function (n) { native.burn(this.model.handle, Math.floor(n)); };
  AmwgSampler.prototype.sample = function (n) { return this.model.sample(n, this.thinning_interval, this.monitored_params); };
  // Not in the reference: sample(n) without the reshaping into nested arrays -- for millions of chains the nested form is impractical.
  // -> {data: flat array (Float64Array under Node) laid out [row][entry][chain], shape: [rows, entries, chains], entries: [{name, index}]}
  AmwgSampler.prototype.sample_raw = function (n) {
    var m = this.model, monitored = this.monitored_params === null ? m.state_keys() : this.monitored_params, entries = [], labels = [], i, j, e, thin, rows;
    for (i = 0; i < monitored.length; i++) { e = m.entries(monitored[i]); for (j = 0; j < e.length; j++) { entries.push(e[j]); labels.push({name: monitored[i], index: j}); } }
    thin = Math.abs(Math.floor(this.thinning_interval));
    if (!(thin >= 1)) { throw "sample_raw needs thin >= 1"; }
    rows = n <= 0 ? 0 : Math.ceil(Math.floor(n) / thin);
    return {data: native.sample(m.handle, Math.floor(n), thin, entries), shape: [rows, entries.length, m.n_cold], entries: labels};
  };
  AmwgSampler.prototype.step = function () { this.burn(1); return this.model.state(); };
  AmwgSampler.prototype.state = function () { return this.model.state(); };
  // Not in the reference: place the chains (from a previous run, prior draws, an optimiser). Shapes as state() returns them, or one
  // chain's value for all chains; parameters not named keep their values; adaptation and the random streams carry on untouched.
  AmwgSampler.prototype.set_state = function (values) { this.model.set_state(values); };
  // Not in the reference: checkpoints (DESIGN.md §2). checkpoint() -> the image of this sampler's chains (a Buffer under Node);
  // restore(image or [image, ...]) resumes, bit for bit, the run the images were taken from: same model, data and options, and
  // images that together cover this sampler's chains (from any number of samplers). The sampler adopts the images' seed.
  AmwgSampler.prototype.checkpoint = function () {
    var img = native.checkpoint(this.model.handle);
    return typeof Buffer === "function" ? Buffer.from(img.buffer, img.byteOffset, img.length) : img;
  };
  AmwgSampler.prototype.restore = function (images) {
    this.model.seed = native.restore(this.model.handle, is_array(images) ? images : [images], 0);
  };
  AmwgSampler.prototype.log_post = function () { var lp = native.get_log_post(this.model.handle); return this.n_chains === 1 ? lp[0] : lp; };
  AmwgSampler.prototype.start_adaptation = function () { native.set_adapting(this.model.handle, 1); };
  AmwgSampler.prototype.stop_adaptation = function () { native.set_adapting(this.model.handle, 0); };
  AmwgSampler.prototype.info = function () {
    // the reference returns the thin / monitor METHODS under those keys (mcmc.js:977-980, a bug); the values are returned here
    var out = {state: this.model.state(), thin: this.thinning_interval, monitor: this.monitored_params, steppers: [this.model.info()]}, m = this.model, K, li, r, k, att = [], rate = [];
    if (m.betas !== null) {               // options.temperatures: swap rounds, and per rung pair the swaps accepted / attempted over this sampler's ladders
      K = m.betas.length; li = native.ladder_info(m.handle); k = li.rounds;
      for (r = 0; r < K - 1; r++) { att.push((m.n_chains / K) * Math.floor((k + 1 - (r % 2)) / 2)); rate.push(att[r] > 0 ? li.accepts[r] / att[r] : NaN); }
      out.tempering = {temperatures: m.temperatures.slice(), rounds: k, swap_accepts: li.accepts, swap_attempts: att, swap_rate: rate};
    }
    return out;
  };
  AmwgSampler.prototype.close = function () { if (this.model && this.model.handle !== null) { native.destroy(this.model.handle); this.model.handle = null; } };
  AmwgSampler.prototype.sweep_kernel = function () { return native.jit_status(this.model.handle); };

  // ---------------------------------------------------------------------------------------------- stand-alone steppers (mcmc.js:433-912)
  // A zero-argument log_post that closes over the caller's `state` object cannot be recorded from its source alone: the steppers
  // take the same closure the reference takes PLUS read the parameters they step from `state`; the recording binds `state` by name
  // (options.scope.state, set here), so log_post must refer to the state object as `state` or receive it in options.scope.
  function Stepper(params, state, log_post) { this.params = params; this.state = state; this.log_post = log_post; }
  Stepper.prototype.step = function () { throw "Every Stepper need to implement step()"; };
  Stepper.prototype.start_adaptation = function () {};
  Stepper.prototype.stop_adaptation = function () {};
  Stepper.prototype.info = function () { return {}; };

  function device_stepper(who, forced_type, check) {
    function S(params, state, log_post, options) {
      var names = own_keys(params), p, i, self = this, scope, wrapped;
      Stepper.call(this, params, state, log_post);
      check(names, params);
      this.param_name = names.length === 1 ? names[0] : null;
      p = complete_params(params);
      for (i = 0; i < names.length; i++) {
        if (forced_type !== null) { p[names[i]].type = forced_type; if (forced_type === "binary") { p[names[i]].lower = 0; p[names[i]].upper = 1; } }
        p[names[i]].init = deep_clone(state[names[i]]);             // a stepper starts from the state it is given, not from params.init
      }
      options = options || {};
      scope = {};
      if (options.scope) { for (i in options.scope) { if (options.scope.hasOwnProperty(i)) { scope[i] = options.scope[i]; } } }
      // record log_post() with the stepped parameters symbolic: the zero-argument closure becomes function (state, data) by naming
      // the object it closes over `state`
      wrapped = new Function("return function (state, data) { return (" + log_post.toString() + ")(); };")();
      var opts = {};
      for (i in options) { if (options.hasOwnProperty(i)) { opts[i] = options[i]; } }
      opts.scope = scope;
      opts.base_state = state;
      this.names = names;
      this.model = new DeviceModel(p, names, wrapped, null, opts, resolve_stepper_options(p, names, options, who !== "AmwgStepper"));
    }
    S.prototype = Object.create(Stepper.prototype);
    S.prototype.constructor = S;
    S.prototype.step = function () {
      var st, i, n;
      native.burn(this.model.handle, 1);
      st = this.model.state();
      for (i = 0; i < this.names.length; i++) { n = this.names[i]; this.state[n] = st[n]; }
      return this.param_name !== null ? this.state[this.param_name] : this.state;
    };
    S.prototype.start_adaptation = function () { native.set_adapting(this.model.handle, 1); };
    S.prototype.stop_adaptation = function () { native.set_adapting(this.model.handle, 0); };
    S.prototype.info = function () {
      var per = this.model.info(), out = {}, i;
      if (who !== "AmwgStepper") { return per[this.param_name]; }
      for (i = 0; i < this.names.length; i++) { out[this.names[i]] = per[this.names[i]]; }
      return out;
    };
    return S;
  }
  function one_param(msg) { return function (names) { if (names.length !== 1) { throw msg; } }; }
  function onedim_check(names, params) {
    var dim;
    if (names.length !== 1) { throw "OnedimMetropolisStepper can only handle one parameter."; }
    dim = params[names[0]].hasOwnProperty("dim") ? params[names[0]].dim : [1];
    if (!array_equal(is_number(dim) ? [dim] : dim, [1])) { throw "OnedimMetropolisStepper can only handle one one-dimensional parameter."; }
  }
  var multi_msg = "MultidimComponentMetropolisStepper can't handle more than one parameter.";

  return {
    runif: runif, runif_discrete: runif_discrete, rnorm: rnorm, set_random_stream: set_random_stream,
    param_init_fixed: param_init_fixed, complete_params: complete_params,
    RealMetropolisStepper: device_stepper("OnedimMetropolisStepper", "real", onedim_check),
    IntMetropolisStepper: device_stepper("OnedimMetropolisStepper", "int", onedim_check),
    MultiRealComponentMetropolisStepper: device_stepper("MultidimComponentMetropolisStepper", "real", one_param(multi_msg)),
    MultiIntComponentMetropolisStepper: device_stepper("MultidimComponentMetropolisStepper", "int", one_param(multi_msg)),
    BinaryStepper: device_stepper("BinaryStepper", "binary", one_param("BinaryStepper can't handle more than one parameter.")),
    BinaryComponentStepper: device_stepper("BinaryComponentStepper", "binary", one_param("BinaryComponentStepper can't handle more than one parameter.")),
    AmwgStepper: device_stepper("AmwgStepper", null, function () {}),
    AmwgSampler: AmwgSampler,
    where: tracer.where
  };
}));
