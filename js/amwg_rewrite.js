// amwg_rewrite.js -- turn the SOURCE of a log_post closure into a function that can be run on symbolic values.
//
// The reference calls an opaque JS closure per step (mcmc.js:958-960, 524-526). The H100 sampler needs that closure as a
// program (include/amwg.h), and JavaScript has no operator overloading: `log_post += ld.norm(data[i], state.mu, state.sigma)`
// cannot be intercepted at run time. So the closure is recorded FROM ITS SOURCE: `log_post.toString()` is parsed (ES5), every
// operator, property read, method call and truth test is rewritten into a call on a runtime object `__r`, and the rewritten
// text is instantiated with `new Function`. Control flow, scoping and closures stay with the JavaScript engine; only the
// places where a parameter value can appear go through `__r`, which builds an expression tree when an operand is symbolic and
// computes the plain JavaScript result when none is (amwg_trace.js).
//
//   a + b            ->  __r.add(a, b)                a.b / a[k]       ->  __r.get(a, "b") / __r.get(a, k)
//   -a, !a           ->  __r.neg(a), !__r.t(a)        f.g(x, y)        ->  __r.call(f, "g", [x, y])
//   a < b, a === b   ->  __r.lt(a, b), __r.eq(a, b)   a.b = v, a.b += v ->  __r.set(a, "b", v), __r.set(a, "b", __r.add(__r.get(a, "b"), v))
//   if (c) / c ? x:y ->  if (__r.t(c)) / (__r.t(c) ? x : y)             x += v, x++      ->  x = __r.add(x, v), x = __r.add(x, 1)
//   a && b, a || b   ->  __r.and(a, function () { return b; }), __r.or(...)
//
// Free identifiers of the closure (names it uses but does not declare: `ld`, `Math`, helper functions such as `logit` in
// tests/test_data.js:195) are returned to the caller, which supplies their values as arguments of the instantiated function.
(function (root, factory) {
  if (typeof define === "function" && define.amd) { define([], factory); }
  else if (typeof module === "object" && module.exports) { module.exports = factory(); }
  else { root.amwg_rewrite = factory(); }
}(this, function () {
  "use strict";

  // ---------------------------------------------------------------------------------------------------- tokenizer
  var KEYWORDS = {"var": 1, "function": 1, "return": 1, "if": 1, "else": 1, "for": 1, "while": 1, "do": 1, "break": 1, "continue": 1,
                  "new": 1, "delete": 1, "typeof": 1, "instanceof": 1, "in": 1, "this": 1, "null": 1, "true": 1, "false": 1,
                  "throw": 1, "try": 1, "catch": 1, "finally": 1, "switch": 1, "case": 1, "default": 1, "void": 1};
  var PUNCT = [">>>=", "===", "!==", ">>>", "<<=", ">>=", "&&", "||", "==", "!=", "<=", ">=", "++", "--", "+=", "-=", "*=", "/=", "%=",
               "&=", "|=", "^=", "<<", ">>", "{", "}", "(", ")", "[", "]", ";", ",", "<", ">", "+", "-", "*", "/", "%", "&", "|", "^",
               "!", "~", "?", ":", "=", "."];

  function is_id_start(c) { return (c >= "a" && c <= "z") || (c >= "A" && c <= "Z") || c === "_" || c === "$"; }
  function is_digit(c) { return c >= "0" && c <= "9"; }

  function tokenize(src) {
    var toks = [], i = 0, n = src.length, c, j, k, p, text;
    while (i < n) {
      c = src.charAt(i);
      if (c === " " || c === "\t" || c === "\n" || c === "\r") { i++; continue; }
      if (c === "/" && src.charAt(i + 1) === "/") { while (i < n && src.charAt(i) !== "\n") { i++; } continue; }
      if (c === "/" && src.charAt(i + 1) === "*") { i += 2; while (i < n && !(src.charAt(i) === "*" && src.charAt(i + 1) === "/")) { i++; } i += 2; continue; }
      if (is_id_start(c)) {
        j = i + 1;
        while (j < n && (is_id_start(src.charAt(j)) || is_digit(src.charAt(j)))) { j++; }
        text = src.substring(i, j);
        toks.push({t: KEYWORDS.hasOwnProperty(text) ? "kw" : "id", v: text});
        i = j; continue;
      }
      if (is_digit(c) || (c === "." && is_digit(src.charAt(i + 1)))) {
        j = i;
        if (c === "0" && (src.charAt(i + 1) === "x" || src.charAt(i + 1) === "X")) {
          j = i + 2;
          while (j < n && (is_digit(src.charAt(j)) || (src.charAt(j) >= "a" && src.charAt(j) <= "f") || (src.charAt(j) >= "A" && src.charAt(j) <= "F"))) { j++; }
        } else {
          while (j < n && is_digit(src.charAt(j))) { j++; }
          if (src.charAt(j) === ".") { j++; while (j < n && is_digit(src.charAt(j))) { j++; } }
          if (src.charAt(j) === "e" || src.charAt(j) === "E") {
            k = j + 1;
            if (src.charAt(k) === "+" || src.charAt(k) === "-") { k++; }
            if (is_digit(src.charAt(k))) { j = k; while (j < n && is_digit(src.charAt(j))) { j++; } }
          }
        }
        toks.push({t: "num", v: src.substring(i, j)});
        i = j; continue;
      }
      if (c === "\"" || c === "'") {
        j = i + 1;
        while (j < n && src.charAt(j) !== c) { if (src.charAt(j) === "\\") { j++; } j++; }
        toks.push({t: "str", v: src.substring(i, j + 1)});       // kept verbatim, quotes included
        i = j + 1; continue;
      }
      text = null;
      for (p = 0; p < PUNCT.length; p++) {
        if (src.substring(i, i + PUNCT[p].length) === PUNCT[p]) { text = PUNCT[p]; break; }
      }
      if (text === null) { throw "log_post source: unexpected character '" + c + "'"; }
      toks.push({t: "op", v: text});
      i += text.length;
    }
    toks.push({t: "eof", v: null});
    return toks;
  }

  // ------------------------------------------------------------------------------------------------------- parser
  var BINPREC = {"||": 1, "&&": 2, "|": 3, "^": 4, "&": 5, "==": 6, "!=": 6, "===": 6, "!==": 6, "<": 7, ">": 7, "<=": 7, ">=": 7,
                 "instanceof": 7, "in": 7, "<<": 8, ">>": 8, ">>>": 8, "+": 9, "-": 9, "*": 10, "/": 10, "%": 10};
  var ASSIGN_OPS = {"=": 1, "+=": 1, "-=": 1, "*=": 1, "/=": 1, "%=": 1, "&=": 1, "|=": 1, "^=": 1, "<<=": 1, ">>=": 1, ">>>=": 1};

  function Parser(toks) { this.t = toks; this.i = 0; }
  Parser.prototype.peek = function () { return this.t[this.i]; };
  Parser.prototype.next = function () { return this.t[this.i++]; };
  Parser.prototype.at = function (type, v) { var k = this.t[this.i]; return k.t === type && (v === undefined || k.v === v); };
  Parser.prototype.eat = function (type, v) { if (this.at(type, v)) { return this.next(); } return null; };
  Parser.prototype.expect = function (type, v) {
    if (!this.at(type, v)) { throw "log_post source: expected " + (v === undefined ? type : v) + " but found " + this.peek().v; }
    return this.next();
  };
  Parser.prototype.semicolon = function () { this.eat("op", ";"); };

  Parser.prototype.func_rest = function (name) {
    var params = [], body;
    this.expect("op", "(");
    while (!this.eat("op", ")")) { params.push(this.expect("id").v); this.eat("op", ","); }
    body = this.block();
    return {k: "func", name: name, params: params, body: body};
  };
  Parser.prototype.block = function () {
    var body = [];
    this.expect("op", "{");
    while (!this.eat("op", "}")) { body.push(this.statement()); }
    return body;
  };
  Parser.prototype.var_decls = function (no_in) {
    var decls = [], name, init;
    do {
      name = this.expect("id").v;
      init = this.eat("op", "=") ? this.assignment(no_in) : null;
      decls.push({name: name, init: init});
    } while (this.eat("op", ","));
    return {k: "var", decls: decls};
  };
  Parser.prototype.statement = function () {
    var s, test, cons, alt, init, update, body, name, e, cases, c, block, param, handler, fin;
    if (this.at("op", "{")) { return {k: "block", body: this.block()}; }
    if (this.eat("op", ";")) { return {k: "empty"}; }
    if (this.at("kw")) {
      switch (this.peek().v) {
      case "var": this.next(); s = this.var_decls(false); this.semicolon(); return s;
      case "function": this.next(); name = this.expect("id").v; return {k: "funcdecl", fn: this.func_rest(name)};
      case "return":
        this.next();
        e = (this.at("op", ";") || this.at("op", "}") || this.at("eof")) ? null : this.expression();
        this.semicolon();
        return {k: "return", e: e};
      case "if":
        this.next(); this.expect("op", "("); test = this.expression(); this.expect("op", ")");
        cons = this.statement();
        alt = this.eat("kw", "else") ? this.statement() : null;
        return {k: "if", test: test, cons: cons, alt: alt};
      case "for":
        this.next(); this.expect("op", "(");
        init = null;
        if (this.eat("kw", "var")) { init = this.var_decls(true); }
        else if (!this.at("op", ";")) { init = {k: "expr", e: this.expression(true)}; }
        if (this.eat("kw", "in")) {
          e = this.expression(); this.expect("op", ")");
          return {k: "forin", left: init, right: e, body: this.statement()};
        }
        this.expect("op", ";");
        test = this.at("op", ";") ? null : this.expression();
        this.expect("op", ";");
        update = this.at("op", ")") ? null : this.expression();
        this.expect("op", ")");
        return {k: "for", init: init, test: test, update: update, body: this.statement()};
      case "while":
        this.next(); this.expect("op", "("); test = this.expression(); this.expect("op", ")");
        return {k: "while", test: test, body: this.statement()};
      case "do":
        this.next(); body = this.statement(); this.expect("kw", "while"); this.expect("op", "(");
        test = this.expression(); this.expect("op", ")"); this.semicolon();
        return {k: "dowhile", test: test, body: body};
      case "break": this.next(); this.semicolon(); return {k: "break"};
      case "continue": this.next(); this.semicolon(); return {k: "continue"};
      case "throw": this.next(); e = this.expression(); this.semicolon(); return {k: "throw", e: e};
      case "try":
        this.next(); block = this.block(); param = null; handler = null; fin = null;
        if (this.eat("kw", "catch")) { this.expect("op", "("); param = this.expect("id").v; this.expect("op", ")"); handler = this.block(); }
        if (this.eat("kw", "finally")) { fin = this.block(); }
        return {k: "try", block: block, param: param, handler: handler, fin: fin};
      case "switch":
        this.next(); this.expect("op", "("); e = this.expression(); this.expect("op", ")"); this.expect("op", "{");
        cases = [];
        while (!this.eat("op", "}")) {
          if (this.eat("kw", "case")) { c = {test: this.expression(), body: []}; } else { this.expect("kw", "default"); c = {test: null, body: []}; }
          this.expect("op", ":");
          while (!this.at("kw", "case") && !this.at("kw", "default") && !this.at("op", "}")) { c.body.push(this.statement()); }
          cases.push(c);
        }
        return {k: "switch", e: e, cases: cases};
      default: break;
      }
    }
    e = this.expression();
    this.semicolon();
    return {k: "expr", e: e};
  };
  Parser.prototype.expression = function (no_in) {
    var e = this.assignment(no_in);
    while (this.eat("op", ",")) { e = {k: "comma", a: e, b: this.assignment(no_in)}; }
    return e;
  };
  Parser.prototype.assignment = function (no_in) {
    var left = this.conditional(no_in), op;
    if (this.at("op") && ASSIGN_OPS.hasOwnProperty(this.peek().v)) {
      op = this.next().v;
      if (left.k !== "ident" && left.k !== "member") { throw "log_post source: invalid assignment target"; }
      return {k: "assign", op: op, target: left, value: this.assignment(no_in)};
    }
    return left;
  };
  Parser.prototype.conditional = function (no_in) {
    var test = this.binary(1, no_in), a, b;
    if (this.eat("op", "?")) {
      a = this.assignment(false); this.expect("op", ":"); b = this.assignment(no_in);
      return {k: "cond", test: test, a: a, b: b};
    }
    return test;
  };
  Parser.prototype.binary = function (minprec, no_in) {
    var left = this.unary(), tok, op, prec, right;
    for (;;) {
      tok = this.peek();
      op = (tok.t === "op" || (tok.t === "kw" && (tok.v === "instanceof" || tok.v === "in"))) ? tok.v : null;
      if (op === null || !BINPREC.hasOwnProperty(op) || (no_in && op === "in")) { break; }
      prec = BINPREC[op];
      if (prec < minprec) { break; }
      this.next();
      right = this.binary(prec + 1, no_in);
      left = (op === "&&" || op === "||") ? {k: "logical", op: op, a: left, b: right} : {k: "bin", op: op, a: left, b: right};
    }
    return left;
  };
  Parser.prototype.unary = function () {
    var tok = this.peek(), op;
    if (tok.t === "op" && (tok.v === "!" || tok.v === "-" || tok.v === "+" || tok.v === "~")) { this.next(); return {k: "unary", op: tok.v, e: this.unary()}; }
    if (tok.t === "kw" && (tok.v === "typeof" || tok.v === "delete" || tok.v === "void")) { this.next(); return {k: "unary", op: tok.v, e: this.unary()}; }
    if (tok.t === "op" && (tok.v === "++" || tok.v === "--")) { op = this.next().v; return {k: "update", op: op, prefix: true, target: this.unary()}; }
    return this.postfix();
  };
  Parser.prototype.postfix = function () {
    var e = this.call_member(), tok = this.peek();
    if (tok.t === "op" && (tok.v === "++" || tok.v === "--")) { this.next(); return {k: "update", op: tok.v, prefix: false, target: e}; }
    return e;
  };
  Parser.prototype.arguments = function () {
    var args = [];
    this.expect("op", "(");
    while (!this.eat("op", ")")) { args.push(this.assignment(false)); this.eat("op", ","); }
    return args;
  };
  Parser.prototype.call_member = function () {
    var e, name, callee;
    if (this.eat("kw", "new")) {
      callee = this.member_only();
      e = {k: "new", callee: callee, args: this.at("op", "(") ? this.arguments() : []};
    } else {
      e = this.primary();
    }
    for (;;) {
      if (this.eat("op", ".")) { name = this.next().v; e = {k: "member", obj: e, prop: {k: "str", v: "\"" + name + "\""}, dot: name}; }
      else if (this.eat("op", "[")) { name = this.expression(); this.expect("op", "]"); e = {k: "member", obj: e, prop: name, dot: null}; }
      else if (this.at("op", "(")) { e = {k: "call", callee: e, args: this.arguments()}; }
      else { break; }
    }
    return e;
  };
  Parser.prototype.member_only = function () {
    var e = this.primary(), name;
    for (;;) {
      if (this.eat("op", ".")) { name = this.next().v; e = {k: "member", obj: e, prop: {k: "str", v: "\"" + name + "\""}, dot: name}; }
      else if (this.eat("op", "[")) { name = this.expression(); this.expect("op", "]"); e = {k: "member", obj: e, prop: name, dot: null}; }
      else { break; }
    }
    return e;
  };
  Parser.prototype.primary = function () {
    var tok = this.next(), items, props, key, e, name;
    if (tok.t === "num") { return {k: "num", v: tok.v}; }
    if (tok.t === "str") { return {k: "str", v: tok.v}; }
    if (tok.t === "id") { return {k: "ident", name: tok.v}; }
    if (tok.t === "kw") {
      if (tok.v === "this" || tok.v === "null" || tok.v === "true" || tok.v === "false") { return {k: "lit", v: tok.v}; }
      if (tok.v === "function") { name = this.at("id") ? this.next().v : ""; return this.func_rest(name); }
    }
    if (tok.t === "op") {
      if (tok.v === "(") { e = this.expression(); this.expect("op", ")"); return {k: "paren", e: e}; }
      if (tok.v === "[") {
        items = [];
        while (!this.eat("op", "]")) { items.push(this.assignment(false)); this.eat("op", ","); }
        return {k: "array", items: items};
      }
      if (tok.v === "{") {
        props = [];
        while (!this.eat("op", "}")) {
          key = this.next();
          this.expect("op", ":");
          props.push({key: key.t === "str" ? key.v : "\"" + key.v + "\"", value: this.assignment(false)});
          this.eat("op", ",");
        }
        return {k: "object", props: props};
      }
    }
    throw "log_post source: unexpected token " + tok.v;
  };

  // ---------------------------------------------------------------------------------------------------- generator
  var BIN_NAME = {"+": "add", "-": "sub", "*": "mul", "/": "div", "%": "mod", "<": "lt", "<=": "le", ">": "gt", ">=": "ge",
                  "==": "eq", "===": "eq", "!=": "ne", "!==": "ne"};
  var GLOBAL_NAMES = {"undefined": 1, "NaN": 1, "Infinity": 1, "isNaN": 1, "isFinite": 1, "parseFloat": 1, "parseInt": 1, "Array": 1, "Object": 1,
                      "Number": 1, "String": 1, "Boolean": 1, "arguments": 1, "JSON": 1, "console": 1};

  function Gen() { this.scopes = [{}]; this.free = {}; this.ntmp = 0; }
  Gen.prototype.declare = function (name) { this.scopes[this.scopes.length - 1][name] = 1; };
  Gen.prototype.declared = function (name) {
    var i;
    for (i = this.scopes.length - 1; i >= 0; i--) { if (this.scopes[i].hasOwnProperty(name)) { return true; } }
    return false;
  };
  // `var` and function declarations are hoisted to the enclosing function: collect them before generating its body
  Gen.prototype.hoist = function (stmts) {
    var i, j, s;
    for (i = 0; i < stmts.length; i++) {
      s = stmts[i];
      if (!s) { continue; }
      switch (s.k) {
      case "var": for (j = 0; j < s.decls.length; j++) { this.declare(s.decls[j].name); } break;
      case "funcdecl": this.declare(s.fn.name); break;
      case "block": this.hoist(s.body); break;
      case "if": this.hoist([s.cons, s.alt]); break;
      case "for": this.hoist([s.init, s.body]); break;
      case "forin": this.hoist([s.left, s.body]); break;
      case "while": case "dowhile": this.hoist([s.body]); break;
      case "try": this.hoist(s.block); if (s.handler) { this.hoist(s.handler); } if (s.fin) { this.hoist(s.fin); } break;
      case "switch": for (j = 0; j < s.cases.length; j++) { this.hoist(s.cases[j].body); } break;
      default: break;
      }
    }
  };
  Gen.prototype.func = function (f) {
    var i, out;
    this.scopes.push({});
    if (f.name) { this.declare(f.name); }
    for (i = 0; i < f.params.length; i++) { this.declare(f.params[i]); }
    this.hoist(f.body);
    out = "function " + f.name + "(" + f.params.join(", ") + ") {\n" + this.stmts(f.body) + "}";
    this.scopes.pop();
    return out;
  };
  Gen.prototype.stmts = function (list) {
    var i, out = "";
    for (i = 0; i < list.length; i++) { out += this.stmt(list[i]) + "\n"; }
    return out;
  };
  Gen.prototype.truth = function (e) { return "__r.t(" + this.expr(e) + ")"; };
  Gen.prototype.stmt = function (s) {
    var i, out, d;
    switch (s.k) {
    case "empty": return ";";
    case "block": return "{\n" + this.stmts(s.body) + "}";
    case "var":
      out = [];
      for (i = 0; i < s.decls.length; i++) { d = s.decls[i]; out.push(d.name + (d.init ? " = " + this.expr(d.init) : "")); }
      return "var " + out.join(", ") + ";";
    case "funcdecl": return this.func(s.fn);
    case "return": return "return" + (s.e ? " " + this.expr(s.e) : "") + ";";
    case "if": return "if (" + this.truth(s.test) + ") " + this.stmt(s.cons) + (s.alt ? " else " + this.stmt(s.alt) : "");
    case "for":
      out = "for (";
      if (s.init) { out += s.init.k === "var" ? this.stmt(s.init) : this.expr(s.init.e) + ";"; } else { out += ";"; }
      out += " " + (s.test ? this.truth(s.test) : "") + "; " + (s.update ? this.expr(this.void_context(s.update)) : "") + ") ";
      return out + this.stmt(s.body);
    case "forin":
      return "for (" + (s.left.k === "var" ? "var " + s.left.decls[0].name : this.expr(s.left.e)) + " in __r.keys(" + this.expr(s.right) + ")) " + this.stmt(s.body);
    case "while": return "while (" + this.truth(s.test) + ") " + this.stmt(s.body);
    case "dowhile": return "do " + this.stmt(s.body) + " while (" + this.truth(s.test) + ");";
    case "break": return "break;";
    case "continue": return "continue;";
    case "throw": return "throw " + this.expr(s.e) + ";";
    case "try":
      out = "try {\n" + this.stmts(s.block) + "}";
      if (s.handler) { this.scopes.push({}); this.declare(s.param); out += " catch (" + s.param + ") {\n" + this.stmts(s.handler) + "}"; this.scopes.pop(); }
      if (s.fin) { out += " finally {\n" + this.stmts(s.fin) + "}"; }
      return out;
    case "switch":
      out = "switch (__r.concrete(" + this.expr(s.e) + ")) {\n";
      for (i = 0; i < s.cases.length; i++) {
        out += (s.cases[i].test ? "case " + this.expr(s.cases[i].test) : "default") + ":\n" + this.stmts(s.cases[i].body);
      }
      return out + "}";
    case "expr": return this.expr(this.void_context(s.e)) + ";";
    default: throw "log_post source: statement " + s.k + " is not supported";
    }
  };
  // `i++` whose value is not used: the same as `++i`
  Gen.prototype.void_context = function (e) {
    if (e.k === "update" && !e.prefix) { return {k: "update", op: e.op, prefix: true, target: e.target}; }
    if (e.k === "comma") { return {k: "comma", a: this.void_context(e.a), b: this.void_context(e.b)}; }
    return e;
  };
  Gen.prototype.args = function (list) {
    var i, out = [];
    for (i = 0; i < list.length; i++) { out.push(this.expr(list[i])); }
    return out.join(", ");
  };
  Gen.prototype.read_target = function (t) {
    if (t.k === "ident") { return this.expr(t); }
    return "__r.get(" + this.expr(t.obj) + ", " + this.expr(t.prop) + ")";
  };
  Gen.prototype.write_target = function (t, value) {
    if (t.k === "ident") {
      if (!this.declared(t.name)) { this.declare(t.name); this.implicit = this.implicit || {}; this.implicit[t.name] = 1; }
      return t.name + " = " + value;
    }
    return "__r.set(" + this.expr(t.obj) + ", " + this.expr(t.prop) + ", " + value + ")";
  };
  Gen.prototype.expr = function (e) {
    var op, i, out, one;
    switch (e.k) {
    case "num": case "str": return e.v;
    case "lit": return e.v;
    case "paren": return "(" + this.expr(e.e) + ")";
    case "ident":
      if (!this.declared(e.name) && !GLOBAL_NAMES.hasOwnProperty(e.name)) { this.free[e.name] = 1; }
      return e.name;
    case "member": return "__r.get(" + this.expr(e.obj) + ", " + this.expr(e.prop) + ")";
    case "call":
      if (e.callee.k === "member") { return "__r.call(" + this.expr(e.callee.obj) + ", " + this.expr(e.callee.prop) + ", [" + this.args(e.args) + "])"; }
      return this.expr(e.callee) + "(" + this.args(e.args) + ")";
    case "new": return "new " + this.expr(e.callee) + "(" + this.args(e.args) + ")";
    case "func": return "(" + this.func(e) + ")";
    case "array": return "[" + this.args(e.items) + "]";
    case "object":
      out = [];
      for (i = 0; i < e.props.length; i++) { out.push(e.props[i].key + ": " + this.expr(e.props[i].value)); }
      return "{" + out.join(", ") + "}";
    case "bin":
      if (BIN_NAME.hasOwnProperty(e.op)) { return "__r." + BIN_NAME[e.op] + "(" + this.expr(e.a) + ", " + this.expr(e.b) + ")"; }
      return "(__r.concrete(" + this.expr(e.a) + ") " + e.op + " __r.concrete(" + this.expr(e.b) + "))";      // in, instanceof, bit operators
    case "logical":
      return "__r." + (e.op === "&&" ? "and" : "or") + "(" + this.expr(e.a) + ", function () { return " + this.expr(e.b) + "; })";
    case "unary":
      if (e.op === "-") { return "__r.neg(" + this.expr(e.e) + ")"; }
      if (e.op === "+") { return "__r.pos(" + this.expr(e.e) + ")"; }
      if (e.op === "!") { return "(!" + this.truth(e.e) + ")"; }
      if (e.op === "typeof" && e.e.k === "ident") { return "(typeof " + e.e.name + ")"; }
      if (e.op === "delete") { return e.e.k === "member" ? "__r.del(" + this.expr(e.e.obj) + ", " + this.expr(e.e.prop) + ")" : "true"; }
      return "(" + e.op + " __r.concrete(" + this.expr(e.e) + "))";
    case "update":
      one = "__r." + (e.op === "++" ? "add" : "sub") + "(" + this.read_target(e.target) + ", 1)";
      if (e.prefix) { return "(" + this.write_target(e.target, one) + ")"; }
      // postfix: the old value is the result
      return "(" + this.write_target(e.target, one) + ", __r." + (e.op === "++" ? "sub" : "add") + "(" + this.read_target(e.target) + ", 1))";
    case "assign":
      if (e.op === "=") { return "(" + this.write_target(e.target, this.expr(e.value)) + ")"; }
      op = e.op.substring(0, e.op.length - 1);
      if (!BIN_NAME.hasOwnProperty(op)) { throw "log_post source: operator " + e.op + " is not supported"; }
      return "(" + this.write_target(e.target, "__r." + BIN_NAME[op] + "(" + this.read_target(e.target) + ", " + this.expr(e.value) + ")") + ")";
    case "cond": return "(" + this.truth(e.test) + " ? " + this.expr(e.a) + " : " + this.expr(e.b) + ")";
    case "comma": return "(" + this.expr(e.a) + ", " + this.expr(e.b) + ")";
    default: throw "log_post source: expression " + e.k + " is not supported";
    }
  };

  // Source text of a function (expression or declaration) -> {source: rewritten function expression, free: [names]}
  function rewrite(fn_source) {
    var p = new Parser(tokenize("(" + fn_source + ")")), ast, g, name, free = [];
    ast = p.expression();
    while (ast.k === "paren") { ast = ast.e; }
    if (ast.k !== "func") { throw "log_post is not a function"; }
    g = new Gen();
    var text = g.func(ast);
    for (name in g.free) { if (g.free.hasOwnProperty(name)) { free.push(name); } }
    free.sort();
    return {source: "(" + text + ")", free: free, implicit: g.implicit || {}};
  }

  return {tokenize: tokenize, rewrite: rewrite};
}));
