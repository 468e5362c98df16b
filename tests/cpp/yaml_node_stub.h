// yaml_node_stub.h — the part of YAML::Node (yaml-cpp) that the facade's yaml_to_* templates use: operator[] with a
// key (a node that converts to false when the key is absent), IsMap / IsSequence / IsScalar / IsNull, Scalar(), size(),
// as<T>() and range-for iteration. Scalars convert by the rules ct_icp_b200/config.py states for yaml-cpp's as<T>
// (DESIGN.md §5.13). A tree is read from the length-prefixed text tests/test_config_facade.py writes:
//   M <n> then n × (K <len> <key bytes>, node) | S <n> then n nodes | V <len> <bytes> | N (null)
#pragma once
#include <cctype>
#include <cerrno>
#include <cmath>
#include <cstdlib>
#include <istream>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

namespace yaml_stub {

class Node {
public:
    enum Kind { Undefined, Null, Scalar_, Sequence, Map };
    Node() = default;

    static Node Read(std::istream &is) {
        char tag = 0;
        is >> tag;
        Node n;
        n.d_ = std::make_shared<Data>();
        if (tag == 'N') {
            n.d_->kind = Null;
        } else if (tag == 'V') {
            n.d_->kind = Scalar_;
            n.d_->text = ReadBytes(is);
        } else if (tag == 'S' || tag == 'M') {
            size_t count = 0;
            is >> count;
            n.d_->kind = tag == 'S' ? Sequence : Map;
            for (size_t i = 0; i < count; ++i) {
                std::string key;
                if (tag == 'M') {
                    char k = 0;
                    is >> k;
                    if (k != 'K') throw std::runtime_error("stub: bad key tag");
                    key = ReadBytes(is);
                }
                n.d_->items.emplace_back(key, Read(is));
                n.d_->children.push_back(tag == 'S' ? n.d_->items.back().second : Node());
            }
        } else {
            throw std::runtime_error("stub: bad node tag");
        }
        return n;
    }

    explicit operator bool() const { return d_ && d_->kind != Undefined; }
    bool IsDefined() const { return bool(*this); }
    bool IsNull() const { return d_ && d_->kind == Null; }
    bool IsScalar() const { return d_ && d_->kind == Scalar_; }
    bool IsSequence() const { return d_ && d_->kind == Sequence; }
    bool IsMap() const { return d_ && d_->kind == Map; }
    const std::string &Scalar() const { return d_->text; }
    size_t size() const { return d_ ? d_->items.size() : 0; }

    Node operator[](const std::string &key) const {   // the first occurrence of the key; absent: an undefined node
        if (IsScalar() || IsSequence()) throw std::runtime_error("operator[] call on a scalar or a sequence");
        if (IsMap())
            for (const auto &kv : d_->items)
                if (kv.first == key) return kv.second;
        return Node();
    }

    // range-for: a sequence's items; a map's entries iterate as pairs, which as nodes are undefined
    std::vector<Node>::const_iterator begin() const { return d_ ? d_->children.begin() : Empty().begin(); }
    std::vector<Node>::const_iterator end() const { return d_ ? d_->children.end() : Empty().end(); }

    template <class T> T as() const;

private:
    struct Data {
        Kind kind = Undefined;
        std::string text;
        std::vector<std::pair<std::string, Node>> items;
        std::vector<Node> children;
    };
    static const std::vector<Node> &Empty() {
        static const std::vector<Node> none;
        return none;
    }
    std::shared_ptr<Data> d_;

    static std::string ReadBytes(std::istream &is) {
        size_t len = 0;
        is >> len;
        is.get();   // the separator
        std::string s(len, '\0');
        is.read(&s[0], (std::streamsize) len);
        return s;
    }
    [[noreturn]] void Bad(const char *what) const {
        throw std::runtime_error(std::string("bad conversion: not ") + what + ": '" + (d_ ? d_->text : "") + "'");
    }
    const std::string &Text(const char *what) const {
        if (!IsScalar()) Bad(what);
        return d_->text;
    }
    long long Integer(long long lo, long long hi, const char *what) const {
        const std::string &s = Text(what);
        // [+-]? then 0x hex, 0 octal or decimal, the whole text consumed (std::stringstream with the base unset)
        size_t i = (!s.empty() && (s[0] == '+' || s[0] == '-')) ? 1 : 0;
        if (i >= s.size() || !std::isdigit((unsigned char) s[i])) Bad(what);
        errno = 0;
        char *end = nullptr;
        const long long v = std::strtoll(s.c_str(), &end, 0);
        if (errno || *end || v < lo || v > hi) Bad(what);
        return v;
    }
    double Real(const char *what) const {
        const std::string &s = Text(what);
        for (const char *inf : {".inf", ".Inf", ".INF", "+.inf", "+.Inf", "+.INF"})
            if (s == inf) return HUGE_VAL;
        for (const char *inf : {"-.inf", "-.Inf", "-.INF"})
            if (s == inf) return -HUGE_VAL;
        for (const char *nan : {".nan", ".NaN", ".NAN"})
            if (s == nan) return std::nan("");
        // [+-]? (digits [. digits*] | . digits) ([eE] [+-]? digits)?
        size_t i = (!s.empty() && (s[0] == '+' || s[0] == '-')) ? 1 : 0, d = 0;
        while (i < s.size() && std::isdigit((unsigned char) s[i])) ++i, ++d;
        if (i < s.size() && s[i] == '.') {
            ++i;
            while (i < s.size() && std::isdigit((unsigned char) s[i])) ++i, ++d;
        }
        if (!d) Bad(what);
        if (i < s.size() && (s[i] == 'e' || s[i] == 'E')) {
            ++i;
            if (i < s.size() && (s[i] == '+' || s[i] == '-')) ++i;
            size_t e = 0;
            while (i < s.size() && std::isdigit((unsigned char) s[i])) ++i, ++e;
            if (!e) Bad(what);
        }
        if (i != s.size()) Bad(what);
        const double v = std::strtod(s.c_str(), nullptr);
        if (std::isinf(v)) Bad(what);
        return v;
    }
};

template <> inline int Node::as<int>() const { return (int) Integer(-2147483648LL, 2147483647LL, "an int"); }
template <> inline double Node::as<double>() const { return Real("a double"); }
template <> inline float Node::as<float>() const {
    const double v = Real("a float");
    const float f = (float) v;
    if (std::isinf(f) && !std::isinf(v)) Bad("a float");
    return f;
}
template <> inline bool Node::as<bool>() const {
    const std::string &s = Text("a bool");
    std::string lo = s, up = s, cap = s;
    for (auto &c : lo) c = (char) std::tolower((unsigned char) c);
    for (auto &c : up) c = (char) std::toupper((unsigned char) c);
    for (size_t i = 0; i < cap.size(); ++i)
        cap[i] = (char) (i ? std::tolower((unsigned char) cap[i]) : std::toupper((unsigned char) cap[i]));
    if (s != lo && s != up && s != cap) Bad("a bool");
    for (const char *t : {"y", "yes", "true", "on"})
        if (lo == t) return true;
    for (const char *f : {"n", "no", "false", "off"})
        if (lo == f) return false;
    Bad("a bool");
}
template <> inline std::string Node::as<std::string>() const {
    if (IsNull()) return "null";
    return Text("a string");
}

}  // namespace yaml_stub
