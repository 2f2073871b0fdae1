// cli_flags.h -- command-line flags with the semantics of the reference's CMDLine
// (reference src/util/cmdline.h:67-237): every flag is `-name [value]` or
// `--name [value]`, values never start with '-', lists split on ';' or ','.
// Error texts match the reference so wrapper scripts keep working.
#pragma once
#include <cstdlib>
#include <iostream>
#include <map>
#include <string>
#include <vector>

namespace host {

class CmdLine {
 public:
  CmdLine(int argc, char** argv) {
    for (int i = 1; i < argc; i++) {
      std::string name(argv[i]);
      if (!strip_dashes(name)) throw "cannot parse " + name;  // cmdline.h:100-102
      if (values_.count(name)) throw "the parameter " + name + " is already specified";
      std::string value;
      if (i + 1 < argc) {
        std::string next(argv[i + 1]);
        if (!strip_dashes(next)) {  // a value, not another flag
          value = argv[i + 1];
          i++;
        }
      }
      values_[name] = value;
    }
  }

  const std::string& add(const std::string& name, const std::string& help) {
    help_[name] = help;
    return help_.find(name)->first;
  }

  bool has(const std::string& name) const { return values_.count(name) != 0; }
  void set(const std::string& name, const std::string& value) { values_[name] = value; }

  // cmdline.h:150-157
  void check() const {
    for (const auto& kv : values_)
      if (!help_.count(kv.first)) throw "the parameter " + kv.first + " does not exist";
  }

  std::string str(const std::string& name, const std::string& dflt = "") const {
    auto it = values_.find(name);
    return it == values_.end() ? dflt : it->second;
  }
  double num(const std::string& name, double dflt) const {
    auto it = values_.find(name);
    return it == values_.end() ? dflt : atof(it->second.c_str());
  }
  long integer(const std::string& name, long dflt) const {
    auto it = values_.find(name);
    return it == values_.end() ? dflt : atoi(it->second.c_str());
  }
  // a 64-bit count (byte sizes past 2^31-1, which atoi cannot read)
  long long integer64(const std::string& name, long long dflt) const {
    auto it = values_.find(name);
    return it == values_.end() ? dflt : strtoll(it->second.c_str(), nullptr, 10);
  }

  std::vector<std::string> list(const std::string& name) const {
    std::vector<std::string> out;
    const std::string s = str(name);
    const std::string delim = ";,";  // cmdline.h:81
    size_t a = s.find_first_not_of(delim, 0);
    while (a != std::string::npos) {
      size_t b = s.find_first_of(delim, a);
      out.push_back(s.substr(a, b == std::string::npos ? std::string::npos : b - a));
      if (b == std::string::npos) break;
      a = s.find_first_not_of(delim, b);
    }
    return out;
  }
  std::vector<double> num_list(const std::string& name) const {
    std::vector<double> out;
    for (const auto& t : list(name)) out.push_back(atof(t.c_str()));
    return out;
  }
  std::vector<int> int_list(const std::string& name) const {
    std::vector<int> out;
    for (const auto& t : list(name)) out.push_back(atoi(t.c_str()));
    return out;
  }

  // cmdline.h:118-142: "-name" padded to 16 columns, help wrapped at 72
  void print_help() const {
    for (const auto& kv : help_) {
      std::cout << "-" << kv.first;
      for (int i = (int)kv.first.size() + 1; i < 16; i++) std::cout << " ";
      std::string rest = kv.second;
      while (!rest.empty()) {
        if (rest.size() > 72 - 16) {
          size_t p = rest.substr(0, 72 - 16).find_last_of(" \t");
          if (p == 0 || p == std::string::npos) p = 72 - 16;
          std::cout << rest.substr(0, p) << std::endl;
          rest = p + 1 <= rest.size() ? rest.substr(p + 1) : "";
        } else {
          std::cout << rest << std::endl;
          rest.clear();
        }
        if (!rest.empty())
          for (int i = 0; i < 16; i++) std::cout << " ";
      }
    }
  }

 private:
  static bool strip_dashes(std::string& s) {
    if (s.empty() || s[0] != '-') return false;
    s = (s.size() > 1 && s[1] == '-') ? s.substr(2) : s.substr(1);
    return true;
  }
  std::map<std::string, std::string> help_;
  std::map<std::string, std::string> values_;
};

}  // namespace host
