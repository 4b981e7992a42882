// bf_cli.cpp — the brainfuck prover and verifier on the command line (examples/brainfuck/main.rs), over the C++ host layer:
//
//   ministark_bf prove SRC --dst FILE [--input STR] [--memory-budget GIB] [--host-memory GIB] [--device K]
//   ministark_bf verify SRC --proof FILE [--input STR] --output STR
//
// prove builds the execution trace on the device (bf::simulate_device), proves it with mshost::GpuProver in whichever
// residency fits (resident, else streamed, else, with --host-memory, streamed with the Merkle node heaps in that much
// pinned host memory, else it refuses) and writes the reference's (claim, proof).serialize_compressed:
// claim_bytes(source, input, output) followed by the proof bytes.  verify needs no GPU: it parses the claim, checks it
// against the arguments and runs mshost::verify at the reference's 96-bit security level.  Either exits non-zero with a
// message where the reference panics.
#include <chrono>
#include <cstdio>
#include <fstream>
#include <iostream>
#include <iterator>

#include "ministark_prover.hpp"
#include "ministark_verifier.hpp"

using namespace mshost;

namespace {

constexpr ProofOptions OPTIONS{19, 16, 20, 16, 16};     // main.rs:92-105
constexpr u32 SECURITY_LEVEL = 96;                       // main.rs:89

struct Failure : std::runtime_error {
    using std::runtime_error::runtime_error;
};

int usage() {
    fprintf(stderr,
            "usage: ministark_bf prove SRC --dst FILE [--input STR] [--memory-budget GIB] [--host-memory GIB] [--device K]\n"
            "       ministark_bf verify SRC --proof FILE [--input STR] --output STR\n");
    return 2;
}

Bytes read_file(const std::string &path) {
    std::ifstream f(path, std::ios::binary);
    if (!f) throw Failure("cannot read " + path);
    return Bytes(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
}

double seconds_since(std::chrono::steady_clock::time_point t0) {
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

int run_prove(const std::string &src_path, const std::string &dst, const std::string &input_str, double budget_gib, double host_gib,
              int device) {
    const Bytes src_bytes = read_file(src_path);
    const std::string source(src_bytes.begin(), src_bytes.end());
    const Bytes input(input_str.begin(), input_str.end());
    GpuProver prover(device);
    if (budget_gib > 0) prover.memory_budget = (u64)(budget_gib * (double)((u64)1 << 30));
    if (host_gib > 0) prover.host_memory_budget = (u64)(host_gib * (double)((u64)1 << 30));

    const u64 free_before = prover.free_memory();
    auto t0 = std::chrono::steady_clock::now();
    bf::DeviceTrace trace = bf::simulate_device(prover.context(), source, input);
    printf("Generated execution trace (cols=17, rows=%llu) in %.3fs\n", (unsigned long long)trace.n, seconds_since(t0));
    printf("Program output: \"%s\"\n", std::string(trace.output.begin(), trace.output.end()).c_str());
    fflush(stdout);

    const std::vector<Fq> initial = bf::test_rng_fq3(2);    // the permutation start values of the extension columns
    const Bytes claim = bf::claim_bytes(source, input, trace.output);
    const u64 n = trace.n;
    t0 = std::chrono::steady_clock::now();
    const Proof proof = prover.prove(bf::air_config(source, input, trace.output), OPTIONS, std::move(trace.base), n, {}, claim,
                                     [&](ms_ctx *ctx, const u64 *base_dev, u64 rows, const std::vector<Fq> &ch) {
                                         return bf::device_extension(ctx, rows, base_dev, ch, initial[0], initial[1]);
                                     });
    printf("Proof generated in: %.3fs\n", seconds_since(t0));
    printf("Residency: %s\n", prover.last_residency.c_str());
    if (prover.pinned_bytes())
        printf("Pinned host memory: %llu bytes (%s), pinned in %.3fs\n", (unsigned long long)prover.pinned_bytes(),
               gib(prover.pinned_bytes()).c_str(), prover.last_pin_seconds);
    if (free_before != SIZE_MAX) {
        printf("Free device memory before the trace: %llu bytes (%s)\n", (unsigned long long)free_before, gib(free_before).c_str());
        printf("Lowest free device memory between phases: %llu bytes (%s)\n", (unsigned long long)prover.lowest_free_bytes,
               gib(prover.lowest_free_bytes).c_str());
    }
    printf("Proof security (conjectured): %ubit\n", security_level_bits(OPTIONS, n, 3));

    Bytes file = claim;
    const Bytes p = proof.to_bytes(3);
    file.insert(file.end(), p.begin(), p.end());
    printf("Proof size: %zuKB\n", file.size() / 1024);
    std::ofstream f(dst, std::ios::binary);
    if (!f.write(reinterpret_cast<const char *>(file.data()), (std::streamsize)file.size()) || !f.flush()) throw Failure("cannot write " + dst);
    printf("Proof written to %s\n", dst.c_str());
    return 0;
}

int run_verify(const std::string &src_path, const std::string &proof_path, const std::string &input_str, const std::string &output_str) {
    const Bytes src_bytes = read_file(src_path), file = read_file(proof_path);
    const std::string source(src_bytes.begin(), src_bytes.end());
    const Bytes input(input_str.begin(), input_str.end()), output(output_str.begin(), output_str.end());
    // the claim: String, Vec<u8>, Vec<u8>, each a u64 little-endian length and its bytes
    size_t at = 0;
    auto field = [&](const char *what) {
        if (file.size() - at < 8) throw Failure(std::string("truncated claim (") + what + ")");
        u64 len = 0;
        for (int k = 7; k >= 0; k--) len = (len << 8) | file[at + k];
        at += 8;
        if (len > file.size() - at) throw Failure(std::string("truncated claim (") + what + ")");
        Bytes v(file.begin() + at, file.begin() + at + len);
        at += len;
        return v;
    };
    const Bytes c_source = field("source code"), c_input = field("input"), c_output = field("output");
    if (c_input != input) throw Failure("the proof's claim has a different input");
    if (c_output != output) throw Failure("the proof's claim has a different output");
    if (c_source != src_bytes) throw Failure("the proof's claim has different source code");
    const Bytes proof(file.begin() + at, file.end());
    const auto t0 = std::chrono::steady_clock::now();
    try {
        mshost::verify(bf::air_config(source, input, output), proof, {}, bf::claim_bytes(source, input, output), SECURITY_LEVEL);
    } catch (const VerificationError &e) {
        throw Failure(std::string("verification failed: ") + e.what());
    }
    printf("Proof verified in: %.3fs\n", seconds_since(t0));
    return 0;
}

}  // namespace

int main(int argc, char **argv) {
    if (argc < 3) return usage();
    const std::string cmd = argv[1], src = argv[2];
    std::string dst, proof, input, output;
    bool has_output = false;
    double budget = 0, host_memory = 0;
    int device = 0;
    for (int i = 3; i < argc; i++) {
        const std::string a = argv[i];
        if (i + 1 >= argc) return usage();
        const std::string v = argv[++i];
        if (a == "--dst") dst = v;
        else if (a == "--proof") proof = v;
        else if (a == "--input") input = v;
        else if (a == "--output") { output = v; has_output = true; }
        else if (a == "--memory-budget") {
            char *end = nullptr;
            budget = strtod(v.c_str(), &end);
            if (*end || !(budget > 0)) return usage();
        } else if (a == "--host-memory") {
            char *end = nullptr;
            host_memory = strtod(v.c_str(), &end);
            if (*end || !(host_memory > 0)) return usage();
        } else if (a == "--device") device = atoi(v.c_str());
        else return usage();
    }
    try {
        if (cmd == "prove" && !dst.empty()) return run_prove(src, dst, input, budget, host_memory, device);
        if (cmd == "verify" && !proof.empty() && has_output) return run_verify(src, proof, input, output);
    } catch (const std::exception &e) {
        fprintf(stderr, "ministark_bf %s: %s\n", cmd.c_str(), e.what());
        return 1;
    }
    return usage();
}
