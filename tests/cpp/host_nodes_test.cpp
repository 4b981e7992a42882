// Driver for the "streamed_host" residency of include/ministark_prover.hpp (Merkle node heaps in pinned host memory).
// Linked against the CPU build of the ABI (tests/test_host_nodes_cpu.py) or the product library
// (tests/test_gpu_host_nodes.py).  Prints one line per command:
//   host_nodes_test peak <n> <beta> <nbase> <next> <lanes> <ce_blowup> <ff>   -> resident streamed streamed_host host bytes
//   host_nodes_test fib <log_rows> <5 options> <budget> <host budget> [<host budget 2>]
//                                                                             -> <residency> <pinned bytes> <proof hex>
//                                                                                [<pinned bytes once a second proof has
//                                                                                 started under host budget 2>]
//   host_nodes_test bf hello|burner:a:b:c <5 options> <budget> <host budget>  -> <residency> <pinned bytes> out:<hex> <proof hex>
// <budget>: GpuProver::memory_budget, <host budget>: GpuProver::host_memory_budget, in bytes (0: unset).  The bf trace is
// built on the device.  Every proof is checked by the C++ verifier before it is printed; a refusal goes to stderr, exit 1.
#include <cstdio>
#include <iostream>

#include "ministark_prover.hpp"
#include "ministark_verifier.hpp"

using namespace mshost;

static std::string hex(const Bytes &b) {
    static const char *d = "0123456789abcdef";
    std::string s;
    for (u8 c : b) { s.push_back(d[c >> 4]); s.push_back(d[c & 15]); }
    return s;
}

static const char *HELLO = "++++++++++[>+++++++>++++++++++>+++>+<<<<-]>++.>+.+++++++..+++.>++.<<+++++++++++++++.>.+++.------.--------.";

int main(int argc, char **argv) {
    if (argc < 3) { fprintf(stderr, "usage: see the header of host_nodes_test.cpp\n"); return 2; }
    const std::string kind = argv[1];
    auto opt = [&](int i) { return ProofOptions{(u8)atoi(argv[i]), (u8)atoi(argv[i + 1]), (u8)atoi(argv[i + 2]), (u8)atoi(argv[i + 3]), (u8)atoi(argv[i + 4])}; };
    try {
        if (kind == "peak" && argc == 9) {
            u64 a[7];
            for (int i = 0; i < 7; i++) a[i] = strtoull(argv[2 + i], nullptr, 10);
            const PeakBytes p = peak_bytes(a[0], a[1], a[2], a[3], a[4], a[5], a[6]);
            std::cout << p.resident << " " << p.streamed << " " << p.streamed_host << " " << p.host << "\n";
        } else if (kind == "fib" && (argc == 10 || argc == 11)) {
            const u64 n = (u64)1 << atoi(argv[2]);
            GpuProver prover(0);
            prover.memory_budget = strtoull(argv[8], nullptr, 10);
            prover.host_memory_budget = strtoull(argv[9], nullptr, 10);
            std::vector<u64> trace;
            const u64 last = fib_gen_trace(n, trace);
            const Bytes proof = prover.prove(fib_air_config(), opt(3), trace.data(), n, {Fq(last)}).to_bytes(1);
            verify(fib_air_config(), proof, {Fq(last)}, {}, 10);
            std::cout << prover.last_residency << " " << prover.pinned_bytes() << " " << hex(proof);
            if (argc == 11) {                   // a second proof under another host budget: what the prover still holds
                prover.host_memory_budget = strtoull(argv[10], nullptr, 10);
                try {
                    prover.prove(fib_air_config(), opt(3), trace.data(), n, {Fq(last)});
                } catch (const std::runtime_error &) {
                }
                std::cout << " " << prover.pinned_bytes();
            }
            std::cout << "\n";
        } else if (kind == "bf" && argc == 10) {
            const std::string which = argv[2];
            std::string src = HELLO;
            unsigned a, b, c;
            if (sscanf(which.c_str(), "burner:%u:%u:%u", &a, &b, &c) == 3) src = bf::cycle_burner(a, b, c);
            GpuProver prover(0);
            prover.memory_budget = strtoull(argv[8], nullptr, 10);
            prover.host_memory_budget = strtoull(argv[9], nullptr, 10);
            const std::vector<Fq> init = bf::test_rng_fq3(2);
            bf::DeviceTrace t = bf::simulate_device(prover.context(), src);
            const Bytes output = t.output;
            const u64 n = t.n;
            const Bytes proof = prover.prove(bf::air_config(src, {}, output), opt(3), std::move(t.base), n, {}, bf::claim_bytes(src, {}, output),
                                             [&](ms_ctx *ctx, const u64 *base_dev, u64 rows, const std::vector<Fq> &ch) {
                                                 return bf::device_extension(ctx, rows, base_dev, ch, init[0], init[1]);
                                             }).to_bytes(3);
            verify(bf::air_config(src, {}, output), proof, {}, bf::claim_bytes(src, {}, output), 10);
            std::cout << prover.last_residency << " " << prover.pinned_bytes() << " out:" << hex(output) << " " << hex(proof) << "\n";
        } else {
            fprintf(stderr, "unknown command or wrong arguments: %s\n", kind.c_str());
            return 2;
        }
    } catch (const std::exception &e) {
        fprintf(stderr, "host_nodes_test: %s\n", e.what());
        return 1;
    }
    return 0;
}
