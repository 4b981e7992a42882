// Driver for the residency selection, the streamed residency and the device-built brainfuck trace of
// include/ministark_prover.hpp.  Linked against the CPU build of the ABI (tests/test_cpp_stream_prover_cpu.py) or the
// product library (tests/test_gpu_cpp_stream_prover.py).  Prints one line per command:
//   stream_prover_test peak <n> <beta> <nbase> <next> <lanes> <ce_blowup> <ff>      -> <resident bytes> <streamed bytes>
//   stream_prover_test rng <count>                                                 -> c0 c1 c2 per draw, canonical
//   stream_prover_test fib <log_rows> <5 options> <budget>                         -> <residency> <proof hex>
//   stream_prover_test bf hello|burner:a:b:c <5 options> <budget> host|device      -> <residency> out:<hex> <proof hex>
//   stream_prover_test refuse <budget> host|device                                 -> the refusal, whether the trace was
//                                                                                     read, the allocations it made
// <budget>: GpuProver::memory_budget in bytes (0: unset).  Every proof is checked by the C++ verifier before it is printed.
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
    if (argc < 3) { fprintf(stderr, "usage: see the header of stream_prover_test.cpp\n"); return 2; }
    const std::string kind = argv[1];
    auto opt = [&](int i) { return ProofOptions{(u8)atoi(argv[i]), (u8)atoi(argv[i + 1]), (u8)atoi(argv[i + 2]), (u8)atoi(argv[i + 3]), (u8)atoi(argv[i + 4])}; };
    try {
        if (kind == "peak") {
            u64 a[7];
            for (int i = 0; i < 7; i++) a[i] = strtoull(argv[2 + i], nullptr, 10);
            const PeakBytes p = peak_bytes(a[0], a[1], a[2], a[3], a[4], a[5], a[6]);
            std::cout << p.resident << " " << p.streamed << "\n";
        } else if (kind == "rng") {
            for (const Fq &v : bf::test_rng_fq3(strtoull(argv[2], nullptr, 10))) std::cout << v.c[0] << " " << v.c[1] << " " << v.c[2] << "\n";
        } else if (kind == "fib") {
            const u64 n = (u64)1 << atoi(argv[2]);
            const ProofOptions o = opt(3);
            GpuProver prover(0);
            prover.memory_budget = strtoull(argv[8], nullptr, 10);
            std::vector<u64> trace;
            const u64 last = fib_gen_trace(n, trace);
            const Bytes proof = prover.prove(fib_air_config(), o, trace.data(), n, {Fq(last)}).to_bytes(1);
            verify(fib_air_config(), proof, {Fq(last)}, {}, 10);
            std::cout << prover.last_residency << " " << hex(proof) << "\n";
        } else if (kind == "bf") {
            const std::string which = argv[2];
            std::string src = HELLO;
            unsigned a, b, c;
            if (sscanf(which.c_str(), "burner:%u:%u:%u", &a, &b, &c) == 3) src = bf::cycle_burner(a, b, c);
            const ProofOptions o = opt(3);
            GpuProver prover(0);
            prover.memory_budget = strtoull(argv[8], nullptr, 10);
            const std::vector<Fq> init = bf::test_rng_fq3(2);
            Bytes output, proof;
            if (std::string(argv[9]) == "device") {
                bf::DeviceTrace t = bf::simulate_device(prover.context(), src);
                output = t.output;
                const u64 n = t.n;
                proof = prover.prove(bf::air_config(src, {}, output), o, std::move(t.base), n, {}, bf::claim_bytes(src, {}, output),
                                     [&](ms_ctx *ctx, const u64 *base_dev, u64 rows, const std::vector<Fq> &ch) {
                                         return bf::device_extension(ctx, rows, base_dev, ch, init[0], init[1]);
                                     }).to_bytes(3);
            } else {
                const bf::VmTrace t = bf::simulate(src);
                output = t.output;
                std::vector<u64> words(t.base.size());
                for (size_t i = 0; i < words.size(); i++) words[i] = to_mont(t.base[i]);
                proof = prover.prove(bf::air_config(src, {}, output), o, words.data(), t.n, {}, bf::claim_bytes(src, {}, output),
                                     [&](ms_ctx *ctx, const u64 *base_dev, u64, const std::vector<Fq> &ch) {
                                         return bf::device_extension(ctx, t, base_dev, ch, init[0], init[1]);
                                     }).to_bytes(3);
            }
            verify(bf::air_config(src, {}, output), proof, {}, bf::claim_bytes(src, {}, output), 10);
            std::cout << prover.last_residency << " out:" << hex(output) << " " << hex(proof) << "\n";
        } else if (kind == "refuse") {
            // a brainfuck-shaped proof (17 + 9 columns) of 2^20 rows that cannot fit the budget: the host trace is a null
            // pointer and the extension builder records a call, so a refusal that read either would show
            GpuProver prover(0);
            prover.memory_budget = strtoull(argv[2], nullptr, 10);
            const u64 n = (u64)1 << 20;
            bool built = false;
            auto builder = [&](ms_ctx *, const u64 *, u64, const std::vector<Fq> &) { built = true; return DeviceBuf(); };
            const std::string src = bf::cycle_burner(40, 40, 60);
            const AirConfig cfg = bf::air_config(src, {}, {});
            const ProofOptions o{19, 16, 20, 16, 16};
            u64 allocations = 0;
            try {
                if (std::string(argv[3]) == "device") {
                    DeviceBuf base(prover.context(), 8);
                    allocations = device_allocations();
                    prover.prove(cfg, o, std::move(base), n, {}, bf::claim_bytes(src, {}, {}), builder);
                } else {
                    allocations = device_allocations();
                    prover.prove(cfg, o, nullptr, n, {}, bf::claim_bytes(src, {}, {}), builder);
                }
                std::cout << "proved\n";
                return 1;
            } catch (const std::runtime_error &e) {
                std::cout << e.what() << "\n" << "extension built: " << built << "\n"
                          << "allocations: " << device_allocations() - allocations << "\n";
            }
        } else {
            fprintf(stderr, "unknown command %s\n", kind.c_str());
            return 2;
        }
    } catch (const std::exception &e) {
        fprintf(stderr, "stream_prover_test: %s\n", e.what());
        return 1;
    }
    return 0;
}
