// Golden-digest and timing harness for the REAL SharpZipLib (BASELINE.md section 2.1): runs the reference's own
// Deflater / Inflater over buffer files written by tools/csharp_harness/export_inputs.py and prints, per buffer, the
// SHA-256 of the compressed bytes, plus single-thread and N-thread throughput.  Needs a .NET SDK (>= 6.0), so it ships as
// source:
//   dotnet run -c Release --project tools/csharp_harness -- <dir with *.bin> <level> <threads> > reference_digests.json
// tests/test_oracle.py::test_reference_digests compares oracle and GPU output with that file when it exists.
using System;
using System.Collections.Generic;
using System.Diagnostics;
using System.IO;
using System.Linq;
using System.Security.Cryptography;
using System.Threading.Tasks;
using ICSharpCode.SharpZipLib.Zip.Compression;

static class Program
{
	static byte[] DeflateAll(byte[] input, int level)
	{
		// the call pattern of SURVEY.md 8(d): SetInput(all) -> Finish() -> drain with a 512-byte buffer
		var d = new Deflater(level, true);
		d.SetInput(input);
		d.Finish();
		var ms = new MemoryStream(input.Length / 2 + 64);
		var buf = new byte[512];
		while (!d.IsFinished)
		{
			int n = d.Deflate(buf);
			ms.Write(buf, 0, n);
		}
		return ms.ToArray();
	}

	static byte[] InflateAll(byte[] comp, int size)
	{
		var inf = new Inflater(true);
		inf.SetInput(comp);
		var outb = new byte[size];
		int pos = 0;
		while (!inf.IsFinished && pos < size)
		{
			int n = inf.Inflate(outb, pos, size - pos);
			if (n == 0 && inf.IsNeedingInput) break;
			pos += n;
		}
		return outb;
	}

	static int Main(string[] args)
	{
		if (args.Length < 1) { Console.Error.WriteLine("usage: harness <dir> [level=6] [threads=cores]"); return 2; }
		int level = args.Length > 1 ? int.Parse(args[1]) : 6;
		int threads = args.Length > 2 ? int.Parse(args[2]) : Environment.ProcessorCount;
		var files = Directory.GetFiles(args[0], "*.bin").OrderBy(f => f, StringComparer.Ordinal).ToArray();
		var inputs = files.Select(File.ReadAllBytes).ToArray();
		var outputs = new byte[inputs.Length][];
		long total = inputs.Sum(b => (long)b.Length);
		// warm-up + single thread, best of 5
		double best1 = double.MaxValue;
		for (int rep = 0; rep < 6; rep++)
		{
			var sw = Stopwatch.StartNew();
			for (int i = 0; i < inputs.Length; i++) outputs[i] = DeflateAll(inputs[i], level);
			sw.Stop();
			if (rep > 0) best1 = Math.Min(best1, sw.Elapsed.TotalSeconds);
		}
		double bestN = double.MaxValue;
		var po = new ParallelOptions { MaxDegreeOfParallelism = threads };
		for (int rep = 0; rep < 6; rep++)
		{
			var sw = Stopwatch.StartNew();
			Parallel.For(0, inputs.Length, po, i => { outputs[i] = DeflateAll(inputs[i], level); }); // one Deflater per call: not thread safe
			sw.Stop();
			if (rep > 0) bestN = Math.Min(bestN, sw.Elapsed.TotalSeconds);
		}
		double bestI = double.MaxValue;
		for (int rep = 0; rep < 6; rep++)
		{
			var sw = Stopwatch.StartNew();
			Parallel.For(0, inputs.Length, po, i =>
			{
				var back = InflateAll(outputs[i], inputs[i].Length);
				if (!back.AsSpan().SequenceEqual(inputs[i])) throw new InvalidDataException("round trip failed: " + files[i]);
			});
			sw.Stop();
			if (rep > 0) bestI = Math.Min(bestI, sw.Elapsed.TotalSeconds);
		}
		var lines = new List<string>();
		using (var sha = SHA256.Create())
			for (int i = 0; i < inputs.Length; i++)
				lines.Add($"    \"{Path.GetFileName(files[i])}\": {{\"in_sha256\": \"{Convert.ToHexString(sha.ComputeHash(inputs[i])).ToLowerInvariant()}\", " +
				          $"\"out_sha256\": \"{Convert.ToHexString(sha.ComputeHash(outputs[i])).ToLowerInvariant()}\", \"in_len\": {inputs[i].Length}, \"out_len\": {outputs[i].Length}}}");
		Console.WriteLine("{");
		Console.WriteLine($"  \"sharpziplib\": \"{typeof(Deflater).Assembly.GetName().Version}\", \"level\": {level}, \"threads\": {threads}, \"bytes\": {total},");
		Console.WriteLine($"  \"deflate_gbs_1_thread\": {total / best1 / 1e9:F4}, \"deflate_gbs_n_threads\": {total / bestN / 1e9:F4}, \"inflate_gbs_n_threads\": {total / bestI / 1e9:F4},");
		Console.WriteLine("  \"buffers\": {");
		Console.WriteLine(string.Join(",\n", lines));
		Console.WriteLine("  }\n}");
		return 0;
	}
}
